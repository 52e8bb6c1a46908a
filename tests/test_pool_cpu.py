"""dist.pool_sum / pool_max / pool_min / pool_cat over a gloo group of spawned CPU processes: the partials combine in
ascending rank order (three ranks, so that float64 addition order shows), every rank gets the same bytes, int64
partials sum exactly, ragged last axes concatenate in rank order, and a one-rank group returns the partial itself, as
the sample-processing helper `_pooled` does without a group (while the pools read None as the world group)."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from madrl_b200.dist import _pooled, pool_cat, pool_max, pool_min, pool_sum

WORLD = 3
# in rank order (1e16 + 1) + -1e16 = 0 (1e16 + 1 rounds back to 1e16); in another order the sum is 1
VALS = (1e16, 1.0, -1e16)


def _partials(rank):
    f = torch.tensor([[VALS[rank], 0.25 * rank], [rank - 1.0, 3.0 + rank]], dtype=torch.float64)
    i = torch.tensor([2 ** 40 + rank, -rank, 7], dtype=torch.int64)
    return f, i


def _worker(rank, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=WORLD)
    try:
        f, i = _partials(rank)
        out = dict(sum=pool_sum(f, None), isum=pool_sum(i, None), max=pool_max(f, None), min=pool_min(f, None),
                   imax=pool_max(i, None), cat=pool_cat(torch.arange(rank + 1, dtype=torch.int64).view(1, -1)
                                                        .repeat(2, 1) * 10 + rank, None))
        try:
            pool_sum(f.float(), None)
            out["refused_f32"] = False
        except ValueError:
            out["refused_f32"] = True
        own, _ = dist.new_subgroups(group_size=1)                     # this rank alone
        out["one_rank_identity"] = pool_sum(f, own) is f and pool_min(i, own) is i and pool_cat(f, own) is f
        out["no_group_identity"] = all(_pooled(p, f, None) is f for p in (pool_sum, pool_max, pool_min, pool_cat))
        q.put((rank, {k: (v.numpy().tobytes(), tuple(v.shape)) if torch.is_tensor(v) else v for k, v in out.items()}))
    finally:
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_pool_helpers_over_three_gloo_ranks():
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, q)) for r in range(WORLD)]
    try:
        for p in procs:
            p.start()
        for p in procs:
            p.join(180)
            assert p.exitcode == 0
        got = dict(q.get() for _ in range(WORLD))
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
                p.join()
    for r in range(1, WORLD):
        assert got[r] == got[0]                                        # the same bytes on every rank
    res = got[0]
    assert res["refused_f32"] and res["one_rank_identity"] and res["no_group_identity"]
    parts = [_partials(r) for r in range(WORLD)]
    want = parts[0][0].clone()
    for r in range(1, WORLD):
        want = want + parts[r][0]
    as_t = lambda k, dt: torch.frombuffer(bytearray(res[k][0]), dtype=dt).view(res[k][1])     # noqa: E731
    s = as_t("sum", torch.float64)
    assert s.numpy().tobytes() == want.numpy().tobytes()
    assert float(s[0, 0]) == 0.0                                       # (1e16 + 1) + -1e16: rank order
    assert torch.equal(as_t("isum", torch.int64), sum(p[1] for p in parts))
    fs = torch.stack([p[0] for p in parts])
    assert torch.equal(as_t("max", torch.float64), fs.max(0).values)
    assert torch.equal(as_t("min", torch.float64), fs.min(0).values)
    assert torch.equal(as_t("imax", torch.int64), torch.stack([p[1] for p in parts]).max(0).values)
    cat = torch.cat([torch.arange(r + 1, dtype=torch.int64).view(1, -1).repeat(2, 1) * 10 + r for r in range(WORLD)],
                    dim=1)
    assert torch.equal(as_t("cat", torch.int64), cat)
