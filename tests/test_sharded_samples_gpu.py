"""Sample processing and evaluation pooled over the ranks of a sharded batch (``group=``), on the GPU:

  * with a one-rank group every pooled call returns the bits of ``group=None``;
  * an evaluation over several ranks refuses an engine not built by ``dist.make_sharded``;
  * two processes, each holding half of a C2-like Waterworld batch through ``dist.make_sharded`` (ragged: 31 and 32
    envs), over gloo on one GPU -- and over NCCL on two GPUs where the box has them: every pooled output has the
    same bytes on both ranks and matches the unsharded single-process call (counts, lengths, path counts, bin
    counts and the fallback decision exactly; float32 standardiser state and simplev within one float32 ulp;
    float64 moments, explained variances and mean returns at rtol 1e-12; the rltools baseline with obsnorm within
    1e-9 of the unsharded fit; evaluate_heuristic on Waterworld and Pursuit exactly).
"""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from conftest import ROOT

pytestmark = pytest.mark.gpu

E_G, T, MPL, D_CFG = 63, 60, 25, dict(n_poison=10, n_sensors=30)


def _np(x):
    if torch.is_tensor(x):
        return x.detach().cpu().numpy()
    if isinstance(x, dict):
        return {k: _np(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(_np(v) for v in x)
    return x


def compute(dev, group, rank=0, world=1):
    """Every pooled entry point on this rank's shard of one rollout (group=None, world=1: the unsharded batch)."""
    from madrl_b200 import BatchedMAWaterWorld, BatchedPursuitEvade, evaluate_heuristic
    from madrl_b200 import postproc as pp
    from madrl_b200 import rltools_sampler as rs
    from madrl_b200.dist import make_sharded
    kw = {} if group is None else dict(group=group)
    out = {}
    eng = make_sharded(BatchedMAWaterWorld, E_G, 5, 5, rank=rank, world=world, seed=3, device=dev,
                       max_path_length=MPL, **D_CFG)
    lo = eng.shard[0]
    obs0 = eng.reset().clone()
    act, obs, rew, done, _ = eng.rollout_heuristic(T, obs0.clone(), auto_reset=True, norm="env")
    E, A = eng.n_envs, eng._n_acting
    obs, obs0 = obs.reshape(T, E, A, -1).float().contiguous(), obs0.reshape(E, A, -1).float().contiguous()
    D = obs.shape[-1]
    out["lo"], out["rew"], out["done"] = lo, rew, done
    st, sa = rs.RunningStandardizer(D, dev), rs.RunningStandardizer(D, dev, n_agents=A)
    sr = rs.RunningStandardizer(1, dev)
    st.update(obs, obs0, **kw)
    sa.update(obs, obs0, **kw)
    sr.update_per_agent(rew.unsqueeze(-1), **kw)
    out["std"] = [s.get_param_values() for s in (st, sa, sr)]
    q = pp.gae(rew, torch.zeros_like(rew), done, 0.99, 1.0)[1]
    for pa in (False, True):
        out["tb", pa] = rs.time_baseline(q, done, None, pa, **kw)
    simplev = out["tb", False][0]
    out["mom"] = pp.moments(q, simplev, **kw)
    out["moma"] = pp.moments_agents(q, simplev, **kw)
    out["ev"] = (pp.explained_variance(simplev, q, **kw), pp.explained_variance(simplev, q, per_agent=True, **kw))
    out["ca"] = (pp.center_advantages(q, **kw), pp.center_advantages(q, True, True, per_agent=True, **kw))
    out["fields"] = [rs.sample_fields(rew, done, m, **kw) for m in ("decentralized", "concurrent", "centralized")]
    out["pstats"] = [pp.path_statistics(rew, q, done, pa, **kw) for pa in (False, True)]
    bl, rn = rs.LinearFeatureBaseline(D, dev, True), rs.RunningStandardizer(1, dev)
    bl.update_obsnorm(obs, obs0, **kw)
    rn.update(rew.unsqueeze(-1), **kw)
    out["ps"] = []
    for _ in range(2):
        r = rs.process_samples(bl, obs, done, rew, 0.99, 0.97, rewnorm=rn, obs_before=obs0, **kw)
        out["ps"].append((r["v_r"], r["tv_r"], r["fallback"], r["advantages"], bl.get_param_values()[0]))
    cb = pp.LinearFeatureBaseline(D, dev, n_agents=A)
    out["conc"] = [pp.process_samples_concurrent(cb, obs, done, rew, 0.99, 0.97, obs_before=obs0, **kw)
                   for _ in range(2)]
    rb = pp.LinearFeatureBaseline(D, dev)
    rec = pp.process_samples_recurrent(rb, obs, act, rew, done, 0.99, 0.97, "decentralized", obs_before=obs0, **kw)
    out["rec"] = {k: rec[k] for k in ("ExplainedVariance", "AverageReturn", "StdReturn", "MaxReturn", "MinReturn",
                                      "AverageDiscountedReturn", "NumTrajs")}
    ww = make_sharded(BatchedMAWaterWorld, E_G, 5, 5, rank=rank, world=world, seed=8, device=dev,
                      max_path_length=MPL, **D_CFG)
    out["eval_ww"] = evaluate_heuristic(ww, 100, 0.99, "decentralized", chunk=24, **kw)
    pe = make_sharded(BatchedPursuitEvade, 21, np.load(os.path.join(ROOT, "maps", "map_pool16.npy")), rank=rank,
                      world=world, n_evaders=30, n_pursuers=8, obs_range=7, surround=True, sample_maps=True, seed=6,
                      device=dev, max_path_length=40)
    out["eval_pe"] = evaluate_heuristic(pe, 50, 0.99, "decentralized", chunk=24, py2_division=True, **kw)
    torch.cuda.synchronize(dev)
    return _np(out)


def _bits_equal(a, b, path="out"):
    """The same keys, types and bytes all the way down."""
    if isinstance(a, dict):
        assert sorted(a, key=str) == sorted(b, key=str), path
        for k in a:
            _bits_equal(a[k], b[k], "%s[%r]" % (path, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _bits_equal(x, y, "%s[%d]" % (path, i))
    elif isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), path
    else:
        assert type(a) is type(b) and (a == b or (a != a and b != b)), (path, a, b)


# ---- one rank -------------------------------------------------------------------------------------------------


@pytest.fixture(scope="module")
def one_rank_group():
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        yield dist.group.WORLD
    finally:
        dist.destroy_process_group()


def test_one_rank_group_gives_the_bits_of_no_group(one_rank_group):
    _bits_equal(compute("cuda:0", one_rank_group), compute("cuda:0", None))


# ---- two ranks ------------------------------------------------------------------------------------------------


def _worker(rank, world, port, backend, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = "cuda:%d" % (rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    try:
        res = compute(dev, dist.group.WORLD, rank, world)
        from madrl_b200 import BatchedMAWaterWorld, evaluate_heuristic
        unsharded = BatchedMAWaterWorld(4, 5, 5, device=dev, seed=1, max_path_length=5, **D_CFG)
        try:                          # every rank refuses an engine that does not know its shard, before exchanging
            evaluate_heuristic(unsharded, 4, 0.99, "decentralized", group=dist.group.WORLD)
            res["refused"] = False
        except ValueError as ex:
            res["refused"] = "make_sharded" in str(ex)
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run_two(backend):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, backend, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        got = {}
        for _ in range(2):
            r, res = q.get(timeout=600)        # raises (and the workers are killed below) if a rank fails
            got[r] = res
        for p in procs:
            p.join(300)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
            p.join()
    return got


def _ulps(a, b):
    return int(np.abs(a.view(np.int32).astype(np.int64) - b.view(np.int32).astype(np.int64)).max())


def _check_sharded(got, full):
    """got: {rank: compute(...)} of two ranks; full: the unsharded compute."""
    r0, r1 = got[0], got[1]
    assert r0["refused"] and r1["refused"]
    his = [(r["lo"], r["lo"] + r["done"].shape[1]) for r in (r0, r1)]
    assert his == [(0, 31), (31, 63)]
    for r, (lo, hi) in zip((r0, r1), his):                    # the shards hold the unsharded batch's envs
        assert np.array_equal(r["rew"], full["rew"][:, lo:hi]) and np.array_equal(r["done"], full["done"][:, lo:hi])
    pooled = ("std", "mom", "moma", "ev", "fields", "pstats", "rec", "eval_ww", "eval_pe")
    for k in pooled:
        _bits_equal(r0[k], r1[k], k)
    for k in (("tb", False), ("tb", True)):
        _bits_equal(r0[k][1:], r1[k][1:], str(k))
    for i in range(2):
        _bits_equal([x for j, x in enumerate(r0["ps"][i]) if j != 3], [x for j, x in enumerate(r1["ps"][i]) if j != 3])
        _bits_equal(r0["conc"][i][3], r1["conc"][i][3])
    # against the unsharded batch
    for (g, w) in zip(r0["std"], full["std"]):
        assert np.array_equal(g[0], w[0]) and _ulps(g[1], w[1]) <= 1 and _ulps(g[2], w[2]) <= 1
    for pa in (False, True):
        s, bs, bc = full["tb", pa]
        assert np.array_equal(r0["tb", pa][2], bc)
        np.testing.assert_allclose(r0["tb", pa][1], bs, rtol=1e-12)
        for r, (lo, hi) in zip((r0, r1), his):
            assert _ulps(r["tb", pa][0], s[:, lo:hi]) <= 1
    for k in ("mom", "moma"):     # the mean of q - simplev cancels to ~1e-10: an absolute floor at 1e-14 of the scale
        np.testing.assert_allclose(r0[k], full[k], rtol=1e-12, atol=1e-14 * np.abs(full[k]).max())
    np.testing.assert_allclose(r0["ev"][0], full["ev"][0], rtol=1e-12)
    np.testing.assert_allclose(r0["ev"][1], full["ev"][1], rtol=1e-12)
    for r, (lo, hi) in zip((r0, r1), his):
        for c in range(2):                   # centred values near 0 carry the means' rounding: an absolute bound
            np.testing.assert_allclose(r["ca"][c], full["ca"][c][:, lo:hi], rtol=1e-6, atol=1e-6)
    for g, w in zip(r0["fields"], full["fields"]):
        assert sorted(g) == sorted(w)
        for k in ("batch", "avglen", "maxlen", "minlen"):
            assert g[k] == w[k], k
        for k in ("ret", "ravg"):
            assert g[k] == pytest.approx(w[k], rel=1e-12), k
    for g, w in zip(r0["pstats"], full["pstats"]):
        for gd, wd in zip(g if isinstance(g, list) else [g], w if isinstance(w, list) else [w]):
            assert gd["NumTrajs"] == wd["NumTrajs"] and gd["MaxReturn"] == wd["MaxReturn"]
            assert gd["MinReturn"] == wd["MinReturn"]
            for k in ("AverageReturn", "StdReturn", "AverageDiscountedReturn"):
                assert gd[k] == pytest.approx(wd[k], rel=1e-12), k
    for i in range(2):
        v_r, tv_r, fb, _, coef = r0["ps"][i]
        wv, wtv, wfb, _, wcoef = full["ps"][i]
        assert fb == wfb
        assert v_r == pytest.approx(wv, rel=1e-12, abs=1e-12) and tv_r == pytest.approx(wtv, rel=1e-12, abs=1e-12)
        assert np.array_equal(coef, r1["ps"][i][4])
        assert np.abs(coef - wcoef).max() <= 1e-9 * np.abs(wcoef).max()
        np.testing.assert_allclose(r0["conc"][i][3], full["conc"][i][3], rtol=1e-12, atol=1e-12)
    for k in ("NumTrajs", "MaxReturn", "MinReturn"):
        assert r0["rec"][k] == full["rec"][k], k
    for k in ("ExplainedVariance", "AverageReturn", "StdReturn", "AverageDiscountedReturn"):
        assert r0["rec"][k] == pytest.approx(full["rec"][k], rel=1e-12), k
    _bits_equal(r0["eval_ww"], full["eval_ww"], "eval_ww")
    _bits_equal(r0["eval_pe"], full["eval_pe"], "eval_pe")


def test_two_gloo_ranks_on_one_gpu_pool_to_the_unsharded_batch():
    got = _run_two("gloo")
    _check_sharded(got, compute("cuda:0", None))


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_two_nccl_ranks_pool_to_the_unsharded_batch():
    got = _run_two("nccl")
    _check_sharded(got, compute("cuda:0", None))
