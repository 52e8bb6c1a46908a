"""Times the whole-path selection across ranks (WholePathSampler with ``group=``, DESIGN §4.9) at C2: Waterworld,
E = 4096 envs, max_path_length 500, batch_size 12000, an MLP policy (64-64 tanh), launches of 64 steps.

One process (``python scripts/whole_paths_sharded_rate.py``):
  * per launch, from CUDA events over many reps of one call's launches: madrl_whole_paths_fold (the unsharded fold)
    against madrl_whole_paths_steps + madrl_whole_paths_fold_pooled as a sharded sampler runs them (steps while t* is
    unknown, the pooled fold on every launch), on the done columns of a real call;
  * the sampler call over 2 gloo ranks that share the one GPU (each rank half the envs) against the unsharded call.
    The ranks exchange through host memory and compete for the same GPU: this is the functional overhead of the
    exchange, not a multi-GPU result.

Under ``torchrun --nproc-per-node N`` (N GPUs, NCCL): the sampler call over the N ranks, one GPU each, E sharded.

Every number is the median over rounds; the card's name and power limit are read in the same run.
Usage:  python scripts/whole_paths_sharded_rate.py [--rounds 5] [--reps 200] [--envs 4096] [--out FILE]
"""
import argparse
import datetime
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from madrl_b200 import BatchedMAWaterWorld, WholePathSampler  # noqa: E402
from madrl_b200 import _lib  # noqa: E402
from madrl_b200._lib import _ptr  # noqa: E402
from madrl_b200.whole_paths import _Selection  # noqa: E402

MPL, CHUNK, BATCH = 500, 64, 12000
WW = dict(n_pursuers=5, n_evaders=5, max_path_length=MPL)


def card(dev_index):
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                           str(dev_index)], capture_output=True, text=True).stdout.strip()


def mlp_policy(eng, dev):
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(eng.obs_dim, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64),
                              torch.nn.Tanh(), torch.nn.Linear(64, 2)).to(dev)
    for p in net.parameters():
        p.requires_grad_(False)

    def policy(o, s):
        m = net(o)
        return torch.tanh(m), {"mean": m}, s
    return policy


def med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def call_ms(sampler, rounds, dev, group=None):
    """The median wall time of a sampler call (every rank of `group` starts each call together)."""
    import torch.distributed as dist
    sampler()                                                        # capture and warm-up
    out = []
    for _ in range(rounds):
        torch.cuda.synchronize(dev)
        if group is not None:
            dist.barrier(group=group)
        t0 = time.perf_counter()
        sampler()
        torch.cuda.synchronize(dev)
        out.append(time.perf_counter() - t0)
    return 1e3 * med(out)


def kernel_times(E, rounds, reps, dev):
    """Per-launch microseconds of the unsharded fold and of steps + pooled fold over one call's launches."""
    eng = BatchedMAWaterWorld(E, device=dev, **WW)
    sampler = WholePathSampler(eng, mlp_policy(eng, dev), BATCH, MPL, chunk=CHUNK)
    sel = _Selection(E, CHUNK, BATCH, sampler.max_steps(), dev)
    obs0 = eng.reset()
    while True:
        r = sampler.loop(obs0, None)
        pobs = r.policy_obs.clone()
        if sel.add(obs0, pobs, r.actions.clone(), r.rew.clone(), r.done, r.info.clone(), {}):
            break
        obs0 = pobs[-1]
    L, n, s = _lib.lib(), len(sel.launches), _lib.stream(dev)
    pooled_launches = int(sel.status[1]) // CHUNK + 1                # the launches a sharded call exchanges in
    carry0 = torch.tensor([-1, -1, 0], dtype=torch.int32, device=dev).repeat_interleave(E)
    acc0 = torch.tensor([0, -1, 0, 0, 0], dtype=torch.int64, device=dev)
    want = (sel.carry.clone(), sel.acc.clone())
    inc = torch.empty(CHUNK, dtype=torch.int64, device=dev)

    def d(j):
        return _ptr(sel.done_stage[j * CHUNK:])

    def fold():
        for j in range(n):
            _lib.check(L.madrl_whole_paths_fold(CHUNK, E, j * CHUNK, BATCH, d(j), _ptr(sel.carry), _ptr(sel.acc), s))

    def pooled():
        for j in range(n):
            if j < pooled_launches:
                _lib.check(L.madrl_whole_paths_steps(CHUNK, E, j * CHUNK, d(j), _ptr(sel.carry), _ptr(inc), s))
            _lib.check(L.madrl_whole_paths_fold_pooled(CHUNK, E, j * CHUNK, BATCH, d(j), _ptr(inc), _ptr(sel.carry),
                                                       _ptr(sel.acc), s))

    def steps_only():
        for j in range(n):
            _lib.check(L.madrl_whole_paths_steps(CHUNK, E, j * CHUNK, d(j), _ptr(carry0), _ptr(inc), s))

    def timed(body):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ts = []
        for _ in range(rounds):
            torch.cuda.synchronize(dev)
            a.record()
            for _ in range(reps):
                sel.carry.copy_(carry0)
                sel.acc.copy_(acc0)
                body()
            b.record()
            torch.cuda.synchronize(dev)
            ts.append(a.elapsed_time(b) * 1e3 / reps / n)
        return med(ts)

    def reset_only():
        pass
    out = dict(launches=n, pooled_launches=pooled_launches, t_star=int(sel.status[1]))
    out["reset_us_per_launch"] = timed(reset_only)                   # the two carry / acc copies per rep
    out["fold_us_per_launch"] = timed(fold)
    assert torch.equal(sel.carry, want[0]) and torch.equal(sel.acc, want[1])
    out["steps_pooled_fold_us_per_launch"] = timed(pooled)
    assert torch.equal(sel.carry, want[0]) and torch.equal(sel.acc[:2], want[1][:2]) and int(sel.acc[2]) == 1
    out["steps_us_per_launch_every_launch"] = timed(steps_only)
    return out


def rank_main(rank, world, port, E, rounds, q):
    import torch.distributed as dist
    from madrl_b200.dist import make_sharded
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world, timeout=datetime.timedelta(seconds=600))
    try:
        eng = make_sharded(BatchedMAWaterWorld, E, rank=rank, world=world, device=dev, **WW)
        sampler = WholePathSampler(eng, mlp_policy(eng, dev), BATCH, MPL, chunk=CHUNK, group=dist.group.WORLD)
        q.put((rank, call_ms(sampler, rounds, dev, dist.group.WORLD)))
    finally:
        dist.destroy_process_group()


def gloo_two_ranks(E, rounds):
    import socket
    import torch.multiprocessing as mp
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=rank_main, args=(r, 2, port, E, rounds, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=1800) for _ in procs)
    finally:
        for p in procs:
            p.join(120)
            if p.is_alive():
                p.kill()
                p.join()
    return max(got.values())


def torchrun_main(args):
    import torch.distributed as dist
    from madrl_b200.dist import make_sharded, world_info
    rank, world, local = world_info()
    dev = torch.device("cuda", local)
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl")
    try:
        eng = make_sharded(BatchedMAWaterWorld, args.envs, rank=rank, world=world, device=dev, **WW)
        sampler = WholePathSampler(eng, mlp_policy(eng, dev), BATCH, MPL, chunk=CHUNK, group=dist.group.WORLD)
        ms = torch.tensor([call_ms(sampler, args.rounds, dev, dist.group.WORLD)], device=dev)
        dist.all_reduce(ms, op=dist.ReduceOp.MAX)
        if rank == 0:
            emit(dict(card=card(local), mode="nccl", ranks=world, E=args.envs, batch_size=BATCH, chunk=CHUNK,
                      sharded_call_ms=float(ms[0])), args.out)
    finally:
        dist.destroy_process_group()


def emit(res, out):
    line = json.dumps(res)
    print(line)
    if out:
        os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
        with open(out, "w") as f:
            f.write(line + "\n")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("whole_paths_sharded_rate needs a CUDA device")
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        return torchrun_main(args)
    dev = torch.device("cuda", 0)
    res = dict(card=card(0), E=args.envs, batch_size=BATCH, chunk=CHUNK)
    res.update(kernel_times(args.envs, args.rounds, args.reps, dev))
    eng = BatchedMAWaterWorld(args.envs, device=dev, **WW)
    res["unsharded_call_ms"] = call_ms(WholePathSampler(eng, mlp_policy(eng, dev), BATCH, MPL, chunk=CHUNK),
                                       args.rounds, dev)
    del eng
    torch.cuda.empty_cache()
    res["gloo_2_ranks_one_gpu_call_ms"] = gloo_two_ranks(args.envs, args.rounds)
    emit(res, args.out)


if __name__ == "__main__":
    main()
