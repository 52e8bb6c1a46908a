"""ReplayPool's kernels against the same work composed from PyTorch operations (one GPU command).

    python scripts/replay_rate.py [--rounds R] [--reps N] [--only c2 c5] [--out FILE]

Shapes: Waterworld C2 (4096 envs x 5 pursuers, D = 213, T = 256) and Hostage C5 (8192 envs x 10 rescuers, T = 64)
at the runner's DDPG defaults: replay_pool_size = 500 000, batch_size = 12 000.  The rollout tensors are synthetic
(random rows, 1 % done steps, no horizon cut), so every transition is kept and one add keeps far more than the pool
holds: only the last 500 000 land, as in a DDPG loop fed by whole rollouts.
  * add: ReplayPool.add (plan, scan, insert) against cumsum compaction + index_select / index_copy_ of the landing
    rows (the composition needs a host read for the number of landing rows);
  * sample: ReplayPool.random_batches(n, B) at B = 12 000 and 100 000, n = 1 and 8, against randint + index_select
    of the five arrays.
Variants alternate round by round, N calls per round, timed with CUDA events; reported: the median ms per call, the
spread over rounds, the algorithmic bytes computed from the shapes (each source row read once, plus the writes) and
bytes / time as a share of the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the
same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
HBM = 3.35e12
M = 500000
SHAPES = {"c2": ("waterworld", 256), "c5": ("hostage", 64)}


def card():
    import torch
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            stdout=subprocess.PIPE, text=True).stdout.strip()
    except OSError:
        pl = "unknown"
    return dict(name=torch.cuda.get_device_name(0), power_limit=pl)


def timed(fns, rounds, reps):
    """{name: (median ms per call, min, max over rounds)}, the variants alternating round by round."""
    import numpy as np
    import torch
    per = {k: [] for k in fns}
    for f in fns.values():   # warm-up: every shape, allocations, lazy initialisation
        f()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, f in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(reps):
                f()
            b.record()
            b.synchronize()
            per[k].append(a.elapsed_time(b) / reps)
    return {k: (float(np.median(v)), float(min(v)), float(max(v))) for k, v in per.items()}


def torch_add(pool, obs, act, rew, done, obs_before, term, scale):
    """The add composed from PyTorch operations: the same landing rows at the same slots."""
    import torch
    T, E, A, D = obs.shape
    EA = E * A
    Mp = pool.max_pool_size
    keep = done.new_ones(done.shape, dtype=torch.bool)   # no horizon cut in this workload
    keep_a = keep[:, :, None].expand(T, E, A).reshape(-1)
    pos = torch.cumsum(keep_a, 0) - 1
    K = pos[-1] + 1
    land = keep_a & (pos >= K - Mp)
    rows = land.nonzero().squeeze(1)                       # host read
    top = pool._ctl[0].clone()
    slots = (top + pos.index_select(0, rows)) % Mp
    of, tf = obs.view(-1, D), term.view(-1, D)
    prev = of.index_select(0, (rows - EA).clamp(min=0))
    first = rows < EA
    prev[first] = obs_before.view(-1, D).index_select(0, rows[first])
    d = done[:, :, None].expand(T, E, A).reshape(-1).index_select(0, rows).bool()
    nxt = torch.where(d[:, None], tf.index_select(0, rows), of.index_select(0, rows))
    pool.observations.index_copy_(0, slots, prev)
    pool.next_observations.index_copy_(0, slots, nxt)
    pool.actions.index_copy_(0, slots, act.view(-1, act.shape[-1]).index_select(0, rows))
    pool.rewards.index_copy_(0, slots, (rew.view(-1).index_select(0, rows).double() * scale).float())
    pool.terminals.index_copy_(0, slots, d.to(torch.uint8))
    size = pool._ctl[2].clone()
    pool._ctl[0] = (top + K) % Mp
    pool._ctl[1] = (pool._ctl[1] + (size + K - Mp).clamp(min=0)) % Mp
    pool._ctl[2] = (size + K).clamp(max=Mp)


def torch_sample(pool, n, B, gen):
    import torch
    idx = torch.randint(0, M - 1, (n * B,), device=pool.device, generator=gen)
    return [t.index_select(0, idx) for t in (pool.observations, pool.next_observations, pool.actions, pool.rewards,
                                             pool.terminals)]


def run_shape(name, rounds, reps):
    import bench
    import torch
    from madrl_b200 import ReplayPool
    wl, T = SHAPES[name]
    w = bench.WORKLOADS[wl]
    E, A = w["envs"], w["agents"]
    D = bench.make_engine(wl, 8, "cuda", 0).obs_dim
    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev).manual_seed(0)
    obs = torch.randn((T, E, A, D), device=dev, generator=g)
    term = torch.randn((T, E, A, D), device=dev, generator=g)
    act = torch.randn((T, E, A, 2), device=dev, generator=g)
    rew = torch.randn((T, E, A), device=dev, generator=g)
    done = (torch.rand((T, E), device=dev, generator=g) < 0.01).to(torch.uint8)
    obs_before = torch.randn((E, A, D), device=dev, generator=g)
    z = torch.zeros(E, dtype=torch.int32, device=dev)
    pools = [ReplayPool(M, A, D, 2, dev, scale_reward=0.01, seed=1) for _ in range(2)]
    fns = {"cuda_add": lambda: pools[0].add(obs, act, rew, done, obs_before, term, z, z, 0, 10 ** 9),
           "torch_add": lambda: torch_add(pools[1], obs, act, rew, done, obs_before, term, 0.01)}
    res = timed(fns, rounds, reps)
    torch.cuda.synchronize()
    same = all(torch.equal(getattr(pools[0], k), getattr(pools[1], k))
               for k in ("observations", "next_observations", "actions", "rewards", "terminals"))
    s = 4
    add_bytes = (M + E * A) * D * s + 2 * M * D * s + M * 2 * (2 * 4 + 4) + M + T * E
    out = dict(shape=name, E=E, A=A, D=D, T=T, pool=M, transitions=T * E * A, same_pool_contents=same,
               add_bytes=add_bytes)
    for k, (med, lo, hi) in res.items():
        out[k] = dict(ms=round(med, 4), min=round(lo, 4), max=round(hi, 4),
                      hbm_share=round(add_bytes / (med * 1e-3) / HBM, 3))
    del obs, term
    torch.cuda.empty_cache()
    sample = {}
    for n, B in ((1, 12000), (8, 12000), (1, 100000)):
        sg = torch.Generator(device=dev).manual_seed(1)
        fns = {"cuda": lambda: pools[0].random_batches(n, B), "torch": lambda: torch_sample(pools[1], n, B, sg)}
        r = timed(fns, rounds, reps)
        b = n * B * (2 * (2 * D * s + 2 * 4 + 4 + 1) + 8)
        sample["n%d_B%d" % (n, B)] = {k: dict(ms=round(m, 4), min=round(lo, 4), max=round(hi, 4),
                                              hbm_share=round(b / (m * 1e-3) / HBM, 3)) for k, (m, lo, hi) in r.items()}
        sample["n%d_B%d" % (n, B)]["bytes"] = b
    out["sample"] = sample
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--only", nargs="*", default=list(SHAPES))
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("replay_rate.py measures on a CUDA device; none is visible")
    res = dict(card=card(), shapes=[run_shape(n, a.rounds, a.reps) for n in a.only])
    js = json.dumps(res, indent=1)
    print(js)
    if a.out:
        with open(a.out, "w") as f:
            f.write(js + "\n")


if __name__ == "__main__":
    main()
