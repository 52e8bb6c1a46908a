"""What pooling over the ranks of a sharded batch (``group=``) adds to sample processing and evaluation, on one GPU.

At the C2 (Waterworld 4096 x 256 x 5) and C5 (Hostage 8192 x 64 x 10) rollout shapes of
scripts/linear_baseline_rate.py, each call is timed with ``group=None`` and with a one-rank gloo group, alternating,
over the same rollout:

  * rltools' ``process_samples`` (decentralized, obsnorm baseline, reward normaliser);
  * rllab's ``process_samples_concurrent`` (per-agent baseline, centring);
  * ``path_statistics`` (decentralized);
  * ``evaluate_heuristic`` (C2 only: Hostage has no heuristic policy), 100 episodes of at most 100 steps.

A one-rank group exchanges nothing (the pooling helpers return the partial itself), so the added time is the split
passes and the host-side combination, not collective latency.  The partial bytes each rank would send per call are
counted from the pooled tensors; with W ranks each receives W times that.  Multi-GPU collective time is not
measured here.

    python scripts/sharded_samples_rate.py [--rounds 5] [--reps 3] [--out FILE]
"""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from linear_baseline_rate import card, make, timed  # noqa: E402


class ByteCount(object):
    """Counts the bytes of every partial handed to the pooling helpers (what one rank contributes)."""

    def __init__(self):
        import madrl_b200.dist as md
        from madrl_b200 import rltools_sampler as rs
        self.n = 0
        pool, cat = md._pool, md.pool_cat

        def counted_pool(t, group, combine):
            self.n += t.numel() * t.element_size()
            return pool(t, group, combine)

        def counted_cat(t, group):
            self.n += t.numel() * t.element_size()
            return cat(t, group)
        md._pool, md.pool_cat, rs.pool_cat = counted_pool, counted_cat, counted_cat

    def of(self, fn):
        self.n = 0
        fn()
        torch.cuda.synchronize()
        return self.n


def rollout(shape):
    eng, T = make(shape)
    obs0 = eng.reset()
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    act_shape = (T, eng.n_envs, eng._n_acting) + eng._act_tail
    if eng._act_dtype == torch.int32:
        act = torch.randint(0, 5, act_shape, dtype=torch.int32, device="cuda", generator=g)
    else:
        act = torch.randn(act_shape, device="cuda", generator=g) * 0.5
    obs, rew, done, _ = eng.rollout(act)
    del eng
    T, E, A = rew.shape
    return obs.reshape(T, E, A, -1).float().contiguous(), obs0.reshape(E, A, -1).float().contiguous(), rew, done


def calls(shape):
    """{name: fn(kw)} over one rollout of `shape`; kw is {} or {"group": g}."""
    from madrl_b200 import BatchedMAWaterWorld, evaluate_heuristic
    from madrl_b200 import postproc as pp
    from madrl_b200 import rltools_sampler as rs
    from madrl_b200.dist import make_sharded
    obs, obs0, rew, done = rollout(shape)
    T, E, A, D = obs.shape
    bl, rn = rs.LinearFeatureBaseline(D, "cuda", True), rs.RunningStandardizer(1, "cuda")
    bl.update_obsnorm(obs, obs0)
    rn.update(rew.unsqueeze(-1))
    cb = pp.LinearFeatureBaseline(D, "cuda", n_agents=A)
    q = pp.gae(rew, torch.zeros_like(rew), done, 0.99, 1.0)[1]
    out = dict(
        rltools_process_samples=lambda kw: rs.process_samples(bl, obs, done, rew, 0.99, 0.97, rewnorm=rn,
                                                              obs_before=obs0, **kw),
        rllab_process_samples_concurrent=lambda kw: pp.process_samples_concurrent(cb, obs, done, rew, 0.99, 0.97,
                                                                                  obs_before=obs0, **kw),
        path_statistics=lambda kw: pp.path_statistics(rew, q, done, **kw))
    if shape == "C2":
        eng = make_sharded(BatchedMAWaterWorld, 4096, 5, 5, rank=0, world=1, seed=0, device="cuda",
                           max_path_length=100, n_poison=10, n_sensors=30)
        out["evaluate_heuristic"] = lambda kw: evaluate_heuristic(eng, 100, 0.99, "decentralized", **kw)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="C2,C5")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: nothing to measure")
    dist.init_process_group("gloo", store=dist.HashStore(), rank=0, world_size=1)
    try:
        counter = ByteCount()
        name, limits = card()
        res = dict(gpu=name, power_limit_and_max_sm_clock=limits, rounds=args.rounds, reps=args.reps, calls={})
        for shape in args.shapes.split(","):
            for call, fn in calls(shape).items():
                variants = {"none": {}, "one_rank_group": dict(group=dist.group.WORLD)}
                for kw in variants.values():
                    fn(kw)                                            # warm-up: modules, allocator
                times = {k: [] for k in variants}
                for _ in range(args.rounds):                          # alternate, so drift hits both alike
                    for k, kw in variants.items():
                        times[k].append(timed(lambda: fn(kw), args.reps)[0])
                med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
                spread = {k: (max(v) - min(v)) / med[k] for k, v in times.items()}
                row = dict(ms_none=med["none"] * 1e3, ms_one_rank_group=med["one_rank_group"] * 1e3,
                           added_ms=(med["one_rank_group"] - med["none"]) * 1e3,
                           spread_none=spread["none"], spread_group=spread["one_rank_group"],
                           partial_bytes_per_rank=counter.of(lambda: fn(variants["one_rank_group"])))
                res["calls"]["%s %s" % (shape, call)] = row
                print("%s %-34s none %8.3f ms  group %8.3f ms  added %+7.3f ms  partials %7d B" % (
                    shape, call, row["ms_none"], row["ms_one_rank_group"], row["added_ms"],
                    row["partial_bytes_per_rank"]), flush=True)
        print(json.dumps(res))
        if args.out:
            with open(args.out, "w") as f:
                json.dump(res, f, indent=1)
    finally:
        dist.destroy_process_group()


if __name__ == "__main__":
    main()
