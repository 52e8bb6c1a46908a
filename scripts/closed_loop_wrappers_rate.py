"""Closed-loop rollouts with the observation wrappers (PolicyRollout's frame_stack= / standardizer=) on bench.py's
workloads, and the per-step wrapper kernel against the two whole-trajectory passes it fuses (one GPU command).

    python scripts/closed_loop_wrappers_rate.py [--rounds R] [--reps N] [--launches L] [--only NAME ...] [--out FILE]

Shapes: Waterworld C2, Pursuit C3 and Hostage C5 at bench.py's env counts, T = 256 / 16 / 64, with the policies of
scripts/closed_loop_rate.py over the flattened stack [E, A, D * B].  For each shape:
  * rollout variants, each on an engine of its own built from the same seed, run alternately round by round, N calls
    per round timed with a host clock around work that ends in a device synchronise: no wrappers, B = 4, obsnorm,
    and B = 4 with obsnorm.  Reported: median ms per PolicyRollout call and the spread over the rounds.
  * kernel variants on one step's inputs (the rows, terminal rows and done flags of a real rollout step), L launches
    per round timed with CUDA events, alternated round by round: the fused madrl_obs_wrap_step_* (B = 4, with and
    without obsnorm) against madrl_standardize_obs_terminal_* + madrl_frame_stack_* at T = 1 (and frame_stack alone
    without obsnorm).  Reported: median us per step, the spread, the bytes per step computed from the shapes, and
    that over the time as a fraction of the H100 SXM data sheet's 3.35 TB/s.
The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))
SHAPES = {"c2": ("waterworld", 256), "c3": ("pursuit", 16), "c5": ("hostage", 64)}
ROLLOUTS = {"none": (1, False), "stack4": (4, False), "obsnorm": (1, True), "stack4_obsnorm": (4, True)}
B = 4
HBM = 3.35e12


def kernel_bytes(n, s, obsnorm, fused):
    """Bytes one step moves (n elements of s bytes, B = 4), the terminal rows of done envs aside."""
    stats = 32 if obsnorm else 0                       # float64 mean and var, read and written
    if fused:
        return n * ((2 * s if obsnorm else s) + stats + 2 * B * s)          # obs (+ write-back), prev, out
    std = n * (2 * s + stats) if obsnorm else 0
    return std + n * (s + 3 * B * s)                   # frame_stack: obs, carry read and written, out


def run_shape(name, rounds, reps, launches):
    import bench
    import numpy as np
    import torch
    from closed_loop_rate import CategoricalMLP, GaussianMLP, timed
    from madrl_b200 import _lib
    from madrl_b200._lib import _ptr
    from madrl_b200.closed_loop import PolicyRollout
    from madrl_b200.postproc import FrameStack, Standardizer
    wl, T = SHAPES[name]
    w = bench.WORKLOADS[wl]
    E, A = w["envs"], w["agents"]
    pe = w["family"] == "pe"
    engs = {v: bench.make_engine(wl, E, "cuda", 0) for v in ROLLOUTS}
    D = engs["none"].obs_dim
    ros, obs0 = {}, {}
    for v, (b, obsnorm) in ROLLOUTS.items():
        eng = engs[v]
        pol = (CategoricalMLP if pe else GaussianMLP)(D * b, 5 if pe else 2)
        flat = (lambda p: lambda o, s: p(o.reshape(E, A, -1), s))(pol)
        std = Standardizer(E, A, D, "cuda", enable_obsnorm=True) if obsnorm else None
        o = eng.reset()
        if std is not None:
            std.obs(o)
        obs0[v] = FrameStack(E, A, D, b, "cuda", eng.obs_dtype).reset(o) if b > 1 else o
        ros[v] = PolicyRollout(eng, flat, T, frame_stack=b, standardizer=std)

    def rollout(v):
        def go():
            obs0[v] = ros[v](obs0[v]).policy_obs[-1].clone()
        return go

    fns = {v: rollout(v) for v in ROLLOUTS}
    first = {}
    for v in ROLLOUTS:                                 # capture and warm-up
        first[v] = timed(fns[v], 1)
        timed(fns[v], 1)
    per = {v: [] for v in ROLLOUTS}
    for _ in range(rounds):
        for v in ROLLOUTS:
            per[v].append(timed(fns[v], reps))
    res = dict(rollout_ms={})
    for v in ROLLOUTS:
        res["rollout_ms"][v] = dict(median=round(float(np.median(per[v])), 4), min=round(min(per[v]), 4),
                                    max=round(max(per[v]), 4), first_call=round(first[v], 1))

    # one real step's inputs: the rows and done flags of the last step of the stack4_obsnorm rollout; terminal rows
    # from a one-step open-loop launch with set_terminal_obs
    eng = engs["none"]
    term = torch.zeros((1, E, A, D), device="cuda")
    eng.set_terminal_obs(term)
    step = eng.rollout(torch.zeros((1, E, A) + eng._act_tail, dtype=eng._act_dtype, device="cuda"))
    eng.set_terminal_obs(None)
    done = ros["stack4_obsnorm"]._traj[2][-1].clone()
    x = step[0][0].contiguous()
    t1 = term[0].contiguous()
    mean = torch.zeros((E, A, D), dtype=torch.float64, device="cuda")
    var = torch.ones_like(mean)
    bufs = [torch.zeros((E, A, D, B), device="cuda") for _ in range(2)]
    L = _lib.lib()
    st = _lib.stream(torch.device("cuda", torch.cuda.current_device()))
    flip = [0]

    def fused(obsnorm):
        def go():
            p, o = bufs[flip[0]], bufs[1 - flip[0]]
            flip[0] ^= 1
            _lib.check(L.madrl_obs_wrap_step_f32(E, A, D, B, _ptr(x), _ptr(t1), _ptr(done), _ptr(p), _ptr(o),
                                                 _ptr(mean if obsnorm else None), _ptr(var if obsnorm else None),
                                                 0.001, 1e-8, st))
        return go

    def composed(obsnorm):
        def go():
            if obsnorm:
                _lib.check(L.madrl_standardize_obs_terminal_f32(1, E, A * D, _ptr(x), _ptr(t1), _ptr(done), _ptr(mean),
                                                                _ptr(var), 0.001, 1e-8, st))
            _lib.check(L.madrl_frame_stack_f32(1, E, A, D, B, _ptr(x), _ptr(done), _ptr(bufs[0]), _ptr(bufs[1]), st))
        return go

    kfns = {"fused_obsnorm": (fused(True), True, True), "composed_obsnorm": (composed(True), True, False),
            "fused_stack": (fused(False), False, True), "composed_stack": (composed(False), False, False)}

    def events(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) * 1e3 / launches

    for fn, _, _ in kfns.values():
        events(fn)
    kper = {k: [] for k in kfns}
    for _ in range(rounds):
        for k, (fn, _, _) in kfns.items():
            kper[k].append(events(fn))
    res["kernel_us"] = {}
    n = E * A * D
    for k, (_, obsnorm, is_fused) in kfns.items():
        us = float(np.median(kper[k]))
        nb = kernel_bytes(n, 4, obsnorm, is_fused)
        res["kernel_us"][k] = dict(median=round(us, 2), min=round(min(kper[k]), 2), max=round(max(kper[k]), 2),
                                   bytes_per_step=nb, bytes_per_elem=nb // n,
                                   hbm_fraction=round(nb / (us * 1e-6) / HBM, 3))
    return dict(shape=name, workload=wl, envs=E, agents=A, obs_dim=D, T=T, elems_per_step=n, **res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--only", nargs="*", default=sorted(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("closed_loop_wrappers_rate.py needs a CUDA device")
    from closed_loop_rate import card
    report = dict(card=card(), torch=torch.__version__, rounds=args.rounds, reps=args.reps, launches=args.launches,
                  shapes=[])
    print(json.dumps(report["card"]), flush=True)
    t0 = time.time()
    for name in args.only:
        r = run_shape(name, args.rounds, args.reps, args.launches)
        report["shapes"].append(r)
        print("%s (%s, %d envs x %d agents x %d dims, T=%d)" % (name, r["workload"], r["envs"], r["agents"],
                                                                 r["obs_dim"], r["T"]))
        for v, x in r["rollout_ms"].items():
            print("  rollout %-16s %9.3f ms [%9.3f, %9.3f]" % (v, x["median"], x["min"], x["max"]))
        for k, x in r["kernel_us"].items():
            print("  kernel  %-16s %9.2f us [%9.2f, %9.2f]  %3d B/elem  %.2f of 3.35 TB/s" % (
                k, x["median"], x["min"], x["max"], x["bytes_per_elem"], x["hbm_fraction"]), flush=True)
        torch.cuda.empty_cache()
    print("total %.0f s" % (time.time() - t0))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
