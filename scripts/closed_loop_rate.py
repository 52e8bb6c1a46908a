"""Closed-loop rollouts with a learned-policy shape on bench.py's workloads (one GPU command).

    python scripts/closed_loop_rate.py [--rounds R] [--reps N] [--only NAME ...] [--out FILE]

The policy is rllab's default GaussianMLPPolicy shape: one tanh hidden layer of 32 and a learned, state-independent
log_std, sampled with torch.randn (Pursuit: a categorical MLP policy with one tanh hidden layer of 32, sampled by
Gumbel-max).  Shapes: Waterworld C2, Pursuit C3 and Hostage C5 at bench.py's env counts, T = 256 / 16 / 64.

For each shape the variants below run alternately, round by round, each on an engine of its own built from the same
seed, and each round times N calls with a host clock around work that ends in a device synchronise:
  * eager_step       the Python loop a caller writes today: BatchedEngine.step + the policy per step, the per-step
                     outputs stacked at the end;
  * eager_rollout    PolicyRollout(graph=False): the same loop into fixed buffers;
  * graph_stream     PolicyRollout, one CUDA graph, observations stored evict-first (MADRL_OBS_CACHE_STREAM);
  * graph_keep       PolicyRollout, one CUDA graph, observations stored at normal L2 priority (MADRL_OBS_CACHE_KEEP);
  * open_loop        for reference: one rollout() launch of T steps with precomputed actions (no policy);
  * heuristic        for reference: rollout_heuristic, the hand-written policy inside the kernel (not Hostage).
Reported per variant: median ms per T-step rollout over the rounds, the spread (min and max of the round medians),
agent-env-steps/s at the median, and for the graph variants the time of the first call (side-stream warm-up,
capture and the first replay).  The card's name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
SHAPES = {"c2": ("waterworld", 256), "c3": ("pursuit", 16), "c5": ("hostage", 64)}
VARIANTS = ("eager_step", "eager_rollout", "graph_stream", "graph_keep", "open_loop", "heuristic")


def card():
    import torch
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(), "power.limit": "unknown"}


class GaussianMLP(object):
    """rllab's GaussianMLPPolicy(hidden_sizes=(32,), tanh) forward pass and sample."""

    def __init__(self, D, n_act, seed=0):
        import torch
        g = torch.Generator().manual_seed(seed)
        self.W1 = (torch.randn(D, 32, generator=g) / D ** 0.5).cuda()
        self.b1 = torch.zeros(32).cuda()
        self.W2 = (torch.randn(32, n_act, generator=g) * 0.1).cuda()
        self.b2 = torch.zeros(n_act).cuda()
        self.log_std = torch.zeros(n_act).cuda()

    def __call__(self, obs, state):
        import torch
        mean = torch.tanh(obs.float() @ self.W1 + self.b1) @ self.W2 + self.b2
        log_std = self.log_std.expand_as(mean)
        return mean + torch.randn_like(mean) * log_std.exp(), {"mean": mean, "log_std": log_std}, state


class CategoricalMLP(GaussianMLP):
    """rllab's CategoricalMLPPolicy(hidden_sizes=(32,), tanh): softmax probabilities, one sample per agent."""

    def __call__(self, obs, state):
        import torch
        logits = torch.tanh(obs.float() @ self.W1 + self.b1) @ self.W2 + self.b2
        u = torch.rand_like(logits).clamp_(min=1e-20)
        return (logits - torch.log(-torch.log(u))).argmax(-1), {"prob": torch.softmax(logits, -1)}, state


def timed(fn, reps):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / reps


def run_shape(name, rounds, reps):
    import bench
    import numpy as np
    import torch
    from madrl_b200 import _lib
    from madrl_b200.closed_loop import PolicyRollout
    wl, T = SHAPES[name]
    w = bench.WORKLOADS[wl]
    E, A = w["envs"], w["agents"]
    pe = w["family"] == "pe"
    variants = [v for v in VARIANTS if not (v == "heuristic" and w["family"] == "hw")]
    engs = {v: bench.make_engine(wl, E, "cuda", 0) for v in variants}
    pol = (CategoricalMLP if pe else GaussianMLP)(engs[variants[0]].obs_dim, 5 if pe else 2)
    obs0 = {v: e.reset() for v, e in engs.items()}
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    act = bench.make_actions(wl, T, E, "cuda", g)

    def eager_step():
        eng, prev = engs["eager_step"], obs0["eager_step"]
        steps = []
        for _ in range(T):
            a, _, _ = pol(prev, None)
            o, r, d, info = eng.step(a, auto_reset=True)
            steps.append((a, o, r, d, info))
            prev = o
        obs0["eager_step"] = prev
        return [torch.stack([s[i] for s in steps]) for i in range(4)]

    ros = {"eager_rollout": PolicyRollout(engs["eager_rollout"], pol, T, graph=False),
           "graph_stream": PolicyRollout(engs["graph_stream"], pol, T, obs_cache=_lib.OBS_CACHE_STREAM),
           "graph_keep": PolicyRollout(engs["graph_keep"], pol, T, obs_cache=_lib.OBS_CACHE_KEEP)}

    def policy_rollout(v):
        def go():
            out = ros[v](obs0[v])
            obs0[v] = out.obs[-1].clone()
        return go

    bufs = engs["open_loop"]._outputs(T, None, True)
    heur = engs["heuristic"]._outputs(T, None, True) if "heuristic" in engs else None
    fns = {"eager_step": eager_step, "open_loop": lambda: engs["open_loop"].rollout(act, out=bufs)}
    for v in ros:
        fns[v] = policy_rollout(v)
    if heur is not None:
        def heuristic():
            engs["heuristic"].rollout_heuristic(T, obs0["heuristic"], out=heur, record_actions=False)
            obs0["heuristic"] = heur[0][-1].clone()
        fns["heuristic"] = heuristic
    first = {}
    for v in variants:   # warm-up; the graph variants capture here
        first[v] = timed(fns[v], 1)
        timed(fns[v], 1)
    per = {v: [] for v in variants}
    for _ in range(rounds):
        for v in variants:
            per[v].append(timed(fns[v], reps))
    res = {}
    for v in variants:
        ms = float(np.median(per[v]))
        res[v] = dict(ms_median=round(ms, 4), ms_min=round(min(per[v]), 4), ms_max=round(max(per[v]), 4),
                      agent_env_steps_per_s=round(T * E * A / (ms * 1e-3)))
        if v in ros and ros[v].graph:
            res[v]["first_call_ms"] = round(first[v], 1)
    return dict(shape=name, workload=wl, envs=E, agents=A, T=T, obs_dim=engs[variants[0]].obs_dim, variants=res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--only", nargs="*", default=sorted(SHAPES))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("closed_loop_rate.py needs a CUDA device")
    report = dict(card=card(), torch=torch.__version__, rounds=args.rounds, reps=args.reps, shapes=[])
    print(json.dumps(report["card"]), flush=True)
    for name in args.only:
        r = run_shape(name, args.rounds, args.reps)
        report["shapes"].append(r)
        print("%s (%s, %d envs x %d agents, T=%d)" % (name, r["workload"], r["envs"], r["agents"], r["T"]))
        for v, x in r["variants"].items():
            print("  %-14s %9.3f ms [%9.3f, %9.3f]  %.3g agent-env-steps/s%s" % (
                v, x["ms_median"], x["ms_min"], x["ms_max"], x["agent_env_steps_per_s"],
                "  first call %.1f ms" % x["first_call_ms"] if "first_call_ms" in x else ""), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(report, f, indent=1)


if __name__ == "__main__":
    main()
