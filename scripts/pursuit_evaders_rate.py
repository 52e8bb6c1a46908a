"""Pursuit C3 with the evaders under a caller's controller (one GPU command).

    python scripts/pursuit_evaders_rate.py [--envs E] [--t T] [--reps N]

Prints the card (name, power limit, SM clock), then:
  * open loop: ms per T-step rollout launch from CUDA events (median over N launches), the random controller
    (the flagship kernel) and the EVC kernel fed an int32 [T, E, Ne] action tensor, one after the other;
  * the same for set_evader_controller(4) (one constant, no action tensor) and for model_state on;
  * closed loop: ms per PolicyRollout call of T steps (CUDA graph replay) with a small pursuer MLP, without and with
    an evader_policy (a linear map of model_state's evader channel to Ne x 5 logits, argmax).
Agent-env-steps/s are pursuers x envs x steps over that time.

Numbers: not measured yet.  Run it on an H100 and record the card and its power limit beside them.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
          catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)


def card():
    import torch
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {}


def timed(fn, reps):
    """Median ms of `fn` over `reps` calls, from CUDA events, after two warm-up calls."""
    import torch
    for _ in range(2):
        fn()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return sorted(ms)[len(ms) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, default=65536)
    ap.add_argument("--t", type=int, default=16)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    import numpy as np
    import torch
    from madrl_b200 import BatchedPursuitEvade, PolicyRollout
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    maps = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
    E, T, Np, Ne = args.envs, args.t, C3["n_pursuers"], C3["n_evaders"]
    dev = torch.device("cuda")
    rate = lambda ms, steps=T: Np * E * steps / (ms * 1e-3)
    out = dict(card=card(), envs=E, t=T, config="C3")

    eng = BatchedPursuitEvade(E, maps, device=dev, seed=1, **C3)
    eng.reset()
    act = torch.randint(0, 5, (T, E, Np), dtype=torch.int32, device=dev)
    ev = torch.randint(0, 5, (T, E, Ne), dtype=torch.int32, device=dev)
    bufs = eng._outputs(T, None, True)
    res = {}
    for name, kw in (("random", {}), ("evc_tensor", dict(evader_actions=ev))):
        res[name] = timed(lambda: eng.rollout(act, out=bufs, **kw), args.reps)
    eng.set_evader_controller(4)
    res["evc_fixed"] = timed(lambda: eng.rollout(act, out=bufs), args.reps)
    eng.set_evader_controller(None)
    eng.set_model_state(torch.zeros((E, 4, 16, 16), device=dev))
    res["random_model_state"] = timed(lambda: eng.rollout(act, out=bufs), args.reps)
    out["open_loop_ms"] = res
    out["open_loop_agent_steps_per_s"] = {k: rate(v) for k, v in res.items()}

    D = eng.obs_dim
    pol = torch.nn.Sequential(torch.nn.Linear(D, 64), torch.nn.Tanh(), torch.nn.Linear(64, 5)).to(dev)
    evnet = torch.nn.Linear(16 * 16, Ne * 5).to(dev)

    def policy(obs, state):
        with torch.no_grad():
            return pol(obs).argmax(-1), {}, state

    def ev_policy(ms):
        with torch.no_grad():
            return evnet(ms[:, 2].flatten(1)).view(-1, Ne, 5).argmax(-1)

    closed = {}
    for name, evp in (("pursuers_only", None), ("with_evader_policy", ev_policy)):
        obs0 = eng.reset()
        loop = PolicyRollout(eng, policy, T, evader_policy=evp)
        closed[name] = timed(lambda: loop(obs0), args.reps)
    out["closed_loop_ms"] = closed
    out["closed_loop_agent_steps_per_s"] = {k: rate(v) for k, v in closed.items()}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
