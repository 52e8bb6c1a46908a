"""Waterworld launch geometry across batch sizes (one GPU command).

    python scripts/ww_launch_cap.py [--shapes c2,c4] [--envs E1,E2,...] [--steps T1,T2,...] [--rounds R] [--reps N]

Prints the card (name, power limit, SM clock), then, for the C2 (5 pursuers, T = 256) and C4 (20 pursuers,
T = 64) configs at each batch size E, times with CUDA events (median of N launches) a launch of each length
in --steps (default: the config's T, and 1) with the persistent wave at as many one-warp blocks per SM as fit
(set_launch(blocks_per_sm=32)) and at 16.  The two settings alternate within the process for R rounds; the
median over the rounds and the min-max spread are printed, and the ratio 16 / as many as fit.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from ww_write_path import card, event_ms  # noqa: E402  (same directory)

SHAPES = {"c2": (dict(n_pursuers=5, n_evaders=5, n_poison=10, n_sensors=30), 256),
          "c4": (dict(n_pursuers=20, n_evaders=50, n_poison=50, n_sensors=30), 64)}
SETTINGS = (32, 16)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c2,c4")
    ap.add_argument("--envs", default="2200,2640,3000,4096,6000,8192")
    ap.add_argument("--steps", default="", help="launch lengths (default: the config's T, and 1)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    a = ap.parse_args()
    import torch
    from madrl_b200 import BatchedMAWaterWorld
    if not torch.cuda.is_available():
        raise SystemExit("ww_launch_cap.py needs a CUDA device")
    print("card:", json.dumps(card()))
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    for name in a.shapes.split(","):
        cfg, T = SHAPES[name]
        Ts = [int(x) for x in a.steps.split(",")] if a.steps else [T, 1]
        for E in [int(x) for x in a.envs.split(",")]:
            eng = BatchedMAWaterWorld(E, device="cuda", seed=0, **cfg)
            eng.reset()
            Np, D = cfg["n_pursuers"], eng.obs_dim
            g = torch.Generator(device="cuda")
            g.manual_seed(1234)
            act = torch.randn(max(Ts), E, Np, 2, device="cuda", generator=g) * 0.5
            bufs = lambda t: (torch.empty((t, E, Np, D), device="cuda"), torch.empty((t, E, Np), device="cuda"),  # noqa: E731
                              torch.empty((t, E), dtype=torch.uint8, device="cuda"),
                              torch.empty((t, E, 2), dtype=torch.int32, device="cuda"))
            runs = {t: (act[:t].contiguous(), bufs(t)) for t in Ts}
            res = {(t, b): [] for t in Ts for b in SETTINGS}
            for _ in range(a.rounds):
                for b in SETTINGS:
                    eng.set_launch(blocks_per_sm=b)
                    for t, (at, out) in runs.items():
                        res[t, b].append(event_ms(lambda: eng.rollout(at, auto_reset=True, out=out), 3,
                                                  max(a.reps, a.reps * 64 // t)))
            del runs, act, eng
            torch.cuda.empty_cache()
            for t in Ts:
                med = {}
                txt = []
                for b in SETTINGS:
                    v = sorted(res[t, b])
                    med[b] = v[len(v) // 2]
                    txt.append("%s %.4f ms (spread %.1f%%)" % ("fit" if b == 32 else "16", med[b],
                                                              100 * (v[-1] - v[0]) / med[b]))
                print("%s E=%5d (%.2f envs per SM) T=%3d: %s; 16/fit = %.3f"
                      % (name, E, E / sms, t, ", ".join(txt), med[16] / med[32]), flush=True)


if __name__ == "__main__":
    main()
