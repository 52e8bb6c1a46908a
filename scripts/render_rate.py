"""Times the frame kernels (render_frames, csrc/render.cu) on one GPU against the host path:

  * Waterworld C2 and C4 and Hostage C5 at 800 x 800, Pursuit C3 (16 x 16 maps) at cell 16, for K = 1, 16 and 256
    envs per call, on engines stepped 200 steps with random actions: frames per second and GB/s of frames written,
    from CUDA events around back-to-back calls into one out= tensor;
  * the host path for K = 1: read the state back, draw the frame with the NumPy oracle (oracle/render_oracle.py):
    frames per second of the wall clock.

Every number is the median over rounds; the card's name and power limit are read in the same run.
Usage:  python scripts/render_rate.py [--rounds 5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade  # noqa: E402
from oracle import render_oracle as R  # noqa: E402

KS = (1, 16, 256)


def make(name, dev):
    if name == "ww_c2":
        eng = BatchedMAWaterWorld(4096, n_pursuers=5, n_evaders=5, device=dev)
    elif name == "ww_c4":
        eng = BatchedMAWaterWorld(4096, n_pursuers=20, n_evaders=50, n_poison=50, device=dev)
    elif name == "hw_c5":
        eng = BatchedHostageWorld(8192, 10, 16, 16, 4, 2, device=dev)
    else:
        eng = BatchedPursuitEvade(65536, np.load(os.path.join(ROOT, "maps", "map_pool16.npy")), n_evaders=30,
                                  n_pursuers=8, obs_range=7, surround=True, sample_maps=True, device=dev)
    g = torch.Generator(device=dev).manual_seed(0)
    E, A = eng.n_envs, eng._n_acting
    eng.reset()
    for _ in range(4):   # 200 steps in launches of 50
        if name == "pe_c3":
            act = torch.randint(0, 5, (50, E, A), generator=g, device=dev, dtype=torch.int32)
        else:
            act = torch.randn((50, E, A, 2), generator=g, device=dev)
        eng.rollout(act)
    torch.cuda.synchronize()
    return eng


def draw_fn(name, eng):
    if name == "pe_c3":
        return lambda ids, out=None: eng.render_frames(ids, cell=16, out=out)
    return lambda ids, out=None: eng.render_frames(ids, screen_size=800, out=out)


def host_frame(name, eng, e):
    st = {k: v.cpu() for k, v in eng.state.items()}   # the read-back is part of the host path
    if name == "pe_c3":
        return R.pe_frames(st, eng.map_pool, [e], eng.obs_range, 16)
    if name == "hw_c5":
        return R.hw_frames(st, [e], 800, eng.cfg)
    return R.ww_frames(st, [e], 800, eng.cfg, eng.n_pursuers, eng.n_evaders)


def device_rate(draw, ids, rounds):
    out = draw(ids)
    per = []
    for _ in range(rounds):
        reps = max(4, 2048 // ids.numel())
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            draw(ids, out=out)
        t1.record()
        t1.synchronize()
        per.append(t0.elapsed_time(t1) / 1e3 / reps)
    s = float(np.median(per))
    return dict(ms_per_call=s * 1e3, frames_per_s=ids.numel() / s, gb_per_s=out.numel() / s / 1e9)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("render_rate.py needs a CUDA device")
    dev = "cuda:0"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None)
    print("card: %s (%s)" % (res["gpu"], res["nvidia_smi"]))
    print("%-6s %4s %10s %12s %9s" % ("config", "K", "ms/call", "frames/s", "GB/s"))
    for name in ("ww_c2", "ww_c4", "hw_c5", "pe_c3"):
        eng = make(name, dev)
        draw = draw_fn(name, eng)
        res[name] = {}
        for K in KS:
            ids = torch.arange(K, dtype=torch.int32, device=dev) * (eng.n_envs // K)
            r = res[name]["K%d" % K] = device_rate(draw, ids, a.rounds)
            print("%-6s %4d %10.3f %12.0f %9.1f" % (name, K, r["ms_per_call"], r["frames_per_s"], r["gb_per_s"]),
                  flush=True)
        per = []
        for i in range(max(1, min(a.rounds, 3))):
            t0 = time.perf_counter()
            want = host_frame(name, eng, i)
            per.append(time.perf_counter() - t0)
        got = draw(torch.tensor([i], dtype=torch.int32, device=dev)).cpu().numpy()
        assert np.array_equal(got, want), "%s: the kernel's frame differs from the oracle's" % name
        res[name]["host_K1_frames_per_s"] = 1.0 / float(np.median(per))
        print("%-6s %4d %10.3f %12.1f %9s  (host: state read-back + NumPy oracle)"
              % (name, 1, 1e3 * float(np.median(per)), res[name]["host_K1_frames_per_s"], "-"), flush=True)
        del eng
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
