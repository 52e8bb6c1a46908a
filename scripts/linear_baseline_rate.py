"""Throughput of the linear feature baseline (csrc/baseline.cu) on full rollout launches, against the obvious
PyTorch implementation (features built per chunk of 65 536 rows in float64, G.addmm_(F^T, F) = cuBLAS DGEMM,
F @ c for predict; oracle/baseline_oracle.py).  The two are timed alternately in one process with CUDA events.

Shapes are the benchmark's rollout launches, filled by a real auto-reset rollout of each engine:
  C2 Waterworld 4096 x 256 x 5, C3 Pursuit 65536 x 16 x 8, C4 Waterworld 4096 x 64 x 20, C5 Hostage 8192 x 64 x 10.
Reported: normal equations (+ solve) time and useful FP64 rate 2 N (Df+1)(Df+2)/2 / t (the upper triangle of
[F y]^T [F y]) with its share of the 67 TFLOP/s FP64 tensor-core data-sheet figure, and predict time with its
observation read rate N D elem / t.  The card's name and power limit are read in the same run.

    python scripts/linear_baseline_rate.py [--rounds 5] [--shapes C2,C3,C4,C5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import baseline_oracle as bo  # noqa: E402

FP64_TC_PEAK = 67e12     # H100 SXM data sheet, FP64 tensor core, dense
PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)


def make(shape):
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    kw = dict(seed=0, device="cuda", max_path_length=500)
    if shape == "C2":
        return BatchedMAWaterWorld(4096, 5, 5, n_poison=10, n_sensors=30, **kw), 256
    if shape == "C4":
        return BatchedMAWaterWorld(4096, 20, 50, n_poison=50, n_sensors=30, **kw), 64
    if shape == "C3":
        return BatchedPursuitEvade(65536, np.load(os.path.join(ROOT, "maps", "map_pool16.npy")), **PE_C3, **kw), 16
    return BatchedHostageWorld(8192, 10, 16, 16, 4, 2, **kw), 64


def rollout(shape):
    from madrl_b200.postproc import gae
    eng, T = make(shape)
    obs0 = eng.reset()
    t0 = eng.state["path_len"].clone()
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    act_shape = (T, eng.n_envs, eng._n_acting) + eng._act_tail
    if eng._act_dtype == torch.int32:
        act = torch.randint(0, 5, act_shape, dtype=torch.int32, device="cuda", generator=g)
    else:
        act = torch.randn(act_shape, device="cuda", generator=g) * 0.5
    obs, rew, done, _ = eng.rollout(act)
    ret = gae(rew, torch.zeros_like(rew), done, 0.99, 1.0)[1]
    del eng, act
    return obs, obs0, done, ret, t0


def timed(fn, reps):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3, out


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader",
                            "-i", str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30)
        return name, q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        return name, "unknown (%s)" % e


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="C2,C3,C4,C5")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("linear_baseline_rate.py measures on a GPU; none is visible")
    from madrl_b200.postproc import LinearFeatureBaseline
    name, power = card()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power), flush=True)
    results = []
    for shape in args.shapes.split(","):
        obs, obs0, done, ret, t0 = rollout(shape)
        T, E, A, D = obs.shape
        N, Dc = T * E * A, 2 * D + 5
        flop = 2.0 * N * Dc * (Dc + 1) / 2
        obs_bytes = N * D * obs.element_size()
        b = LinearFeatureBaseline(D, "cuda")
        b.fit(obs, done, ret, obs0, t0)                      # warm-up: module load, solver workspaces
        c = torch.from_numpy(b.get_param_values()).cuda()
        bo.torch_normal_equations(obs, done, ret, obs0, t0)
        bo.torch_predict(obs, done, c, obs0, t0)
        t = {k: [] for k in ("gram", "fit", "predict", "torch_gram", "torch_predict")}
        for _ in range(args.rounds):                          # alternate the implementations
            t["gram"].append(timed(lambda: b.normal_equations(obs, done, ret, obs0, t0), args.reps)[0])
            t["torch_gram"].append(timed(lambda: bo.torch_normal_equations(obs, done, ret, obs0, t0), args.reps)[0])
            t["fit"].append(timed(lambda: b.fit(obs, done, ret, obs0, t0), args.reps)[0])
            t["predict"].append(timed(lambda: b.predict(obs, done, obs0, t0), args.reps)[0])
            t["torch_predict"].append(timed(lambda: bo.torch_predict(obs, done, c, obs0, t0), args.reps)[0])
        med = {k: float(np.median(v)) for k, v in t.items()}
        spread = {k: float((max(v) - min(v)) / np.median(v)) for k, v in t.items()}
        r = dict(shape=shape, T=T, E=E, A=A, D=D, rows=N, cols=Dc, card=name, power=power,
                 gram_ms=med["gram"] * 1e3, fit_ms=med["fit"] * 1e3, predict_ms=med["predict"] * 1e3,
                 torch_gram_ms=med["torch_gram"] * 1e3, torch_predict_ms=med["torch_predict"] * 1e3,
                 gram_tflops=flop / med["gram"] / 1e12, gram_share_of_67tf=flop / med["gram"] / FP64_TC_PEAK,
                 torch_gram_tflops=flop / med["torch_gram"] / 1e12,
                 predict_gbs=obs_bytes / med["predict"] / 1e9, torch_predict_gbs=obs_bytes / med["torch_predict"] / 1e9,
                 spread=spread)
        results.append(r)
        print(json.dumps(r), flush=True)
        del obs, obs0, done, ret, t0, b
        torch.cuda.empty_cache()
    print("\n| shape | rows | Df+1 | normal eq ms | FP64 TFLOP/s | of 67 | +solve ms | PyTorch ms | predict ms | GB/s |"
          " PyTorch predict ms |")
    print("|---|---|---|---|---|---|---|---|---|---|---|")
    for r in results:
        print("| %s | %d | %d | %.2f | %.1f | %.0f %% | %.2f | %.2f | %.3f | %.0f | %.2f |" % (
            r["shape"], r["rows"], r["cols"], r["gram_ms"], r["gram_tflops"], 100 * r["gram_share_of_67tf"],
            r["fit_ms"], r["torch_gram_ms"], r["predict_ms"], r["predict_gbs"], r["torch_predict_ms"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
