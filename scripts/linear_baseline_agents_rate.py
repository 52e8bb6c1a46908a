"""Throughput of the per-agent linear feature baseline (concurrent mode, csrc/baseline.cu madrl_lfb_*_agents) on
full rollout launches, against what a user can do without it:
  pooled x A   A calls of the pooled baseline, each on contiguous copies of one agent's obs / obs_before / returns
               (the copies are timed with the calls);
  torch        the chunked PyTorch float64 Gram (G.addmm_ = cuBLAS DGEMM, oracle/baseline_oracle.py) per agent.
The three are timed alternately in one process with CUDA events, on the shapes and rollouts of
scripts/linear_baseline_rate.py (C2 Waterworld 4096 x 256 x 5, C3 Pursuit 65536 x 16 x 8, C4 Waterworld
4096 x 64 x 20, C5 Hostage 8192 x 64 x 10).  Reported: per-agent normal equations, fit (+ batched solve) and
predict times; the pooled-x-A fit and predict; the PyTorch Gram of every agent; the pooled single fit over all
rows, for scale.  The card's name and power limit are read in the same run.

    python scripts/linear_baseline_agents_rate.py [--rounds 5] [--shapes C2,C3,C4,C5] [--out FILE]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from linear_baseline_rate import card, rollout, timed  # noqa: E402
from oracle import baseline_oracle as bo  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="C2,C3,C4,C5")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("linear_baseline_agents_rate.py measures on a GPU; none is visible")
    from madrl_b200.postproc import LinearFeatureBaseline
    name, power = card()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power), flush=True)
    results = []
    for shape in args.shapes.split(","):
        obs, obs0, done, ret, t0 = rollout(shape)
        T, E, A, D = obs.shape
        per = LinearFeatureBaseline(D, "cuda", n_agents=A)
        pooled = LinearFeatureBaseline(D, "cuda")

        def pooled_fit():
            for a in range(A):
                pooled.fit(obs[:, :, a:a + 1].contiguous(), done, ret[:, :, a:a + 1].contiguous(),
                           obs0[:, a:a + 1].contiguous(), t0)

        def pooled_predict():
            for a in range(A):
                pooled.predict(obs[:, :, a:a + 1].contiguous(), done, obs0[:, a:a + 1].contiguous(), t0)

        def torch_grams():
            return [bo.torch_normal_equations(obs[:, :, a:a + 1], done, ret[:, :, a:a + 1], obs0[:, a:a + 1], t0)
                    for a in range(A)]

        fns = dict(gram=lambda: per.normal_equations(obs, done, ret, obs0, t0),
                   fit=lambda: per.fit(obs, done, ret, obs0, t0),
                   predict=lambda: per.predict(obs, done, obs0, t0),
                   pooled_x_a_fit=pooled_fit, pooled_x_a_predict=pooled_predict, torch_grams=torch_grams,
                   pooled_one_fit=lambda: pooled.fit(obs, done, ret, obs0, t0))
        for fn in fns.values():                                    # warm-up: module load, solver workspaces
            fn()
        t = {k: [] for k in fns}
        for _ in range(args.rounds):                               # alternate the implementations
            for k, fn in fns.items():
                t[k].append(timed(fn, args.reps)[0])
        med = {k: float(np.median(v)) * 1e3 for k, v in t.items()}
        spread = {k: float((max(v) - min(v)) / np.median(v)) for k, v in t.items()}
        r = dict(shape=shape, T=T, E=E, A=A, D=D, rows=T * E * A, card=name, power=power,
                 **{k + "_ms": v for k, v in med.items()}, spread=spread)
        results.append(r)
        print(json.dumps(r), flush=True)
        del obs, obs0, done, ret, t0, per, pooled
        torch.cuda.empty_cache()
    print("\n| shape | A | per-agent normal eq ms | per-agent fit ms | pooled x A fit ms | PyTorch x A Gram ms |"
          " pooled 1 fit ms | per-agent predict ms | pooled x A predict ms |")
    print("|---|---|---|---|---|---|---|---|---|")
    for r in results:
        print("| %s | %d | %.2f | %.2f | %.2f | %.2f | %.2f | %.3f | %.3f |" % (
            r["shape"], r["A"], r["gram_ms"], r["fit_ms"], r["pooled_x_a_fit_ms"], r["torch_grams_ms"],
            r["pooled_one_fit_ms"], r["predict_ms"], r["pooled_x_a_predict_ms"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()
