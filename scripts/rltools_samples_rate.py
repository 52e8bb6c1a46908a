"""Throughput of rltools' sample processing on the device (madrl_b200.rltools_sampler, csrc/postproc.cu
madrl_running_moments_* / madrl_time_baseline_*_f32, csrc/baseline.cu madrl_lfbr_*) on full rollout launches, against
the PyTorch implementation of the same steps (oracle/rltools_oracle.py torch_process_samples: float64 features
materialised, a backward loop over time, scatter_add bins for the time baseline, a DGEMM Gram and
torch.linalg.cholesky).

At the C2, C3, C4 and C5 rollout shapes of scripts/linear_baseline_rate.py, decentralized control with an obsnorm and
a reward normaliser, each timed with CUDA events, alternating the device path and PyTorch over the rounds; the median
and the min-max spread are printed:
  process     process_samples (predict with a fitted baseline, q, simplev, explained variances, GAE, fit) against
              torch_process_samples
  rewnorm     RunningStandardizer(1).update over the rewards (D = 1), against torch's float64 sums
  obsnorm     the baseline's obsnorm update over the observation rows (D = the obs width), against torch's sums
  time_bl     time_baseline, against the scatter_add bins
  gram        the rltools normal equations, against the DGEMM on materialised features
Bytes: the rows each pass reads (float32), over the 3 350 GB/s HBM3 data sheet of the H100 SXM; FP64 FLOP of the Gram
(2 N Dc^2, the whole square) over the 67 TFLOP/s FP64 tensor-core data sheet.  The card's name and power limit are read
in the same run.

    python scripts/rltools_samples_rate.py [--rounds 5] [--reps 3] [--shapes C2,C3,C4,C5] [--out FILE]
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

from linear_baseline_rate import card, make, timed  # noqa: E402
from oracle import rltools_oracle as ro  # noqa: E402

DATASHEET_GBS, DATASHEET_FP64 = 3350.0, 67e12


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


def torch_bins(q, done):
    """simplev by scatter_add over the time index (pooled over every agent's rows)."""
    idx = ro.torch_index(done).unsqueeze(-1).expand(q.shape).reshape(-1)
    L = int(idx.max()) + 1
    s = torch.zeros(L, dtype=torch.float64, device=q.device).scatter_add_(0, idx, q.double().reshape(-1))
    c = torch.zeros(L, dtype=torch.float64, device=q.device).scatter_add_(0, idx, torch.ones_like(s[idx]))
    return (s / c)[idx].view(q.shape).float()


def stats(xs):
    xs = sorted(xs)
    med = xs[len(xs) // 2]
    return med, (xs[-1] - xs[0]) / med if med > 0 else 0.0


def main():
    from madrl_b200 import rltools_sampler as rs
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="C2,C3,C4,C5")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this script measures the GPU")
    name, power = card()
    print("card: %s, power limit / max SM clock: %s" % (name, power))
    rows = []
    for shape in args.shapes.split(","):
        obs, ob, rew, done = rollout(shape)
        T, E, A, D = obs.shape
        bl = rs.LinearFeatureBaseline(D, "cuda", True)
        rn = rs.RunningStandardizer(1, "cuda")
        bl.update_obsnorm(obs, ob)
        rn.update(rew.unsqueeze(-1))
        rs.process_samples(bl, obs, done, rew, 0.99, 0.97, rn, obs_before=ob)      # a fitted baseline
        w, norm = bl._coeffs.clone(), bl.obsnorm.norm_table.unsqueeze(0)
        q = rs.process_samples(None, obs, done, rew, 0.99, 0.97, rn)["q"]

        def torch_gram():
            F = ro.torch_features(obs, ob, done, norm)
            Fy = torch.cat([F, q.double().unsqueeze(-1)], -1).reshape(-1, D + 4)
            return Fy.t() @ Fy

        pairs = dict(
            process=(lambda: rs.process_samples(bl, obs, done, rew, 0.99, 0.97, rn, obs_before=ob),
                     lambda: ro.torch_process_samples(obs, ob, done, rew, 0.99, 0.97, rn.denom, w, norm, False)),
            rewnorm=(lambda: rn._sums(rew.unsqueeze(-1), None, 1),
                     lambda: (rew.double().sum((0, 1, 2)), (rew.double() ** 2).sum((0, 1, 2)))),
            obsnorm=(lambda: bl.obsnorm._sums(obs, ob, 1),
                     lambda: (obs.double().sum((0, 1, 2)), (obs.double() ** 2).sum((0, 1, 2)))),
            time_bl=(lambda: rs.time_baseline(q, done), lambda: torch_bins(q, done)),
            gram=(lambda: bl.normal_equations(obs, done, q, ob), torch_gram))
        n = T * E * A
        nbytes = dict(process=n * (2 * D * 4 + 4 * 4), rewnorm=n * 4, obsnorm=n * D * 4, time_bl=n * 12,
                      gram=n * (D + 1) * 4)
        times = {k: ([], []) for k in pairs}
        for k, (dev_fn, torch_fn) in pairs.items():          # warm-up
            dev_fn(), torch_fn()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for k, (dev_fn, torch_fn) in pairs.items():
                times[k][0].append(timed(dev_fn, args.reps)[0])
                times[k][1].append(timed(torch_fn, args.reps)[0])
        for k in pairs:
            (md, sd), (mt, st) = stats(times[k][0]), stats(times[k][1])
            gbs = nbytes[k] / md / 1e9
            row = dict(shape=shape, part=k, T=T, E=E, A=A, D=D, device_ms=md * 1e3, device_spread=sd,
                       torch_ms=mt * 1e3, torch_spread=st, gbs=gbs, frac_hbm=gbs / DATASHEET_GBS)
            if k == "gram":
                row["fp64_frac"] = 2.0 * n * (D + 4) ** 2 / md / DATASHEET_FP64
            rows.append(row)
            print("%s %-8s T%d E%d A%d D%d  device %8.3f ms (%4.1f%%)  torch %8.3f ms (%4.1f%%)  %7.1f GB/s (%4.1f%% "
                  "of the data sheet)%s" % (shape, k, T, E, A, D, md * 1e3, sd * 100, mt * 1e3, st * 100, gbs,
                                            100 * gbs / DATASHEET_GBS,
                                            ("  FP64 %.1f%% of 67 TFLOP/s" % (100 * row["fp64_frac"])
                                             if "fp64_frac" in row else "")))
        del obs, ob, rew, done, bl, q
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            json.dump(dict(card=name, power=power, rows=rows), f, indent=1)


if __name__ == "__main__":
    np.seterr(all="ignore")
    main()
