"""Throughput of the recurrent sample batch (madrl_b200.postproc.pad_paths / process_samples_recurrent,
csrc/postproc.cu madrl_paths_pad_*) on full rollout launches, against what a user can do without it:
  torch      a PyTorch gather of the source rows through a [P, L] index into zeros (oracle/recurrent_oracle.py
             torch_pad), for the same observations, actions and rewards;
  host       pack_paths(...).to_list() and rllab-style NumPy padding (pad_tensor_n) of the same three arrays -- every
             observation crosses PCIe -- at one reduced size (C2 with 256 envs), timed with a host clock.
pad_paths and the PyTorch gather are timed alternately in one process with CUDA events, with process_samples_recurrent
(decentralized, pooled baseline: predict, GAE, explained variance, centring, padding of obs / actions / rewards /
returns / advantages, fit), at the C2, C3, C4 and C5 rollout shapes of scripts/linear_baseline_rate.py; the median
over the rounds and the min-max spread are printed, and the padded tensors of the two implementations are compared
bit for bit.  Bytes of a pad = the source rows read + P * L * row bytes written, for the three tensors; reported next
to the card's streaming-write rate (fill_ of a float32 tensor the size of the C2 observations) and the 3 350 GB/s
HBM3 data sheet of the H100 SXM.  The card's name and power limit are read in the same run.

    python scripts/recurrent_samples_rate.py [--rounds 5] [--shapes C2,C3,C4,C5] [--out FILE]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from linear_baseline_rate import card, make, timed  # noqa: E402
from oracle import recurrent_oracle as ro  # noqa: E402

DATASHEET_GBS = 3350.0


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
    return obs, obs0, act, rew, done


def fill_rate(reps=20):
    x = torch.empty((256, 4096, 5, 213), dtype=torch.float32, device="cuda")
    x.fill_(0.0)
    s = timed(lambda: x.fill_(1.0), reps)[0]
    nbytes = x.numel() * 4
    del x
    torch.cuda.empty_cache()
    return nbytes / s / 1e9


def host_pad(obs, obs0, act, rew, done):
    """pack_paths(...).to_list() and NumPy padding, as a user of the host path would."""
    from madrl_b200.postproc import pack_paths
    torch.cuda.synchronize()
    t = time.perf_counter()
    paths = pack_paths(obs, act, rew, done, obs_before=obs0).to_list()
    L = max(len(p["rewards"]) for p in paths)
    out = [ro.pad_tensor_n([p[k] for p in paths], L) for k in ("observations", "actions", "rewards")]
    return time.perf_counter() - t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--shapes", default="C2,C3,C4,C5")
    ap.add_argument("--host-envs", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("recurrent_samples_rate.py measures on a GPU; none is visible")
    from madrl_b200.postproc import LinearFeatureBaseline, pad_paths, process_samples_recurrent
    name, power = card()
    print("# %s, power.limit / clocks.max.sm: %s" % (name, power), flush=True)
    fill_gbs = fill_rate()
    print("# fill_ streaming-write rate: %.0f GB/s (data sheet %.0f GB/s)" % (fill_gbs, DATASHEET_GBS), flush=True)
    results = []
    for shape in args.shapes.split(","):
        obs, obs0, act, rew, done = rollout(shape)
        T, E, A, D = obs.shape
        bl = LinearFeatureBaseline(D, "cuda")
        pp = pad_paths(obs, act, rew, done, obs_before=obs0)
        rec = torch.stack([pp.env, pp.agent, pp.start, pp.length], dim=-1)
        P, L = rec.shape[0], pp.valids.shape[1]
        row_bytes = D * obs.element_size() + act[0, 0, 0].numel() * act.element_size() + rew.element_size()
        nbytes = T * E * A * row_bytes + P * L * row_bytes

        def torch_pad():
            return (ro.torch_pad(obs, rec, L, first=obs0), ro.torch_pad(act, rec, L), ro.torch_pad(rew, rec, L))

        want = torch_pad()
        same = all(torch.equal(a, b) for a, b in zip((pp.observations, pp.actions, pp.rewards), want))
        del pp, want
        fns = dict(pad_paths=lambda: pad_paths(obs, act, rew, done, obs_before=obs0), torch_gather=torch_pad,
                   process_samples_recurrent=lambda: process_samples_recurrent(
                       bl, obs, act, rew, done, 0.99, 0.97, "decentralized", obs_before=obs0))
        for fn in fns.values():                                      # warm-up
            fn()
        t = {k: [] for k in fns}
        for _ in range(args.rounds):                                 # alternate the implementations
            for k, fn in fns.items():
                t[k].append(timed(fn, args.reps)[0])
        med = {k: float(np.median(v)) * 1e3 for k, v in t.items()}
        spread = {k: float((max(v) - min(v)) / np.median(v)) for k, v in t.items()}
        r = dict(shape=shape, T=T, E=E, A=A, D=D, P=P, L=L, padded_over_rollout=P * L / (T * E * A), bytes=nbytes,
                 bitwise_equal_torch=same, card=name, power=power, fill_gbs=fill_gbs,
                 **{k + "_ms": v for k, v in med.items()}, spread=spread,
                 pad_gbs=nbytes / (med["pad_paths"] * 1e-3) / 1e9)
        results.append(r)
        print(json.dumps(r), flush=True)
        del obs, obs0, act, rew, done, bl
        torch.cuda.empty_cache()
    # the host path, at a reduced size: the C2 configuration with --host-envs envs
    from madrl_b200 import BatchedMAWaterWorld
    eng = BatchedMAWaterWorld(args.host_envs, 5, 5, n_poison=10, n_sensors=30, seed=0, device="cuda",
                              max_path_length=500)
    obs0 = eng.reset()
    g = torch.Generator(device="cuda")
    g.manual_seed(1)
    act = torch.randn((256, args.host_envs, 5, 2), device="cuda", generator=g) * 0.5
    obs, rew, done, _ = eng.rollout(act)
    host_s = []
    dev_s = []
    for _ in range(args.rounds):
        s, out = host_pad(obs, obs0, act, rew, done)
        host_s.append(s)
        dev_s.append(timed(lambda: pad_paths(obs, act, rew, done, obs_before=obs0), args.reps)[0])
    pp = pad_paths(obs, act, rew, done, obs_before=obs0)
    same = all(np.array_equal(a, b.cpu().numpy()) for a, b in zip(out, (pp.observations, pp.actions, pp.rewards)))
    host = dict(shape="C2/%d envs" % args.host_envs, host_ms=float(np.median(host_s)) * 1e3,
                host_spread=float((max(host_s) - min(host_s)) / np.median(host_s)),
                pad_paths_ms=float(np.median(dev_s)) * 1e3, bitwise_equal_host=same, card=name, power=power)
    print(json.dumps(host), flush=True)
    print("\n| shape | P x L / rows | pad_paths ms | GB/s (%% of fill_ %.0f, %% of 3350) | torch gather ms |"
          " process_samples_recurrent ms | bitwise |" % fill_gbs)
    print("|---|---|---|---|---|---|---|")
    for r in results:
        print("| %s | %.2f | %.2f (+-%.0f%%) | %.0f (%.0f%%, %.0f%%) | %.2f | %.2f | %s |" % (
            r["shape"], r["padded_over_rollout"], r["pad_paths_ms"], 100 * r["spread"]["pad_paths"], r["pad_gbs"],
            100 * r["pad_gbs"] / fill_gbs, 100 * r["pad_gbs"] / DATASHEET_GBS, r["torch_gather_ms"],
            r["process_samples_recurrent_ms"], r["bitwise_equal_torch"]))
    print("| %s host | | %.2f | | host: %.1f ms (+-%.0f%%) | | %s |" % (
        host["shape"], host["pad_paths_ms"], host["host_ms"], 100 * host["host_spread"], host["bitwise_equal_host"]))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(results=results, host=host, fill_gbs=fill_gbs), f, indent=1)


if __name__ == "__main__":
    main()
