"""Times whole-episode evaluation (madrl_b200.evaluate) on one GPU at the product shapes, max_traj_len 500:

  * evaluate_policy with an MLP policy and evaluate_heuristic (Waterworld: one norm per env; Pursuit), K = 1 and 2
    episodes per env: ms per evaluation (reset, K * 500 steps in launches of 64, records, one host read) and
    episodes per second;
  * madrl_eval_episodes_* on one 64-step chunk, from CUDA events: time, and bytes moved over time against the
    H100 SXM's 3.35 TB/s; against the same records composed from PyTorch operations (one group of elementwise
    kernels per step), whose records must be the kernel's bits;
  * C2's rollout_heuristic launch (64 and 256 steps) with norm="env" against norm="agent".

Every number is the median over rounds that alternate the variants; the card's name and power limit are read in
the same run.  Usage:  python scripts/evaluate_rate.py [--rounds 5] [--configs c2,c3,c5] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from madrl_b200 import (BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade, evaluate_heuristic,  # noqa: E402
                        evaluate_policy)
from madrl_b200 import evaluate as ev  # noqa: E402

HBM = 3.35e12
MPL, CHUNK = 500, 64


def make(name, dev):
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if name == "c2":
        return BatchedMAWaterWorld(4096, n_pursuers=5, n_evaders=5, device=dev, max_path_length=MPL)
    if name == "c3":
        return BatchedPursuitEvade(65536, np.load(os.path.join(root, "maps", "map_pool16.npy")), n_evaders=30,
                                   n_pursuers=8, obs_range=7, surround=True, sample_maps=True, device=dev,
                                   max_path_length=MPL)
    return BatchedHostageWorld(8192, 10, 16, 16, 4, 2, device=dev, max_path_length=MPL)


def mlp_policy(eng, dev):
    out = 5 if eng._abi == "pursuit" else 2
    net = torch.nn.Sequential(torch.nn.Linear(eng.obs_dim, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64),
                              torch.nn.Tanh(), torch.nn.Linear(64, out)).to(dev)
    for p in net.parameters():
        p.requires_grad_(False)
    if out == 5:
        return lambda o, s: (net(o).argmax(-1), {}, s)
    return lambda o, s: (torch.tanh(net(o)), {}, s)


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0


def composed(rew, done, info, disc, K, state, out):
    """The records of madrl_eval_episodes_* from PyTorch operations; `state` (ret, qsum, G, pw, len, k, isum) and
    `out` (ret, qsum, len, info rows, each with one spare row that absorbs the steps that record nothing)."""
    ret, qsum, G, pw, ln, k, isum = state
    T, E, A = rew.shape
    C = isum.shape[1]
    ar = torch.arange(E, device=rew.device)
    for t in range(T):
        r = rew[t].double()
        ret += r
        G += pw
        qsum += r * G
        pw *= disc
        ln += 1
        isum += info[t].view(E, C)
        d = done[t].bool()
        idx = torch.where(d & (k < K), k * E + ar, K * E)
        out[0].index_copy_(0, idx, ret)
        out[1].index_copy_(0, idx, qsum)
        out[2].index_copy_(0, idx, ln.int())
        out[3].index_copy_(0, idx, isum)
        k += d.long()
        keep = (~d).double()[:, None]
        ret *= keep
        qsum *= keep
        G *= keep
        pw.copy_(torch.where(d[:, None], torch.ones_like(pw), pw))
        ln *= (~d).long()
        isum *= (~d).long()[:, None]


def kernel_rates(eng, rounds, dev):
    """madrl_eval_episodes_* on one CHUNK-step chunk against the PyTorch composition, CUDA events, medians."""
    E, A, K, disc = eng.n_envs, eng._n_acting, 2, 0.99
    g = torch.Generator(device=dev).manual_seed(0)
    rew = torch.randn((CHUNK, E, A), generator=g, device=dev, dtype=eng.dtype)
    done = (torch.rand((CHUNK, E), generator=g, device=dev) < 0.05).to(torch.uint8)
    C = int(np.prod(eng._info_tail))
    info = torch.randint(0, 3, (CHUNK, E, C), generator=g, device=dev, dtype=torch.int32)
    rec = ev.EpisodeRecords(eng, K, disc)

    def state():
        z = lambda *s, dt=torch.float64: torch.zeros(s, dtype=dt, device=dev)  # noqa: E731
        return [z(E, A), z(E, A), z(E, A), torch.ones(E, A, dtype=torch.float64, device=dev),
                z(E, dt=torch.int64), z(E, dt=torch.int64), z(E, C, dt=torch.int64)]

    def outs():
        z = lambda *s, dt=torch.float64: torch.zeros(s, dtype=dt, device=dev)  # noqa: E731
        return [z(K * E + 1, A), z(K * E + 1, A), z(K * E + 1, dt=torch.int32), z(K * E + 1, C, dt=torch.int64)]

    # the two give the same bits on the same chunk
    st, o = state(), outs()
    composed(rew, done, info, disc, K, st, o)
    rec.add(rew, done, info)
    got = rec.read(K * E)
    same = all(np.array_equal(a, b[:K * E].cpu().numpy()) for a, b in zip(got, (o[0], o[1], o[2], o[3])))
    reps, tk, tc = 20, [], []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    st, o = state(), outs()
    for _ in range(rounds):
        ev0.record()
        for _ in range(reps):
            rec.add(rew, done, info)
        ev1.record()
        torch.cuda.synchronize()
        tk.append(ev0.elapsed_time(ev1) / reps)
        ev0.record()
        composed(rew, done, info, disc, K, st, o)
        ev1.record()
        torch.cuda.synchronize()
        tc.append(ev0.elapsed_time(ev1))
    rb = rew.element_size()
    # rewards, done and info read once; the carry read and written once (records: at most K E rows, negligible)
    nbytes = CHUNK * E * (A * rb + 1 + 4 * C) + 2 * E * A * 8 * 8
    ms = float(np.median(tk))
    return dict(chunk_steps=CHUNK, kernel_ms=ms, kernel_bytes=nbytes, kernel_GBps=nbytes / ms / 1e6,
                kernel_share_of_3_35TBps=nbytes / ms / 1e-3 / HBM, torch_composed_ms=float(np.median(tc)),
                same_bits_as_composed=bool(same))


def eval_rates(name, rounds, dev):
    eng = make(name, dev)
    pol = mlp_policy(eng, dev)
    variants = [("mlp", K) for K in (1, 2)]
    if eng._abi != "hostage":
        variants += [("heuristic", K) for K in (1, 2)]

    def run(kind, K):
        n = K * eng.n_envs
        if kind == "mlp":
            return evaluate_policy(eng, pol, n, 0.99, "decentralized", chunk=CHUNK)
        return evaluate_heuristic(eng, n, 0.99, "decentralized", chunk=CHUNK)

    for v in variants:          # warm-up: captures, module loads
        run(*v)
    times = {v: [] for v in variants}
    for _ in range(rounds):
        for v in variants:
            times[v].append(wall(lambda: run(*v)))
    out = {}
    for (kind, K), ts in times.items():
        s = float(np.median(ts))
        out["%s_K%d" % (kind, K)] = dict(ms_per_evaluation=s * 1e3, episodes_per_s=K * eng.n_envs / s,
                                         steps=K * MPL, rounds=[t * 1e3 for t in ts])
    out["eval_episodes_kernel"] = kernel_rates(eng, rounds, dev)
    del eng
    torch.cuda.empty_cache()
    return out


def heuristic_norm_rates(rounds, dev):
    eng = make("c2", dev)
    obs0 = eng.reset()
    res = {}
    for T in (64, 256):
        bufs = eng._outputs(T, None, True)
        times = {"agent": [], "env": []}
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for norm in times:      # warm-up
            eng.rollout_heuristic(T, obs0, out=bufs, record_actions=False, norm=norm)
        for _ in range(rounds):
            for norm in times:
                ev0.record()
                for _ in range(5):
                    eng.rollout_heuristic(T, obs0, out=bufs, record_actions=False, norm=norm)
                ev1.record()
                torch.cuda.synchronize()
                times[norm].append(ev0.elapsed_time(ev1) / 5)
        res["T%d" % T] = {k: dict(ms_per_launch=float(np.median(v)), rounds=v) for k, v in times.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--configs", default="c2,c3,c5")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("evaluate_rate.py needs a CUDA device")
    dev = "cuda:0"
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    res = dict(gpu=torch.cuda.get_device_name(0), nvidia_smi=q[0] if q else None, max_traj_len=MPL, chunk=CHUNK)
    for name in a.configs.split(","):
        res[name] = eval_rates(name, a.rounds, dev)
        print(json.dumps({name: res[name]}), flush=True)
    res["c2_rollout_heuristic_norm"] = heuristic_norm_rates(a.rounds, dev)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
