"""Times whole-path sampling (madrl_b200.whole_paths) at C2: Waterworld, E = 4096 envs, max_path_length 500,
batch_size = E * 500, an MLP policy (64-64 tanh), launches of 64 steps:

  * the sampler's call (reset, the launches, the fold after each launch and its status read, the copies of each
    launch's outputs, the finish and the gathers) against the bare PolicyRollout launches over the same steps;
  * the fold (per launch) and the finish + gathers of the batch, from CUDA events, and the gathers' bytes (each
    kept row read once and written once) over the H100 SXM's 3.35 TB/s;
  * process_samples_concurrent on the flat batch (path-parallel kernels) against the same pass on a continuing
    rollout [500, 4096] of the same N rows (serial kernels).

Every number is the median over rounds; the card's name and power limit are read in the same run.
Usage:  python scripts/whole_paths_rate.py [--rounds 5] [--envs 4096] [--out FILE]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from madrl_b200 import BatchedMAWaterWorld, WholePathSampler, postproc  # noqa: E402
from madrl_b200 import _lib  # noqa: E402
from madrl_b200._lib import _ptr  # noqa: E402
from madrl_b200.whole_paths import _Selection  # noqa: E402

HBM = 3.35e12
MPL, CHUNK = 500, 64


def mlp_policy(eng, dev):
    net = torch.nn.Sequential(torch.nn.Linear(eng.obs_dim, 64), torch.nn.Tanh(), torch.nn.Linear(64, 64),
                              torch.nn.Tanh(), torch.nn.Linear(64, 2)).to(dev)
    for p in net.parameters():
        p.requires_grad_(False)

    def policy(o, s):
        m = net(o)
        return torch.tanh(m), {"mean": m}, s
    return policy


def wall(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def events(fn, reps=1):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / 1e3 / reps


def med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--envs", type=int, default=4096)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("whole_paths_rate needs a CUDA device")
    dev = torch.device("cuda", 0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True).stdout.strip()
    E = args.envs
    eng = BatchedMAWaterWorld(E, n_pursuers=5, n_evaders=5, device=dev, max_path_length=MPL)
    pol = mlp_policy(eng, dev)
    sampler = WholePathSampler(eng, pol, E * MPL, MPL, chunk=CHUNK)
    res = dict(card=card, E=E, batch_size=E * MPL, chunk=CHUNK)
    sampler()                                                        # capture and warm-up
    t_sample, t_bare, t_fold, t_gather, t_proc_flat, t_proc_cont = [], [], [], [], [], []
    for _ in range(args.rounds):
        dt, batch = wall(sampler)
        t_sample.append(dt)
        n_launch = batch.n_steps // CHUNK

        def bare():
            obs0 = eng.reset()
            for _ in range(n_launch):
                r = sampler.loop(obs0, None)
                obs0 = r.policy_obs[-1]
        t_bare.append(wall(bare)[0])
        del batch
    batch = sampler()
    N, P, A = len(batch), batch.n_paths, batch.rew.shape[1]
    row_bytes = sum(x[0].numel() * x.element_size() for x in
                    [batch.obs, batch.actions, batch.rew, batch.infos] + list(batch.extras.values()))
    res.update(N=N, P=P, n_steps=batch.n_steps, t_star=batch.t_star, gather_bytes=2 * N * row_bytes)
    # the fold and the finish + gathers, replayed on the launches of one more call
    sel = _Selection(E, CHUNK, E * MPL, sampler.max_steps(), dev)
    obs0 = eng.reset()
    while True:
        r = sampler.loop(obs0, None)
        pobs = r.policy_obs.clone()
        if sel.add(obs0, pobs, r.actions.clone(), r.rew.clone(), r.done, r.info.clone(),
                   {k: v.clone() for k, v in r.extras.items()}):
            break
        obs0 = pobs[-1]
    L = _lib.lib()
    carry0, acc0 = sel.carry.clone(), sel.acc.clone()

    def fold_all():
        sel.carry.copy_(torch.tensor([-1, -1, 0], dtype=torch.int32, device=dev).repeat_interleave(E))
        sel.acc.copy_(torch.tensor([0, -1, 0, 0, 0], dtype=torch.int64, device=dev))
        for j in range(len(sel.launches)):
            _lib.check(L.madrl_whole_paths_fold(CHUNK, E, j * CHUNK, E * MPL, _ptr(sel.done_stage[j * CHUNK:]),
                                                _ptr(sel.carry), _ptr(sel.acc), _lib.stream(dev)))
    for _ in range(args.rounds):
        t_fold.append(events(fold_all) / len(sel.launches))
        assert torch.equal(sel.carry, carry0) and torch.equal(sel.acc, acc0)
        t_gather.append(events(sel.batch))
    # processing: the flat batch against a continuing rollout of the same rows
    o, d, rw, ob = batch.as_rollout()
    D = o.shape[3]
    Tc = N // E
    oc = batch._obs_store[1:Tc * E + 1].view(Tc, E, A, D)
    dc = torch.zeros((Tc, E), dtype=torch.uint8, device=dev)
    dc[-1] = 1
    rc, obc = batch.rew[:Tc * E].view(Tc, E, A), batch.obs[:E].contiguous()
    for _ in range(args.rounds):
        bl = postproc.LinearFeatureBaseline(D, dev, n_agents=A)
        t_proc_flat.append(wall(lambda: postproc.process_samples_concurrent(bl, o, d, rw, 0.99, 0.97,
                                                                            obs_before=ob))[0])
        bl = postproc.LinearFeatureBaseline(D, dev, n_agents=A)
        t_proc_cont.append(wall(lambda: postproc.process_samples_concurrent(bl, oc, dc, rc, 0.99, 0.97,
                                                                            obs_before=obc))[0])
    res.update(sampler_ms=1e3 * med(t_sample), bare_launches_ms=1e3 * med(t_bare),
               fold_us_per_launch=1e6 * med(t_fold), finish_gather_ms=1e3 * med(t_gather),
               gather_share_of_hbm=res["gather_bytes"] / HBM / med(t_gather),
               process_flat_ms=1e3 * med(t_proc_flat), process_continuing_ms=1e3 * med(t_proc_cont),
               continuing_rows=Tc * E)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
