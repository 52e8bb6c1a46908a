"""float32 against bfloat16 observations on bench.py's workloads (one GPU command).

    python scripts/obs_bf16_rate.py [--lib NAME=PATH ...] [--rounds R] [--reps N]

Prints the card (name, power limit, SM clock), then, for each of bench.py's four workloads (Waterworld
C2 and C4, Pursuit C3, Hostage C5; bench.py's env counts and launch lengths):
  * ms per rollout launch from CUDA events around the launches (median over N launches), with the
    float32 and the bfloat16 engine launched alternately in the same process;
  * agent-env-steps/s and algorithmic bytes per env-step over kernel time.  The bytes are bench.py's
    compulsory-traffic formula with the observation values counted at their stored size (2 bytes in
    bfloat16);
  * the end-to-end rate of the host-buffer entry point (madrl_*_rollout_host2, pinned host tensors, wall
    clock around the blocking calls), both formats.
After the timed launches the two engines, which started from the same seed and took the same actions, run
one more launch each: the bfloat16 observations must equal the float32 ones converted with
`.to(torch.bfloat16)` bit for bit, and rewards, dones and infos must be equal.  A mismatch exits non-zero.

Every `--lib` build (default: the in-tree library; a PATH is loaded through MADRL_B200_LIB, e.g. one
made by scripts/build_variant.py from another checkout) runs in a child process of its own, the builds
alternating for R rounds.  A build without madrl_*_set_obs_format is timed in float32 only.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WORKLOADS = ("waterworld", "pursuit", "waterworld_c4", "hostage")   # bench.py's names: C2, C3, C4, C5


def card():
    import torch
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(), "power.limit": "unknown", "clocks.sm": "unknown"}


def alg_bytes(wl, eng):
    """bench.py's algorithmic bytes per env-step, which count 4-byte observations, with the engine's
    observation values (acting agents x obs_dim) counted at their stored size."""
    import bench
    obs_values = eng._n_acting * eng.obs_dim
    return bench.bytes_per_env_step(wl) - (4 - eng.obs_dtype.itemsize) * obs_values


def engine(wl, obs_dtype):
    import bench
    import torch
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    w = bench.WORKLOADS[wl]
    E, kw = w["envs"], {} if obs_dtype == torch.float32 else dict(obs_dtype=obs_dtype)
    if w["family"] == "ww":
        return BatchedMAWaterWorld(E, device="cuda", seed=0, **w["cfg"], **kw)
    if w["family"] == "pe":
        import numpy as np
        maps = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
        return BatchedPursuitEvade(E, maps, device="cuda", seed=0, max_path_length=500, **w["cfg"], **kw)
    return BatchedHostageWorld(E, *w["cfg"], device="cuda", seed=0, **kw)


def kernel_rates(wl, fmts, reps):
    """fmt -> ms per launch; the engines alternate launch by launch.  Returns (rates, mismatch or None)."""
    import bench
    import torch
    w = bench.WORKLOADS[wl]
    E, T, A = w["envs"], w["t"], w["agents"]
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    act = bench.make_actions(wl, T, E, "cuda", g)
    engs = {f: engine(wl, dt) for f, dt in fmts.items()}
    outs = {f: e._outputs(T, None, True) for f, e in engs.items()}
    for e in engs.values():
        e.reset()
    for _ in range(3):
        for f, e in engs.items():
            e.rollout(act, auto_reset=True, out=outs[f])
    torch.cuda.synchronize()
    ev = {f: [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
          for f in engs}
    for i in range(reps):
        for f, e in engs.items():
            ev[f][i][0].record()
            e.rollout(act, auto_reset=True, out=outs[f])
            ev[f][i][1].record()
    torch.cuda.synchronize()
    res = {}
    for f in engs:
        ms = sorted(s.elapsed_time(t) for s, t in ev[f])[reps // 2]
        nb = alg_bytes(wl, engs[f])
        res[f] = {"ms": ms, "agent_steps_per_sec": E * A * T / (ms * 1e-3), "alg_bytes_per_env_step": nb,
                  "alg_gbs": nb * E * T / (ms * 1e-3) / 1e9}
    bad = None
    if "bf16" in engs:   # both engines took the same actions from the same seed: check the last launch
        for f, e in engs.items():
            e.rollout(act, auto_reset=True, out=outs[f])
        (o32, r32, d32, i32), (o16, r16, d16, i16) = outs["fp32"], outs["bf16"]
        if not torch.equal(o32.to(torch.bfloat16).view(torch.int16), o16.view(torch.int16)):
            bad = "observations differ from fp32.to(bfloat16)"
        elif not (torch.equal(r32, r16) and torch.equal(d32, d16) and torch.equal(i32, i16)):
            bad = "rewards / dones / infos differ"
    del engs, outs
    torch.cuda.empty_cache()
    return res, bad


def e2e_rate(wl, obs_dtype):
    """Agent-env-steps/s of madrl_*_rollout_host2 (pinned buffers; <= 1 GB of observations per call)."""
    import bench
    import torch
    w = bench.WORKLOADS[wl]
    E, A, T = w["envs"], w["agents"], w["t"]
    eng = engine(wl, obs_dtype)
    eng.reset()
    Te = max(1, min(T, (1 << 30) // (E * A * eng.obs_dim * 4)))
    h_act = [bench.make_actions(wl, Te, E, "cuda", None, host=True).pin_memory() for _ in range(2)]
    h_out = (torch.empty((Te, E, A, eng.obs_dim), dtype=obs_dtype).pin_memory(), torch.empty((Te, E, A)).pin_memory(),
             torch.empty((Te, E), dtype=torch.uint8).pin_memory(),
             torch.empty((Te, E) + eng._info_tail, dtype=torch.int32).pin_memory())
    for i in range(2):
        eng.rollout_host(h_act[i % 2], *h_out)
    torch.cuda.synchronize()
    n = 5
    t0 = time.perf_counter()
    for i in range(n):
        eng.rollout_host(h_act[i % 2], *h_out)
    dt = time.perf_counter() - t0
    d2h = sum(x.numel() * x.element_size() for x in h_out)
    del eng
    torch.cuda.empty_cache()
    return {"agent_steps_per_sec": E * A * Te * n / dt, "t_inner": Te, "d2h_gbs": d2h * n / dt / 1e9}


def child(reps, e2e):
    import torch
    sys.path.insert(0, ROOT)
    from madrl_b200 import _lib
    fmts = {"fp32": torch.float32}
    if hasattr(_lib.lib(), "madrl_ww_set_obs_format"):
        fmts["bf16"] = torch.bfloat16
    rec = {}
    for wl in WORKLOADS:
        rates, bad = kernel_rates(wl, fmts, reps)
        rec[wl] = {"kernel": rates, "mismatch": bad}
        if e2e:
            rec[wl]["e2e"] = {f: e2e_rate(wl, dt) for f, dt in fmts.items()}
    print(json.dumps(rec), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build to time (PATH is loaded through MADRL_B200_LIB; 'NAME=' = the in-tree library)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10, help="timed launches per workload, format and round")
    ap.add_argument("--no-e2e", action="store_true", help="skip the host-buffer rates")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    sys.path.insert(0, ROOT)
    if a.child:
        return child(a.reps, not a.no_e2e)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("obs_bf16_rate.py needs a CUDA device")
    libs = [tuple(s.split("=", 1)) for s in a.lib] or [("new", "")]
    print("card:", json.dumps(card()), flush=True)
    res = {n: [] for n, _ in libs}
    failed = False
    for r in range(a.rounds):
        for n, path in libs:
            env = dict(os.environ)
            env.pop("MADRL_B200_LIB", None)
            if path:
                env["MADRL_B200_LIB"] = os.path.abspath(path)
            cmd = [sys.executable, os.path.abspath(__file__), "--child", "--reps", str(a.reps)]
            p = subprocess.run(cmd + (["--no-e2e"] if a.no_e2e else []), env=env, cwd=ROOT, capture_output=True, text=True)
            if p.returncode:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit("round %d, build %s failed" % (r, n))
            rec = json.loads(p.stdout.strip().splitlines()[-1])
            res[n].append(rec)
            for wl in WORKLOADS:
                for f, k in rec[wl]["kernel"].items():
                    line = "round %d %-8s %-14s %s: %.3f ms/launch, %.3f G agent-steps/s, %d B/env-step, %.0f GB/s" % (
                        r, n, wl, f, k["ms"], k["agent_steps_per_sec"] / 1e9, k["alg_bytes_per_env_step"], k["alg_gbs"])
                    if "e2e" in rec[wl]:
                        x = rec[wl]["e2e"][f]
                        line += "; e2e %.3f G agent-steps/s (D2H %.1f GB/s)" % (x["agent_steps_per_sec"] / 1e9, x["d2h_gbs"])
                    print(line, flush=True)
                if rec[wl]["mismatch"]:
                    print("MISMATCH %s %s: %s" % (n, wl, rec[wl]["mismatch"]), flush=True)
                    failed = True
    print("summary (median over %d rounds; spread = (max - min) / median):" % a.rounds)
    for n, _ in libs:
        for wl in WORKLOADS:
            for f in res[n][0][wl]["kernel"]:
                ms = sorted(rec[wl]["kernel"][f]["ms"] for rec in res[n])
                med = ms[len(ms) // 2]
                line = "  %-8s %-14s %s: kernel %.3f ms (spread %.1f%%)" % (n, wl, f, med, 100 * (ms[-1] - ms[0]) / med)
                if "e2e" in res[n][0][wl]:
                    e = sorted(rec[wl]["e2e"][f]["agent_steps_per_sec"] for rec in res[n])
                    line += ", e2e %.3f G agent-steps/s (spread %.1f%%)" % (e[len(e) // 2] / 1e9,
                                                                             100 * (e[-1] - e[0]) / e[len(e) // 2])
                print(line)
    if failed:
        raise SystemExit("bfloat16 observations are not the rounded float32 ones")


if __name__ == "__main__":
    main()
