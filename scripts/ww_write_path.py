"""Waterworld observation write path against the card's streaming-write rate (one GPU command).

    python scripts/ww_write_path.py [--lib NAME=PATH ...] [--rounds R] [--blocks-per-sm N ...]
                                    [--obs-writer MODE ...] [--envs E1,E2,...]

Prints the card (name, power limit, SM clock), then times with CUDA events
  * `fill_` of a float32 tensor the size of one headline launch's observations ([256, 4096, 5, 213]):
    the rate at which this card streams writes to HBM, the ceiling of a kernel that mostly writes;
  * the headline rollout (C2: 4096 envs, 5 pursuers, T = 256) and C4 (4096 envs, 20 pursuers, T = 64),
    reported as kernel time and observation bytes / kernel time next to the fill rate.
Every `--lib` build (default: the library MADRL_B200_LIB names, else the in-tree one; a PATH is loaded
through MADRL_B200_LIB, e.g. one made by scripts/build_variant.py from another checkout) is timed in a
child process of its own, the builds alternating for R rounds, and the median and min-max spread over
the rounds are printed per build.  Each `--blocks-per-sm N` times every build once more with the
persistent wave capped at N one-warp blocks per SM (engine.set_launch): at N = 16 each warp steps about
two envs in turn, which shows how much of a warp's time the other resident warps can absorb.  Each
`--obs-writer on|off` times every build once more with that Waterworld observation write path
(set_obs_writer; builds without the entry point are timed as they are).  `--envs` times C2 at these batch sizes
instead of 4096 only (the sizes scripts/ww_launch_cap.py uses: 2200,2640,3000,4096,6000,8192).  The writer-warp
kernel's geometry is compiled in (MADRL_WW_WRITER_* in csrc/waterworld.cu): its sweep is a list of `--lib` builds
made with scripts/build_variant.py NAME -DMADRL_WW_WRITER_SLOTS=3 ...
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHAPES = {"c2": dict(cfg=dict(n_pursuers=5, n_evaders=5, n_poison=10, n_sensors=30), E=4096, T=256),
          "c4": dict(cfg=dict(n_pursuers=20, n_evaders=50, n_poison=50, n_sensors=30), E=4096, T=64)}
WRITER_MODES = {"auto": 0, "off": 1, "on": 2}   # MADRL_WW_OBS_WRITER_*


def shapes(envs):
    """The timed shapes: C2 at each batch size of `envs` (named c2 at 4096, c2@E otherwise), then C4."""
    out = {}
    for E in envs:
        out["c2" if E == 4096 else "c2@%d" % E] = dict(SHAPES["c2"], E=E)
    out["c4"] = SHAPES["c4"]
    return out


def card():
    import torch
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.strip().split(",")]))
    except (OSError, subprocess.SubprocessError):
        return {"name": torch.cuda.get_device_name(), "power.limit": "unknown", "clocks.sm": "unknown"}


def event_ms(fn, warmup, reps):
    """Median over `reps` calls of fn's device time (CUDA events around each call)."""
    import torch
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(reps)]
    for s, e in ev:
        s.record()
        fn()
        e.record()
    torch.cuda.synchronize()
    return sorted(s.elapsed_time(e) for s, e in ev)[reps // 2]


def fill_rate(reps):
    import torch
    x = torch.empty((256, 4096, 5, 213), dtype=torch.float32, device="cuda")
    ms = event_ms(lambda: x.fill_(1.0), 3, reps)
    nbytes = x.numel() * 4
    del x
    torch.cuda.empty_cache()
    return {"bytes": nbytes, "ms": ms, "gbs": nbytes / (ms * 1e-3) / 1e9}


def rollout_rate(s, reps, bps, writer):
    import torch
    sys.path.insert(0, ROOT)
    from madrl_b200 import BatchedMAWaterWorld, _lib
    E, T, Np = s["E"], s["T"], s["cfg"]["n_pursuers"]
    eng = BatchedMAWaterWorld(E, device="cuda", seed=0, **s["cfg"])
    eng.set_launch(blocks_per_sm=bps)
    if writer != "auto" and hasattr(_lib.lib(), "madrl_ww_set_obs_writer"):
        eng.set_obs_writer(WRITER_MODES[writer])
    eng.reset()
    g = torch.Generator(device="cuda")
    g.manual_seed(1234)
    act = torch.randn(T, E, Np, 2, device="cuda", generator=g) * 0.5
    out = (torch.empty((T, E, Np, eng.obs_dim), device="cuda"), torch.empty((T, E, Np), device="cuda"),
           torch.empty((T, E), dtype=torch.uint8, device="cuda"), torch.empty((T, E, 2), dtype=torch.int32, device="cuda"))
    ms = event_ms(lambda: eng.rollout(act, auto_reset=True, out=out), 3, reps)
    obs_bytes = out[0].numel() * 4
    return {"ms": ms, "obs_bytes": obs_bytes, "obs_gbs": obs_bytes / (ms * 1e-3) / 1e9,
            "agent_steps_per_sec": E * Np * T / (ms * 1e-3)}


def child(reps, bps, writer, envs):
    print(json.dumps({n: rollout_rate(s, reps, bps, writer) for n, s in shapes(envs).items()}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", action="append", default=[], metavar="NAME=PATH",
                    help="a build to time (PATH is loaded through MADRL_B200_LIB; 'NAME=' = the in-tree library)")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10, help="timed launches per shape and round")
    ap.add_argument("--blocks-per-sm", type=int, action="append", default=[], metavar="N",
                    help="also time with at most N resident blocks per SM (0 = the library default)")
    ap.add_argument("--obs-writer", action="append", default=[], choices=["on", "off"],
                    help="also time with this Waterworld observation write path (set_obs_writer)")
    ap.add_argument("--envs", default="4096", help="C2 batch sizes")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--bps", type=int, default=0, help=argparse.SUPPRESS)
    ap.add_argument("--writer", default="auto", help=argparse.SUPPRESS)
    a = ap.parse_args()
    envs = [int(x) for x in a.envs.split(",")]
    if a.child:
        return child(a.reps, a.bps, a.writer, envs)
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("ww_write_path.py needs a CUDA device")
    libs = [tuple(s.split("=", 1)) for s in a.lib] or [("default", os.environ.get("MADRL_B200_LIB", ""))]
    # one timed build per (library, blocks per SM, write path); bps 0 and "auto" = the default launch, named by the
    # library alone
    libs = [(n + ("" if b == 0 else "@%d" % b) + ("" if w == "auto" else "/" + w), path, b, w)
            for w in ["auto"] + a.obs_writer for b in [0] + a.blocks_per_sm for n, path in libs]
    timed = shapes(envs)
    print("card:", json.dumps(card()))
    fill = fill_rate(20)
    print("fill_ float32 %.2f GB: %.3f ms, %.1f GB/s (streaming-write rate)" % (fill["bytes"] / 1e9, fill["ms"], fill["gbs"]))
    res = {n: {s: [] for s in timed} for n, _, _, _ in libs}
    for r in range(a.rounds):
        for n, path, bps, w in libs:
            env = dict(os.environ)
            env.pop("MADRL_B200_LIB", None)
            if path:
                env["MADRL_B200_LIB"] = os.path.abspath(path)
            p = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--reps", str(a.reps),
                                "--bps", str(bps), "--writer", w, "--envs", a.envs],
                               env=env, cwd=ROOT, capture_output=True, text=True)
            if p.returncode:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit("round %d, build %s failed" % (r, n))
            rec = json.loads(p.stdout.strip().splitlines()[-1])
            for s in timed:
                res[n][s].append(rec[s])
                print("round %d %-11s %s: %.3f ms/launch, obs %.1f GB/s (%.1f%% of fill), %.3g agent-steps/s"
                      % (r, n, s, rec[s]["ms"], rec[s]["obs_gbs"], 100 * rec[s]["obs_gbs"] / fill["gbs"],
                         rec[s]["agent_steps_per_sec"]), flush=True)
    print("summary (median over %d rounds; spread = (max - min) / median of the launch time):" % a.rounds)
    for n, _, _, _ in libs:
        for s in timed:
            ms = sorted(x["ms"] for x in res[n][s])
            med = ms[len(ms) // 2]
            gbs = res[n][s][0]["obs_bytes"] / (med * 1e-3) / 1e9
            print("  %-11s %s: %.3f ms (spread %.1f%%), obs %.1f GB/s = %.1f%% of the fill rate"
                  % (n, s, med, 100 * (ms[-1] - ms[0]) / med, gbs, 100 * gbs / fill["gbs"]))


if __name__ == "__main__":
    main()
