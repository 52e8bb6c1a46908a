"""Waterworld's and Hostage's kernels on float32-exact scenes (tests/exact_scenes.py), at every instantiation their
launchers dispatch to (needs a GPU).

Each scene is one teacher-forced step from a hand-placed state at the exact ties, ranges, ray offsets, collision,
rebound and respawn thresholds and walls that the float32 teacher-forced tests exclude as fragile.  Every quantity
the reference compares is exact in float32 there, so nothing is excluded: observations equal the float64 oracle's
rounded to the observation type bit for bit (signed zeros included), and rewards, done, info, the post-step state
and the Philox counter are equal.  The in-kernel heuristic policy (POLICY) is held to the same check on its first
step, taken from an all-zero obs0 (so with zero actions), and the action it then computes from that step's sensing
to 1e-5 of the heuristic on the oracle's observation.  Which kernel each launch ran is read from the launch logs;
the last test runs every launch setting once and asserts that they reach exactly the instantiations written out
there."""
import numpy as np
import pytest
import torch

import exact_scenes as X
from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, _lib

pytestmark = pytest.mark.gpu

WW_TYPES = {"f32": (torch.float32, None), "bf16": (torch.float32, torch.bfloat16), "f64": (torch.float64, None)}


def logged(fam, fields, fn):
    L = _lib.lib()
    log = getattr(L, "madrl_%s_launch_log" % fam)
    assert log(1, None, 0) >= 0
    try:
        out = fn()
    finally:
        recs = np.zeros((64, fields), np.int32)
        n = log(0, recs.ctypes.data, 64)
    assert n == 1, n
    return out, tuple(recs[0, :-1].tolist())


def modes(scene, kind, opl, K):
    out = ["plain", "policy_agent", "policy_env"]
    if kind != "f64":
        out.append("keep")
    if kind == "f32" and X.writer_runs(scene, opl, K):
        out.append("writer")
    return out


def ww_run(scene, kind, opl, kch_kc, mode):
    K = X.K_OF[kch_kc]
    cfg, st, exp = X.ww_expect(scene, X.WW_N[opl], K)
    dtype, obs_dtype = WW_TYPES[kind]
    E = X.ww_envs(scene, K)
    eng = BatchedMAWaterWorld(E, **cfg, device="cuda", dtype=dtype, obs_dtype=obs_dtype, seed=X.SEED)
    s = eng.state
    for k, v in st.items():
        s[k].copy_(torch.as_tensor(np.asarray(v)).to(s[k].dtype).expand_as(s[k]))
    s["sensors"].copy_(torch.as_tensor(exp["S"].T.copy()).to(dtype))
    if mode == "keep":
        eng.set_obs_cache(_lib.OBS_CACHE_KEEP)
    eng.set_obs_writer(_lib.WW_OBS_WRITER_ON if mode == "writer" else _lib.WW_OBS_WRITER_OFF)
    where = (scene.name, kind, opl, kch_kc, mode)
    if mode.startswith("policy"):
        obs0 = torch.zeros((E, cfg["n_pursuers"], eng.obs_dim), dtype=obs_dtype or dtype, device="cuda")
        out, rec = logged("ww", 10, lambda: eng.rollout_heuristic(2, obs0, auto_reset=False, norm=mode[7:]))
        act, obs, rew, done, info = out
        act = act.cpu().numpy()
        assert not act[0].any(), where
        want = X.ww_heuristic(exp["obs"], exp["S"], mode[7:])
        assert np.abs(act[1, 0] - want).max() <= 1e-5, (where, act[1, 0], want)
    else:
        (obs, rew, done, info), rec = logged("ww", 10, lambda: eng.rollout(
            torch.zeros((1, E, cfg["n_pursuers"], 2), dtype=dtype, device="cuda"), auto_reset=False))
    ob = obs[0, 0]
    ob = ob.view(torch.int16).cpu().numpy().view(np.uint16) if kind == "bf16" else ob.cpu().numpy()
    X.check_obs(where, ob, exp, kind)
    X.check_step(where, exp, rew[0, 0].cpu().numpy(), done[0, 0].item(), info[0, 0].cpu().numpy(), kind)
    if not mode.startswith("policy"):
        s = {k: v.cpu().numpy() for k, v in eng.state.items()}
        X.check_state(where, exp, np.stack([s["pos_x"][0], s["pos_y"][0]], 1),
                      np.stack([s["vel_x"][0], s["vel_y"][0]], 1), s["rng_counter"][0], kind)
    return rec


@pytest.mark.parametrize("kch_kc", list(X.K_OF), ids=lambda p: "kch%d_kc%d" % p)
@pytest.mark.parametrize("opl", [1, 2, 4, 8])
@pytest.mark.parametrize("kind", list(WW_TYPES))
def test_waterworld_exact_scenes(kind, opl, kch_kc):
    for scene in X.WW_SCENES:
        for mode in modes(scene, kind, opl, X.K_OF[kch_kc]):
            rec = ww_run(scene, kind, opl, kch_kc, mode)
            assert rec[2:5] == (opl,) + kch_kc and rec[8] == (mode == "writer"), (scene, mode, rec)


HW_TYPES = {"f64": (torch.float64, None, False), "f32": (torch.float32, None, False),
            "f32_keep": (torch.float32, None, True), "bf16": (torch.float32, torch.bfloat16, False),
            "bf16_keep": (torch.float32, torch.bfloat16, True)}


@pytest.mark.parametrize("kch_kc", list(X.K_OF), ids=lambda p: "kch%d_kc%d" % p)
@pytest.mark.parametrize("opl", [1, 2, 4, 8])
@pytest.mark.parametrize("htype", list(HW_TYPES))
def test_hostage_exact_scenes(htype, opl, kch_kc):
    for scene in X.HW_SCENES:
        hw_run(scene, htype, opl, kch_kc)


def hw_run(scene, htype, opl, kch_kc):
    dtype, obs_dtype, keep = HW_TYPES[htype]
    kind = htype.split("_")[0]
    K = X.K_OF[kch_kc]
    args, kw, st, exp = X.hw_expect(scene, X.HW_N[opl], K)
    eng = BatchedHostageWorld(1, *args, **kw, device="cuda", dtype=dtype, obs_dtype=obs_dtype, seed=X.SEED)
    s = eng.state
    for k, v in st.items():
        s[k].copy_(torch.as_tensor(np.asarray(v)).to(s[k].dtype).expand_as(s[k]))
    eng._view(eng.layout.sensors, dtype, (2, K)).copy_(torch.as_tensor(exp["S"].T.copy()).to(dtype))
    if keep:
        eng.set_obs_cache(_lib.OBS_CACHE_KEEP)
    where = (scene.name, htype, opl, kch_kc)
    (obs, rew, done, info), rec = logged("hostage", 7, lambda: eng.rollout(
        torch.zeros((1, 1, args[0], 2), dtype=dtype, device="cuda"), auto_reset=False))
    assert rec[2:6] == (opl,) + kch_kc + (int(keep),), (where, rec)
    ob = obs[0, 0]
    ob = ob.view(torch.int16).cpu().numpy().view(np.uint16) if kind == "bf16" else ob.cpu().numpy()
    X.check_obs(where, ob, exp, kind)
    X.check_step(where, exp, rew[0, 0].cpu().numpy(), done[0, 0].item(), info[0, 0].cpu().numpy(), kind)
    s = {k: v.cpu().numpy() for k, v in eng.state.items()}
    X.check_state(where, exp, np.stack([s["pos_x"][0], s["pos_y"][0]], 1),
                  np.stack([s["vel_x"][0], s["vel_y"][0]], 1), s["rng_counter"][0], kind)
    assert int(s["flags"][0]) == exp["flags"] and np.array_equal(s["saved"][0].astype(bool), exp["saved"]), where
    return rec


def test_launch_logs_name_every_instantiation():
    """Every launch setting the tests above use, on one scene each (the two-pursuer scene, whose whole env-step the
    writer-warp kernel stages at every sensor layout), runs exactly these instantiations, as the launch logs record
    them: (sizeof(real), sizeof(O), OPL, KCH, KC, PEER, POLICY, KEEP, WRITER) for ww_kernel, (sizeof(real),
    sizeof(O), OPL, KCH, KC, KEEP) for hw_kernel."""
    pairs = [(opl, kch, kc) for opl in (1, 2, 4, 8) for kch, kc in ((1, 30), (1, 0), (2, 0))]
    ww = set()
    for opl, kch, kc in pairs:
        for r, o in ((4, 4), (4, 2), (8, 8)):
            ww |= {(r, o, opl, kch, kc, 0, pol, 0, 0) for pol in (0, 1, 2)}
            if r == 4:
                ww.add((r, o, opl, kch, kc, 0, 0, 1, 0))
    ww |= {(4, 4, 1, kch, kc, 0, 0, 0, 1) for kch, kc in ((1, 30), (1, 0), (2, 0))}   # the writer-warp kernel
    hw = {(r, o, opl, kch, kc, keep) for opl, kch, kc in pairs
          for r, o, keep in ((8, 8, 0), (4, 4, 0), (4, 4, 1), (4, 2, 0), (4, 2, 1))}
    assert len(ww) == 12 * 11 + 3 and len(hw) == 60
    scene = next(s for s in X.WW_SCENES if s.name == "np2_corner_ties")
    got = {ww_run(scene, kind, opl, (kch, kc), mode) for kind in WW_TYPES for opl, kch, kc in pairs
           for mode in modes(scene, kind, opl, X.K_OF[(kch, kc)])}
    assert got == ww, (sorted(ww - got), sorted(got - ww))
    got = {hw_run(X.HW_SCENES[0], htype, opl, (kch, kc)) for htype in HW_TYPES for opl, kch, kc in pairs}
    assert got == hw, (sorted(hw - got), sorted(got - hw))
