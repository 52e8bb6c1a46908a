"""Waterworld's and Hostage's kernels on float32-exact scenes (tests/exact_scenes.py), in the warp emulator of
tests/emu: the float32 and fp64 builds at every (OPL, KCH, KC) the launchers dispatch to, the writer-warp kernel and
both norms of the in-kernel heuristic policy.  The checks are tests/test_exact_ties_gpu.py's: nothing is excluded,
observations equal the float64 oracle's bit for bit, and so do rewards, done, info, the post-step state and the
Philox counter."""
import numpy as np
import pytest

import exact_scenes as X
from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)
from emu import driver
from madrl_b200 import _lib as L

pytestmark = driver.needs_cxx


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


def _p(a):
    return driver.ptr(a)


def launch_record(lib, fam, fields, fn):
    log = getattr(lib, "madrl_%s_launch_log" % fam)
    assert log(1, None, 0) >= 0
    out = fn()
    recs = np.zeros((64, fields), np.int32)
    assert log(0, _p(recs), 64) == 1
    return out, tuple(recs[0, :-1].tolist())


def write(eng, st, S, family):
    """The scene's state into every env of `eng` (env 0 is checked)."""
    g, Ly, E = eng, eng.layout, eng.n_envs
    N = int(Ly.n_obj)
    objs = g.view(Ly.objs, g.obs_dtype, (E, 4, N))
    objs[:] = np.stack([st["pos_x"], st["pos_y"], st["vel_x"], st["vel_y"]])
    g.view(Ly.timestep, np.int32, (E,))[:] = st["timestep"]
    g.view(Ly.rng_counter, np.int64, (E,))[:] = st["rng_counter"]
    g.view(Ly.sensors, g.obs_dtype, (2, len(S)))[:] = S.T
    if family == "ww":
        g.view(Ly.obst, g.obs_dtype, (E, 2))[:] = (st["obst_x"], st["obst_y"])
    else:
        fixed = g.view(Ly.fixed, g.obs_dtype, (E, 4))
        fixed[:, 0:2], fixed[:, 2:4] = st["key"], st["bomb"]
        g.view(Ly.flags, np.int32, (E,))[:] = st["flags"]
        g.view(Ly.saved, np.uint8, (E, g.n_hostages))[:] = st["saved"]


def post(eng):
    Ly, E = eng.layout, eng.n_envs
    objs = eng.view(Ly.objs, eng.obs_dtype, (E, 4, int(Ly.n_obj)))[0]
    return objs[0:2].T.copy(), objs[2:4].T.copy(), int(eng.view(Ly.rng_counter, np.int64, (E,))[0])


def ww_modes(scene, kind, opl, K):
    if kind == "f64":
        return ["plain"]
    return ["plain", "policy_agent", "policy_env"] + (["writer"] if X.writer_runs(scene, opl, K) else [])


@pytest.mark.parametrize("kch_kc", list(X.K_OF), ids=lambda p: "kch%d_kc%d" % p)
@pytest.mark.parametrize("opl", [1, 2, 4, 8])
@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_waterworld_exact_scenes(kind, opl, kch_kc):
    K = X.K_OF[kch_kc]
    for scene in X.WW_SCENES:
        cfg, st, exp = X.ww_expect(scene, X.WW_N[opl], K)
        for mode in ww_modes(scene, kind, opl, K):
            E = X.ww_envs(scene, K)
            eng = driver.EmuWaterworld(E, fp64=kind == "f64", seed=X.SEED, **cfg)
            write(eng, st, exp["S"], "ww")
            assert eng.lib.madrl_ww_set_obs_writer(eng._h, L.WW_OBS_WRITER_ON if mode == "writer"
                                                   else L.WW_OBS_WRITER_OFF) == 0
            where = (scene.name, kind, opl, kch_kc, mode)
            Np = cfg["n_pursuers"]
            if mode.startswith("policy"):
                norm = L.HEURISTIC_NORM_ENV if mode == "policy_env" else L.HEURISTIC_NORM_AGENT
                assert eng.lib.madrl_ww_set_heuristic_norm(eng._h, norm) == 0
                obs0 = np.zeros((E, Np, eng.obs_dim), eng.obs_dtype)
                (act, obs, rew, done, info), rec = launch_record(
                    eng.lib, "ww", 10, lambda: eng.rollout_heuristic(2, obs0, auto_reset=False))
                assert not act[0].any(), where
                want = X.ww_heuristic(exp["obs"], exp["S"], mode[7:])
                assert np.abs(act[1, 0] - want).max() <= 1e-5, (where, act[1, 0], want)
            else:
                (obs, rew, done, info), rec = launch_record(
                    eng.lib, "ww", 10, lambda: eng.rollout(np.zeros((1, E, Np, 2)), auto_reset=False))
            assert rec[2:5] == (opl,) + kch_kc and rec[8] == (mode == "writer"), (where, rec)
            X.check_obs(where, obs[0, 0], exp, kind)
            X.check_step(where, exp, rew[0, 0], done[0, 0], info[0, 0], kind)
            if not mode.startswith("policy"):
                X.check_state(where, exp, *post(eng), kind)


@pytest.mark.parametrize("kch_kc", list(X.K_OF), ids=lambda p: "kch%d_kc%d" % p)
@pytest.mark.parametrize("opl", [1, 2, 4, 8])
@pytest.mark.parametrize("kind", ["f32", "f64"])
def test_hostage_exact_scenes(kind, opl, kch_kc):
    K = X.K_OF[kch_kc]
    for scene in X.HW_SCENES:
        args, kw, st, exp = X.hw_expect(scene, X.HW_N[opl], K)
        eng = driver.EmuHostage(1, *args, fp64=kind == "f64", seed=X.SEED, **kw)
        write(eng, st, exp["S"], "hw")
        where = (scene.name, kind, opl, kch_kc)
        (obs, rew, done, info), rec = launch_record(
            eng.lib, "hostage", 7, lambda: eng.rollout(np.zeros((1, 1, args[0], 2)), auto_reset=False))
        assert rec[2:5] == (opl,) + kch_kc, (where, rec)
        X.check_obs(where, obs[0, 0], exp, kind)
        X.check_step(where, exp, rew[0, 0], done[0, 0], info[0, 0], kind)
        X.check_state(where, exp, *post(eng), kind)
        Ly = eng.layout
        assert int(eng.view(Ly.flags, np.int32, (1,))[0]) == exp["flags"], where
        assert np.array_equal(eng.view(Ly.saved, np.uint8, (1, eng.n_hostages))[0].astype(bool), exp["saved"]), where
