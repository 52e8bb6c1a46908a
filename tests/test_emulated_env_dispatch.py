"""Pursuit's and Hostage's rollout kernels at every instantiation their launchers dispatch to, run by the warp
emulator of tests/emu on the CPU: the case table of tests/env_dispatch_edges.py at E = 3 (the emulated device
runs 2 warps, so one warp steps two envs), against the oracles over whole auto-reset trajectories cut into two
launches, with the launch log checked first.  tests/test_env_dispatch_edges_gpu.py runs the same table on the
device."""
import numpy as np
import pytest

import env_dispatch_edges as D
from emu import driver
from emu.driver import Guarded
from emu.driver import ptr as _p
from teacher_forced import EmuAdapter

pytestmark = driver.needs_cxx

E = 3


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


def read_log(lib, fam, fields):
    """Records of madrl_<fam>_launch_log since it was last read, without their grids; the log is left off."""
    recs = np.zeros((4096, fields), np.int32)
    n = getattr(lib, "madrl_%s_launch_log" % fam)(0, _p(recs), 4096)
    assert 0 <= n <= 4096
    return [tuple(r[:-1]) for r in recs[:n].tolist()]


def log_on(lib, fam):
    assert getattr(lib, "madrl_%s_launch_log" % fam)(1, None, 0) >= 0


def split_rollout(eng, act, fam, term):
    """rollout(act) as two launches (a third, then the rest) with auto-reset, terminal observations into `term`
    (NaN where nothing was kept)."""
    T1 = max(1, act.shape[0] // 3)
    outs = []
    for a, tm in ((act[:T1], term[:T1]), (act[T1:], term[T1:])):
        assert getattr(eng.lib, "madrl_%s_set_terminal_obs" % fam)(eng._h, _p(tm)) == 0
        outs.append(eng.rollout(a, auto_reset=True))
    assert getattr(eng.lib, "madrl_%s_set_terminal_obs" % fam)(eng._h, None) == 0
    return [np.concatenate(x) for x in zip(*outs)]


# ------------------------------------------------------------------------------------------------ Hostage
@pytest.mark.parametrize("case", D.H_CASES, ids=repr)
def test_emulated_hostage_dispatch_matches_oracle(case):
    from emu.driver import EmuHostage
    seed, base, mpl, T = 321, 77, 7, min(case.T, 20)
    eng = EmuHostage(E, *case.args, seed=seed, env_id_base=base, max_path_length=mpl, **case.kw)
    log_on(eng.lib, "hostage")
    obs0 = eng.reset()
    act = D.hw_actions(case, E, T)
    term = np.ascontiguousarray(np.full((T, E, case.Nr, eng.obs_dim), np.nan))
    obs, rew, done, info = split_rollout(eng, act, "hostage", term)
    assert read_log(eng.lib, "hostage", 7) == [D.hw_record(case, 8, 8, 0)] * 3
    oracles = D.hw_oracles(case, seed, base, E)
    D.hw_check_trajectory(case, oracles, obs0, act, obs, rew, done, info, mpl, term)
    D.hw_check_state(case, EmuAdapter(eng, "hw").read(), oracles)
    D.hw_check_reach(case, oracles)


# ------------------------------------------------------------------------------------------------ Pursuit
def pe_state(eng):
    Ly, Np, Ne, R = eng.layout, eng.n_pursuers, eng.n_evaders, eng.cfg.obs_range
    pos = eng.view(Ly.pos, np.uint8, (E, 2, Np + Ne))
    return dict(pursuer_x=pos[:, 0, :Np], pursuer_y=pos[:, 1, :Np], evader_x=pos[:, 0, Np:], evader_y=pos[:, 1, Np:],
                gone=eng.view(Ly.gone, np.int64, (E,)), map_id=eng.view(Ly.map_id, np.int32, (E,)),
                rng_counter=eng.view(Ly.rng_counter, np.int64, (E,)),
                stale=eng.view(Ly.stale, np.int16, (E, Np, R * R)))


@pytest.mark.parametrize("case", D.P_CASES, ids=repr)
def test_emulated_pursuit_dispatch_matches_oracle(case):
    from emu.driver import EmuPursuit
    seed, base, mpl, T = 77, 500, 9, min(case.T, 20)
    maps = case.maps()
    eng = EmuPursuit(E, maps, seed=seed, env_id_base=base, max_path_length=mpl, **case.cfg)
    log_on(eng.lib, "pursuit")
    obs0 = eng.reset()
    act = D.pe_actions(case, E, T)
    term = np.full((T, E, case.Np, eng.obs_dim), np.nan, np.float32)
    obs, rew, done, removed = split_rollout(eng, act, "pursuit", term)
    assert read_log(eng.lib, "pursuit", 8) == [D.pe_record(case, 4, 0, 0)] * 3
    oracles = D.pe_oracles(case, maps, seed, base, E)
    D.pe_check_trajectory(case, oracles, obs0, act, obs, rew, done, removed, mpl, term)
    D.pe_check_state(case, pe_state(eng), oracles)


# ------------------------------------------------------------------------------------------------ launch logs
def _launch(eng, fam, obs_bytes, T=1):
    """One rollout launch of T steps into scratch buffers (any observation element size)."""
    A = eng.n_agents
    act = np.zeros((T, eng.n_envs, A) + eng.act_shape, eng.act_dtype)
    obs = np.zeros(T * eng.n_envs * A * eng.obs_dim * obs_bytes, np.uint8)
    rew = np.zeros((T, eng.n_envs, A), np.float64)
    done, info = np.zeros((T, eng.n_envs), np.uint8), np.zeros((T, eng.n_envs, 2), np.int32)
    assert getattr(eng.lib, "madrl_%s_rollout" % fam)(eng._h, T, _p(act), _p(obs), _p(rew), _p(done), _p(info), 1,
                                                     None) == 0


def test_emulated_dispatch_reaches_every_instantiation():
    """Every case launched with every element type, store policy and (Pursuit) the heuristic policy: the logged
    instantiations are exactly the 60 Hostage and 96 Pursuit kernels the dispatchers can reach."""
    from emu.driver import EmuHostage, EmuPursuit
    lib = driver.load()
    log_on(lib, "hostage")
    for case in D.H_CASES:
        for fp64 in (True, False):
            eng = EmuHostage(1, *case.args, fp64=fp64, **case.kw)
            for fmt, cache, ob in ((0, 0, 8 if fp64 else 4), (0, 1, 4), (1, 0, 2), (1, 1, 2)):
                if fp64 and (fmt or cache):
                    continue
                assert lib.madrl_hostage_set_obs_format(eng._h, fmt) == 0
                assert lib.madrl_hostage_set_obs_cache(eng._h, cache) == 0
                _launch(eng, "hostage", ob)
    assert set(read_log(lib, "hostage", 7)) == D.HW_ALL
    log_on(lib, "pursuit")
    for case in D.P_CASES:
        eng = EmuPursuit(1, case.maps(), **case.cfg)
        for fmt, ob in ((0, 4), (1, 2)):
            assert lib.madrl_pursuit_set_obs_format(eng._h, fmt) == 0
            for cache in (0, 1):
                assert lib.madrl_pursuit_set_obs_cache(eng._h, cache) == 0
                _launch(eng, "pursuit", ob)
            obs0, obs = [np.zeros(eng.n_agents * eng.obs_dim * ob, np.uint8) for _ in range(2)]
            rew, done, info = np.zeros(eng.n_agents, np.float32), np.zeros(1, np.uint8), np.zeros(1, np.int32)
            assert lib.madrl_pursuit_rollout_heuristic(eng._h, 1, _p(obs0), None, _p(obs), _p(rew), _p(done), _p(info),
                                                       1, 1, None) == 0
    assert set(read_log(lib, "pursuit", 8)) == D.PE_ALL


def test_emulated_pursuit_and_hostage_launch_logs():
    """madrl_pursuit_launch_log and madrl_hostage_launch_log keep madrl_ww_launch_log's contract: one record per
    launch with its grid, a count that includes launches past the caller's buffer, nothing while off, and
    MADRL_EINVAL for a missing buffer.  The three logs are separate."""
    from emu.driver import EmuHostage, EmuPursuit, EmuWaterworld
    hw = EmuHostage(3, *D.H_BY_NAME["o8_k30"].args, **D.H_BY_NAME["o8_k30"].kw)
    case = D.P_BY_NAME["e2_c2_conv"]
    pe = EmuPursuit(3, case.maps(), **case.cfg)
    ww = EmuWaterworld(3, n_pursuers=5, n_evaders=5)
    lib = hw.lib
    for fam, fields in (("hostage", 7), ("pursuit", 8), ("ww", 10)):
        assert getattr(lib, "madrl_%s_launch_log" % fam)(1, None, 0) >= 0
    hw.reset()
    hw.rollout(np.zeros((2, 3, 1, 2)))
    pe.reset()
    recs = Guarded((2, 8), np.int32, -9)
    assert lib.madrl_ww_launch_log(0, None, 0) == 0
    assert lib.madrl_pursuit_launch_log(1, _p(recs.arr), 1) == 1
    # EPL 2, CPL 2, runtime R, rollout, conv layout, streaming stores; the emulated device's grid is 2 warps
    assert recs.check("records").tolist() == [[4, 2, 2, 0, 0, 0, 0, 2], [-9] * 8]
    hrec = Guarded((3, 7), np.int32, -9)
    assert lib.madrl_hostage_launch_log(0, _p(hrec.arr), 1) == 2
    assert hrec.check("records").tolist() == [[8, 8, 8, 1, 30, 0, 2]] + [[-9] * 7] * 2
    hw.rollout(np.zeros((1, 3, 1, 2)))
    ww.reset()
    assert lib.madrl_hostage_launch_log(0, None, 0) == 0 and lib.madrl_ww_launch_log(0, None, 0) == 0
    pe.rollout(np.zeros((1, 3, case.Np), np.int32))
    assert lib.madrl_pursuit_launch_log(0, None, 0) == 1
    for fam in ("hostage", "pursuit"):
        assert getattr(lib, "madrl_%s_launch_log" % fam)(0, None, 1) == -1
        assert getattr(lib, "madrl_%s_launch_log" % fam)(0, None, -1) == -1
