"""Pursuit's evader-control (EVC) kernels run by the warp emulator of tests/emu on the CPU: both layouts, the
heuristic policy on and off, one and two chunks of evader lanes, resets inside the launch.  A launch fed the random
controller's own actions equals the random launch bit for bit (state included); fixed and per-step actions and
model_state follow the oracle.  tests/test_pursuit_evaders_gpu.py runs the same checks on the device."""
import numpy as np
import pytest

import env_dispatch_edges as D
import pursuit_evaders_edges as V
from emu import driver
from emu.driver import Guarded
from emu.driver import ptr as _p

pytestmark = driver.needs_cxx

E, SEED, BASE, MPL = 3, 41, 900, 6
# EPL 1 flat; EPL 1 conv with surround captures; EPL 2 flat on one cell (every evader caught at once); EPL 2 conv
# with random_opponents
CASES = ["e1_c1_flat", "e1_c2_conv", "e2_c1_flat", "e2_c2_conv"]


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


def make(case, **kw):
    from emu.driver import EmuPursuit
    return EmuPursuit(E, case.maps(), seed=SEED, env_id_base=BASE, max_path_length=MPL, **dict(case.cfg, **kw))


def state(eng):
    Ly = eng.layout
    return eng.view(Ly.rng_counter, np.int64, (E,)).copy(), eng.view(Ly.gone, np.int64, (E,)).copy()


def model_state_buffer(eng):
    ms = Guarded((E, 4, eng.cfg.xs, eng.cfg.ys), np.float32, np.nan)
    assert eng.lib.madrl_pursuit_set_model_state(eng._h, _p(ms.arr)) == 0
    return ms


def launch(eng, policy, T, act, obs0, ev=None, strides=None):
    """One launch of T steps: open loop with `act`, or the heuristic from `obs0`; evaders from `ev` [T, E, Ne]
    (strides as given, or the array's own) or the handle's controller -> (actions, obs, rew, done, info)."""
    Np, D_ = eng.n_agents, eng.obs_dim
    bufs = [Guarded((T, E, Np), np.int32, -7), Guarded((T, E, Np, D_), np.float32, np.nan),
            Guarded((T, E, Np), np.float32, np.nan), Guarded((T, E), np.uint8, 255), Guarded((T, E), np.int32, -1)]
    outs = [_p(b.arr) for b in bufs[1:]]
    if ev is not None:
        st, se = strides if strides is not None else (ev.strides[0] // 4, ev.strides[1] // 4)
    if policy:
        obs0 = np.ascontiguousarray(obs0, np.float32)
        if ev is None:
            rc = eng.lib.madrl_pursuit_rollout_heuristic(eng._h, T, _p(obs0), _p(bufs[0].arr), *outs, 1, 1, None)
        else:
            rc = eng.lib.madrl_pursuit_rollout_heuristic_evaders(eng._h, T, _p(obs0), _p(bufs[0].arr), _p(ev), st, se,
                                                                 *outs, 1, 1, None)
    else:
        act = np.ascontiguousarray(act, np.int32)
        bufs[0].arr[...] = act
        if ev is None:
            rc = eng.lib.madrl_pursuit_rollout(eng._h, T, _p(act), *outs, 1, None)
        else:
            rc = eng.lib.madrl_pursuit_rollout_evaders(eng._h, T, _p(act), _p(ev), st, se, *outs, 1, None)
    eng._check(rc)
    return tuple(b.check(n) for b, n in zip(bufs, ("actions", "obs", "rew", "done", "info")))


def read_log(lib):
    recs = np.zeros((64, 8), np.int32)
    n = lib.madrl_pursuit_launch_log(0, _p(recs), 64)
    return [tuple(r[:-1]) for r in recs[:n].tolist()]


@pytest.mark.parametrize("policy", [0, 1], ids=["open", "heuristic"])
@pytest.mark.parametrize("name", CASES)
def test_emulated_random_actions_reproduce_random_launch(name, policy):
    """Step by step with the random controller, reading each step's actions off the stream; then one launch of all
    T steps fed those actions through the EVC kernel: the same trajectory and the same state blob.  Its
    model_state is the oracle's after the same steps."""
    case = D.P_BY_NAME[name]
    T = 14
    act = D.pe_actions(case, E, T)
    a = make(case)
    obs0 = a.reset()
    ev = np.zeros((T, E, case.Ne), np.int32)
    outs, prev = [], obs0
    for t in range(T):
        ctr, gone = state(a)
        ev[t] = V.random_evader_actions(SEED, BASE, ctr, gone, case.Ne, fill_seed=t)
        o = launch(a, policy, 1, act[t:t + 1], prev)
        outs.append(o)
        prev = o[1][0]
    want = [np.concatenate(x) for x in zip(*outs)]

    b = make(case)
    ms = model_state_buffer(b)
    assert b.lib.madrl_pursuit_launch_log(1, None, 0) >= 0
    assert np.array_equal(b.reset(), obs0)
    got = launch(b, policy, T, act, obs0, ev=ev)
    assert read_log(b.lib) == [(4, case.inst[0], case.inst[1], case.inst[2], 2, case.flat, 0),
                               (4, case.inst[0], case.inst[1], case.inst[2], 2 | policy, case.flat, 0)]
    for w, g, n in zip(want, got, ("actions", "obs", "rew", "done", "info")):
        assert np.array_equal(w, g, equal_nan=True), n
    assert np.array_equal(a.blob, b.blob)

    oracles = V.pe_oracles(case, case.maps(), SEED, BASE, E)
    for o in oracles:
        o.reset()
    V.oracle_trajectory(oracles, got[0], ev, MPL)
    m = ms.check("model_state")
    for e, o in enumerate(oracles):
        assert np.array_equal(m[e], o.model_state), e


@pytest.mark.parametrize("name", ["e1_c2_conv", "e2_c2_conv"])
def test_emulated_fixed_controller(name):
    """SingleActionPolicy(a): the handle's fixed mode, one row of actions read with strides 0 and 0, and an explicit
    [T, E, Ne] tensor all give the oracle's trajectory (whose draws are consumed, unused)."""
    case = D.P_BY_NAME[name]
    T, a_fix = 10, 1
    act = D.pe_actions(case, E, T, seed=3)
    oracles = V.pe_oracles(case, case.maps(), SEED, BASE, E)
    obs0 = np.array([[D.f32(x).reshape(-1) for x in o.reset()] for o in oracles])
    full = np.full((T, E, case.Ne), a_fix, np.int32)
    w_obs, w_rew, w_done, w_rem = V.oracle_trajectory(oracles, act, full, MPL)
    row = np.full(case.Ne, a_fix, np.int32)
    runs = []
    for kind in ("fixed", "row", "full"):
        eng = make(case)
        assert np.array_equal(eng.reset().reshape(obs0.shape), obs0)
        if kind == "fixed":
            assert eng.lib.madrl_pursuit_set_evader_control(eng._h, 1, a_fix) == 0
            runs.append(launch(eng, 0, T, act, None))
        elif kind == "row":
            runs.append(launch(eng, 0, T, act, None, ev=row, strides=(0, 0)))
        else:
            runs.append(launch(eng, 0, T, act, None, ev=full))
        runs[-1] = runs[-1] + (eng.blob.copy(),)
    for r in runs:
        assert np.array_equal(r[1].reshape(w_obs.shape), w_obs)
        assert np.array_equal(r[2], w_rew) and np.array_equal(r[3].astype(bool), w_done)
        assert np.array_equal(r[4], w_rem)
        assert np.array_equal(r[5], runs[0][5])


def test_emulated_model_state_reset_and_capture_step():
    """model_state after reset(), and after a step whose removals end the episode: every evader caught on the one
    free cell is still counted (the reference updates model_state before remove_agents)."""
    case = D.P_BY_NAME["e2_c1_flat"]
    eng = make(case)
    ms = model_state_buffer(eng)
    oracles = V.pe_oracles(case, case.maps(), SEED, BASE, E)
    eng.reset()
    for e, o in enumerate(oracles):
        o.reset()
        assert np.array_equal(ms.arr[e], o.model_state), e
    assert ms.arr[0, 2, 0, 1] == case.Ne and ms.arr[0, 1, 0, 1] == case.Np and (ms.arr[0, 0] == [[-1, 0], [-1, -1]]).all()
    act = np.full((1, E, case.Np), 4, np.int32)
    ev = np.full((1, E, case.Ne), 4, np.int32)
    bufs = [Guarded((1, E, case.Np, eng.obs_dim), np.float32, np.nan), Guarded((1, E, case.Np), np.float32, np.nan),
            Guarded((1, E), np.uint8, 255), Guarded((1, E), np.int32, -1)]
    eng._check(eng.lib.madrl_pursuit_rollout_evaders(eng._h, 1, _p(act), _p(ev), ev.strides[0] // 4, ev.strides[1] // 4,
                                                     *[_p(b.arr) for b in bufs], 0, None))
    assert (bufs[2].check("done") == 1).all() and (bufs[3].check("info") == case.Ne).all()
    V.oracle_trajectory(oracles, act, ev, MPL, auto_reset=False)
    m = ms.check("model_state")
    for e, o in enumerate(oracles):
        assert o.gone.all() and np.array_equal(m[e], o.model_state), e
    assert (m[:, 2, 0, 1] == case.Ne).all()


def test_emulated_evader_control_refusals():
    case = D.P_BY_NAME["e1_c1_flat"]
    eng = make(case)
    for mode in (-1, 2):
        assert eng.lib.madrl_pursuit_set_evader_control(eng._h, mode, 0) != 0
    assert eng.lib.madrl_pursuit_set_evader_control(None, 0, 0) != 0
    assert eng.lib.madrl_pursuit_set_model_state(None, None) != 0
    assert eng.lib.madrl_pursuit_rollout_evaders(eng._h, 0, None, None, 0, 0, None, None, None, None, 1, None) != 0
    assert eng.lib.madrl_pursuit_set_evader_control(eng._h, 0, 0) == 0
    assert eng.lib.madrl_pursuit_set_model_state(eng._h, None) == 0
