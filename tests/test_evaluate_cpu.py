"""Whole-episode evaluation without a GPU:

  * madrl_eval_episodes_* (csrc/postproc.cu), run by the warp emulator (tests/emu), equals its NumPy restatement
    (oracle/eval_oracle.py) bit for bit, for any cut of the rollout into launches;
  * the records' statistics (madrl_b200.evaluate.statistics) equal rltools' evaluate_policy statistics computed from
    the padded reward arrays;
  * Waterworld's in-kernel heuristic with one norm per env (madrl_ww_set_heuristic_norm) takes the reference's
    joint-norm actions and closes the loop as the oracle env does;
  * the refusals of the C entry points and of madrl_b200.evaluate.
"""
import types

import numpy as np
import pytest

import replay_eval_edges as RE
from emu.driver import Guarded, needs_cxx, ptr
from madrl_b200 import evaluate as ev
from madrl_b200 import _lib
from oracle import eval_oracle as eo
from oracle.philox import Stream
from oracle.waterworld_oracle import WaterworldOracle


def scripted(T, E, A, C, seed, ends=(), p_done=0.15, f64=False):
    """Rewards, done flags and info of a T-step rollout: random ends plus the (t, e) in `ends`."""
    rs = np.random.RandomState(seed)
    rew = (rs.randn(T, E, A) * 2 + 0.3).astype(np.float64 if f64 else np.float32)
    done = (rs.rand(T, E) < p_done).astype(np.uint8)
    for t, e in ends:
        done[t, e] = 1
    info = rs.randint(0, 4, size=(T, E, C)).astype(np.int32)
    return rew, done, info


def run_kernel(lib, rew, done, info, disc, K, cuts):
    """The emulated kernel over the rollout cut at `cuts` -> (records, carry)."""
    T, E, A = rew.shape
    C = info.shape[2]
    carry = Guarded((E, A, _lib.EVAL_CARRY_WORDS), np.int64, 0)
    recs = [Guarded((K * E, A), np.float64, 0), Guarded((K * E, A), np.float64, 0), Guarded((K * E,), np.int32, 0),
            Guarded((K * E, C), np.int64, 0)]
    fn = lib.madrl_eval_episodes_f64 if rew.dtype == np.float64 else lib.madrl_eval_episodes_f32
    for t0, t1 in zip((0,) + tuple(cuts), tuple(cuts) + (T,)):
        r, d, i = (np.ascontiguousarray(x[t0:t1]) for x in (rew, done, info))
        rc = fn(t1 - t0, E, A, C, ptr(r), ptr(d), ptr(i) if C else None, disc, K, ptr(carry.arr),
                *[ptr(x.arr) for x in recs], None)
        assert rc == 0, lib.madrl_last_error().decode()
    return [x.check("record") for x in recs], carry.check("carry")


def run_oracle(rew, done, info, disc, K, cuts):
    T, E, A = rew.shape
    carry, recs = eo.new_carry(E, A), eo.new_records(E, A, info.shape[2], K)
    for t0, t1 in zip((0,) + tuple(cuts), tuple(cuts) + (T,)):
        eo.eval_episodes(rew[t0:t1], done[t0:t1], info[t0:t1], disc, K, carry, recs)
    return recs, carry


CASES = {
    # name: T, E, A, C, K, discount, float64, forced ends
    "c2like": (40, 6, 5, 2, 3, 0.99, False, [(6, 0), (7, 0), (13, 2), (0, 3), (39, 4)]),
    "a1_c0": (30, 5, 1, 0, 2, 0.95, False, [(0, 0), (1, 0), (2, 0)]),
    "c1_f64": (35, 4, 3, 1, 4, 0.9, True, [(6, 1), (7, 1), (20, 3)]),
    "gamma0": (25, 3, 2, 2, 5, 0.0, False, [(5, 0), (6, 0)]),
    "gamma1": (25, 3, 2, 2, 5, 1.0, True, [(13, 2), (14, 2)]),
}


@needs_cxx
@pytest.mark.parametrize("name", sorted(CASES))
def test_emulated_eval_episodes_equal_the_oracle_for_every_cut(name):
    """Chunks of 1, 7 and the whole rollout give the same bits as the oracle; ends fall on chunk boundaries
    (t = 6, 7 with chunk 7), at t = 0 and on consecutive steps (episodes of length 1)."""
    from emu.driver import load
    T, E, A, C, K, disc, f64, ends = CASES[name]
    rew, done, info = scripted(T, E, A, C, seed=len(name), ends=ends, f64=f64)
    lib = load()
    want, want_carry = run_oracle(rew, done, info, disc, K, ())
    assert (want[2] > 0).any() and (want[2] == 1).any()
    for step in (1, 7, T):
        cuts = tuple(range(step, T, step))
        got, carry = run_kernel(lib, rew, done, info, disc, K, cuts)
        for g, w in zip(got, want):
            assert np.array_equal(g, w), (name, step)
        assert np.array_equal(carry, want_carry), (name, step)
        o_recs, o_carry = run_oracle(rew, done, info, disc, K, cuts)
        assert all(np.array_equal(a, b) for a, b in zip(o_recs, want)) and np.array_equal(o_carry, want_carry)


@needs_cxx
@pytest.mark.parametrize("C", [0, 1, 2])
@pytest.mark.parametrize("run", range(len(RE.RECORD_RUNS)),
                         ids=["T%d_K%d_g%s" % (r[0], r[1], r[2]) for r in RE.RECORD_RUNS])
@pytest.mark.parametrize("shape", RE.RECORD_SHAPES[:3] + RE.RECORD_SHAPES[4:6] + RE.RECORD_SHAPES[7:9],
                         ids=lambda s: "E%d_A%d" % s)
def test_emulated_records_at_the_edge_cases(shape, run, C):
    """The cases of tests/test_evaluate_edges_gpu.py (tests/replay_eval_edges.py): records filled with sentinels
    first, carry and records bit for bit after every launch."""
    from emu.driver import load
    lib = load()
    E, A = shape
    T, K, disc, launch_len = RE.RECORD_RUNS[run]
    f64 = (RE.RECORD_SHAPES.index(shape) + C + run) % 2 == 1
    rew, done, info, cuts = RE.record_case(T, E, A, C, K, 17 * E + A + run, f64, launch_len)
    carry = Guarded((E, A, _lib.EVAL_CARRY_WORDS), np.int64, 0)
    recs = [Guarded(x.shape, x.dtype, 0) for x in RE.record_sentinels(E, A, C, K)]
    for g, x in zip(recs, RE.record_sentinels(E, A, C, K)):
        g.arr[...] = x
    fn = lib.madrl_eval_episodes_f64 if f64 else lib.madrl_eval_episodes_f32
    want = RE.record_sentinels(E, A, C, K)
    for t0, t1, w_carry, w_recs in RE.run_records_oracle(rew, done, info, disc, K, cuts, want):
        r, d, i = (np.ascontiguousarray(x[t0:t1]) for x in (rew, done, info))
        assert fn(t1 - t0, E, A, C, ptr(r), ptr(d), ptr(i) if C else None, disc, K, ptr(carry.arr),
                  *[ptr(x.arr) for x in recs[:3]], ptr(recs[3].arr) if C else None, None) == 0
        assert np.array_equal(carry.check("carry"), w_carry), (t0, t1)
        assert RE.records_equal([x.check("record") for x in recs], w_recs), (t0, t1)


def episodes_of(rew, done, info, K):
    """Each env's first K complete episodes in record order k * E + e: (rewards [L, A], info sums [C])."""
    T, E, A = rew.shape
    per_env = [[] for _ in range(E)]
    for e in range(E):
        s = 0
        for t in range(T):
            if done[t, e]:
                per_env[e].append((rew[s:t + 1, e].astype(np.float64), info[s:t + 1, e].sum(axis=0)))
                s = t + 1
    return [per_env[e][k] for k in range(K) for e in range(E)]


@needs_cxx
@pytest.mark.parametrize("n", [2, 7, 9])
@pytest.mark.parametrize("mode", ["decentralized", "centralized"])
def test_statistics_of_the_records_equal_rltools(n, mode):
    """n < E, n not a multiple of E, n = K E: the statistics of records 0 .. n-1 equal evaluate_policy's from the
    padded reward arrays.  Centralized: every agent has the same reward."""
    from emu.driver import load
    T, E, A, C, K = 60, 3, 4, 2, 3
    rs = np.random.RandomState(n)
    done = np.zeros((T, E), np.uint8)
    for e in range(E):                                   # K episodes per env of varied lengths, then one running
        done[np.sort(rs.choice(np.arange(e, 45), K, replace=False)), e] = 1
    rew = (rs.randn(T, E, A) + 0.2).astype(np.float32)
    if mode == "centralized":
        rew[:] = rew[..., :1]
    info = rs.randint(0, 3, size=(T, E, C)).astype(np.int32)
    (ret, qsum, ln, isum), _ = run_kernel(load(), rew, done, info, 0.95, K, (17, 40))
    got = ev.statistics(ret[:n], qsum[:n], ln[:n], isum[:n], mode, ("a", "b"))
    want = eo.reference_statistics(episodes_of(rew, done, info, K)[:n], 0.95, mode, ("a", "b"))
    assert sorted(got) == sorted(want)
    for k in want:
        assert np.allclose(got[k], want[k], rtol=1e-12, atol=1e-12), k
    if mode == "centralized":
        ret[0, 1] += 1e-3
        with pytest.raises(ValueError, match="same reward"):
            ev.statistics(ret[:n], qsum[:n], ln[:n], isum[:n], mode, ("a", "b"))


# ----------------------------------------------------------------- Waterworld's heuristic with one norm per env
def set_env_norm(eng, norm):
    rc = eng.lib.madrl_ww_set_heuristic_norm(eng._h, norm)
    assert rc == 0, eng.lib.madrl_last_error().decode()


@needs_cxx
@pytest.mark.parametrize("name,cfg,E,T", [
    ("c2", dict(n_pursuers=5, n_evaders=5), 3, 40),
    ("dense", dict(n_pursuers=5, n_evaders=5, n_coop=1, radius=0.04, sensor_range=0.3), 3, 40),
    ("k40", dict(n_pursuers=4, n_evaders=40, n_poison=3, n_sensors=40, radius=0.03, addid=False), 2, 16)])
def test_emulated_env_norm_policy_closes_the_loop_fp64(name, cfg, E, T):
    """Every action is the reference's on the env's Np observations as one batch, and the env it drives is the
    oracle env; chained launches equal one launch."""
    from emu.driver import EmuWaterworld
    seed, base, mpl = 3, 70, 13
    eng = EmuWaterworld(E, seed=seed, env_id_base=base, max_path_length=mpl, **cfg)
    set_env_norm(eng, _lib.HEURISTIC_NORM_ENV)
    obs0 = eng.reset()
    act, obs, rew, done, info = eng.rollout_heuristic(T, obs0, auto_reset=True)
    joint = np.linalg.norm(act.reshape(T, E, -1), axis=-1)
    assert np.all((np.abs(joint - 1) < 1e-12) | (joint == 0))
    for e in range(E):
        o = WaterworldOracle(rng=Stream(seed, base + e), **cfg)
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < 1e-9
        prev, ts = obs0[e], 0
        for t in range(T):
            want, _ = eo.waterworld_env_action(prev)
            assert np.abs(want - act[t, e]).max() < 1e-12, (t, e)
            oo, rr, dd, ii = o.step(act[t, e].astype(np.float64))
            ts += 1
            dd = dd or ts >= mpl
            assert bool(done[t, e]) == dd and [ii['evcatches'], ii['pocatches']] == list(info[t, e])
            assert np.abs(rr - rew[t, e]).max() < 1e-9
            if dd:
                oo, ts = o.reset(), 0
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9
            prev = obs[t, e]
    assert done.any()
    eng2 = EmuWaterworld(E, seed=seed, env_id_base=base, max_path_length=mpl, **cfg)
    set_env_norm(eng2, _lib.HEURISTIC_NORM_ENV)
    o0 = eng2.reset()
    a1 = eng2.rollout_heuristic(T // 2, o0, auto_reset=True)
    a2 = eng2.rollout_heuristic(T - T // 2, a1[1][-1], auto_reset=True)
    for x, y1, y2 in zip((act, obs, rew, done, info), a1, a2):
        assert np.array_equal(x, np.concatenate([y1, y2]))


@needs_cxx
def test_emulated_env_norm_policy_fp32_and_agent_norm_unchanged():
    """float32: the joint-norm actions within 1e-5 of the float64 reference on the same observations (norms below
    1e-2 skipped, all-zero where the norm is 0).  Switching back to AGENT gives the default kernel's bits."""
    from emu.driver import EmuWaterworld
    cfg, seed, E, T = dict(n_pursuers=5, n_evaders=5), 5, 5, 30
    eng = EmuWaterworld(E, seed=seed, fp64=False, **cfg)
    set_env_norm(eng, _lib.HEURISTIC_NORM_ENV)
    obs0 = eng.reset()
    act, obs = eng.rollout_heuristic(T, obs0, auto_reset=False)[:2]
    prev = np.concatenate([obs0[None], obs[:-1]]).astype(np.float64)
    checked = 0
    for t in range(T):
        for e in range(E):
            want, n = eo.waterworld_env_action(prev[t, e])
            if n == 0:
                assert not act[t, e].any()
            elif n > 1e-2:
                checked += 1
                assert np.abs(want - act[t, e]).max() < 1e-5, (t, e)
    assert checked > 0.8 * T * E
    runs = []
    for norm in (None, _lib.HEURISTIC_NORM_AGENT):
        e2 = EmuWaterworld(E, seed=seed, fp64=False, **cfg)
        if norm is not None:
            set_env_norm(e2, _lib.HEURISTIC_NORM_ENV)
            set_env_norm(e2, norm)
        runs.append(e2.rollout_heuristic(T, e2.reset(), auto_reset=False))
    assert all(np.array_equal(a, b) for a, b in zip(*runs))


# ----------------------------------------------------------------------------------------------- refusals
@needs_cxx
def test_c_entry_points_refuse_bad_arguments():
    from emu.driver import EmuWaterworld, load
    lib = load()
    z = np.zeros(64, np.float64)
    good = dict(T=2, E=2, A=2, C=1, disc=0.9, K=1, info=ptr(np.zeros(64, np.int32)), isum=ptr(np.zeros(64, np.int64)))

    def call(**kw):
        a = dict(good, **kw)
        return lib.madrl_eval_episodes_f32(a["T"], a["E"], a["A"], a["C"], ptr(z), ptr(z), a["info"], a["disc"],
                                           a["K"], ptr(z), ptr(z), ptr(z), ptr(z), a["isum"], None)
    assert call() == 0
    for bad in (dict(T=0), dict(E=0), dict(A=0), dict(K=0), dict(C=-1), dict(C=3), dict(disc=1.5), dict(disc=-0.1),
                dict(info=None), dict(isum=None)):
        assert call(**bad) == -1, bad
    assert call(C=0, info=None, isum=None) == 0
    eng = EmuWaterworld(1, n_pursuers=2, n_evaders=2)
    assert eng.lib.madrl_ww_set_heuristic_norm(eng._h, 2) == -1
    assert b"heuristic norm" in eng.lib.madrl_last_error()
    assert eng.lib.madrl_ww_set_heuristic_norm(None, 0) == -1


def fake_engine(abi="ww", mpl=20, E=4):
    return types.SimpleNamespace(_abi=abi, n_envs=E, cfg=types.SimpleNamespace(max_path_length=mpl))


@pytest.mark.parametrize("call,match", [
    (lambda: ev.evaluate_heuristic(fake_engine(mpl=0), 4, 0.99, "decentralized"), "max_path_length"),
    (lambda: ev.evaluate_heuristic(fake_engine(), 4, 0.99, "joint"), "mode"),
    (lambda: ev.evaluate_heuristic(fake_engine(), 0, 0.99, "decentralized"), "n_trajs"),
    (lambda: ev.evaluate_heuristic(fake_engine(), 4, 1.5, "decentralized"), "discount"),
    (lambda: ev.evaluate_heuristic(fake_engine(), 4, 0.99, "decentralized", chunk=0), "chunk"),
    (lambda: ev.evaluate_heuristic(fake_engine(), 4, 0.99, "decentralized", norm="batch"), "norm"),
    (lambda: ev.evaluate_heuristic(fake_engine("hostage"), 4, 0.99, "decentralized"), "Hostage"),
    (lambda: ev.evaluate_policy(fake_engine(mpl=0), None, 4, 0.99, "decentralized"), "max_path_length"),
    (lambda: ev.evaluate_policy(fake_engine(), None, 4, 0.99, "centralised"), "mode"),
])
def test_evaluate_refuses_before_any_work(call, match):
    with pytest.raises(ValueError, match=match):
        call()


def test_rollout_heuristic_refuses_an_unknown_norm():
    from madrl_b200.waterworld import BatchedMAWaterWorld
    eng = object.__new__(BatchedMAWaterWorld)
    with pytest.raises(ValueError, match="norm"):
        eng.rollout_heuristic(4, None, norm="batch")


@needs_cxx
def test_emulated_fp64_heuristic_evaluation_reproduces_the_reference():
    """The golden case of tests/golden/eval_ww_heuristic.npz (the reference's decrollout, heuristic, TrajBatch and
    discount on the same streams) through the emulated env-norm rollout and records kernels."""
    import json
    import os
    from conftest import GOLDEN_DIR
    from emu.driver import EmuWaterworld, load
    g = np.load(os.path.join(GOLDEN_DIR, "eval_ww_heuristic.npz"))
    c = json.loads(str(g["case"]))
    E, K, L, n = c["E"], c["K"], c["max_traj_len"], c["n_trajs"]
    eng = EmuWaterworld(E, seed=c["seed"], env_id_base=c["env_id_base"], max_path_length=L, **c["config"])
    set_env_norm(eng, _lib.HEURISTIC_NORM_ENV)
    _, obs, rew, done, info = eng.rollout_heuristic(K * L, eng.reset(), auto_reset=True)
    (ret, qsum, ln, isum), _ = run_kernel(load(), rew, done, info, c["discount"], K, (L, 2 * L))
    assert np.array_equal(ln[:n], g["ep_len"]) and np.array_equal(isum[:n], g["ep_info"])
    assert np.abs(ret[:n] - g["ep_ret"]).max() < 1e-9
    got = ev.statistics(ret[:n], qsum[:n], ln[:n], isum[:n], "decentralized", ("evcatches", "pocatches"))
    for k in ("ret", "retstd", "disc_ret"):
        assert np.abs(got[k] - g[k]).max() < 1e-9, k
    for j, k in enumerate(g["info_keys"]):
        assert np.array_equal(got[str(k)], g["info"][:, j]), k
