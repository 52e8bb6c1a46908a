"""Pursuit's and Hostage's rollout kernels at every instantiation their launchers dispatch to, at the largest maps
and object counts they accept (needs a GPU).  The cases are tests/env_dispatch_edges.py's table.

Every test first reads, from the library's launch logs (madrl_pursuit_launch_log, madrl_hostage_launch_log), which
instantiation each launch ran, and checks it against the case's: a wider kernel usually gives the same numbers, so
only the log can show that a shape was dispatched to the wrong one.  Then:
  * Hostage fp64 and Pursuit float32 follow the oracle over whole auto-reset trajectories with a horizon, cut into
    two launches, with terminal observations, and end in the oracle's per-env state and draw counters;
  * Hostage float32 matches the oracle by teacher forcing, with the fragility exclusions of oracle/fragility.py;
  * bfloat16 observations equal the float32 engine's rounded, and KEEP stores equal streaming ones, all else
    identical, state blob included;
  * one persistent wave of 2 x SMs + 7 envs (set_launch(blocks_per_sm=1)) equals the default launch;
  * Pursuit's in-kernel heuristic policy closes the loop as the oracle policy does, for both window centres.
The last test launches every case every way and compares the logged set with all 60 Hostage and 96 Pursuit
kernels, written out."""
import numpy as np
import pytest
import torch

import env_dispatch_edges as D
import teacher_forced as TF
from madrl_b200 import BatchedHostageWorld, BatchedPursuitEvade, _lib
from test_heuristics import check_pursuit_closed_loop

pytestmark = pytest.mark.gpu

KEEP, STREAM = _lib.OBS_CACHE_KEEP, _lib.OBS_CACHE_STREAM


def launched(fam, fields, fn):
    """fn() with the family's launch log on -> (its result, [record without grid], [grid]) of its launches."""
    L, most = _lib.lib(), 4096
    log = getattr(L, "madrl_%s_launch_log" % fam)
    assert log(1, None, 0) >= 0
    try:
        out = fn()
        torch.cuda.synchronize()
    finally:
        recs = np.zeros((most, fields), np.int32)
        n = log(0, recs.ctypes.data, most)
    assert 0 <= n <= most, n
    return out, [tuple(r[:-1]) for r in recs[:n].tolist()], [r[-1] for r in recs[:n].tolist()]


def np_(xs):
    return [x.float().cpu().numpy() if x.dtype == torch.bfloat16 else x.cpu().numpy() for x in xs]


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def split_rollout(eng, act, term=False):
    """rollout(act) with auto-reset as two launches (a third, then the rest) -> (obs, rew, done, info, term or
    None); `term`: terminal observations kept in NaN-filled tensors."""
    T1 = max(1, act.shape[0] // 3)
    outs, terms = [], []
    for a in (act[:T1], act[T1:]):
        if term:
            # float32's NaN, rounded: the bfloat16 of the float32 fill, as the comparisons round
            terms.append(torch.full((a.shape[0], eng.n_envs, eng._n_acting, eng.obs_dim), float("nan"),
                                    device="cuda").to(eng.obs_dtype))
            eng.set_terminal_obs(terms[-1])
        outs.append(eng.rollout(a, auto_reset=True))
    eng.set_terminal_obs(None)
    cat = [torch.cat(x) for x in zip(*outs)]
    return cat + [torch.cat(terms) if term else None]


def bits(x):
    return x.view({torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}.get(x.dtype, x.dtype))


def assert_same_rollout(got, want, obs_dtype, case):
    """[reset obs, obs, rew, done, info, terminal obs, state blob] of a bf16 / KEEP engine against the float32
    STREAM engine's, bit for bit; bfloat16 observations against the float32 ones rounded."""
    for i, (g, w) in enumerate(zip(got, want)):
        if i in (0, 1, 5) and obs_dtype is not None:
            w = w.to(obs_dtype)
        assert torch.equal(bits(g), bits(w)), (case, i)


# ------------------------------------------------------------------------------------------------ Hostage
def hw_make(case, E, dtype=torch.float32, **kw):
    return BatchedHostageWorld(E, *case.args, dtype=dtype, **case.kw, **kw)


@pytest.mark.parametrize("case", D.H_CASES, ids=repr)
def test_hostage_fp64_trajectories_match_oracle(case):
    seed, base, mpl = 321, 77, 15
    eng = hw_make(case, case.E, torch.float64, seed=seed, env_id_base=base, max_path_length=mpl)
    act = D.hw_actions(case, case.E, case.T)

    def run():
        return eng.reset(), split_rollout(eng, torch.as_tensor(act), term=True)
    (obs0, outs), recs, _ = launched("hostage", 7, run)
    assert recs == [D.hw_record(case, 8, 8, 0)] * 3, recs
    obs0, (obs, rew, done, info, term) = obs0.cpu().numpy(), np_(outs)
    oracles = D.hw_oracles(case, seed, base, case.E)
    seen = D.hw_check_trajectory(case, oracles, obs0, act, obs, rew, done, info, mpl, term)
    D.hw_check_state(case, TF.TorchAdapter(eng).read(), oracles)
    D.hw_check_reach(case, oracles)
    assert "done" in seen and set(case.events) <= seen, (case, seen)


@pytest.mark.parametrize("case", D.H_CASES, ids=repr)
def test_hostage_fp32_teacher_forced(case):
    E, T, seed = 24, 6, 99
    eng = hw_make(case, E, seed=seed)
    eng.reset()
    ad = TF.TorchAdapter(eng)
    log, recs, _ = launched("hostage", 7, lambda: TF.hw_self_teacher_forced(
        ad, case.args, case.kw, seed, T, 3.0, "hw_dispatch_" + case.name,
        lambda done: eng.reset(mask=torch.as_tensor(done))))
    assert set(recs) == {D.hw_record(case, 4, 4, 0)}, recs
    log.dump()
    assert log.checked_frac >= 0.98 and log.obs_frac >= 0.999, log.d


def hw_variant(case, E, T, obs_dtype, cache, seed=3, mpl=11, **kw):
    eng = hw_make(case, E, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **kw)
    eng.set_obs_cache(cache)
    act = torch.as_tensor(D.hw_actions(case, E, T, seed=4), dtype=torch.float32)

    def run():
        return [eng.reset()] + split_rollout(eng, act, term=True) + [eng._blob.clone()]
    return launched("hostage", 7, run)


@pytest.mark.parametrize("case", D.H_CASES, ids=repr)
def test_hostage_bf16_and_keep_equal_fp32_stream(case):
    E, T = 64, 30
    want, recs, _ = hw_variant(case, E, T, None, STREAM)
    assert set(recs) == {D.hw_record(case, 4, 4, 0)}, recs
    assert want[3].any()
    for obs_dtype, cache, ob, keep in ((None, KEEP, 4, 1), (torch.bfloat16, STREAM, 2, 0), (torch.bfloat16, KEEP, 2, 1)):
        got, recs, _ = hw_variant(case, E, T, obs_dtype, cache)
        # the reset launches stream whatever the cache mode
        assert recs == [D.hw_record(case, 4, ob, 0), D.hw_record(case, 4, ob, keep), D.hw_record(case, 4, ob, keep)]
        assert_same_rollout(got, want, obs_dtype, case)


@pytest.mark.parametrize("case", D.H_CASES, ids=repr)
def test_hostage_persistent_wave_equals_default_launch(case):
    E, T = 2 * sms() + 7, 25
    runs = []
    for bps in (0, 1):
        eng = hw_make(case, E, seed=8, max_path_length=9)
        eng.set_launch(blocks_per_sm=bps)
        act = torch.as_tensor(D.hw_actions(case, E, T, seed=6), dtype=torch.float32)
        out, recs, grids = launched("hostage", 7, lambda: [eng.reset()] + list(eng.rollout(act)) + [eng._blob])
        assert set(recs) == {D.hw_record(case, 4, 4, 0)} and grids == [E if bps == 0 else sms()] * 2, (recs, grids)
        runs.append(out)
    assert runs[0][3].any()
    for a, b in zip(*runs):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------ Pursuit
def pe_make(case, maps, E, **kw):
    return BatchedPursuitEvade(E, maps, **case.cfg, **kw)


@pytest.mark.parametrize("case", D.P_CASES, ids=repr)
def test_pursuit_trajectories_bit_exact(case):
    seed, base, mpl = 77, 500, 13
    maps = case.maps()
    eng = pe_make(case, maps, case.E, seed=seed, env_id_base=base, max_path_length=mpl)
    act = D.pe_actions(case, case.E, case.T)
    (obs0, outs), recs, _ = launched("pursuit", 8, lambda: (eng.reset(), split_rollout(eng, torch.as_tensor(act),
                                                                                      term=True)))
    assert recs == [D.pe_record(case, 4, 0, 0)] * 3, recs
    obs0, (obs, rew, done, removed, term) = obs0.cpu().numpy(), np_(outs)
    oracles = D.pe_oracles(case, maps, seed, base, case.E)
    n_removed, hi = D.pe_check_trajectory(case, oracles, obs0, act, obs, rew, done, removed, mpl, term)
    D.pe_check_state(case, {k: v.cpu().numpy() for k, v in eng.state.items()}, oracles)
    assert done.any()
    if case.gone_hi:
        assert hi, case


def pe_variant(case, maps, E, T, obs_dtype, cache, seed=3, mpl=11, **kw):
    eng = pe_make(case, maps, E, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **kw)
    eng.set_obs_cache(cache)
    act = torch.as_tensor(D.pe_actions(case, E, T, seed=4))
    return launched("pursuit", 8, lambda: [eng.reset()] + split_rollout(eng, act, term=True) + [eng._blob.clone()])


@pytest.mark.parametrize("case", D.P_CASES, ids=repr)
def test_pursuit_bf16_and_keep_equal_fp32_stream(case):
    E, T = 64, 30
    maps = case.maps()
    want, recs, _ = pe_variant(case, maps, E, T, None, STREAM)
    assert set(recs) == {D.pe_record(case, 4, 0, 0)}, recs
    for obs_dtype, cache, ob, keep in ((None, KEEP, 4, 1), (torch.bfloat16, STREAM, 2, 0), (torch.bfloat16, KEEP, 2, 1)):
        got, recs, _ = pe_variant(case, maps, E, T, obs_dtype, cache)
        assert recs == [D.pe_record(case, ob, 0, 0), D.pe_record(case, ob, 0, keep), D.pe_record(case, ob, 0, keep)]
        assert_same_rollout(got, want, obs_dtype, case)


@pytest.mark.parametrize("case", D.P_CASES, ids=repr)
def test_pursuit_persistent_wave_equals_default_launch(case):
    E, T = 2 * sms() + 7, 25
    maps = case.maps()
    runs = []
    for bps in (0, 1):
        eng = pe_make(case, maps, E, seed=8, max_path_length=9)
        eng.set_launch(blocks_per_sm=bps)
        act = torch.as_tensor(D.pe_actions(case, E, T, seed=6))
        out, recs, grids = launched("pursuit", 8, lambda: [eng.reset()] + list(eng.rollout(act)) + [eng._blob])
        assert set(recs) == {D.pe_record(case, 4, 0, 0)} and grids[-1] == (E if bps == 0 else sms()), (recs, grids)
        runs.append(out)
    for a, b in zip(*runs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("py2", [True, False])
@pytest.mark.parametrize("case", D.P_CASES, ids=repr)
def test_pursuit_heuristic_policy_closes_the_loop(case, py2):
    """The POLICY kernels against the oracle policy; two chained launches equal one; bfloat16 observations change
    no action and equal the float32 ones rounded."""
    E, T, seed, base, mpl = 6, 24, 21, 900, 13
    maps = case.maps()

    def engine(obs_dtype=None):
        return pe_make(case, maps, E, seed=seed, env_id_base=base, max_path_length=mpl, obs_dtype=obs_dtype)
    eng = engine()
    (obs0, outs), recs, _ = launched("pursuit", 8, lambda: (lambda o: (o, eng.rollout_heuristic(
        T, o, auto_reset=True, py2_division=py2)))(eng.reset()))
    assert recs == [D.pe_record(case, 4, 0, 0), D.pe_record(case, 4, 1, 0)], recs
    act, obs, rew, done, removed = np_(outs)
    check_pursuit_closed_loop(maps, case.cfg, seed, base, obs0.cpu().numpy(), act, obs, rew, done, removed, mpl, py2)
    e2 = engine()
    o0 = e2.reset()
    a1 = e2.rollout_heuristic(T // 3, o0, auto_reset=True, py2_division=py2)
    a2 = e2.rollout_heuristic(T - T // 3, a1[1][-1], auto_reset=True, py2_division=py2)
    for x, y1, y2 in zip(outs, a1, a2):
        assert torch.equal(x, torch.cat([y1, y2]))
    eb = engine(torch.bfloat16)
    got, recs, _ = launched("pursuit", 8, lambda: eb.rollout_heuristic(T, eb.reset(), auto_reset=True,
                                                                       py2_division=py2))
    assert recs == [D.pe_record(case, 2, 0, 0), D.pe_record(case, 2, 1, 0)], recs
    assert torch.equal(got[1].view(torch.int16), outs[1].to(torch.bfloat16).view(torch.int16))
    for x, y in zip(got[:1] + got[2:], outs[:1] + outs[2:]):
        assert torch.equal(x, y)


# ------------------------------------------------------------------------------------------------ coverage
def test_dispatch_reaches_every_instantiation():
    """Every case launched with every element type, store policy and (Pursuit) the heuristic policy: the logged
    instantiations are exactly the 60 Hostage and 96 Pursuit kernels the dispatchers can reach."""
    def hostage():
        for case in D.H_CASES:
            act = torch.zeros(2, 4, case.Nr, 2)
            hw_make(case, 4, torch.float64).rollout(act.double())
            for obs_dtype in (None, torch.bfloat16):
                for cache in (STREAM, KEEP):
                    eng = hw_make(case, 4, obs_dtype=obs_dtype)
                    eng.set_obs_cache(cache)
                    eng.rollout(act)
    _, recs, _ = launched("hostage", 7, hostage)
    assert set(recs) == D.HW_ALL, sorted(D.HW_ALL ^ set(recs))

    def pursuit():
        for case in D.P_CASES:
            maps = case.maps()
            act = torch.zeros(2, 4, case.Np, dtype=torch.int32)
            for obs_dtype in (None, torch.bfloat16):
                for cache in (STREAM, KEEP):
                    eng = pe_make(case, maps, 4, obs_dtype=obs_dtype)
                    eng.set_obs_cache(cache)
                    eng.rollout(act)
                    eng.rollout_heuristic(2, eng.reset())
    _, recs, _ = launched("pursuit", 8, pursuit)
    assert set(recs) == D.PE_ALL, sorted(D.PE_ALL ^ set(recs))
