"""Whole-episode evaluation on the GPU at its edges (cases in tests/replay_eval_edges.py):

* madrl_eval_episodes_f32 / _f64 equal oracle/eval_oracle.py bit for bit -- ret, qsum, len, info sums and the
  carry after every launch -- at E A around the 128-thread block with A = 1, 5 and 32, C = 0, 1 and 2 with int64
  info sums past the int32 range, discount 0, 1 and 0.5 over an episode of 1 199 steps, episodes of one step,
  done on the first step of a launch, launches of one step, and envs finishing more and fewer than K episodes
  (records the kernel must not write keep a sentinel);
* Waterworld's in-kernel heuristic with one norm per env (kWwPolicyEnv) at every instantiation the launch picks:
  each objects-per-lane count (1, 2, 4, 8) with each sensor form (K = 30 at compile time, run-time K <= 32,
  K in 33..64), with Np = 1 and Np = 32 among them: fp64 closes the loop with the oracle env, fp32 decisions are
  the float64 reference's, and bfloat16 observations leave the float32 launch's decisions unchanged; the same
  grid with norm="agent";
* evaluate_heuristic end to end at a non-C2 cell with reward_mech='global' against the statistics of an
  oracle-driven loop."""
import math

import numpy as np
import pytest
import torch

import replay_eval_edges as RE
from madrl_b200 import BatchedMAWaterWorld, evaluate_heuristic
from madrl_b200 import _lib
from madrl_b200._lib import _ptr
from oracle import eval_oracle as eo
from oracle.heuristics_oracle import waterworld_action
from oracle.philox import Stream
from oracle.waterworld_oracle import WaterworldOracle

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def n(t):
    return t.cpu().numpy()


def dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), device=DEV)


# ------------------------------------------------------------------------------------------------ episode records

@pytest.mark.parametrize("C", [0, 1, 2])
@pytest.mark.parametrize("run", range(len(RE.RECORD_RUNS)),
                         ids=["T%d_K%d_g%s" % (r[0], r[1], r[2]) for r in RE.RECORD_RUNS])
@pytest.mark.parametrize("shape", RE.RECORD_SHAPES, ids=["E%d_A%d" % s for s in RE.RECORD_SHAPES])
def test_records_are_the_oracle_bit_for_bit(shape, run, C):
    E, A = shape
    T, K, disc, launch_len = RE.RECORD_RUNS[run]
    f64 = (RE.RECORD_SHAPES.index(shape) + C + run) % 2 == 1
    rew, done, info, cuts = RE.record_case(T, E, A, C, K, 17 * E + A + run, f64, launch_len)
    assert 1 in np.diff((0,) + cuts) and done[list(cuts)].any()
    rew_d, done_d, info_d = dev(rew), dev(done), dev(info)
    carry = torch.zeros((E, A, _lib.EVAL_CARRY_WORDS), dtype=torch.int64, device=DEV)
    recs = [dev(x) for x in RE.record_sentinels(E, A, C, K)]
    fn = _lib.lib().madrl_eval_episodes_f64 if f64 else _lib.lib().madrl_eval_episodes_f32
    want = RE.record_sentinels(E, A, C, K)
    for t0, t1, w_carry, w_recs in RE.run_records_oracle(rew, done, info, disc, K, cuts, want):
        _lib.check(fn(t1 - t0, E, A, C, _ptr(rew_d[t0:t1]), _ptr(done_d[t0:t1]), _ptr(info_d[t0:t1]) if C else None,
                      disc, K, _ptr(carry), _ptr(recs[0]), _ptr(recs[1]), _ptr(recs[2]),
                      _ptr(recs[3]) if C else None, _lib.stream(DEV)))
        assert np.array_equal(n(carry), w_carry), (t0, t1)
        assert RE.records_equal([n(x) for x in recs], w_recs), (t0, t1)
    ln = want[2].reshape(K, E)
    assert (ln[:, np.arange(E) % 6 == 1] == RE.RECORD_SENTINEL_INT).all()      # never done: no record
    assert (ln[:, np.arange(E) % 6 == 0] == 1).all()                           # K episodes of one step
    if C:                                                                      # int64 sums past int32
        assert (want[3][want[2] >= 2] > 2 ** 31).all()
    if E > 5:
        assert (ln[0, np.arange(E) % 6 == 5] == T - 1).all()                  # the long episode's record


# ------------------------------------------------------------------------------------------------ env-norm heuristic

# objects-per-lane class x sensor form: (n_pursuers, n_evaders, n_poison, n_sensors, n_coop)
ENV_CELLS = {
    "o1_k30_np1": (1, 5, 10, 30, 1),
    "o1_k8": (3, 4, 6, 8, 2),
    "o1_k40": (2, 6, 5, 40, 1),
    "o2_k30_np32": (32, 10, 10, 30, 2),
    "o2_k17": (5, 20, 15, 17, 2),
    "o2_k64": (4, 30, 10, 64, 2),
    "o4_k30": (6, 50, 40, 30, 2),
    "o4_k31_np1": (1, 60, 40, 31, 1),
    "o4_k33": (8, 40, 40, 33, 2),
    "o8_k30": (20, 100, 100, 30, 2),
    "o8_k12_np32": (32, 100, 124, 12, 2),
    "o8_k50_np1": (1, 150, 100, 50, 1),
}
SEED, BASE, MPL = 13, 500, 9


def cell_cfg(name):
    Np, Ne, Npo, K, coop = ENV_CELLS[name]
    return dict(n_pursuers=Np, n_evaders=Ne, n_poison=Npo, n_sensors=K, n_coop=coop)


def test_the_cells_cover_every_instantiation():
    """Each objects-per-lane count with each sensor form, and Np = 1 and 32."""
    seen = set()
    for name in ENV_CELLS:
        Np, Ne, Npo, K, _ = ENV_CELLS[name]
        opl = 1 << max(0, math.ceil(math.log2(math.ceil((Np + Ne + Npo) / 32))))
        form = "k30" if K == 30 else ("k<=32" if K <= 32 else "k<=64")
        assert name.startswith("o%d_" % opl)
        seen.add((opl, form))
    assert len(seen) == 12
    assert {ENV_CELLS[c][0] for c in ENV_CELLS} >= {1, 32}


def engine(name, E, dtype=torch.float64, **kw):
    return BatchedMAWaterWorld(E, device=DEV, seed=SEED, env_id_base=BASE, max_path_length=MPL, dtype=dtype,
                               **dict(cell_cfg(name), **kw))


@pytest.mark.parametrize("name", sorted(ENV_CELLS))
def test_env_norm_closes_the_loop_fp64(name):
    """Every action is the reference's on the env's previous observations as one batch (1e-12), zero exactly
    where the joint norm is 0; the env those actions drive is the oracle env (1e-9, events equal) across
    auto-resets; two chained launches equal one."""
    cfg, E, T = cell_cfg(name), 3, 2 * MPL + 4
    eng = engine(name, E)
    obs0 = eng.reset()
    out = eng.rollout_heuristic(T, obs0, auto_reset=True, norm="env")
    act, obs, rew, done, info = [n(x) for x in out]
    for e in range(E):
        o = WaterworldOracle(rng=Stream(SEED, BASE + e), **cfg)
        assert np.abs(np.array(o.reset()) - n(obs0)[e]).max() < 1e-9
        prev, ts = n(obs0)[e], 0
        for t in range(T):
            want, nrm = eo.waterworld_env_action(prev)
            if nrm == 0:
                assert not act[t, e].any(), (t, e)
            assert np.abs(want - act[t, e]).max() < 1e-12, (t, e)
            oo, rr, dd, ii = o.step(act[t, e].astype(np.float64))
            ts += 1
            dd = dd or ts >= MPL
            assert bool(done[t, e]) == dd and [ii['evcatches'], ii['pocatches']] == list(info[t, e]), (t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9, (t, e)
            if dd:
                oo, ts = o.reset(), 0
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (t, e)
            prev = obs[t, e]
    assert done.any()
    eng2 = engine(name, E)
    a1 = eng2.rollout_heuristic(T // 2, eng2.reset(), auto_reset=True, norm="env")
    a2 = eng2.rollout_heuristic(T - T // 2, a1[1][-1].contiguous(), auto_reset=True, norm="env")
    for x, y1, y2 in zip(out, a1, a2):
        assert torch.equal(x, torch.cat([y1, y2]))


def test_env_norm_of_a_blind_env_is_exactly_zero():
    """Sensors that reach nothing: every joint norm is 0 and every action exactly 0, at Np = 1 and Np = 32."""
    for name in ("o1_k30_np1", "o8_k12_np32"):
        eng = engine(name, 4, sensor_range=1e-6)
        act = eng.rollout_heuristic(6, eng.reset(), auto_reset=True, norm="env")[0]
        assert not act.any(), name


@pytest.mark.parametrize("name", sorted(ENV_CELLS))
def test_env_norm_decisions_fp32(name):
    """The float32 instantiation: each decision within 1e-5 of the float64 reference on the engine's own previous
    observations; joint norms below 1e-2 amplify float32 rounding and are skipped (counted)."""
    E, T = 16, 12
    eng = engine(name, E, dtype=torch.float32)
    obs0 = eng.reset()
    act, obs = [n(x) for x in eng.rollout_heuristic(T, obs0, auto_reset=True, norm="env")[:2]]
    prev = np.concatenate([n(obs0)[None], obs[:-1]]).astype(np.float64)
    checked = skipped = zero = 0
    for t in range(T):
        for e in range(E):
            want, nrm = eo.waterworld_env_action(prev[t, e])
            if nrm == 0:
                zero += 1
                assert not act[t, e].any(), (t, e)
            elif nrm > 1e-2:
                checked += 1
                assert np.abs(want - act[t, e]).max() < 1e-5, (t, e)
            else:
                skipped += 1
    assert checked > 0.5 * (T * E - zero) and checked > 0, (checked, skipped, zero)


@pytest.mark.parametrize("name", sorted(ENV_CELLS))
def test_env_norm_bf16_observations_keep_the_fp32_decisions(name):
    """One launch of the bfloat16-observation engine from its bfloat16 reset observation, and one of the float32
    engine (same seed) from that observation widened: actions, rewards, dones and infos bit-identical, and the
    observations the float32 ones rounded to bfloat16."""
    E, T = 16, 2 * MPL
    bf = engine(name, E, dtype=torch.float32, obs_dtype=torch.bfloat16)
    f32 = engine(name, E, dtype=torch.float32)
    o_bf = bf.reset()
    f32.reset()
    rb = bf.rollout_heuristic(T, o_bf, auto_reset=True, norm="env")
    rf = f32.rollout_heuristic(T, o_bf.float(), auto_reset=True, norm="env")
    for k, x, y in zip(("actions", "rew", "done", "info"), (rb[0],) + tuple(rb[2:]), (rf[0],) + tuple(rf[2:])):
        assert torch.equal(x, y), k
    assert torch.equal(rb[1], rf[1].to(torch.bfloat16))
    assert rb[3].any()


@pytest.mark.parametrize("name", sorted(ENV_CELLS))
def test_agent_norm_closes_the_loop_fp64(name):
    """norm="agent" at the same cells: each pursuer's action is the reference's per-agent heuristic."""
    cfg, E, T = cell_cfg(name), 2, MPL + 3
    eng = engine(name, E)
    obs0 = eng.reset()
    act, obs, rew, done, info = [n(x) for x in eng.rollout_heuristic(T, obs0, auto_reset=True, norm="agent")]
    for e in range(E):
        o = WaterworldOracle(rng=Stream(SEED, BASE + e), **cfg)
        o.reset()
        prev, ts = n(obs0)[e], 0
        for t in range(T):
            for i in range(cfg["n_pursuers"]):
                assert np.abs(waterworld_action(prev[i]) - act[t, e, i]).max() < 1e-12, (t, e, i)
            oo, rr, dd, ii = o.step(act[t, e].astype(np.float64))
            ts += 1
            dd = dd or ts >= MPL
            assert bool(done[t, e]) == dd and [ii['evcatches'], ii['pocatches']] == list(info[t, e]), (t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9
            if dd:
                oo, ts = o.reset(), 0
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (t, e)
            prev = obs[t, e]


@pytest.mark.parametrize("mode", ["decentralized", "centralized"])
def test_evaluate_heuristic_matches_an_oracle_loop(mode):
    """evaluate_heuristic at o2_k17 (fp64, reward_mech='global', chunks that do not divide the horizon) against
    rltools' statistics of the episodes an oracle env driven by the reference heuristic produces on the same
    streams."""
    name, E, n_trajs, disc, L = "o2_k17", 3, 7, 0.97, 11
    cfg = dict(cell_cfg(name), reward_mech="global")
    got = evaluate_heuristic(BatchedMAWaterWorld(E, device=DEV, seed=SEED, env_id_base=BASE, max_path_length=L,
                                                 dtype=torch.float64, **cfg), n_trajs, disc, mode, chunk=5)
    K = -(-n_trajs // E)
    per_env = []
    for e in range(E):
        o = WaterworldOracle(rng=Stream(SEED, BASE + e), **cfg)
        prev, eps, rews, infos = np.array(o.reset()), [], [], []
        for _ in range(K * L):
            a, _ = eo.waterworld_env_action(prev)
            oo, rr, dd, ii = o.step(a)
            rews.append(np.asarray(rr, np.float64))
            infos.append([ii['evcatches'], ii['pocatches']])
            if dd or len(rews) >= L:
                eps.append((np.array(rews), np.sum(infos, axis=0)))
                rews, infos = [], []
                oo = o.reset()
            prev = np.array(oo)
        per_env.append(eps)
    episodes = [per_env[e][k] for k in range(K) for e in range(E)][:n_trajs]
    want = eo.reference_statistics(episodes, disc, mode, ("evcatches", "pocatches"))
    assert sorted(got) == sorted(want)
    for k in want:
        assert np.allclose(got[k], want[k], rtol=1e-9, atol=1e-9), (k, got[k], want[k])
