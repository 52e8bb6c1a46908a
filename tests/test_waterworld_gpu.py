"""Parity of the CUDA MAWaterWorld engine with the oracle / golden vectors (needs a GPU).

 * fp64 verification build: whole trajectories must agree with the float64 oracle (same discrete
   events, observations within 1e-9) -- including the golden vectors recorded from the real
   reference.
 * fp32 production build: single-step teacher forcing from the engine's own fp32 states; every
   transition whose branch decisions are not within EPS of a threshold must match within 1e-5
   (the tolerance BASELINE.json's north_star states).
"""
import json
import os

import numpy as np
import pytest
import torch

import teacher_forced as TF
from conftest import GOLDEN_DIR
from oracle.philox import Stream
from oracle.waterworld_oracle import WaterworldOracle

pytestmark = pytest.mark.gpu

TOL32 = TF.TOL32


def make(cfg, E, dtype, **kw):
    from madrl_b200 import BatchedMAWaterWorld
    return BatchedMAWaterWorld(E, dtype=dtype, **cfg, **kw)


def engine_state(eng, e):
    st = {k: v.cpu().numpy() for k, v in eng.state.items()}
    Np, Ne = eng.n_pursuers, eng.n_evaders
    X = np.stack([st['pos_x'][e], st['pos_y'][e]], 1).astype(np.float64)
    V = np.stack([st['vel_x'][e], st['vel_y'][e]], 1).astype(np.float64)
    return dict(px=X[:Np], pv=V[:Np], ex=X[Np:Np + Ne], ev=V[Np:Np + Ne], ox=X[Np + Ne:],
                ov=V[Np + Ne:], obst=np.array([[st['obst_x'][e], st['obst_y'][e]]], dtype=np.float64),
                t=int(st['timestep'][e]), counter=int(st['rng_counter'][e]))


CFGS = {
    "c2": dict(n_pursuers=5, n_evaders=5),
    "dense": dict(n_pursuers=5, n_evaders=5, n_coop=1, radius=0.04, sensor_range=0.3),
    "global_nospeed_randobst": dict(n_pursuers=3, n_evaders=4, n_poison=2, n_sensors=7, n_coop=1,
                                    radius=0.05, reward_mech='global', speed_features=False,
                                    addid=False, obstacle_loc=None),
    "c4": dict(n_pursuers=20, n_evaders=50, n_poison=50),
    "k40": dict(n_pursuers=4, n_evaders=40, n_poison=3, n_sensors=40, n_coop=2, radius=0.03),
    "big200": dict(n_pursuers=6, n_evaders=120, n_poison=74, n_coop=2, radius=0.02),   # 8 objects per lane
}


@pytest.mark.parametrize("name,E,T", [("c2", 48, 150), ("dense", 32, 150),
                                      ("global_nospeed_randobst", 40, 200), ("c4", 8, 30),
                                      ("k40", 8, 60), ("big200", 3, 25)])
def test_fp64_trajectories_match_oracle(name, E, T):
    cfg = CFGS[name]
    seed, base = 1234, 1000
    eng = make(cfg, E, torch.float64, seed=seed, env_id_base=base)
    obs0 = eng.reset().cpu().numpy()
    oracles = [WaterworldOracle(rng=Stream(seed, base + e), **cfg) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < 1e-9, e
    Np = cfg['n_pursuers']
    act = (np.random.RandomState(5).randn(T, E, Np, 2) * 0.7)
    obs, rew, done, info = [x.cpu().numpy() for x in eng.rollout(torch.as_tensor(act), auto_reset=False)]
    catches = 0
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert [ii['evcatches'], ii['pocatches']] == list(info[t, e]), (t, e)
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9, (t, e)
            assert bool(done[t, e]) == dd
            catches += ii['evcatches'] + ii['pocatches']
    for e, o in enumerate(oracles):
        s = engine_state(eng, e)
        assert s['counter'] == o.np_random.counter and s['t'] == o.t
        assert np.abs(s['ex'] - o.ex).max() < 1e-9 and np.abs(s['pv'] - o.pv).max() < 1e-9
    assert catches > 0


@pytest.mark.parametrize("name", ["ww_c2", "ww_dense", "ww_c4", "ww_global_nospeed"])
def test_fp64_matches_reference_golden(name):
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    cfg = json.loads(str(g["config"]))
    if cfg.get("obstacle_loc", 0) is not None and "obstacle_loc" in cfg:
        cfg["obstacle_loc"] = np.array(cfg["obstacle_loc"])
    eng = make(cfg, 1, torch.float64, seed=int(g["seed"]), env_id_base=int(g["env_id"]))
    assert np.abs(eng.reset().cpu().numpy()[0] - g["obs0"]).max() < 1e-9
    act = torch.as_tensor(g["actions"][:, None])
    obs, rew, done, info = [x.cpu().numpy() for x in eng.rollout(act, auto_reset=False)]
    assert np.array_equal(info[:, 0], g["info"])
    assert np.abs(obs[:, 0] - g["obs"]).max() < 1e-9
    assert np.abs(rew[:, 0] - g["rew"]).max() < 1e-9
    assert np.array_equal(done[:, 0].astype(bool), g["done"])
    assert int(eng.state['rng_counter'][0].item()) == int(g["counter"])


@pytest.mark.parametrize("name,E,T,min_frac", [("c2", 256, 24, 0.98), ("dense", 128, 30, 0.98),
                                               ("c4", 16, 12, 0.98),  # 72 600 predicates per step
                                               ("global_nospeed_randobst", 128, 30, 0.98)])
def test_fp32_single_step_teacher_forced(name, E, T, min_frac):
    """fp32 production build, one step at a time from its own states, vs the float64 oracle; per-predicate
    exclusion (oracle/fragility.py): `min_frac` of the transitions and 99.9 % of the observation
    elements of those must be compared (counts written to $MADRL_PARITY_DIR when set)."""
    cfg = CFGS[name]
    eng = make(cfg, E, torch.float32, seed=99)
    eng.reset()
    log = TF.ww_self_teacher_forced(TF.TorchAdapter(eng), cfg, 99, T, 0.7, "ww_fp32_self_" + name)
    log.dump()
    assert log.checked_frac >= min_frac and log.obs_frac >= 0.999, log.d


@pytest.mark.parametrize("name", ["ww_c2", "ww_dense", "ww_c4", "ww_c4_long", "ww_global_nospeed"])
def test_fp32_teacher_forced_from_reference_states(name):
    """The benched instantiation against the REAL reference: every step of every golden is replayed
    from the reference's recorded float64 state (cast to fp32) and compared with the reference's
    recorded obs / reward / events / next state."""
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    cfg = json.loads(str(g["config"]))
    if cfg.get("obstacle_loc", 0) is not None and "obstacle_loc" in cfg:
        cfg["obstacle_loc"] = np.array(cfg["obstacle_loc"])
    eng = make(cfg, 1, torch.float32, seed=int(g["seed"]), env_id_base=int(g["env_id"]))
    eng.reset()
    log = TF.ww_golden_teacher_forced(TF.TorchAdapter(eng), g, cfg, "ww_fp32_golden_" + name)
    log.dump()
    assert log.checked_frac >= 0.98 and log.obs_frac >= 0.999, log.d


def test_fp32_multi_step_tracks_fp64_build():
    """Free-running (not teacher-forced) comparison of the fp32 production build with the fp64
    verification build (which itself follows the float64 oracle): trajectories may only separate
    where a comparison flips, so after 60 steps the large majority of envs must still show the
    same discrete events, with observations still within 1e-4, and the batch statistics must agree."""
    cfg = CFGS["c2"]
    E, T = 2048, 60
    a32 = make(cfg, E, torch.float32, seed=17)
    a64 = make(cfg, E, torch.float64, seed=17)
    assert (a32.reset().double() - a64.reset()).abs().max() < 1e-6
    act = torch.randn(T, E, 5, 2, generator=torch.Generator().manual_seed(3)) * 0.7
    o32, r32, d32, i32 = a32.rollout(act.cuda(), auto_reset=False)
    o64, r64, d64, i64 = a64.rollout(act.cuda().double(), auto_reset=False)
    same = (i32 == i64).all(dim=2).cumprod(dim=0).bool()              # [T, E] still identical events
    close = ((o32.double() - o64).abs().amax(dim=(2, 3)) < 1e-4)
    tracking = (same & close).cumprod(dim=0).bool()
    assert tracking[-1].float().mean() > 0.80, tracking.float().mean(dim=1)[[0, 9, 29, 59]]
    # batch statistics agree even where single envs separated
    assert abs(int(i32.sum()) - int(i64.sum())) <= 0.05 * int(i64.sum()) + 5
    assert abs(float(r32.sum()) - float(r64.sum())) <= 0.05 * abs(float(r64.sum())) + 5.0


def test_auto_reset_and_horizon_follow_vec_env_executor():
    """VecEnvExecutor.step: done at timestep_limit or at max_path_length; the done env is reset in
    place and that step's obs slot holds the reset observation (vec_env_executor.py:16-28)."""
    cfg = CFGS["c2"]
    E, T, mpl, seed = 6, 23, 9, 4
    eng = make(cfg, E, torch.float64, seed=seed, max_path_length=mpl)
    eng.reset()
    act = np.random.RandomState(0).randn(T, E, 5, 2) * 0.5
    obs, rew, done, info = [x.cpu().numpy() for x in eng.rollout(torch.as_tensor(act), auto_reset=True)]
    oracles = [WaterworldOracle(rng=Stream(seed, e), **cfg) for e in range(E)]
    for o in oracles:
        o.reset()
    ts = np.zeros(E, int)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            ts[e] += 1
            dd = dd or ts[e] >= mpl
            assert bool(done[t, e]) == dd
            if dd:
                oo = o.reset()
                ts[e] = 0
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9
    assert done.sum() == E * (T // mpl)


def test_sharding_is_invisible_and_launch_geometry_is_irrelevant():
    cfg = CFGS["dense"]
    E, T = 64, 40
    act = torch.as_tensor(np.random.RandomState(1).randn(T, E, 5, 2).astype(np.float32))
    full = make(cfg, E, torch.float32, seed=7)
    full.reset()
    ref = [x.cpu() for x in full.rollout(act)]
    half = E // 2
    for base in (0, half):
        sh = make(cfg, half, torch.float32, seed=7, env_id_base=base)
        sh.set_launch(warps_per_block=3, blocks_per_sm=1)  # override accepted; warps_per_block is ignored
        sh.reset()
        out = [x.cpu() for x in sh.rollout(act[:, base:base + half].contiguous())]
        for a, b in zip(ref, out):
            assert torch.equal(a[:, base:base + half], b)


def test_dropin_env_surface():
    import pickle
    from madrl_b200 import MAWaterWorld
    env = MAWaterWorld(5, 5, seed=21, env_id=2)
    assert len(env.agents) == 5 and env.agents[0].observation_space.shape == (213,)
    assert env.agents[0].action_space.shape == (2,) and env.reward_mech == 'local'
    assert env.timestep_limit == 1000
    obs = env.reset()
    assert len(obs) == 5 and obs[0].shape == (213,) and not env.is_terminal
    orc = WaterworldOracle(5, 5, rng=Stream(21, 2))
    o0 = orc.reset()
    assert np.abs(np.array(o0) - np.array(obs)).max() <= TOL32
    a = np.random.RandomState(0).randn(10) * 0.5       # flat (2*Np,) centralized action format
    o1, r1, d1, i1 = env.step(a)
    assert len(o1) == 5 and r1.shape == (5,) and d1 is False and set(i1) == {'evcatches', 'pocatches'}
    with pytest.raises(ValueError):
        env.step(np.zeros(7))
    env2 = pickle.loads(pickle.dumps(env))              # EzPickle: rebuilt from ctor args
    assert env2.n_pursuers == 5 and len(env2.reset()) == 5
    ex = env.vec_env_executor(n_envs=3, max_path_length=5)
    assert ex.num_envs == 3 and len(ex.reset()) == 3
    for _ in range(5):
        obs_n, rew_n, done_n, infos = ex.step(np.zeros((3, 10)))
    assert done_n.all() and rew_n.shape == (3, 5) and infos['evcatches'].shape == (3,)
