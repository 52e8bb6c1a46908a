"""The KERNEL SOURCE (madrl_b200/csrc/*.cu) executed on the CPU by the warp emulator of tests/emu
(g++ + a fake <cuda_runtime.h>; every CUDA thread is a fiber, warp collectives are rendezvous
points) and compared with the oracle.  This is test infrastructure: it checks the C++ semantics of
the kernels and of the host launch code without a GPU, for the default build and for the
experiment flags that are still off in the product; the `-m gpu` tests remain the parity proof of
what nvcc makes of the same source.  Nothing in madrl_b200/ can load the emulator library."""
import os

import numpy as np
import pytest

from conftest import ROOT
from emu import driver
from emu.driver import Guarded
from emu.driver import ptr as _p
from oracle.hostage_oracle import HostageOracle
from oracle.philox import Stream
from oracle.pursuit_oracle import PursuitOracle
from oracle.waterworld_oracle import WaterworldOracle

pytestmark = driver.needs_cxx

# build variants: the product defaults
VARIANTS = {"default": ()}
if os.environ.get("MADRL_EMU_DEFINES"):   # ad-hoc check of an experiment build: MADRL_EMU_DEFINES="-DFOO=1 -DBAR=1"
    VARIANTS["env"] = tuple(os.environ["MADRL_EMU_DEFINES"].split())
PE_VARIANTS = sorted(VARIANTS)


def f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32)


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    """Every emulated launch is also race-checked: two lanes touching the same shared-memory byte,
    one of them writing, without a __syncwarp / __syncthreads in between, fail the test."""
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


# ------------------------------------------------------------------------------------ Waterworld
WW = {
    "c2": dict(n_pursuers=5, n_evaders=5),
    "dense": dict(n_pursuers=5, n_evaders=5, n_coop=1, radius=0.04, sensor_range=0.3),
    "global_nospeed_randobst": dict(n_pursuers=3, n_evaders=4, n_poison=2, n_sensors=7, n_coop=1, radius=0.05,
                                    reward_mech='global', speed_features=False, addid=False, obstacle_loc=None),
    "c4": dict(n_pursuers=20, n_evaders=50, n_poison=50),                                     # 4 objects per lane
    "k40": dict(n_pursuers=4, n_evaders=40, n_poison=3, n_sensors=40, n_coop=2, radius=0.03),  # 2 sensors per lane
    "big200": dict(n_pursuers=6, n_evaders=120, n_poison=74, n_coop=2, radius=0.02),          # 8 objects per lane
    "minimum": dict(n_pursuers=1, n_evaders=1, n_poison=1, n_sensors=1, n_coop=1, radius=0.05),
    # K = 30 WITHOUT speed features: must not take the compile-time (K = 30, speed features) instantiation
    "k30_nospeed": dict(n_pursuers=3, n_evaders=4, n_poison=5, n_sensors=30, speed_features=False, radius=0.03),
    "np32_k64": dict(n_pursuers=32, n_evaders=3, n_poison=2, n_sensors=64, n_coop=3, radius=0.03),
}


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("name,E,T", [("c2", 5, 60), ("dense", 5, 80), ("global_nospeed_randobst", 5, 80),
                                      ("c4", 3, 8), ("k40", 3, 25), ("big200", 2, 6), ("minimum", 5, 60), ("k30_nospeed", 3, 40),
                                      ("np32_k64", 2, 6)])
def test_waterworld_fp64_trajectories_match_oracle(variant, name, E, T):
    from emu.driver import EmuWaterworld
    cfg = WW[name]
    seed, base = 1234, 1000
    eng = EmuWaterworld(E, seed=seed, env_id_base=base, defines=VARIANTS[variant], **cfg)
    obs0 = eng.reset()
    oracles = [WaterworldOracle(rng=Stream(seed, base + e), **cfg) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < 1e-9, e
    Np = cfg['n_pursuers']
    act = np.random.RandomState(5).randn(T, E, Np, 2) * 0.7
    obs, rew, done, info = eng.rollout(act, auto_reset=False)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert [ii['evcatches'], ii['pocatches']] == list(info[t, e]), (t, e)
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9, (t, e)
            assert bool(done[t, e]) == dd
    for e, o in enumerate(oracles):
        s = eng.state(e)
        assert s['counter'] == o.np_random.counter and s['t'] == o.t
        assert np.abs(s['ex'] - o.ex).max() < 1e-9 and np.abs(s['pv'] - o.pv).max() < 1e-9


@pytest.mark.parametrize("variant", sorted(VARIANTS))
def test_waterworld_auto_reset_horizon_mask_and_host_path(variant):
    from emu.driver import EmuWaterworld
    cfg = WW["c2"]
    E, T, mpl, seed = 5, 20, 7, 4
    eng = EmuWaterworld(E, seed=seed, max_path_length=mpl, defines=VARIANTS[variant], **cfg)
    eng.reset()
    act = np.random.RandomState(0).randn(T, E, 5, 2) * 0.5
    obs, rew, done, info = eng.rollout(act, auto_reset=True)
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
    # the host-buffer entry point gives the same trajectory as the device one
    a, b = [EmuWaterworld(E, seed=9, defines=VARIANTS[variant], **cfg) for _ in range(2)]
    a.reset(), b.reset()
    for x, y in zip(a.rollout(act, host=False), b.rollout(act, host=True)):
        assert np.array_equal(x, y)
    # masked reset re-initialises only the selected envs
    before = [a.state(e) for e in range(E)]
    mask = np.array([1, 0, 0, 1, 0], np.uint8)
    obs_r = a.reset(mask)
    for e in range(E):
        s = a.state(e)
        if mask[e]:
            assert s['t'] == 1 and np.abs(obs_r[e]).sum() > 0
        else:
            assert s['t'] == before[e]['t'] and np.array_equal(s['px'], before[e]['px']) and not obs_r[e].any()


def test_waterworld_fp32_build_tracks_fp64_build():
    from emu.driver import EmuWaterworld
    cfg, E, T = WW["c2"], 4, 12
    act = np.random.RandomState(3).randn(T, E, 5, 2) * 0.5
    outs = []
    for fp64 in (True, False):
        eng = EmuWaterworld(E, seed=11, fp64=fp64, **cfg)
        o0 = eng.reset()
        outs.append((o0,) + eng.rollout(act, auto_reset=False))
    assert outs[1][0].dtype == np.float32
    assert np.abs(outs[0][0] - outs[1][0]).max() < 1e-5
    same_events = np.array_equal(outs[0][4], outs[1][4])
    if same_events:   # no threshold flipped in fp32: the trajectories stay within rounding noise
        assert np.abs(outs[0][1] - outs[1][1]).max() < 1e-3


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("name,E,T,min_frac", [("c2", 12, 12, 0.95), ("dense", 10, 12, 0.95), ("c4", 2, 4, 0.85)])
def test_waterworld_fp32_single_step_teacher_forced(variant, name, E, T, min_frac):
    """The fp32 instantiation, one step at a time from its own fp32 states, against the float64 oracle
    (tolerance 1e-5, per-predicate exclusion of comparisons within 3e-7 of their threshold) -- the
    GPU test's methodology (tests/teacher_forced.py) at small size."""
    import teacher_forced as TF
    from emu.driver import EmuWaterworld
    cfg = WW[name]
    eng = EmuWaterworld(E, seed=99, fp64=False, defines=VARIANTS[variant], **cfg)
    eng.reset()
    log = TF.ww_self_teacher_forced(TF.EmuAdapter(eng, "ww"), cfg, 99, T, 0.7, "emu_ww_" + name)
    assert log.checked_frac >= min_frac and log.obs_frac >= 0.999, log.d


@pytest.mark.parametrize("name", ["ww_c2", "ww_dense", "ww_c4", "ww_global_nospeed"])
def test_waterworld_fp32_teacher_forced_from_reference_states(name):
    """fp32 instantiation replayed from the REAL reference's recorded float64 states (tests/golden)."""
    import teacher_forced as TF
    from emu.driver import EmuWaterworld
    g, cfg = _golden(name)
    if cfg.get("obstacle_loc", 0) is not None and "obstacle_loc" in cfg:
        cfg["obstacle_loc"] = np.array(cfg["obstacle_loc"])
    eng = EmuWaterworld(1, seed=int(g["seed"]), env_id_base=int(g["env_id"]), fp64=False, **cfg)
    eng.reset()
    log = TF.ww_golden_teacher_forced(TF.EmuAdapter(eng, "ww"), g, cfg, "emu_golden_" + name)
    assert log.checked_frac >= 0.95 and log.obs_frac >= 0.999, log.d


@pytest.mark.parametrize("name", ["hw_c5", "hw_c5_local", "hw_dense", "hw_k12"])
def test_hostage_fp32_teacher_forced_from_reference_states(name):
    import teacher_forced as TF
    from emu.driver import EmuHostage
    g, kw = _golden(name)
    if 'key_loc' in kw:
        kw['key_loc'] = np.array(kw['key_loc'])
    args = tuple(int(a) for a in g["args"])
    eng = EmuHostage(1, *args, seed=int(g["seed"]), env_id_base=int(g["env_id"]), fp64=False, **kw)
    eng.reset()
    log = TF.hw_golden_teacher_forced(TF.EmuAdapter(eng, "hw"), g, args, kw, "emu_golden_" + name)
    assert log.checked_frac >= 0.95 and log.obs_frac >= 0.999, log.d


# ------------------------------------------------------------------------------------ Pursuit
def pool16():
    return np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))


def small_map():
    m = np.zeros((1, 5, 5), dtype=np.int32)
    m[0, 2, 2] = -1
    return m


C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
          catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
PE = {
    "c3": (pool16, C3),
    "c3_global": (pool16, dict(C3, reward_mech='global', urgency_reward=-0.1)),
    "ncatch": (pool16, dict(C3, surround=False, n_evaders=20, n_pursuers=12, obs_range=5)),
    "window_r9": (pool16, dict(C3, constraint_window=0.5, n_evaders=6, n_pursuers=10, obs_range=9, include_id=False)),
    "many_evaders": (pool16, dict(C3, n_evaders=50, n_pursuers=30, obs_range=11, catchr=0.01)),
    "crowd": (small_map, dict(n_evaders=4, n_pursuers=10, obs_range=3, surround=True, reward_mech='local',
                              catchr=0.1, term_pursuit=5.0)),
    "conv_small": (small_map, dict(n_evaders=3, n_pursuers=3, obs_range=4, surround=False, n_catch=1,
                                   reward_mech='global', flatten=False)),
    "random_opp": (small_map, dict(n_evaders=5, n_pursuers=6, obs_range=3, surround=False, n_catch=1,
                                   reward_mech='local', catchr=0.1, random_opponents=True, max_opponents=6)),
}


def check_pursuit_state(eng, oracles):
    for e, o in enumerate(oracles):
        s = eng.state(e)
        assert np.array_equal(s['pursuers'], o.ppos)
        live = ~o.gone
        assert np.array_equal(s['evaders'][live], o.epos[live])
        assert [(s['gone'] >> j) & 1 for j in range(o.Ne)] == [int(x) for x in o.gone]
        assert s['counter'] == o.rng.counter


@pytest.mark.parametrize("variant", PE_VARIANTS)
@pytest.mark.parametrize("name,E,T", [("c3", 5, 40), ("c3_global", 3, 30), ("ncatch", 5, 40), ("window_r9", 5, 40),
                                      ("many_evaders", 2, 12), ("crowd", 6, 120), ("conv_small", 6, 80),
                                      ("random_opp", 8, 60)])
def test_pursuit_trajectories_bit_exact(variant, name, E, T):
    from emu.driver import EmuPursuit
    mk, cfg = PE[name]
    maps = mk()
    seed, base = 77, 500
    eng = EmuPursuit(E, maps, seed=seed, env_id_base=base, defines=VARIANTS[variant], **cfg)
    obs0 = eng.reset()
    oracles = [PursuitOracle(maps, rng=Stream(seed, base + e), **cfg) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.array_equal(f32(o.reset()).reshape(obs0[e].shape), obs0[e]), e
    check_pursuit_state(eng, oracles)
    act = np.random.RandomState(9).randint(0, 5, size=(T, E, cfg['n_pursuers'])).astype(np.int32)
    obs, rew, done, removed = eng.rollout(act, auto_reset=False)
    total = 0
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert ii['removed'] == removed[t, e] and dd == bool(done[t, e]), (t, e)
            assert np.array_equal(f32(oo).reshape(obs[t, e].shape), obs[t, e]), (t, e)
            assert np.array_equal(f32(rr), rew[t, e]), (t, e)
            total += ii['removed']
    check_pursuit_state(eng, oracles)
    if name in ("ncatch", "crowd"):
        assert total > 0


@pytest.mark.parametrize("variant", PE_VARIANTS)
@pytest.mark.parametrize("name", ["crowd", "random_opp"])
def test_pursuit_auto_reset(variant, name):
    from emu.driver import EmuPursuit
    mk, cfg = PE[name]
    maps, E, T, mpl, seed = mk(), 5, 40, 9, 3
    eng = EmuPursuit(E, maps, seed=seed, max_path_length=mpl, defines=VARIANTS[variant], **cfg)
    eng.reset()
    act = np.random.RandomState(1).randint(0, 5, size=(T, E, cfg['n_pursuers'])).astype(np.int32)
    obs, rew, done, removed = eng.rollout(act, auto_reset=True)
    oracles = [PursuitOracle(maps, rng=Stream(seed, e), **cfg) for e in range(E)]
    for o in oracles:
        o.reset()
    ts = np.zeros(E, int)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            ts[e] += 1
            dd = dd or ts[e] >= mpl
            assert bool(done[t, e]) == dd and ii['removed'] == removed[t, e]
            if dd:
                oo = o.reset()
                ts[e] = 0
            assert np.array_equal(f32(oo).reshape(obs[t, e].shape), obs[t, e]), (t, e)
            assert np.array_equal(f32(rr), rew[t, e])


# ------------------------------------------------------------------------------------ Hostage
HW = {
    "c5": ((10, 16, 16, 4, 2), {}),
    "c5_local": ((10, 16, 16, 4, 2), dict(reward_mech='local')),
    "dense": ((3, 10, 5, 1, 2), dict(radius=0.05, sensor_range=0.35, key_radius=0.06, reward_mech='local', addid=False)),
    "k12_fixed_key": ((4, 6, 8, 2, 1), dict(radius=0.04, n_sensors=12, key_radius=0.05, bomb_radius=0.02,
                                            key_loc=np.array([[0.93, 0.97]]))),
    "big": ((12, 40, 30, 2, 2), dict(radius=0.03, n_sensors=40, key_radius=0.04)),
    "minimum": ((1, 1, 1, 1, 1), dict(n_sensors=1, radius=0.05, key_radius=0.05)),
}


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("name,E,T,std", [("c5", 4, 50, 1.0), ("c5_local", 3, 50, 2.0), ("dense", 6, 150, 3.0),
                                          ("k12_fixed_key", 6, 150, 3.0), ("big", 2, 12, 2.0),
                                          ("minimum", 5, 80, 3.0)])
def test_hostage_fp64_trajectories_match_oracle(variant, name, E, T, std):
    from emu.driver import EmuHostage
    args, kw = HW[name]
    seed, base = 321, 77
    eng = EmuHostage(E, *args, seed=seed, env_id_base=base, defines=VARIANTS[variant], **kw)
    obs0 = eng.reset()
    oracles = [HostageOracle(*args, rng=Stream(seed, base + e), **kw) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < 1e-9, e
    act = np.random.RandomState(5).randn(T, E, args[0], 2) * std
    obs, rew, done, info = eng.rollout(act, auto_reset=True)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert [ii['ho_saved'], ii['cr_encs']] == list(info[t, e]), (t, e)
            assert bool(done[t, e]) == dd, (t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9, (t, e)
            if dd:                       # auto-reset: the slot holds the reset observation
                oo = o.reset()
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (t, e)
    for e, o in enumerate(oracles):
        s = eng.state(e)
        assert s['counter'] == o.np_random.counter and s['t'] == o.t
        assert np.array_equal(s['saved'], np.asarray(o.saved, bool))


# ------------------------------------------------------------------ golden vectors of the REAL reference
# (tests/golden/*.npz, recorded by oracle/make_golden.py from the imported reference classes)
def _golden(name):
    import json
    from conftest import GOLDEN_DIR
    g = np.load(os.path.join(GOLDEN_DIR, name + ".npz"), allow_pickle=False)
    return g, json.loads(str(g["config"]))


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("name", ["ww_c2", "ww_dense", "ww_c4", "ww_global_nospeed"])
def test_waterworld_reproduces_reference_golden(variant, name):
    from emu.driver import EmuWaterworld
    g, cfg = _golden(name)
    if cfg.get("obstacle_loc", 0) is not None and "obstacle_loc" in cfg:
        cfg["obstacle_loc"] = np.array(cfg["obstacle_loc"])
    eng = EmuWaterworld(1, seed=int(g["seed"]), env_id_base=int(g["env_id"]), defines=VARIANTS[variant], **cfg)
    assert np.abs(eng.reset()[0] - g["obs0"]).max() < 1e-9
    obs, rew, done, info = eng.rollout(g["actions"][:, None], auto_reset=False)
    assert np.array_equal(info[:, 0], g["info"])
    assert np.abs(obs[:, 0] - g["obs"]).max() < 1e-9
    assert np.abs(rew[:, 0] - g["rew"]).max() < 1e-9
    assert np.array_equal(done[:, 0].astype(bool), g["done"])
    assert eng.state(0)['counter'] == int(g["counter"])


@pytest.mark.parametrize("variant", PE_VARIANTS)
@pytest.mark.parametrize("name", ["pe_c3", "pe_c3_global", "pe_ncatch", "pe_window", "pe_small", "pe_even_range", "pe_random_opp",
                                  "pe_crowd"])
def test_pursuit_reproduces_reference_golden(variant, name):
    from emu.driver import EmuPursuit
    g, cfg = _golden(name)
    maps = pool16() if str(g["maps"]) == "pool16" else small_map()
    eng = EmuPursuit(1, maps, seed=int(g["seed"]), env_id_base=int(g["env_id"]), defines=VARIANTS[variant], **cfg)
    assert np.array_equal(eng.reset()[0], f32(g["obs0"]))
    resets = list(g["reset_at"])
    t0, k, T = 0, 0, g["actions"].shape[0]
    while t0 < T:                      # segment by segment between the recorded reset() calls
        t1 = (resets[k] + 1) if k < len(resets) else T
        obs, rew, done, removed = eng.rollout(g["actions"][t0:t1, None], auto_reset=False)
        assert np.array_equal(obs[:, 0], f32(g["obs"][t0:t1]))
        assert np.array_equal(rew[:, 0], f32(g["rew"][t0:t1]))
        assert np.array_equal(done[:, 0].astype(bool), g["done"][t0:t1])
        assert np.array_equal(removed[:, 0], g["removed"][t0:t1])
        if k < len(resets):
            assert np.array_equal(eng.reset()[0], f32(g["reset_obs"][k]))
            k += 1
        t0 = t1
    assert eng.state(0)['counter'] == int(g["counter"])


@pytest.mark.parametrize("variant", sorted(VARIANTS))
@pytest.mark.parametrize("name", ["hw_c5", "hw_c5_local", "hw_dense", "hw_k12"])
def test_hostage_reproduces_reference_golden(variant, name):
    from emu.driver import EmuHostage
    g, kw = _golden(name)
    if 'key_loc' in kw:
        kw['key_loc'] = np.array(kw['key_loc'])
    args = tuple(int(a) for a in g["args"])
    eng = EmuHostage(1, *args, seed=int(g["seed"]), env_id_base=int(g["env_id"]), defines=VARIANTS[variant], **kw)
    assert np.abs(eng.reset()[0] - g["obs0"]).max() < 1e-9
    obs, rew, done, info = eng.rollout(g["actions"][:, None], auto_reset=True)
    assert np.array_equal(info[:, 0], g["info"])
    assert np.array_equal(done[:, 0].astype(bool), g["done"])
    assert np.abs(rew[:, 0] - g["rew"]).max() < 1e-9
    expect = g["obs"].copy()
    for k, t in enumerate(g["reset_at"]):          # the reference driver reset() where done
        expect[t] = g["reset_obs"][k]
    assert np.abs(obs[:, 0] - expect).max() < 1e-9
    assert eng.state(0)['counter'] == int(g["counter"])


# ------------------------------------------------------------------ seeded random configurations
def _ww_random_cfg(rs):
    return dict(n_pursuers=int(rs.randint(1, 33)), n_evaders=int(rs.randint(1, 70)), n_poison=int(rs.randint(1, 70)),
                n_sensors=int(rs.randint(1, 65)), n_coop=int(rs.randint(1, 4)), radius=float(rs.uniform(0.01, 0.06)),
                sensor_range=float(rs.uniform(0.1, 0.45)), obstacle_radius=float(rs.uniform(0.05, 0.3)),
                ev_speed=float(rs.uniform(0.005, 0.03)), poison_speed=float(rs.uniform(0.005, 0.03)),
                reward_mech=['local', 'global'][rs.randint(2)], addid=bool(rs.randint(2)),
                speed_features=bool(rs.randint(2)),
                obstacle_loc=None if rs.randint(3) == 0 else rs.uniform(0.2, 0.8, size=2))


@pytest.mark.parametrize("variant", ["default"])
@pytest.mark.parametrize("case", range(10))
def test_waterworld_random_configurations(variant, case):
    from emu.driver import EmuWaterworld
    rs = np.random.RandomState(1000 + case)
    cfg = _ww_random_cfg(rs)
    n_obj = cfg['n_pursuers'] + cfg['n_evaders'] + cfg['n_poison']
    E, T = 2, max(4, min(40, 1200 // n_obj))
    seed, base = int(rs.randint(1 << 30)), int(rs.randint(1000))
    eng = EmuWaterworld(E, seed=seed, env_id_base=base, defines=VARIANTS[variant], **cfg)
    obs0 = eng.reset()
    oracles = [WaterworldOracle(rng=Stream(seed, base + e), **cfg) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < 1e-9, (cfg, e)
    act = rs.randn(T, E, cfg['n_pursuers'], 2) * 0.8
    obs, rew, done, info = eng.rollout(act, auto_reset=False)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert [ii['evcatches'], ii['pocatches']] == list(info[t, e]), (cfg, t, e)
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (cfg, t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9, (cfg, t, e)
    for e, o in enumerate(oracles):
        assert eng.state(e)['counter'] == o.np_random.counter


@pytest.mark.parametrize("variant", ["default"])
@pytest.mark.parametrize("case", range(10))
def test_hostage_random_configurations(variant, case):
    from emu.driver import EmuHostage
    rs = np.random.RandomState(2000 + case)
    n_good, n_host, n_bad = int(rs.randint(1, 33)), int(rs.randint(1, 50)), int(rs.randint(1, 50))
    args = (n_good, n_host, n_bad, int(rs.randint(1, 4)), int(rs.randint(1, 3)))
    kw = dict(radius=float(rs.uniform(0.01, 0.06)), n_sensors=int(rs.randint(1, 65)),
              sensor_range=float(rs.uniform(0.1, 0.4)), key_radius=float(rs.uniform(0.005, 0.08)),
              bomb_radius=float(rs.uniform(0.01, 0.08)), bad_speed=float(rs.uniform(0.005, 0.03)),
              reward_mech=['local', 'global'][rs.randint(2)], addid=bool(rs.randint(2)))
    if rs.randint(2):
        kw['key_loc'] = rs.uniform(0.9, 1.0, size=(1, 2))
    E, T = 2, max(6, min(60, 2400 // (n_good + n_host + n_bad)))
    seed, base = int(rs.randint(1 << 30)), int(rs.randint(1000))
    eng = EmuHostage(E, *args, seed=seed, env_id_base=base, defines=VARIANTS[variant], **kw)
    obs0 = eng.reset()
    oracles = [HostageOracle(*args, rng=Stream(seed, base + e), **kw) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < 1e-9, (args, kw, e)
    act = rs.randn(T, E, n_good, 2) * 2.5
    obs, rew, done, info = eng.rollout(act, auto_reset=True)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert [ii['ho_saved'], ii['cr_encs']] == list(info[t, e]), (args, kw, t, e)
            assert bool(done[t, e]) == dd and np.abs(rr - rew[t, e]).max() < 1e-9, (args, kw, t, e)
            if dd:
                oo = o.reset()
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (args, kw, t, e)


@pytest.mark.parametrize("variant", ["default"])
@pytest.mark.parametrize("case", range(10))
def test_pursuit_random_configurations(variant, case):
    from emu.driver import EmuPursuit
    rs = np.random.RandomState(3000 + case)
    if rs.randint(3) == 0:
        xs, ys = int(rs.randint(2, 12)), int(rs.randint(2, 12))
        maps = (rs.rand(int(rs.randint(1, 4)), xs, ys) < 0.15).astype(np.int32) * -1
        maps[:, 0, 0] = 0
    else:
        maps = pool16()
    cfg = dict(n_evaders=int(rs.randint(1, 65)), n_pursuers=int(rs.randint(1, 33)), obs_range=int(rs.randint(1, 12)),
               surround=bool(rs.randint(2)), n_catch=int(rs.randint(1, 4)), flatten=bool(rs.randint(4) != 0),
               reward_mech=['local', 'global'][rs.randint(2)], catchr=float(rs.choice([0.01, 0.1, 0.37])),
               term_pursuit=float(rs.choice([5.0, 1.5])), urgency_reward=float(rs.choice([0.0, -0.1])),
               include_id=bool(rs.randint(2)), sample_maps=bool(rs.randint(2)),
               constraint_window=float(rs.choice([1.0, 0.6])), layer_norm=int(rs.choice([10, 7])))
    E, T = 2, 25
    seed, base = int(rs.randint(1 << 30)), int(rs.randint(1000))
    eng = EmuPursuit(E, maps, seed=seed, env_id_base=base, defines=VARIANTS[variant], **cfg)
    obs0 = eng.reset()
    oracles = [PursuitOracle(maps, rng=Stream(seed, base + e), **cfg) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.array_equal(f32(o.reset()).reshape(obs0[e].shape), obs0[e]), (cfg, e)
    act = rs.randint(0, 5, size=(T, E, cfg['n_pursuers'])).astype(np.int32)
    obs, rew, done, removed = eng.rollout(act, auto_reset=False)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert ii['removed'] == removed[t, e] and dd == bool(done[t, e]), (cfg, t, e)
            assert np.array_equal(f32(oo).reshape(obs[t, e].shape), obs[t, e]), (cfg, t, e)
            assert np.array_equal(f32(rr), rew[t, e]), (cfg, t, e)
    check_pursuit_state(eng, oracles)


def test_integration_md_ctypes_stub_runs():
    """The ctypes stub printed in INTEGRATION.md section 4 (config struct, create, reset_host,
    rollout_host, destroy) is executed verbatim -- at 6 envs, against the emulator library, which
    exports the same C ABI."""
    import re
    from emu import build_emu
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    code = re.search(r"## 4\. C ABI without PyTorch.*?```python\n(.*?)```", doc, re.S).group(1)
    assert 'C.CDLL("madrl_b200/libmadrl_b200.so")' in code
    code = code.replace('C.CDLL("madrl_b200/libmadrl_b200.so")', 'C.CDLL(%r)' % build_emu.build([]))
    code = code.replace("4096", "6").replace("T = 16", "T = 4")
    ns = {}
    exec(compile(code, "INTEGRATION.md", "exec"), ns)
    assert ns["rc"] == 0 and ns["obs"].shape == (4, 6, 5, 213)
    assert np.isfinite(ns["obs"]).all() and ns["done"].max() <= 1 and (ns["info"] >= 0).all()


def test_host_code_validation_seed_and_curriculum_knobs():
    """Host side of the C ABI on the emulator build: argument validation never throws and reports
    through madrl_last_error; seed() re-keys the stream and restarts the counters; Pursuit's
    set_params (catchr, constraint_window: the curriculum knobs of pursuit_evade.py:264-272) takes
    effect at the next step / reset."""
    from emu.driver import EmuPursuit, EmuWaterworld
    with pytest.raises(RuntimeError, match="n_pursuers"):
        EmuWaterworld(4, 40, 5)
    with pytest.raises(RuntimeError, match="n_sensors"):
        EmuWaterworld(4, 5, 5, n_sensors=100)
    eng = EmuWaterworld(3, 5, 5, seed=5)
    lib = eng.lib
    assert lib.madrl_ww_rollout(eng._h, 0, None, None, None, None, None, 0, None) == -1
    assert b"T must be" in lib.madrl_last_error()
    assert lib.madrl_ww_reset(None, None, None, None) == -1
    with pytest.raises(RuntimeError):
        eng.set_launch(warps_per_block=9)
    # seed(): same seed -> same episode, different seed -> different episode
    a = eng.reset().copy()
    eng.seed(5)
    assert np.array_equal(eng.reset(), a) and eng.state(0)['counter'] > 0
    eng.seed(6)
    assert not np.array_equal(eng.reset(), a)
    # Pursuit curriculum knobs
    maps = small_map()
    cfg = dict(n_evaders=4, n_pursuers=6, obs_range=3, surround=True, reward_mech='local', catchr=0.1, term_pursuit=5.0)
    pe = EmuPursuit(2, maps, seed=3, **cfg)
    assert lib.madrl_pursuit_set_params(pe._h, 0.25, 1.0) == 0
    pe.reset()
    act = np.random.RandomState(0).randint(0, 5, size=(6, 2, 6)).astype(np.int32)
    obs, rew, done, removed = pe.rollout(act, auto_reset=False)
    oracles = [PursuitOracle(maps, rng=Stream(3, e), **dict(cfg, catchr=0.25)) for e in range(2)]
    for o in oracles:
        o.reset()
    for t in range(6):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert np.array_equal(f32(rr), rew[t, e]) and ii['removed'] == removed[t, e]


@pytest.mark.parametrize("family", ["waterworld", "hostage"])
def test_timestep_limit_horizon_with_auto_reset(family):
    """The env's own 1000-step horizon (waterworld.py:124-126, hostage.py:181-184) followed by the
    in-place reset, one env, 1 010 steps."""
    from emu.driver import EmuHostage, EmuWaterworld
    T, seed = 1010, 21
    rs = np.random.RandomState(4)
    if family == "waterworld":
        cfg = dict(n_pursuers=2, n_evaders=3, n_poison=2, n_sensors=5)
        eng = EmuWaterworld(1, seed=seed, **cfg)
        orc = WaterworldOracle(rng=Stream(seed, 0), **cfg)
        act = rs.randn(T, 1, 2, 2) * 0.3
    else:
        args = (2, 3, 2, 3, 1)
        kw = dict(n_sensors=5, bomb_radius=1e-4)    # a bomb nobody hits and hostages nobody can all save
        eng = EmuHostage(1, *args, seed=seed, **kw)
        orc = HostageOracle(*args, rng=Stream(seed, 0), **kw)
        act = rs.randn(T, 1, 2, 2) * 0.3
    assert np.abs(np.array(orc.reset()) - eng.reset()[0]).max() < 1e-9
    obs, rew, done, info = eng.rollout(act, auto_reset=True)
    n_done = 0
    for t in range(T):
        oo, rr, dd, ii = orc.step(act[t, 0])
        assert bool(done[t, 0]) == dd, t
        assert np.abs(rr - rew[t, 0]).max() < 1e-9, t
        if dd:
            oo = orc.reset()
            n_done += 1
        assert np.abs(np.array(oo) - obs[t, 0]).max() < 1e-9, t
    assert n_done >= 1
    if family == "waterworld":
        assert bool(done[998, 0]) and done.sum() == 1   # reset() consumed step 1: index 998 is the 1000th step


@pytest.mark.parametrize("variant", ["default"])
def test_waterworld_fused_peer_gather_layout(variant):
    """The PEER instantiation of the Waterworld kernel (in-kernel stores into other ranks' gather
    buffers over NVLink, madrl_ww_set_peers): two "ranks" with different env shards write their
    reward / done / info rows into slot `rank` of two destination buffers, env-major
    [n_slots][E][t_max][...], including partial reward runs at the end of the rollout."""
    import ctypes as C
    from emu.driver import EmuWaterworld
    cfg = dict(n_pursuers=5, n_evaders=5)
    E, T, t_max, n_ranks = 3, 37, 40, 2     # 37 steps: a partial 32-step done/info flush and reward run
    dests = [dict(rew=np.full((n_ranks, E, t_max, 5), np.nan), done=np.full((n_ranks, E, t_max), 255, np.uint8),
                  info=np.full((n_ranks, E, t_max, 2), -1, np.int32)) for _ in range(2)]
    outs = []
    for rank in range(n_ranks):
        eng = EmuWaterworld(E, seed=8, env_id_base=rank * E, max_path_length=9, defines=VARIANTS[variant], **cfg)
        arr = lambda k: (C.c_void_p * 2)(*[d[k].ctypes.data for d in dests])   # noqa: E731
        assert eng.lib.madrl_ww_set_peers(eng._h, 2, rank, t_max, arr('rew'), arr('done'), arr('info')) == 0
        eng.reset()
        act = np.random.RandomState(rank).randn(T, E, 5, 2) * 0.5
        outs.append(eng.rollout(act, auto_reset=True))
    for d in dests:
        for rank, (obs, rew, done, info) in enumerate(outs):
            assert np.array_equal(d['rew'][rank, :, :T], rew.transpose(1, 0, 2))
            assert np.array_equal(d['done'][rank, :, :T], done.T)
            assert np.array_equal(d['info'][rank, :, :T], info.transpose(1, 0, 2))
            assert np.isnan(d['rew'][rank, :, T:]).all() and (d['done'][rank, :, T:] == 255).all()


def _peer_dests(n_dest, n_slots, E, t_max, Np):
    """Destination gather buffers filled with sentinels, and the ctypes pointer tables of set_peers."""
    import ctypes as C
    dests = [dict(rew=np.full((n_slots, E, t_max, Np), np.nan), done=np.full((n_slots, E, t_max), 255, np.uint8),
                  info=np.full((n_slots, E, t_max, 2), -1, np.int32)) for _ in range(n_dest)]
    return dests, lambda k: (C.c_void_p * n_dest)(*[d[k].ctypes.data for d in dests])


@pytest.mark.parametrize("name,T,mpl", [("minimum", 1, 0), ("minimum", 33, 11), ("np32_k64", 1, 1)])
def test_waterworld_fused_peer_gather_edge_shapes(name, T, mpl):
    """The peer rows at the staging edges: one pursuer (32-step reward runs: T = 1 is a partial run of one step,
    T = 33 a full run and a partial one, with a reset on the last step) and 32 pursuers (one step per run).  Two
    ranks of 3 envs each write slot `rank` of a 3-slot buffer; the emulated grid has 2 warps, so one warp steps two
    envs.  The rows equal an unsharded rollout of all 6 envs without peers, and the rest stays as it was."""
    from emu.driver import EmuWaterworld
    cfg = WW[name]
    Np, E, W, t_max = cfg["n_pursuers"], 3, 2, T + 3
    dests, arr = _peer_dests(2, W + 1, E, t_max, Np)
    act = np.random.RandomState(T).randn(T, W * E, Np, 2) * 0.6
    ref = EmuWaterworld(W * E, seed=6, max_path_length=mpl, **cfg)
    ref.reset()
    want = ref.rollout(act, auto_reset=mpl > 0)
    for rank in range(W):
        eng = EmuWaterworld(E, seed=6, env_id_base=rank * E, max_path_length=mpl, **cfg)
        assert eng.lib.madrl_ww_set_peers(eng._h, 2, rank, t_max, arr('rew'), arr('done'), arr('info')) == 0
        eng.reset()
        got = eng.rollout(act[:, rank * E:(rank + 1) * E], auto_reset=mpl > 0)
        for x, y in zip(got, want):
            assert np.array_equal(x, y[:, rank * E:(rank + 1) * E])
    for d in dests:
        for rank in range(W):
            s = slice(rank * E, (rank + 1) * E)
            assert np.array_equal(d['rew'][rank, :, :T], want[1][:, s].transpose(1, 0, 2))
            assert np.array_equal(d['done'][rank, :, :T], want[2][:, s].T)
            assert np.array_equal(d['info'][rank, :, :T], want[3][:, s].transpose(1, 0, 2))
        assert np.isnan(d['rew'][:, :, T:]).all() and (d['done'][:, :, T:] == 255).all() and (d['info'][:, :, T:] == -1).all()
        assert np.isnan(d['rew'][W:]).all() and (d['done'][W:] == 255).all() and (d['info'][W:] == -1).all()


def test_waterworld_launch_log():
    """madrl_ww_launch_log records each launch's instantiation and grid while it is on, counts launches past the
    buffer it is given, and records nothing while it is off."""
    from emu.driver import EmuWaterworld
    eng = EmuWaterworld(3, seed=4, **WW["c2"])
    lib, recs = eng.lib, np.full((4, 10), -9, np.int32)
    assert lib.madrl_ww_launch_log(1, None, 0) >= 0
    eng.reset()
    act = np.zeros((2, 3, 5, 2))
    eng.rollout(act)
    dests, arr = _peer_dests(1, 1, 3, 2, 5)
    assert lib.madrl_ww_set_peers(eng._h, 1, 0, 2, arr('rew'), arr('done'), arr('info')) == 0
    eng.rollout(act)
    assert lib.madrl_ww_launch_log(1, _p(recs), 2) == 3
    # fp64, OPL 1, compile-time K = 30; the emulated device has 2 SMs with one resident block each
    assert recs[:2].tolist() == [[8, 8, 1, 1, 30, 0, 0, 0, 0, 2]] * 2 and (recs[2:] == -9).all()
    eng.rollout(act)
    assert lib.madrl_ww_launch_log(0, _p(recs), 4) == 1 and recs[0].tolist() == [8, 8, 1, 1, 30, 1, 0, 0, 0, 2]
    eng.rollout(act)
    assert lib.madrl_ww_launch_log(0, None, 0) == 0
    assert lib.madrl_ww_launch_log(0, None, 1) == -1


def test_waterworld_peer_exchange_refuses_host_rollout():
    """The host-buffer rollout cuts a rollout into chunked launches, and each launch would write its peer rows from
    step 0 of the gather buffers.  With peers set it is refused, with one chunk or several, and writes nothing; once
    the peers are cleared it runs again."""
    from emu.driver import EmuWaterworld
    cfg = WW["c2"]
    E, T, Np = 3, 13, 5
    eng = EmuWaterworld(E, seed=4, max_path_length=7, fp64=False, **cfg)
    eng.reset()
    dests, arr = _peer_dests(1, 1, E, T, Np)
    for d in dests:
        d['rew'] = d['rew'].astype(np.float32)
    assert eng.lib.madrl_ww_set_peers(eng._h, 1, 0, T, arr('rew'), arr('done'), arr('info')) == 0
    act = np.ascontiguousarray(np.random.RandomState(2).randn(T, E, Np, 2).astype(np.float32))
    f = eng.lib.madrl_ww_rollout_host2
    step_bytes = E * Np * eng.obs_dim * 4
    try:
        for chunk in (0, 3 * step_bytes):                 # one chunk (the default size), ~3 steps per chunk
            eng.lib.madrl_set_host_chunk_bytes(chunk)
            for host in (f, eng.lib.madrl_ww_rollout_host):
                bufs = [Guarded((T, E, Np, eng.obs_dim), np.float32, np.nan), Guarded((T, E, Np), np.float32, np.nan),
                        Guarded((T, E), np.uint8, 255), Guarded((T, E, 2), np.int32, -1)]
                args = (eng._h, T, _p(act), *[_p(b.arr) for b in bufs], 1) + ((0,) if host is f else ())
                assert host(*args) == -1
                assert b"set_peers" in eng.lib.madrl_last_error()
                assert all(np.isnan(b.check("host").astype(np.float64)).all() for b in bufs[:2])
                assert (bufs[2].arr == 255).all() and (bufs[3].arr == -1).all()
        d = dests[0]
        assert np.isnan(d['rew']).all() and (d['done'] == 255).all() and (d['info'] == -1).all()
        assert eng.lib.madrl_ww_set_peers(eng._h, 0, 0, 0, None, None, None) == 0
        ref = EmuWaterworld(E, seed=4, max_path_length=7, fp64=False, **cfg)
        ref.reset()
        for x, y in zip(eng.rollout(act, host=True), ref.rollout(act)):
            assert np.array_equal(x, y)
        assert np.isnan(d['rew']).all() and (d['done'] == 255).all() and (d['info'] == -1).all()
    finally:
        eng.lib.madrl_set_host_chunk_bytes(0)


def _vec_executor_check(eng, oracles, act, mpl, exact, info_of):
    """VecEnvExecutor.step semantics (vec_env_executor.py:16-28) against per-env oracles: done at the
    env's own terminal state or at max_path_length, reset in place, obs slot = reset observation."""
    T, E = act.shape[:2]
    obs, rew, done, info = eng.rollout(act, auto_reset=True)
    ts = np.zeros(E, int)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            ts[e] += 1
            dd = dd or ts[e] >= mpl
            assert bool(done[t, e]) == dd, (t, e)
            assert info_of(ii) == list(np.atleast_1d(info[t, e])), (t, e)
            if dd:
                oo = o.reset()
                ts[e] = 0
            if exact:
                assert np.array_equal(f32(oo).reshape(obs[t, e].shape), obs[t, e]) and np.array_equal(f32(rr), rew[t, e])
            else:
                assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9 and np.abs(rr - rew[t, e]).max() < 1e-9, (t, e)


@pytest.mark.parametrize("variant", ["default"])
@pytest.mark.parametrize("case", range(5))
def test_random_configurations_with_horizon_and_auto_reset(variant, case):
    from emu.driver import EmuHostage, EmuPursuit, EmuWaterworld
    rs = np.random.RandomState(7000 + case)
    mpl, seed, base, E, T = int(rs.randint(3, 12)), int(rs.randint(1 << 30)), int(rs.randint(1000)), 3, 30
    # Waterworld
    cfg = _ww_random_cfg(rs)
    cfg.update(n_evaders=min(cfg['n_evaders'], 20), n_poison=min(cfg['n_poison'], 20))
    eng = EmuWaterworld(E, seed=seed, env_id_base=base, max_path_length=mpl, defines=VARIANTS[variant], **cfg)
    orc = [WaterworldOracle(rng=Stream(seed, base + e), **cfg) for e in range(E)]
    eng.reset(); [o.reset() for o in orc]
    _vec_executor_check(eng, orc, rs.randn(T, E, cfg['n_pursuers'], 2) * 0.8, mpl, False,
                        lambda ii: [ii['evcatches'], ii['pocatches']])
    # Hostage
    args = (int(rs.randint(1, 12)), int(rs.randint(1, 20)), int(rs.randint(1, 20)), int(rs.randint(1, 3)), 1)
    kw = dict(radius=float(rs.uniform(0.02, 0.06)), n_sensors=int(rs.randint(1, 40)), key_radius=0.05,
              reward_mech=['local', 'global'][rs.randint(2)])
    eng = EmuHostage(E, *args, seed=seed, env_id_base=base, max_path_length=mpl, defines=VARIANTS[variant], **kw)
    orc = [HostageOracle(*args, rng=Stream(seed, base + e), **kw) for e in range(E)]
    eng.reset(); [o.reset() for o in orc]
    _vec_executor_check(eng, orc, rs.randn(T, E, args[0], 2) * 2.0, mpl, False, lambda ii: [ii['ho_saved'], ii['cr_encs']])
    # Pursuit
    pcfg = dict(n_evaders=int(rs.randint(1, 12)), n_pursuers=int(rs.randint(1, 12)), obs_range=int(rs.randint(1, 8)),
                surround=bool(rs.randint(2)), n_catch=int(rs.randint(1, 3)), reward_mech=['local', 'global'][rs.randint(2)],
                catchr=0.1, sample_maps=True, flatten=bool(rs.randint(2)))
    maps = pool16() if rs.randint(2) else small_map()
    eng = EmuPursuit(E, maps, seed=seed, env_id_base=base, max_path_length=mpl, defines=VARIANTS[variant], **pcfg)
    orc = [PursuitOracle(maps, rng=Stream(seed, base + e), **pcfg) for e in range(E)]
    eng.reset(); [o.reset() for o in orc]
    _vec_executor_check(eng, orc, rs.randint(0, 5, size=(T, E, pcfg['n_pursuers'])).astype(np.int32), mpl, True,
                        lambda ii: [ii['removed']])


def test_host_entry_points_equal_device_entry_points():
    """*_reset_host / *_rollout_host (staging copies inside the library) against the device-pointer
    entry points, Pursuit and Hostage (Waterworld: see the auto-reset test above)."""
    from emu.driver import EmuHostage, EmuPursuit
    maps = pool16()
    mk = [lambda: EmuPursuit(4, maps, seed=3, max_path_length=6, **C3),
          lambda: EmuHostage(4, 10, 16, 16, 4, 2, seed=3, max_path_length=6, fp64=False)]
    acts = [np.random.RandomState(0).randint(0, 5, size=(14, 4, 8)).astype(np.int32),
            np.random.RandomState(1).randn(14, 4, 10, 2).astype(np.float32)]
    for make, act in zip(mk, acts):
        a, b = make(), make()
        oa = a.reset()
        ob = Guarded(oa.shape, oa.dtype, 0)
        assert b._f("reset_host")(b._h, None, _p(ob.arr)) == 0
        assert np.array_equal(oa, ob.check("obs"))
        for x, y in zip(a.rollout(act, host=False), b.rollout(act, host=True)):
            assert np.array_equal(x, y)


def test_pipelined_host_rollout_chunks_and_obs_last_mode():
    """csrc/host_pipeline.cuh: the host-buffer rollout cut into several chunks (chunk size forced down)
    must equal the single device launch for every family, and MADRL_HOST_OBS_LAST returns rewards /
    dones / infos of every step + only the last step's observations."""
    from emu.driver import EmuHostage, EmuPursuit, EmuWaterworld
    maps = pool16()
    mk = [lambda: EmuWaterworld(3, seed=4, max_path_length=7, fp64=False, **WW["c2"]),
          lambda: EmuPursuit(3, maps, seed=4, max_path_length=7, **C3),
          lambda: EmuHostage(3, 10, 16, 16, 4, 2, seed=4, max_path_length=7, fp64=False)]
    T = 13                                   # odd: chunk boundaries must keep the info rows 8-byte aligned
    acts = [np.random.RandomState(2).randn(T, 3, 5, 2).astype(np.float32),
            np.random.RandomState(0).randint(0, 5, size=(T, 3, 8)).astype(np.int32),
            np.random.RandomState(1).randn(T, 3, 10, 2).astype(np.float32)]
    for make, act in zip(mk, acts):
        a, b, c = make(), make(), make()
        for e in (a, b, c):
            e.reset()
        ref = a.rollout(act, host=False)
        b.lib.madrl_set_host_chunk_bytes(ref[0][0].nbytes * 3)          # ~3 steps per chunk -> 5 chunks
        try:
            for x, y in zip(ref, b.rollout(act, host=True)):
                assert np.array_equal(x, y)
            f = getattr(c.lib, "madrl_%s_rollout_host2" % c.fam)
            E, A = c.n_envs, c.n_agents
            bufs = [Guarded((E, A, c.obs_dim), c.obs_dtype, np.nan), Guarded((T, E, A), c.obs_dtype, np.nan),
                    Guarded((T, E), np.uint8, 255), Guarded((T, E) + c.info_shape, np.int32, -1)]
            assert f(c._h, T, _p(np.ascontiguousarray(act)), *[_p(x.arr) for x in bufs], 1, 1) == 0
            last, rew, done, info = [x.check("host2") for x in bufs]
            assert np.array_equal(last, ref[0][-1]) and np.array_equal(rew, ref[1])
            assert np.array_equal(done, ref[2]) and np.array_equal(info, ref[3])
            assert f(c._h, T, _p(np.ascontiguousarray(act)), *[_p(x.arr) for x in bufs], 1, 2) == -1   # unknown flag
        finally:
            b.lib.madrl_set_host_chunk_bytes(0)


@pytest.mark.parametrize("family", ["waterworld", "pursuit", "hostage"])
def test_terminal_observations_are_kept_on_the_side(family):
    """madrl_*_set_terminal_obs: with auto-reset the obs slot of a done step holds the reset observation;
    the side tensor receives the observation the env returned before it was reset (what
    StandardizedEnv.step sees first, madrl_environments/__init__.py:283-291); other slots stay untouched."""
    from emu.driver import EmuHostage, EmuPursuit, EmuWaterworld
    mpl, T, E = 5, 17, 3
    if family == "waterworld":
        mk = lambda **kw: EmuWaterworld(E, seed=6, fp64=True, **WW["c2"], **kw)          # noqa: E731
        act = np.random.RandomState(0).randn(T, E, 5, 2)
    elif family == "pursuit":
        mk = lambda **kw: EmuPursuit(E, pool16(), seed=6, **C3, **kw)                     # noqa: E731
        act = np.random.RandomState(0).randint(0, 5, size=(T, E, 8)).astype(np.int32)
    else:
        mk = lambda **kw: EmuHostage(E, 10, 16, 16, 4, 2, seed=6, fp64=True, **kw)        # noqa: E731
        act = np.random.RandomState(0).randn(T, E, 10, 2)
    a, b = mk(max_path_length=mpl), mk(max_path_length=mpl)
    a.reset(), b.reset()
    obs_a, rew_a, done_a, _ = a.rollout(act, auto_reset=True)
    term = Guarded(obs_a.shape, obs_a.dtype, -7.0)
    f = getattr(b.lib, "madrl_%s_set_terminal_obs" % b.fam)
    assert f(b._h, _p(term.arr)) == 0
    obs_b, rew_b, done_b, _ = b.rollout(act, auto_reset=True)
    assert f(b._h, None) == 0
    t_arr = term.check("terminal obs")
    assert np.array_equal(obs_a, obs_b) and np.array_equal(done_a, done_b) and done_a.sum() >= E * (T // mpl)
    # reference run without auto-reset, reset by hand: its step obs at a done step is the terminal observation
    c = mk(max_path_length=mpl)
    c.reset()
    for t in range(T):
        o, _, d, _ = c.rollout(act[t:t + 1], auto_reset=False)
        for e in range(E):
            if d[0, e]:
                assert np.array_equal(t_arr[t, e], o[0, e]), (t, e)
            else:
                assert (t_arr[t, e] == -7.0).all(), (t, e)
        if d[0].any():
            c.reset(mask=d[0])
