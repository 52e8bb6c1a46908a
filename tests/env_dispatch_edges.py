"""Cases shared by the dispatch-edge tests of Pursuit's and Hostage's rollout kernels (pe_kernel in csrc/pursuit.cu,
hw_kernel in csrc/hostage.cu): tests/test_env_dispatch_edges_gpu.py runs them on the device,
tests/test_emulated_env_dispatch.py in the warp emulator of tests/emu.

hw_launch_t picks OPL (object chunks per lane) from the n_hostages + n_bad non-rescuer objects: 1 for <= 32, 2 for
<= 64, 4 for <= 128, 8 for <= 255; and the sensor layout from K: KC = 30 (compile-time K) for K = 30, KCH = 1 for any
other K <= 32, KCH = 2 for K = 33..64.  pe_launch_t picks EPL (evader chunks per lane) from n_evaders (1 for <= 32,
2 for <= 64) and the window layout from obs_range R: RC = 7 (compile-time R, CPL 2) for R = 7, else CPL =
ceil(R^2 / 32) cells per lane, rounded up to 4 when it is 3.  Each case names the instantiation it must reach, as
the launch-log records (madrl_pursuit_launch_log / madrl_hostage_launch_log) spell it, and every test checks the log
against that name before it compares values: a case that drifted to another kernel fails instead of passing on a
wider kernel's identical numbers.

The Hostage cases put the object and sensor counts on the dispatch boundaries, with radii and sensor ranges large
enough that objects of chunks >= 1 are sensed and hit; `HostageProbe` measures that from the float64 oracle.  The
Pursuit cases cover every (EPL, window layout, flatten) triple on maps up to 255 cells on a side.  No case can hang
the reset's redraw loop: maps with buildings keep free cells and spawn over the whole map (constraint_window = 1),
and constraint_window < 1 is used only on maps without buildings."""
import numpy as np
from scipy.spatial import distance as ssd

from oracle.hostage_oracle import HostageOracle
from oracle.philox import Stream
from oracle.pursuit_oracle import PursuitOracle

TOL64 = 1e-9
KEY_IN_SPAWN = np.array([[0.5, 0.75]])   # inside the rescuers' spawn band: with a large key_radius the gate opens at once


# ------------------------------------------------------------------------------------------------ Hostage
class HCase(object):
    """args = (n_good, n_hostages, n_bad, n_coop_save, n_coop_avoid) as BatchedHostageWorld takes them; `inst` =
    (OPL, KCH, KC) of the kernel the launch must run; `events`: which of "save", "gate" and "bomb" the case's
    trajectory test must see."""

    def __init__(self, name, inst, args, events=(), E=8, T=40, **kw):
        self.name, self.inst, self.args, self.kw, self.events, self.E, self.T = name, inst, args, kw, events, E, T
        self.Nr, self.Nh, self.Nc = args[0], args[1], args[2]
        self.K = kw.get("n_sensors", 30)
        n_obj = self.Nh + self.Nc
        assert 1 <= self.Nr <= 32 and n_obj + self.Nr <= 256, name
        opl = {1: 1, 2: 2, 3: 4, 4: 4}.get(-(-n_obj // 32), 8)
        assert inst == (opl, 1 if self.K <= 32 else 2, 30 if self.K == 30 else 0), name
        # chunk c of a lane holds non-rescuer objects 32 c .. 32 c + 31: the criminals first, then the hostages
        self.crim_hi = self.Nc > 32
        self.host_hi = n_obj > 32

    def __repr__(self):
        return self.name


# At most 30 hostages per case: the float32 teacher-forced test compares rewards within 1e-5, and a finished env's
# not-saved penalty (-3 per unsaved hostage) then stays below 128, where float32 rounds the reward within that.
H_CASES = [
    # OPL 1: 32 non-rescuer objects
    HCase("o1_k30", (1, 1, 30), (3, 12, 20, 1, 1), ("save", "gate"), radius=0.04, sensor_range=0.5,
          key_loc=KEY_IN_SPAWN, key_radius=0.5, reward_mech="local"),
    HCase("o1_k1", (1, 1, 0), (2, 16, 16, 2, 1), ("gate",), n_sensors=1, radius=0.05, sensor_range=0.6,
          key_radius=0.3, addid=False),
    HCase("o1_k64", (1, 2, 0), (4, 10, 22, 1, 1), ("save", "gate", "bomb"), n_sensors=64, radius=0.04,
          sensor_range=0.5, key_loc=KEY_IN_SPAWN, key_radius=0.5, bomb_radius=0.35),
    # OPL 2: 33 (the hostage alone in chunk 1) and 64
    HCase("o2_k30", (2, 1, 30), (5, 1, 32, 1, 1), ("save", "gate"), radius=0.04, sensor_range=0.6,
          key_loc=KEY_IN_SPAWN, key_radius=0.5, reward_mech="local"),
    HCase("o2_k29", (2, 1, 0), (6, 24, 40, 2, 1), ("gate",), n_sensors=29, radius=0.04, sensor_range=0.5,
          key_radius=0.3, addid=False),
    HCase("o2_k33", (2, 2, 0), (3, 20, 13, 3, 1), ("gate",), n_sensors=33, radius=0.05, sensor_range=0.5,
          key_loc=KEY_IN_SPAWN, key_radius=0.5, reward_mech="local"),
    # OPL 4: 65 and 128
    HCase("o4_k30", (4, 1, 30), (4, 25, 40, 1, 1), ("save", "gate", "bomb"), radius=0.03, sensor_range=0.5,
          key_loc=KEY_IN_SPAWN, key_radius=0.5, bomb_radius=0.3),
    HCase("o4_k31", (4, 1, 0), (8, 28, 100, 2, 1), ("save", "gate"), n_sensors=31, radius=0.03, sensor_range=0.4,
          key_loc=KEY_IN_SPAWN, key_radius=0.5, reward_mech="local"),
    HCase("o4_k64", (4, 2, 0), (2, 5, 60, 1, 1), ("gate",), n_sensors=64, radius=0.04, sensor_range=0.5,
          key_radius=0.3, addid=False),
    # OPL 8: 129, 255 (one rescuer, 256 objects in all) and 224 with 32 rescuers (an empty last chunk)
    HCase("o8_k30", (8, 1, 30), (1, 30, 225, 1, 1), ("save", "gate", "bomb"), E=6, T=30, radius=0.04,
          sensor_range=0.5, key_loc=KEY_IN_SPAWN, key_radius=0.5, bomb_radius=0.3),
    HCase("o8_k32", (8, 1, 0), (6, 29, 100, 2, 1), ("save", "gate"), E=6, T=30, n_sensors=32, radius=0.03,
          sensor_range=0.4, key_loc=KEY_IN_SPAWN, key_radius=0.5, reward_mech="local"),
    HCase("o8_k33", (8, 2, 0), (32, 20, 204, 3, 1), ("gate", "bomb"), E=4, T=20, n_sensors=33, radius=0.02,
          sensor_range=0.3, key_loc=KEY_IN_SPAWN, key_radius=0.5),
]
H_BY_NAME = {c.name: c for c in H_CASES}

# every (OPL, KCH, KC) hw_launch_t dispatches to, written out
HW_PAIRS = [(opl, kch, kc) for opl in (1, 2, 4, 8) for kch, kc in ((1, 30), (1, 0), (2, 0))]
# (sizeof(real), sizeof(O), KEEP): fp64, fp32, fp32 KEEP, bf16, bf16 KEEP
HW_TYPES = [(8, 8, 0), (4, 4, 0), (4, 4, 1), (4, 2, 0), (4, 2, 1)]
HW_ALL = {(r, o, opl, kch, kc, keep) for opl, kch, kc in HW_PAIRS for r, o, keep in HW_TYPES}
assert len(HW_ALL) == 60 and {c.inst for c in H_CASES} == set(HW_PAIRS)


def hw_record(case, real, obs, keep):
    """The launch-log record of `case`'s instantiation, without the grid."""
    return (real, obs) + case.inst + (keep,)


def hw_actions(case, E, T, seed=5, std=3.0):
    return np.random.RandomState(seed).randn(T, E, case.Nr, 2) * std


class HostageProbe(HostageOracle):
    """The float64 oracle, recording per step which object chunks the kernel's sensing and criminal respawns reach:
    the chunks of every sensor's nearest criminal, of every sensor's nearest hostage while the gate is open, and of
    the criminals that met a rescuer."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.sensed_c, self.sensed_h, self.hit_chunks = set(), set(), []

    def _sensed(self, i, objx, same=False):
        sv = super()._sensed(i, objx, same)
        if objx is self.cx:
            self._sv_c.append(sv)
        elif objx is self.hx:
            self._sv_h.append(np.where(self._saved_pre[None, :], np.inf, sv))
        return sv

    def step(self, action):
        self._sv_c, self._sv_h, self._saved_pre = [], [], self.saved.copy()
        gate_pre, cx_pre = self.gate_open, self.cx.copy()
        out = super().step(action)
        for sv in self._sv_c:
            j = np.argmin(sv, axis=1)[np.isfinite(sv.min(axis=1))]
            self.sensed_c |= set((j // 32).tolist())
        if gate_pre:
            for sv in self._sv_h:
                j = np.argmin(sv, axis=1)[np.isfinite(sv.min(axis=1))]
                self.sensed_h |= set(((self.Nc + j) // 32).tolist())
        hit = np.where((ssd.cdist(self.rx, cx_pre) <= self.r_r + self.r_c).any(axis=0))[0]
        self.hit_chunks.append(set((hit // 32).tolist()))
        return out


def hw_oracles(case, seed, base, E):
    return [HostageProbe(*case.args, rng=Stream(seed, base + e), **case.kw) for e in range(E)]


def hw_check_trajectory(case, oracles, obs0, act, obs, rew, done, info, mpl, term=None):
    """The engine's auto-reset trajectory (NumPy, float64) against the oracles, within TOL64; `term`: the
    set_terminal_obs tensor, which must hold the oracle's terminal observation at the done slots and its fill (NaN)
    everywhere else.  -> the events seen: {"save", "gate", "bomb", "done"}."""
    T, E = act.shape[:2]
    seen = set()
    for e, o in enumerate(oracles):
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < TOL64, (case, e)
    ts = np.zeros(E, int)
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            seen |= {"save"} if ii['ho_saved'] else set()
            seen |= {"gate"} if o.gate_open else set()
            seen |= {"bomb"} if o.bombed else set()
            ts[e] += 1
            dd = dd or ts[e] >= mpl
            where = (case, t, e)
            assert [ii['ho_saved'], ii['cr_encs']] == list(info[t, e]), where
            assert bool(done[t, e]) == dd, where
            assert np.abs(rr - rew[t, e]).max() < TOL64, where
            if term is not None:
                if dd:
                    assert np.abs(np.array(oo) - term[t, e]).max() < TOL64, where
                else:
                    assert np.isnan(term[t, e]).all(), where
            if dd:
                oo, ts[e] = o.reset(), 0
                seen.add("done")
            assert np.abs(np.array(oo) - obs[t, e]).max() < TOL64, where
    return seen


def hw_check_state(case, arr, oracles):
    """Final per-env state (the dict `Batched*.state` names, as NumPy) against the oracles."""
    Nr, Nc = case.Nr, case.Nc
    for e, o in enumerate(oracles):
        X = np.stack([arr['pos_x'][e], arr['pos_y'][e]], 1).astype(np.float64)
        V = np.stack([arr['vel_x'][e], arr['vel_y'][e]], 1).astype(np.float64)
        flags = int(arr['flags'][e])
        assert int(arr['rng_counter'][e]) == o.np_random.counter and int(arr['timestep'][e]) == o.t, (case, e)
        assert bool(flags & 1) == o.gate_open and bool(flags & 2) == o.bombed, (case, e)
        assert np.array_equal(arr['saved'][e].astype(bool), o.saved), (case, e)
        for got, want in ((X[:Nr], o.rx), (V[:Nr], o.rv), (X[Nr:Nr + Nc], o.cx), (V[Nr:Nr + Nc], o.cv),
                          (X[Nr + Nc:], o.hx)):
            assert np.abs(got - want).max() < TOL64, (case, e)
        assert np.abs(arr['key'][e] - o.key_loc[0]).max() < 1e-12 and np.abs(arr['bomb'][e] - o.bomb[0]).max() < 1e-12


def hw_check_reach(case, oracles):
    """Objects of chunks >= 1 were sensed, a nearest criminal lay in chunk >= 1 (its velocity is read through
    iC >> 5), and criminals of two chunks met rescuers in one step (the respawn draws carry across chunks)."""
    sensed_c = set().union(*[o.sensed_c for o in oracles])
    sensed_h = set().union(*[o.sensed_h for o in oracles])
    if case.crim_hi:
        assert max(sensed_c) >= 1, (case, sensed_c)
        assert any(len(h) >= 2 for o in oracles for h in o.hit_chunks), case
    if case.host_hi:
        assert max(sensed_h, default=-1) >= 1, (case, sensed_h)


# ------------------------------------------------------------------------------------------------ Pursuit
def open_map(xs, ys):
    return np.zeros((1, xs, ys), np.int32)


def building_map(xs, ys, seed=0, n=1, frac=0.15):
    """`n` maps of xs x ys with about `frac` of their cells buildings (-1) and walls along a few rows and columns;
    every map keeps most cells free."""
    rs = np.random.RandomState(seed)
    m = np.where(rs.rand(n, xs, ys) < frac, -1, 0).astype(np.int32)
    for k in range(n):
        m[k, rs.randint(0, xs), rs.randint(0, ys // 2):] = -1
        m[k, rs.randint(0, xs // 2):, rs.randint(0, ys)] = -1
    assert (m == 0).sum(axis=(1, 2)).min() > xs * ys // 2
    return m


def one_cell_map():
    """2 x 2 with one free cell (0, 1): everybody spawns on it and nobody can move."""
    m = np.full((1, 2, 2), -1, np.int32)
    m[0, 0, 1] = 0
    return m


def pool16():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "maps", "map_pool16.npy"))


class PCase(object):
    """`inst` = (EPL, CPL, RC) of the kernel the launch must run; `maps()` builds the map pool; `gone_hi`: the
    trajectory must remove an evader of index >= 32 (chunk 1)."""

    def __init__(self, name, inst, maps, E=8, T=40, gone_hi=False, **cfg):
        self.name, self.inst, self.maps, self.cfg, self.E, self.T, self.gone_hi = name, inst, maps, cfg, E, T, gone_hi
        self.Np, self.Ne, self.R = cfg["n_pursuers"], cfg["n_evaders"], cfg["obs_range"]
        self.flat = int(cfg.get("flatten", True))
        epl = 1 if self.Ne <= 32 else 2
        cpl = {1: 1, 2: 2, 3: 4, 4: 4}[-(-self.R * self.R // 32)]
        assert inst == ((epl, 2, 7) if self.R == 7 else (epl, cpl, 0)), name
        assert not gone_hi or self.Ne > 32

    def __repr__(self):
        return self.name


C3 = dict(n_catch=2, surround=True, reward_mech="local", catchr=0.1, term_pursuit=5.0, include_id=True)
CATCH1 = dict(n_catch=1, surround=False, catchr=0.05, term_pursuit=5.0)
P_CASES = [
    # RC = 7
    PCase("e1_rc7_flat", (1, 2, 7), pool16, n_evaders=32, n_pursuers=8, obs_range=7, sample_maps=True, **C3),
    PCase("e1_rc7_conv", (1, 2, 7), lambda: building_map(255, 16, 1), n_evaders=1, n_pursuers=1, obs_range=7,
          flatten=False, reward_mech="global", **CATCH1),
    PCase("e2_rc7_flat", (2, 2, 7), lambda: building_map(255, 16, 2), gone_hi=True, n_evaders=40, n_pursuers=32,
          obs_range=7, reward_mech="local", **CATCH1),
    PCase("e2_rc7_conv", (2, 2, 7), lambda: building_map(64, 64, 3), gone_hi=True, n_evaders=33, n_pursuers=31,
          obs_range=7, flatten=False, reward_mech="global", urgency_reward=-0.1, **CATCH1),
    # CPL 1: R = 1 .. 5
    PCase("e1_c1_flat", (1, 1, 0), lambda: open_map(64, 64), n_evaders=32, n_pursuers=31, obs_range=1,
          constraint_window=0.15, reward_mech="local", **CATCH1),
    PCase("e1_c1_conv", (1, 1, 0), lambda: building_map(16, 255, 4), n_evaders=1, n_pursuers=32, obs_range=2,
          flatten=False, reward_mech="global", include_id=False, **CATCH1),
    PCase("e2_c1_flat", (2, 1, 0), one_cell_map, gone_hi=True, T=25, n_evaders=64, n_pursuers=32, obs_range=3,
          reward_mech="local", surround=False, n_catch=2, catchr=0.05),
    PCase("e2_c1_conv", (2, 1, 0), lambda: open_map(64, 64), gone_hi=True, n_evaders=64, n_pursuers=32, obs_range=4,
          flatten=False, constraint_window=0.12, random_opponents=True, max_opponents=65, reward_mech="local",
          **CATCH1),
    # CPL 2: R = 6, 8
    PCase("e1_c2_flat", (1, 2, 0), lambda: building_map(64, 64, 5), n_evaders=32, n_pursuers=16, obs_range=8,
          reward_mech="local", **CATCH1),
    PCase("e1_c2_conv", (1, 2, 0), lambda: building_map(16, 255, 6), n_evaders=12, n_pursuers=6, obs_range=6,
          flatten=False, **C3),
    PCase("e2_c2_flat", (2, 2, 0), lambda: building_map(64, 64, 7, n=3), gone_hi=True, n_evaders=40, n_pursuers=32,
          obs_range=6, sample_maps=True, reward_mech="global", **CATCH1),
    PCase("e2_c2_conv", (2, 2, 0), lambda: building_map(64, 64, 8), gone_hi=True, n_evaders=64, n_pursuers=20,
          obs_range=8, flatten=False, random_opponents=True, max_opponents=65, reward_mech="local", **CATCH1),
    # CPL 4: R = 9, 10, 11
    PCase("e1_c4_flat", (1, 4, 0), lambda: building_map(255, 16, 9), n_evaders=5, n_pursuers=4, obs_range=9,
          reward_mech="local", **CATCH1),
    PCase("e1_c4_conv", (1, 4, 0), pool16, n_evaders=32, n_pursuers=32, obs_range=11, flatten=False,
          sample_maps=True, **C3),
    PCase("e2_c4_flat", (2, 4, 0), lambda: open_map(64, 64), gone_hi=True, n_evaders=64, n_pursuers=31,
          obs_range=11, constraint_window=0.2, reward_mech="global", **CATCH1),
    PCase("e2_c4_conv", (2, 4, 0), pool16, gone_hi=True, n_evaders=33, n_pursuers=8, obs_range=10, flatten=False,
          sample_maps=True, reward_mech="local", **CATCH1),
]
P_BY_NAME = {c.name: c for c in P_CASES}

# every (EPL, CPL, RC) pe_launch_t dispatches to, written out
PE_LAYOUTS = [(epl, cpl, rc) for epl in (1, 2) for cpl, rc in ((2, 7), (1, 0), (2, 0), (4, 0))]
# (POLICY, KEEP): rollout, rollout with KEEP stores, heuristic policy (which always streams)
PE_MODES = [(0, 0), (0, 1), (1, 0)]
PE_ALL = {(o, epl, cpl, rc, pol, flat, keep) for epl, cpl, rc in PE_LAYOUTS for flat in (0, 1)
          for pol, keep in PE_MODES for o in (4, 2)}
assert len(PE_ALL) == 96 and {c.inst + (c.flat,) for c in P_CASES} == {l + (f,) for l in PE_LAYOUTS for f in (0, 1)}


def pe_record(case, obs, policy, keep):
    """The launch-log record of `case`'s instantiation, without the grid."""
    epl, cpl, rc = case.inst
    return (obs, epl, cpl, rc, policy, case.flat, keep)


def pe_actions(case, E, T, seed=9):
    return np.random.RandomState(seed).randint(0, 5, size=(T, E, case.Np)).astype(np.int32)


def f32(x):
    return np.asarray(x, dtype=np.float64).astype(np.float32)


def pe_oracles(case, maps, seed, base, E):
    return [PursuitOracle(maps, rng=Stream(seed, base + e), **case.cfg) for e in range(E)]


def pe_check_trajectory(case, oracles, obs0, act, obs, rew, done, removed, mpl, term=None):
    """The engine's auto-reset trajectory against the oracles, bit for bit (observations and rewards as float32);
    `term` as in hw_check_trajectory.  -> (evaders removed in all, whether one of index >= 32 was)."""
    T, E = act.shape[:2]
    for e, o in enumerate(oracles):
        assert np.array_equal(f32(o.reset()).reshape(obs0[e].shape), obs0[e]), (case, e)
    ts = np.zeros(E, int)
    n_removed, hi = 0, False
    for t in range(T):
        for e, o in enumerate(oracles):
            gone_pre = o.gone.copy()
            oo, rr, dd, ii = o.step(act[t, e])
            hi = hi or bool((o.gone & ~gone_pre)[32:].any())
            n_removed += ii['removed']
            ts[e] += 1
            dd = dd or ts[e] >= mpl
            where = (case, t, e)
            assert ii['removed'] == removed[t, e] and dd == bool(done[t, e]), where
            assert np.array_equal(f32(rr), rew[t, e]), where
            if term is not None:
                if dd:
                    assert np.array_equal(f32(oo).reshape(term[t, e].shape), term[t, e]), where
                else:
                    assert np.isnan(term[t, e]).all(), where
            if dd:
                oo, ts[e] = o.reset(), 0
            assert np.array_equal(f32(oo).reshape(obs[t, e].shape), obs[t, e]), where
    return n_removed, hi


def pe_check_state(case, st, oracles):
    """Final per-env state (the dict BatchedPursuitEvade.state names, as NumPy) against the oracles, including the
    never-cleared window channels (pursuit_evade.py:119,438)."""
    for e, o in enumerate(oracles):
        assert np.array_equal(st['pursuer_x'][e], o.ppos[:, 0]) and np.array_equal(st['pursuer_y'][e], o.ppos[:, 1])
        live = ~o.gone
        assert np.array_equal(st['evader_x'][e][live], o.epos[live, 0]), (case, e)
        assert np.array_equal(st['evader_y'][e][live], o.epos[live, 1]), (case, e)
        assert [(int(st['gone'][e]) >> j) & 1 for j in range(o.Ne)] == [int(x) for x in o.gone], (case, e)
        assert int(st['rng_counter'][e]) == o.rng.counter, (case, e)
        assert np.array_equal(o.map_pool[int(st['map_id'][e])], o.map), (case, e)
        stale = st['stale'][e].astype(np.uint16)
        ln = np.float32(o.layer_norm)
        c1 = (stale & 0xff).astype(np.float32) / ln
        c2 = (stale >> 8).astype(np.float32) / ln
        assert np.array_equal(c1.reshape(o.Np, o.R, o.R), o.local_obs[:, 1].astype(np.float32)), (case, e)
        assert np.array_equal(c2.reshape(o.Np, o.R, o.R), o.local_obs[:, 2].astype(np.float32)), (case, e)
