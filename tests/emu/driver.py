"""TEST INFRASTRUCTURE: ctypes drivers for the warp-emulator build of the kernels
(tests/emu/build_emu.py).  The emulator library exports the product's C ABI and is declared with the
product's signature table (madrl_b200/_lib.py); "device" pointers are host pointers, so the entry points
are called directly with NumPy arrays.  The engines take the arguments of
madrl_b200.{waterworld,pursuit,hostage}.Batched* and build their config structs with the same functions
(ww_config / pe_config / hw_config), so the tests read like the GPU ones and check the product's argument
mapping.
"""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from madrl_b200 import _lib as L
from madrl_b200.hostage import hw_config
from madrl_b200.pursuit import map_pool_array, pe_config
from madrl_b200.waterworld import ww_config

from . import build_emu

_libs = {}

needs_cxx = pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="no host C++ compiler")


def open_lib(path):
    """The emulator library at `path`, declared as the product library is."""
    lib = C.CDLL(path)
    L.declare(lib)
    L.check_struct_sizes(lib, path)
    lib.madrl_emu_race_count.restype = C.c_long
    lib.madrl_emu_race_reset.restype = None
    return lib


def load(defines=()):
    key = tuple(sorted(defines))
    if key not in _libs:
        _libs[key] = open_lib(build_emu.build(list(key)))
    return _libs[key]


def races(reset=True):
    """Shared-memory hazards (see smem_access in tests/emu/include/cuda_runtime.h) reported by every
    loaded emulator library since the last call."""
    n = 0
    for lib in _libs.values():
        n += int(lib.madrl_emu_race_count())
        if reset:
            lib.madrl_emu_race_reset()
    return n


def ptr(a):
    """A NumPy array's address as a pointer argument (None -> NULL)."""
    return C.c_void_p(a.ctypes.data) if a is not None else C.c_void_p(0)


def paths_plan(lib, done, A):
    """madrl_paths_plan of done uint8 [T, E] -> (seg_start, seg_len, n_episodes, ep_rec)."""
    T, E = done.shape
    seg_s, seg_l = np.full((T, E), -1, np.int32), np.full((T, E), -1, np.int32)
    n_ep, ep_rec = np.zeros(E, np.int32), np.zeros((E, T, 3), np.int32)
    assert lib.madrl_paths_plan(T, E, A, ptr(done), ptr(seg_s), ptr(seg_l), ptr(n_ep), ptr(ep_rec), None) == 0
    return seg_s, seg_l, n_ep, ep_rec


def moments(lib, rows, A, a, b=None):
    """stats float64 [A, 9] of the columns of a, b [rows, A] as madrl_b200.postproc combines madrl_moments_pass_f32:
    pass 0, its sums divided by the rows in float64, pass 1 about those means, its sums divided by the rows again."""
    st = Guarded((A, 9), np.float64, np.nan)
    ws = np.empty((A, 4096))
    assert lib.madrl_moments_pass_f32(rows, A, ptr(a), ptr(b), 0, ptr(st.arr), ptr(ws), None) == 0
    st.arr[:, 0:3] /= np.float64(rows)
    assert lib.madrl_moments_pass_f32(rows, A, ptr(a), ptr(b), 1, ptr(st.arr), ptr(ws), None) == 0
    st.arr[:, 3:6] /= np.float64(rows)
    return st.check("stats").copy()


def center_advantages(lib, rows, A, x, center, positive):
    """madrl_b200.postproc.center_advantages of x [rows, A] in place: `moments`, then madrl_center_apply_f32 ->
    the statistics it used."""
    stats = moments(lib, rows, A, x)
    assert lib.madrl_center_apply_f32(rows, A, ptr(x), ptr(stats), center, positive, None) == 0
    return stats


GUARD = 1 << 16   # bytes of canary on either side of every output buffer


class Guarded(object):
    """An output array embedded in a canary-filled allocation: out-of-row writes of a kernel show up
    as a failed check instead of silent corruption."""

    def __init__(self, shape, dtype, fill):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        self.raw = np.full(n + 2 * GUARD, 0xA5, np.uint8)
        self.arr = self.raw[GUARD:GUARD + n].view(dtype).reshape(shape)
        self.arr[...] = fill

    def check(self, what):
        assert (self.raw[:GUARD] == 0xA5).all() and (self.raw[-GUARD:] == 0xA5).all(), \
            "kernel wrote outside the %s buffer" % what
        return self.arr


class _Engine(object):
    fam = None

    def _check(self, rc):
        if rc != 0:
            raise RuntimeError("emulated madrl_b200 error %d: %s" % (rc, self.lib.madrl_last_error().decode()))

    def _f(self, name):
        return getattr(self.lib, "madrl_%s_%s" % (self.fam, name))

    def _finish(self, create_args):
        self.layout = self.LayoutT()
        self._check(self._f("state_layout")(C.byref(self.cfg), C.byref(self.layout)))
        self.obs_dim = int(self.layout.obs_dim)
        self.blob = np.zeros(int(self.layout.total_bytes), np.uint8)
        h = C.c_void_p()
        self._check(self._f("create")(C.byref(self.cfg), *create_args, ptr(self.blob), C.byref(h)))
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._f("destroy")(h)

    def view(self, off, dtype, shape):
        n = int(np.prod(shape)) * np.dtype(dtype).itemsize
        return self.blob[off:off + n].view(dtype).reshape(shape)

    def set_launch(self, warps_per_block=0, blocks_per_sm=0):
        self._check(self._f("set_launch")(self._h, warps_per_block, blocks_per_sm))

    def seed(self, seed):
        self._check(self._f("seed")(self._h, int(seed), None))

    def reset(self, mask=None):
        obs = Guarded((self.n_envs, self.n_agents, self.obs_dim), self.obs_dtype, 0)
        m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        self._check(self._f("reset")(self._h, ptr(m), ptr(obs.arr), None))
        return obs.check("obs")

    def rollout(self, actions, auto_reset=True, host=False):
        actions = np.ascontiguousarray(actions, self.act_dtype)
        T = actions.shape[0]
        E, A = self.n_envs, self.n_agents
        bufs = [Guarded((T, E, A, self.obs_dim), self.obs_dtype, np.nan), Guarded((T, E, A), self.obs_dtype, np.nan),
                Guarded((T, E), np.uint8, 255), Guarded((T, E) + self.info_shape, np.int32, -1)]
        ptrs = [ptr(b.arr) for b in bufs]
        if host:
            self._check(self._f("rollout_host")(self._h, T, ptr(actions), *ptrs, int(auto_reset)))
        else:
            self._check(self._f("rollout")(self._h, T, ptr(actions), *ptrs, int(auto_reset), None))
        return tuple(b.check(n) for b, n in zip(bufs, ("obs", "rew", "done", "info")))


    def rollout_heuristic(self, T, obs0, auto_reset=True, **kw):
        """Closed-loop rollout with the in-kernel heuristic policy -> (actions, obs, rew, done, info)."""
        E, A = self.n_envs, self.n_agents
        obs0 = np.ascontiguousarray(obs0, self.obs_dtype)
        assert obs0.shape == (E, A, self.obs_dim)
        bufs = [Guarded((T, E, A) + self.act_shape, self.act_dtype, -7),
                Guarded((T, E, A, self.obs_dim), self.obs_dtype, np.nan), Guarded((T, E, A), self.obs_dtype, np.nan),
                Guarded((T, E), np.uint8, 255), Guarded((T, E) + self.info_shape, np.int32, -1)]
        ptrs = [ptr(b.arr) for b in bufs]
        extra = [int(bool(kw.get("py2_division", True)))] if self.fam == "pursuit" else []
        self._check(self._f("rollout_heuristic")(self._h, T, ptr(obs0), *ptrs, int(auto_reset), *extra, None))
        return tuple(b.check(n) for b, n in zip(bufs, ("actions", "obs", "rew", "done", "info")))


def ww_heuristic_actions(obs, n_sensors, defines=()):
    """madrl_ww_heuristic_actions through the emulator: obs [n, D] float32 / float64 -> actions [n, 2]."""
    lib = load(defines)
    obs = np.ascontiguousarray(obs)
    out = Guarded((obs.shape[0], 2), obs.dtype, np.nan)
    rc = lib.madrl_ww_heuristic_actions(int(obs.dtype == np.float64), obs.shape[0], n_sensors, obs.shape[1], ptr(obs),
                                        ptr(out.arr), None)
    assert rc == 0, lib.madrl_last_error().decode()
    return out.check("actions")


def pursuit_heuristic_actions(obs, obs_range, flatten, fallback, py2_division=True, defines=()):
    """madrl_pursuit_heuristic_actions through the emulator: obs [n, D] float32 -> actions [n] int32."""
    lib = load(defines)
    obs = np.ascontiguousarray(obs, np.float32)
    fb = np.ascontiguousarray(fallback, np.int32)
    lut = np.zeros(128, np.uint8)
    out = Guarded((obs.shape[0],), np.int32, -9)
    rc = lib.madrl_pursuit_heuristic_actions(obs.shape[0], obs_range, int(flatten), obs.shape[1], int(py2_division),
                                             ptr(obs), ptr(fb), ptr(lut), ptr(out.arr), None)
    assert rc == 0, lib.madrl_last_error().decode()
    return out.check("actions")


class EmuWaterworld(_Engine):
    fam, LayoutT, info_shape, act_shape = "ww", L.WWLayout, (2,), (2,)

    def __init__(self, n_envs, *args, fp64=True, defines=(), **kw):
        """The arguments of BatchedMAWaterWorld (without device / dtype)."""
        self.lib = load(defines)
        self.cfg = ww_config(n_envs, *args, fp64=fp64, **kw)
        self.n_envs, self.n_pursuers, self.n_evaders = n_envs, self.cfg.n_pursuers, self.cfg.n_evaders
        self.n_agents = self.n_pursuers
        self.obs_dtype = self.act_dtype = np.float64 if fp64 else np.float32
        self._finish(())

    def state(self, e):
        Ly, N = self.layout, int(self.layout.n_obj)
        objs = self.view(Ly.objs, self.obs_dtype, (self.n_envs, 4, N))[e].astype(np.float64)
        X, V = objs[0:2].T, objs[2:4].T
        Np, Ne = self.n_pursuers, self.n_evaders
        obst = self.view(Ly.obst, self.obs_dtype, (self.n_envs, 2))[e].astype(np.float64)[None]
        return dict(px=X[:Np], pv=V[:Np], ex=X[Np:Np + Ne], ev=V[Np:Np + Ne], ox=X[Np + Ne:], ov=V[Np + Ne:],
                    obst=obst, t=int(self.view(Ly.timestep, np.int32, (self.n_envs,))[e]),
                    counter=int(self.view(Ly.rng_counter, np.int64, (self.n_envs,))[e]))


class EmuHostage(_Engine):
    fam, LayoutT, info_shape, act_shape = "hostage", L.HWLayout, (2,), (2,)

    def __init__(self, n_envs, *args, fp64=True, defines=(), **kw):
        """The arguments of BatchedHostageWorld (without device / dtype)."""
        self.lib = load(defines)
        self.cfg = hw_config(n_envs, *args, fp64=fp64, **kw)
        self.n_envs, self.n_agents, self.n_hostages = n_envs, self.cfg.n_good, self.cfg.n_hostages
        self.obs_dtype = self.act_dtype = np.float64 if fp64 else np.float32
        self._finish(())

    def state(self, e):
        Ly, E = self.layout, self.n_envs
        return dict(counter=int(self.view(Ly.rng_counter, np.int64, (E,))[e]),
                    t=int(self.view(Ly.timestep, np.int32, (E,))[e]),
                    flags=int(self.view(Ly.flags, np.int32, (E,))[e]),
                    saved=self.view(Ly.saved, np.uint8, (E, self.n_hostages))[e].astype(bool))


class EmuPursuit(_Engine):
    fam, LayoutT, info_shape, act_shape = "pursuit", L.PELayout, (), ()
    obs_dtype, act_dtype = np.float32, np.int32

    def __init__(self, n_envs, map_pool, *args, defines=(), **kw):
        """The arguments of BatchedPursuitEvade (without device)."""
        self.lib = load(defines)
        self.map_pool = map_pool_array(map_pool)
        self.cfg = pe_config(n_envs, self.map_pool, *args, **kw)
        self.n_envs, self.n_pursuers, self.n_evaders = n_envs, self.cfg.n_pursuers, self.cfg.n_evaders
        self.n_agents = self.n_pursuers
        self._finish((ptr(self.map_pool),))

    def state(self, e):
        Ly, E, Np = self.layout, self.n_envs, self.n_pursuers
        A = int(Ly.n_agents)
        pos = self.view(Ly.pos, np.uint8, (E, 2, A))[e]
        return dict(pursuers=pos[:, :Np].T.astype(int), evaders=pos[:, Np:].T.astype(int),
                    gone=int(self.view(Ly.gone, np.int64, (E,))[e]),
                    map_id=int(self.view(Ly.map_id, np.int32, (E,))[e]),
                    counter=int(self.view(Ly.rng_counter, np.int64, (E,))[e]))


# ---------------------------------------------------------------------------------------------------
# Test double for the DROP-IN classes (madrl_b200.MAWaterWorld / PursuitEvade / ContinuousHostageWorld):
# those classes talk to a `Batched*` engine (reset / step / seed / set_params returning torch tensors).
# `emulated_dropins()` swaps the engine classes for facades over the emulator engines above, so the
# drop-in code itself -- list-of-arrays returns, float64 conversion, info dicts, spaces, pickling,
# the vec_env_executor hook -- runs unchanged on a CPU box, against what the reference's own callers produced
# (tests/test_reference_callers.py).  On a GPU box the same classes run on the real library.
# ---------------------------------------------------------------------------------------------------
class _TorchFacade(object):
    def __init__(self, emu, info_keys):
        import torch
        self._t, self.emu, self._keys = torch, emu, info_keys
        self.n_envs, self.obs_dim = emu.n_envs, emu.obs_dim
        self.device = torch.device("cpu")
        self.dtype = torch.float64 if emu.obs_dtype == np.float64 else torch.float32

    def seed(self, seed=None):
        self.emu.seed(0 if seed is None else int(seed))
        return [seed]

    def reset(self, mask=None, out=None):
        return self._t.from_numpy(np.array(self.emu.reset(None if mask is None else np.asarray(mask))))

    def step(self, actions, auto_reset=False):
        a = np.asarray(actions).reshape((1, self.n_envs) + self._act_tail)
        obs, rew, done, info = [self._t.from_numpy(np.array(x)) for x in self.emu.rollout(a, auto_reset=auto_reset)]
        if len(self._keys) == 1:
            d = {self._keys[0]: info[0]}
        else:
            d = {k: info[0, :, i] for i, k in enumerate(self._keys)}
        return obs[0], rew[0], done[0], d


def _ww_facade(n_envs, *args, device=None, dtype=None, **kw):
    import torch
    f = _TorchFacade(EmuWaterworld(n_envs, *args, fp64=(dtype == torch.float64), **kw), ("evcatches", "pocatches"))
    f._act_tail = (f.emu.n_pursuers, 2)
    return f


def _hw_facade(n_envs, *args, device=None, dtype=None, **kw):
    import torch
    f = _TorchFacade(EmuHostage(n_envs, *args, fp64=(dtype == torch.float64), **kw), ("ho_saved", "cr_encs"))
    f._act_tail = (f.emu.n_agents, 2)
    return f


def _pe_facade(n_envs, map_pool, device=None, **kw):
    f = _TorchFacade(EmuPursuit(n_envs, map_pool, **kw), ("removed",))
    f._act_tail = (f.emu.n_pursuers,)

    def set_params(catchr, constraint_window):
        f.emu._check(f.emu.lib.madrl_pursuit_set_params(f.emu._h, float(catchr), float(constraint_window)))
    f.set_params = set_params
    import torch
    type(f).state = property(lambda self: {'gone': torch.tensor([self.emu.state(e)['gone'] for e in range(self.n_envs)])})
    return f


class emulated_dropins(object):
    """Context manager: madrl_b200's drop-in env classes run on the emulator engines."""

    def __enter__(self):
        import madrl_b200.hostage as H
        import madrl_b200.pursuit as P
        import madrl_b200.waterworld as W
        self._saved = (W.BatchedMAWaterWorld, P.BatchedPursuitEvade, H.BatchedHostageWorld)
        W.BatchedMAWaterWorld, P.BatchedPursuitEvade, H.BatchedHostageWorld = _ww_facade, _pe_facade, _hw_facade
        return self

    def __exit__(self, *exc):
        import madrl_b200.hostage as H
        import madrl_b200.pursuit as P
        import madrl_b200.waterworld as W
        W.BatchedMAWaterWorld, P.BatchedPursuitEvade, H.BatchedHostageWorld = self._saved
        return False
