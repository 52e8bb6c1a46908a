"""The observation cache policy (madrl_*_set_obs_cache) in the warp emulator of tests/emu: the KEEP instantiations
of the three env kernels against the default (STREAM) ones, with float32 and bfloat16 observations.  The mode only
changes the cache hint of the observation stores, so observations, rewards, dones, infos, terminal observations and
the state blob must be byte-identical.  Also the argument errors of set_obs_cache."""
import os

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)
from emu import driver
from emu.driver import Guarded
from emu.driver import ptr as _p
from madrl_b200 import _lib as L

pytestmark = driver.needs_cxx

WW = {
    "c2": dict(n_pursuers=5, n_evaders=5),                                                    # whole-step staging
    "c4": dict(n_pursuers=20, n_evaders=50, n_poison=50),                                     # two-slot ring
    "k40": dict(n_pursuers=4, n_evaders=40, n_poison=3, n_sensors=40, n_coop=2, radius=0.03),
}
C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
          catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
CONV = dict(n_evaders=3, n_pursuers=3, obs_range=4, surround=False, n_catch=1, reward_mech='global', flatten=False)
HW_ARGS = (10, 16, 16, 4, 2)


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


def pool16():
    return np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))


class Pair(object):
    """The same engine twice: `a` with the default cache mode, `b` with MADRL_OBS_CACHE_KEEP; both with `obs_format`."""

    def __init__(self, make, obs_format):
        self.a, self.b = make(), make()
        for eng in (self.a, self.b):
            assert eng._f("set_obs_format")(eng._h, obs_format) == 0
        assert self.b._f("set_obs_cache")(self.b._h, L.OBS_CACHE_KEEP) == 0
        self.dt = np.uint16 if obs_format == L.OBS_BF16 else np.float32
        self.E, self.A, self.D = self.a.n_envs, self.a.n_agents, self.a.obs_dim

    def reset(self):
        outs = []
        for eng in (self.a, self.b):
            o = Guarded((self.E, self.A, self.D), self.dt, 0)
            assert eng._f("reset")(eng._h, None, _p(o.arr), None) == 0
            outs.append(o.check("obs"))
        assert np.array_equal(outs[0].view(np.uint8), outs[1].view(np.uint8))

    def rollout(self, act, auto_reset=True, term=False):
        T = act.shape[0]
        outs = []
        for eng in (self.a, self.b):
            o = Guarded((T, self.E, self.A, self.D), self.dt, 0x7777)
            r = Guarded((T, self.E, self.A), np.float32, np.nan)
            d = Guarded((T, self.E), np.uint8, 255)
            i = Guarded((T, self.E) + eng.info_shape, np.int32, -1)
            tb = Guarded((T, self.E, self.A, self.D), self.dt, 0x5555) if term else None
            if term:
                assert eng._f("set_terminal_obs")(eng._h, _p(tb.arr)) == 0
            assert eng._f("rollout")(eng._h, T, _p(np.ascontiguousarray(act)), _p(o.arr), _p(r.arr), _p(d.arr),
                                     _p(i.arr), int(auto_reset), None) == 0
            if term:
                assert eng._f("set_terminal_obs")(eng._h, None) == 0
            outs.append([x.check(n) for x, n in ((o, "obs"), (r, "rew"), (d, "done"), (i, "info"))] +
                        ([tb.check("term")] if term else []))
        for x, y in zip(*outs):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8))
        assert np.array_equal(self.a.blob, self.b.blob), "state blobs differ"
        return outs[0]


@pytest.mark.parametrize("fmt", [L.OBS_NATIVE, L.OBS_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("name,E,T", [("c2", 4, 23), ("c4", 2, 9), ("k40", 3, 17)])
def test_waterworld_keep_equals_stream(name, E, T, fmt):
    from emu.driver import EmuWaterworld
    p = Pair(lambda: EmuWaterworld(E, seed=11, env_id_base=3, fp64=False, max_path_length=7, **WW[name]), fmt)
    p.reset()
    act = np.random.RandomState(5).randn(T, E, p.A, 2).astype(np.float32)
    done = p.rollout(act, auto_reset=True, term=True)[2]
    assert done.sum() >= E * (T // 7)
    p.rollout(act[:5], auto_reset=False)


@pytest.mark.parametrize("fmt", [L.OBS_NATIVE, L.OBS_BF16], ids=["f32", "bf16"])
@pytest.mark.parametrize("kind", ["flatten", "conv"])
def test_pursuit_keep_equals_stream(kind, fmt):
    from emu.driver import EmuPursuit
    E, T = 3, 21
    p = Pair(lambda: EmuPursuit(E, pool16(), seed=12, env_id_base=2, max_path_length=6,
                                **(C3 if kind == "flatten" else CONV)), fmt)
    p.reset()
    act = np.random.RandomState(6).randint(0, 5, size=(T, E, p.A)).astype(np.int32)
    assert p.rollout(act, auto_reset=True, term=True)[2].any()
    p.rollout(act[:4], auto_reset=False)


@pytest.mark.parametrize("fmt", [L.OBS_NATIVE, L.OBS_BF16], ids=["f32", "bf16"])
def test_hostage_keep_equals_stream(fmt):
    from emu.driver import EmuHostage
    E, T = 3, 19
    p = Pair(lambda: EmuHostage(E, *HW_ARGS, seed=13, env_id_base=4, fp64=False, max_path_length=8), fmt)
    p.reset()
    act = np.random.RandomState(7).randn(T, E, p.A, 2).astype(np.float32)
    assert p.rollout(act, auto_reset=True, term=True)[2].any()
    p.rollout(act[:4], auto_reset=False)


@pytest.mark.parametrize("fam", ["ww", "pursuit", "hostage"])
def test_set_obs_cache_arguments(fam):
    """Through the declared signature: a NULL handle and unknown modes are refused; KEEP on an fp64 handle too."""
    from emu.driver import EmuHostage, EmuPursuit, EmuWaterworld
    lib = driver.load()
    f = getattr(lib, "madrl_%s_set_obs_cache" % fam)
    assert f.argtypes == list(L.SIGNATURES["madrl_%s_set_obs_cache" % fam][1])
    for mode in (L.OBS_CACHE_STREAM, L.OBS_CACHE_KEEP):
        assert f(None, mode) == -1 and b"NULL" in lib.madrl_last_error()
    if fam == "pursuit":
        eng = EmuPursuit(2, pool16(), **CONV)
    elif fam == "ww":
        eng = EmuWaterworld(2, **WW["c2"], fp64=True)
    else:
        eng = EmuHostage(2, *HW_ARGS, fp64=True)
    for bad in (-1, 2, 1 << 30):
        assert f(eng._h, bad) == -1 and b"unknown observation cache mode" in lib.madrl_last_error()
    assert f(eng._h, L.OBS_CACHE_STREAM) == 0
    if fam != "pursuit":   # the fp64 verification build has no KEEP instantiation
        assert f(eng._h, L.OBS_CACHE_KEEP) == -1 and b"fp32" in lib.madrl_last_error()
    else:
        assert f(eng._h, L.OBS_CACHE_KEEP) == 0
