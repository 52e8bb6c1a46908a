"""The frame kernels' source (csrc/render.cu) on the warp emulator (tests/emu) against the NumPy oracle
(oracle/render_oracle.py), bit for bit, at small sizes, with the emulator's shared-memory race checker on.

The emulator library of tests/emu/build_emu.py is built from a fixed list of sources; this module links the
objects that build leaves with render.cu, compiled with the same flags, into a library of its own
(tests/emu/_build/libmadrl_b200_emu_render.so), and registers it with the driver so that the driver's engines
create their handles in it."""
import os
import subprocess

import numpy as np
import pytest

import env_dispatch_edges as D
from emu import build_emu, driver
from oracle import render_oracle as R

pytestmark = driver.needs_cxx
TAG = ("-DMADRL_EMU_WITH_RENDER",)   # the driver's cache key of the library below; no build uses it
SIZES = (1, 37, 128)


def _render_lib():
    base = build_emu.build()   # also (re)builds the objects of the other sources
    objdir = os.path.join(build_emu.OUT, "obj_default")
    objs = [os.path.join(objdir, s + ".o") for s in build_emu.SOURCES + ["emu_runtime.cpp"]]
    if not all(os.path.exists(o) for o in objs):
        base = build_emu.build(force=True)
    src = os.path.join(build_emu.CSRC, "render.cu")
    robj = os.path.join(build_emu.OUT, "obj_render", "render.cu.o")
    lib = os.path.join(build_emu.OUT, "libmadrl_b200_emu_render.so")
    deps = build_emu._deps() + [base]
    if not os.path.exists(lib) or any(os.path.getmtime(d) > os.path.getmtime(lib) for d in deps):
        os.makedirs(os.path.dirname(robj), exist_ok=True)
        cxx = os.environ.get("CXX", "g++")
        subprocess.check_call([cxx] + build_emu.CXXFLAGS + ["-c", "-o", robj, src])
        tmp = lib + ".%d.tmp" % os.getpid()
        subprocess.check_call([cxx, "-shared", "-o", tmp] + objs + [robj])
        os.replace(tmp, lib)
    return lib


@pytest.fixture(scope="module")
def lib():
    key = tuple(sorted(TAG))
    if key not in driver._libs:
        driver._libs[key] = driver.open_lib(_render_lib())
    driver.races()
    yield driver._libs[key]
    assert driver.races() == 0


def render(eng, ids, size, dirs=None):
    ids = np.ascontiguousarray(ids, np.int32)
    if eng.fam == "pursuit":
        shape = (len(ids), eng.map_pool.shape[2] * size, eng.map_pool.shape[1] * size, 3)
    else:
        shape = (len(ids), size, size, 3)
    out = driver.Guarded(shape, np.uint8, 0x5A)
    args = (size,) if eng.fam == "pursuit" else (size, driver.ptr(dirs))
    eng._check(getattr(eng.lib, "madrl_%s_render" % eng.fam)(eng._h, len(ids), driver.ptr(ids), *args,
                                                             driver.ptr(out.arr), None))
    return out.check("frames")


def stepped(eng, T, seed):
    rs = np.random.RandomState(seed)
    eng.reset()
    if eng.fam == "pursuit":
        eng.rollout(rs.randint(0, 5, (T, eng.n_envs, eng.n_agents)))
    else:
        eng.rollout(rs.randn(T, eng.n_envs, eng.n_agents, 2))
    return eng


def ww_state(eng):
    L, E, N = eng.layout, eng.n_envs, int(eng.layout.n_obj)
    objs = eng.view(L.objs, eng.obs_dtype, (E, 4, N))
    obst = eng.view(L.obst, eng.obs_dtype, (E, 2))
    return dict(pos_x=objs[:, 0], pos_y=objs[:, 1], obst_x=obst[:, 0], obst_y=obst[:, 1])


def hw_state(eng):
    L, E, N = eng.layout, eng.n_envs, int(eng.layout.n_obj)
    objs = eng.view(L.objs, eng.obs_dtype, (E, 4, N))
    fixed = eng.view(L.fixed, eng.obs_dtype, (E, 4))
    return dict(pos_x=objs[:, 0], pos_y=objs[:, 1], key=fixed[:, :2], bomb=fixed[:, 2:],
                saved=eng.view(L.saved, np.uint8, (E, eng.n_hostages)), flags=eng.view(L.flags, np.int32, (E,)))


def pe_state(eng):
    L, E, Np = eng.layout, eng.n_envs, eng.n_pursuers
    pos = eng.view(L.pos, np.uint8, (E, 2, int(L.n_agents)))
    return dict(pursuer_x=pos[:, 0, :Np], pursuer_y=pos[:, 1, :Np], evader_x=pos[:, 0, Np:], evader_y=pos[:, 1, Np:],
                gone=eng.view(L.gone, np.int64, (E,)), map_id=eng.view(L.map_id, np.int32, (E,)))


WW_CASES = {
    "c2": (dict(n_pursuers=5, n_evaders=5), True),
    "c4": (dict(n_pursuers=20, n_evaders=50, n_poison=50), False),
    "random_obstacle": (dict(n_pursuers=3, n_evaders=4, n_poison=2, n_sensors=7, radius=0.05, sensor_range=0.45,
                             obstacle_loc=None), True),
}


@pytest.mark.parametrize("name", sorted(WW_CASES))
def test_waterworld(lib, name):
    kw, fp64 = WW_CASES[name]
    eng = stepped(driver.EmuWaterworld(3, fp64=fp64, defines=TAG, seed=4, **kw), 30, 1)
    blob = eng.blob.copy()
    dirs = R.sensor_dirs(eng.cfg.n_sensors)
    ids = [2, 0, 2]
    for S in SIZES:
        want = R.ww_frames(ww_state(eng), ids, S, eng.cfg, eng.n_pursuers, eng.n_evaders)
        assert np.array_equal(render(eng, ids, S, dirs), want), S
    assert np.array_equal(eng.blob, blob)


@pytest.mark.parametrize("fp64", [False, True])
def test_hostage_c5(lib, fp64):
    eng = stepped(driver.EmuHostage(3, 10, 16, 16, 4, 2, fp64=fp64, defines=TAG, seed=5), 20, 2)
    st = hw_state(eng)
    st["flags"][0] &= ~1   # env 0: gate closed, env 1: open with saved hostages
    st["flags"][1] |= 1
    st["saved"][1, ::2] = 1
    dirs = R.sensor_dirs(eng.cfg.n_sensors)
    for S in SIZES:
        assert np.array_equal(render(eng, [1, 0, 2], S, dirs), R.hw_frames(st, [1, 0, 2], S, eng.cfg)), S


@pytest.mark.parametrize("name", ["e2_c1_conv", "e1_rc7_flat"])
def test_pursuit(lib, name):
    case = D.P_BY_NAME[name]   # e2_c1_conv: random_opponents; both catch evaders within their T steps
    eng = stepped(driver.EmuPursuit(4, case.maps(), defines=TAG, seed=3, **case.cfg), case.T, 3)
    assert (pe_state(eng)["gone"] != 0).any()
    ids = [3, 0, 1, 3]
    for cell in (1, 4, 7):
        want = R.pe_frames(pe_state(eng), eng.map_pool, ids, case.cfg["obs_range"], cell)
        assert np.array_equal(render(eng, ids, cell), want), cell


def test_out_of_range_ids_and_refusals(lib):
    eng = driver.EmuWaterworld(2, 2, 2, n_poison=2, n_sensors=3, fp64=False, defines=TAG)
    eng.reset()
    dirs = R.sensor_dirs(3)
    f = render(eng, [-1, 1, 2], 9, dirs)
    assert f[0].max() == 0 and f[2].max() == 0 and f[1].min() >= 102
    ids, out = np.zeros(1, np.int32), np.zeros((1, 4, 4, 3), np.uint8)
    for n, S, d in ((0, 4, dirs), (1, 0, dirs), (1, 32769, dirs), (1, 4, None)):
        assert lib.madrl_ww_render(eng._h, n, driver.ptr(ids), S, driver.ptr(d), driver.ptr(out), None) == -1
    assert b"screen_size" in lib.madrl_last_error() or b"sensor_dirs" in lib.madrl_last_error()
