"""bfloat16 observations (madrl_*_set_obs_format) in the warp emulator of tests/emu: the bf16 instantiations
of the three env kernels against the fp32 ones.  Observations must be the fp32 ones rounded to nearest
even, bit for bit; state, rewards, dones and infos must not change at all."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)

pytestmark = pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="no host C++ compiler")

OBS_NATIVE, OBS_BF16 = 0, 1

WW = {
    "c2": dict(n_pursuers=5, n_evaders=5),                                                    # whole-step staging
    "c4": dict(n_pursuers=20, n_evaders=50, n_poison=50),                                     # two-slot ring
    "k40": dict(n_pursuers=4, n_evaders=40, n_poison=3, n_sensors=40, n_coop=2, radius=0.03),
    "minimum": dict(n_pursuers=1, n_evaders=1, n_poison=1, n_sensors=1, n_coop=1, radius=0.05),
}
C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
          catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
CONV = dict(n_evaders=3, n_pursuers=3, obs_range=4, surround=False, n_catch=1, reward_mech='global', flatten=False)
HW_ARGS = (10, 16, 16, 4, 2)


def bf16_bits(x):
    """Round-to-nearest-even float32 -> bfloat16 bits (what torch's .to(torch.bfloat16) does)."""
    x = np.ascontiguousarray(x, np.float32)
    assert not np.isnan(x).any()
    u = x.view(np.uint32).astype(np.uint64)
    return ((u + 0x7fff + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def widen(b):
    return (np.ascontiguousarray(b, np.uint16).astype(np.uint32) << 16).view(np.float32)


def pool16():
    return np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    from emu import driver
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


class Pair(object):
    """The same engine twice: `a` with fp32 observations, `b` with bfloat16 ones."""

    def __init__(self, make):
        self.a, self.b = make(), make()
        f = getattr(self.b.lib, "madrl_%s_set_obs_format" % self.b.fam)
        f.argtypes = [C.c_void_p, C.c_int]
        assert f(self.b._h, OBS_BF16) == 0
        self.E, self.A, self.D = self.a.n_envs, self.a.n_agents, self.a.obs_dim

    def obs_bufs(self, shape):
        from emu.driver import Guarded
        return Guarded(shape, np.float32, np.nan), Guarded(shape, np.uint16, 0xFFFF)

    def check_state(self):
        assert np.array_equal(self.a.blob, self.b.blob), "state blobs differ"

    def reset(self, mask=None):
        from emu.driver import _p
        m = None if mask is None else np.ascontiguousarray(mask, np.uint8)
        oa, ob = self.obs_bufs((self.E, self.A, self.D))
        for eng, o in ((self.a, oa), (self.b, ob)):
            assert eng._f("reset")(eng._h, _p(m), _p(o.arr), None) == 0
        return oa.check("obs"), ob.check("obs")

    def rollout(self, act, auto_reset=True, term=False):
        """Both engines, device entry point; with `term`, terminal observations kept on the side."""
        from emu.driver import Guarded, _p
        T = act.shape[0]
        outs, terms = [], []
        for eng, dt in ((self.a, np.float32), (self.b, np.uint16)):
            o = Guarded((T, self.E, self.A, self.D), dt, 0x7777)
            r = Guarded((T, self.E, self.A), np.float32, np.nan)
            d = Guarded((T, self.E), np.uint8, 255)
            i = Guarded((T, self.E) + eng.info_shape, np.int32, -1)
            tb = Guarded((T, self.E, self.A, self.D), dt, -7.0 if dt == np.float32 else 0xFFFF) if term else None
            if term:
                assert eng._f("set_terminal_obs")(eng._h, _p(tb.arr)) == 0
            assert eng._f("rollout")(eng._h, T, _p(np.ascontiguousarray(act)), _p(o.arr), _p(r.arr), _p(d.arr),
                                     _p(i.arr), int(auto_reset), None) == 0
            if term:
                assert eng._f("set_terminal_obs")(eng._h, None) == 0
                terms.append(tb.check("term"))
            outs.append([x.check(n) for x, n in ((o, "obs"), (r, "rew"), (d, "done"), (i, "info"))])
        (oa, ra, da, ia), (ob, rb, db, ib) = outs
        assert np.array_equal(ra, rb) and np.array_equal(da, db) and np.array_equal(ia, ib)
        assert np.array_equal(bf16_bits(oa), ob)
        if term:
            touched = terms[0] != -7.0
            assert touched.any() and np.array_equal(touched, terms[1] != 0xFFFF)   # the same slots were written
            assert np.array_equal(bf16_bits(terms[0][touched]), terms[1][touched])
        self.check_state()
        return oa, ob, da


def ww_pair(name, E, **kw):
    from emu.driver import EmuWaterworld
    p = Pair(lambda: EmuWaterworld(E, seed=11, env_id_base=3, fp64=False, **WW[name], **kw))
    return p, np.random.RandomState(5).randn


@pytest.mark.parametrize("name,E,T", [("c2", 4, 23), ("c4", 2, 9), ("k40", 3, 17), ("minimum", 4, 30)])
def test_waterworld_bf16_equals_rounded_fp32(name, E, T):
    p, randn = ww_pair(name, E, max_path_length=7)
    oa, ob = p.reset()
    assert np.array_equal(bf16_bits(oa), ob)
    p.check_state()
    act = randn(T, E, p.A, 2).astype(np.float32)
    _, _, done = p.rollout(act, auto_reset=True, term=True)
    assert done.sum() >= E * (T // 7)
    p.rollout(act[:5], auto_reset=False)
    mask = np.arange(E) % 2 == 0
    oa, ob = p.reset(mask)
    assert np.array_equal(bf16_bits(oa[mask]), ob[mask])
    p.check_state()


@pytest.mark.parametrize("kind", ["flatten", "conv"])
def test_pursuit_bf16_equals_rounded_fp32(kind):
    from emu.driver import EmuPursuit
    cfg = C3 if kind == "flatten" else CONV
    E, T = 3, 21
    p = Pair(lambda: EmuPursuit(E, pool16(), seed=12, env_id_base=2, max_path_length=6, **cfg))
    oa, ob = p.reset()
    assert np.array_equal(bf16_bits(oa), ob)
    act = np.random.RandomState(6).randint(0, 5, size=(T, E, p.A)).astype(np.int32)
    p.rollout(act, auto_reset=True, term=True)
    p.rollout(act[:4], auto_reset=False)
    oa, ob = p.reset(np.array([1, 0, 1]))
    assert np.array_equal(bf16_bits(oa[[0, 2]]), ob[[0, 2]])
    p.check_state()


def test_hostage_bf16_equals_rounded_fp32():
    from emu.driver import EmuHostage
    E, T = 3, 19
    p = Pair(lambda: EmuHostage(E, *HW_ARGS, seed=13, max_path_length=6, fp64=False))
    oa, ob = p.reset()
    assert np.array_equal(bf16_bits(oa), ob)
    act = np.random.RandomState(7).randn(T, E, p.A, 2).astype(np.float32)
    p.rollout(act, auto_reset=True, term=True)
    p.rollout(act[:3], auto_reset=False)
    p.check_state()


def _host_pair(fam):
    from emu.driver import EmuHostage, EmuPursuit, EmuWaterworld
    E, T = 3, 13
    if fam == "ww":
        mk = lambda: EmuWaterworld(E, seed=4, max_path_length=7, fp64=False, **WW["c2"])   # noqa: E731
        act = np.random.RandomState(2).randn(T, E, 5, 2).astype(np.float32)
    elif fam == "pursuit":
        mk = lambda: EmuPursuit(E, pool16(), seed=4, max_path_length=7, **C3)               # noqa: E731
        act = np.random.RandomState(0).randint(0, 5, size=(T, E, 8)).astype(np.int32)
    else:
        mk = lambda: EmuHostage(E, *HW_ARGS, seed=4, max_path_length=7, fp64=False)         # noqa: E731
        act = np.random.RandomState(1).randn(T, E, 10, 2).astype(np.float32)
    return Pair(mk), act


@pytest.mark.parametrize("fam", ["ww", "pursuit", "hostage"])
def test_host_entry_points_copy_bf16_rows(fam):
    """reset_host and the chunked rollout_host2 (with and without MADRL_HOST_OBS_LAST) move 2-byte rows."""
    from emu.driver import Guarded, _p
    p, act = _host_pair(fam)
    T, E, A, D = act.shape[0], p.E, p.A, p.D
    a, b = p.a, p.b
    oa = Guarded((E, A, D), np.float32, np.nan)
    ob = Guarded((E, A, D), np.uint16, 0)
    assert a._f("reset")(a._h, None, _p(oa.arr), None) == 0
    assert b._f("reset_host")(b._h, None, _p(ob.arr)) == 0
    assert np.array_equal(bf16_bits(oa.check("obs")), ob.check("obs"))
    p.check_state()
    f = b._f("rollout_host2")
    f.argtypes = [C.c_void_p, C.c_int] + [C.c_void_p] * 5 + [C.c_int, C.c_int]
    b.lib.madrl_set_host_chunk_bytes(E * A * D * 2 * 3)          # ~3 steps per chunk
    try:
        for flags in (0, 1):
            a_out = a
            oref = Guarded((T, E, A, D), np.float32, np.nan)
            rref = Guarded((T, E, A), np.float32, np.nan)
            dref = Guarded((T, E), np.uint8, 255)
            iref = Guarded((T, E) + a_out.info_shape, np.int32, -1)
            assert a_out._f("rollout")(a_out._h, T, _p(act), _p(oref.arr), _p(rref.arr), _p(dref.arr), _p(iref.arr),
                                       1, None) == 0
            shape = (E, A, D) if flags else (T, E, A, D)
            bufs = [Guarded(shape, np.uint16, 0x7777), Guarded((T, E, A), np.float32, np.nan),
                    Guarded((T, E), np.uint8, 255), Guarded((T, E) + b.info_shape, np.int32, -1)]
            assert f(b._h, T, _p(act), *[_p(x.arr) for x in bufs], 1, flags) == 0
            o, r, d, i = [x.check("host2") for x in bufs]
            want = bf16_bits(oref.check("obs"))
            assert np.array_equal(o, want[-1] if flags else want)
            assert np.array_equal(r, rref.check("rew")) and np.array_equal(d, dref.check("done"))
            assert np.array_equal(i, iref.check("info"))
            p.check_state()
    finally:
        b.lib.madrl_set_host_chunk_bytes(0)


def _heuristic(eng, T, obs0, act_dtype, act_shape, obs_dtype, extra=()):
    from emu.driver import Guarded, _p
    E, A, D = eng.n_envs, eng.n_agents, eng.obs_dim
    bufs = [Guarded((T, E, A) + act_shape, act_dtype, -7), Guarded((T, E, A, D), obs_dtype, 0x7777),
            Guarded((T, E, A), np.float32, np.nan), Guarded((T, E), np.uint8, 255),
            Guarded((T, E) + eng.info_shape, np.int32, -1)]
    rc = eng._f("rollout_heuristic")(eng._h, T, _p(np.ascontiguousarray(obs0)), *[_p(x.arr) for x in bufs], 1,
                                     *extra, None)
    assert rc == 0, eng.lib.madrl_last_error()
    return [x.check("heuristic") for x in bufs]


def test_waterworld_heuristic_reads_bf16_obs0_widened():
    """A bf16 rollout_heuristic equals an fp32 one whose obs0 is the bf16 obs0 widened to fp32."""
    p, _ = ww_pair("c2", 3, max_path_length=9)
    oa, ob = p.reset()
    ra = _heuristic(p.a, 20, widen(ob), np.float32, (2,), np.float32)
    rb = _heuristic(p.b, 20, ob, np.float32, (2,), np.uint16)
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(bf16_bits(ra[1]), rb[1])
    for x, y in zip(ra[2:], rb[2:]):
        assert np.array_equal(x, y)
    p.check_state()


@pytest.mark.parametrize("kind", ["flatten", "conv"])
def test_pursuit_heuristic_bf16_chained_equals_long(kind):
    """Pursuit's policy only tests which cells hold an evader, which rounding never changes: the bf16
    closed loop equals the fp32 one, and chained bf16 launches equal one long launch."""
    from emu.driver import EmuPursuit
    cfg = C3 if kind == "flatten" else CONV
    E = 3
    p = Pair(lambda: EmuPursuit(E, pool16(), seed=21, max_path_length=8, **cfg))
    q = Pair(lambda: EmuPursuit(E, pool16(), seed=21, max_path_length=8, **cfg))
    oa, ob = p.reset()
    q.reset()
    ra = _heuristic(p.a, 24, oa, np.int32, (), np.float32, (1,))
    rb = _heuristic(p.b, 24, ob, np.int32, (), np.uint16, (1,))
    assert np.array_equal(ra[0], rb[0]) and np.array_equal(bf16_bits(ra[1]), rb[1])
    for x, y in zip(ra[2:], rb[2:]):
        assert np.array_equal(x, y)
    p.check_state()
    first = _heuristic(q.b, 10, ob, np.int32, (), np.uint16, (1,))
    second = _heuristic(q.b, 14, first[1][-1], np.int32, (), np.uint16, (1,))
    for x, y, z in zip(first, second, rb):
        assert np.array_equal(np.concatenate([x, y]), z)
    assert np.array_equal(q.b.blob, p.b.blob)


def test_set_obs_format_rejects_fp64_and_unknown_formats():
    from emu.driver import EmuHostage, EmuPursuit, EmuWaterworld
    for eng in (EmuWaterworld(2, fp64=True, **WW["c2"]), EmuHostage(2, *HW_ARGS, fp64=True)):
        f = eng._f("set_obs_format")
        f.argtypes = [C.c_void_p, C.c_int]
        assert f(eng._h, OBS_BF16) == -1 and b"fp32" in eng.lib.madrl_last_error()
        assert f(eng._h, OBS_NATIVE) == 0
    for eng in (EmuWaterworld(2, fp64=False, **WW["c2"]), EmuPursuit(2, pool16(), **C3),
                EmuHostage(2, *HW_ARGS, fp64=False)):
        f = eng._f("set_obs_format")
        f.argtypes = [C.c_void_p, C.c_int]
        assert f(eng._h, 2) == -1 and b"format" in eng.lib.madrl_last_error()
        assert f(eng._h, -1) == -1
        assert f(eng._h, OBS_BF16) == 0 and f(eng._h, OBS_NATIVE) == 0


def test_bf16_rows_with_peer_exchange_are_rejected():
    """The fused peer exchange is built for native observations only."""
    from emu.driver import EmuWaterworld, Guarded, _p
    p = Pair(lambda: EmuWaterworld(2, seed=1, fp64=False, **WW["c2"]))
    p.reset()
    eng = p.b
    rew = [np.zeros(64, np.float32)]
    done = [np.zeros(64, np.uint8)]
    info = [np.zeros(64, np.int64)]
    arr = lambda xs: (C.c_void_p * 1)(*[x.ctypes.data for x in xs])   # noqa: E731
    assert eng.lib.madrl_ww_set_peers(eng._h, 1, 0, 4, arr(rew), arr(done), arr(info)) == 0
    o = Guarded((1, 2, 5, eng.obs_dim), np.uint16, 0)
    r, d, i = np.zeros((1, 2, 5), np.float32), np.zeros((1, 2), np.uint8), np.zeros((1, 2, 2), np.int32)
    act = np.zeros((1, 2, 5, 2), np.float32)
    assert eng._f("rollout")(eng._h, 1, _p(act), _p(o.arr), _p(r), _p(d), _p(i), 0, None) == -1
    assert b"peer" in eng.lib.madrl_last_error()


def test_bf16_rounding_helper_matches_torch():
    """The NumPy RNE used above is torch's float32 -> bfloat16 conversion."""
    torch = pytest.importorskip("torch")
    x = np.random.RandomState(0).randn(4096).astype(np.float32) * np.float32(3.0)
    x[:8] = [0.0, -0.0, 1.0, 1.00390625, 1.01171875, 3.0e-39, 65504.0, -1.5e-20]
    t = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(bf16_bits(x), t)


# ------------------------------------------------------------------ post-processing on bf16 observations
def _postproc_lib():
    from emu import driver
    L = driver.load(())
    vp, i32, dbl, sz = C.c_void_p, C.c_int, C.c_double, C.c_size_t
    for suf in ("f32", "bf16"):
        getattr(L, "madrl_frame_stack_" + suf).argtypes = [i32] * 5 + [vp] * 5
        getattr(L, "madrl_standardize_" + suf).argtypes = [i32, sz, vp, vp, vp, dbl, dbl, i32, dbl, i32, vp]
        getattr(L, "madrl_standardize_obs_terminal_" + suf).argtypes = [i32, i32, sz] + [vp] * 5 + [dbl, dbl, vp]
    for suf in ("u32", "u16"):
        getattr(L, "madrl_paths_pack_" + suf).argtypes = [i32] * 4 + [vp] * 6
    L.madrl_paths_plan.argtypes = [i32, i32, i32] + [vp] * 6
    return L


def test_bf16_postproc_kernels_equal_f32_on_widened_input():
    """frame_stack / standardize / standardize_obs_terminal / paths_pack_u16 on bf16 observations equal
    the f32 passes run on the widened values, rounded to nearest even (D odd, as C2's 213)."""
    from emu.driver import _p
    L = _postproc_lib()
    rs = np.random.RandomState(3)
    T, E, A, D, B = 9, 3, 2, 13, 4
    xb = bf16_bits(rs.randn(T, E, A, D).astype(np.float32) * np.float32(3))
    xw = widen(xb)
    done = (rs.rand(T, E) < 0.25).astype(np.uint8)
    # frame stack: values are only moved
    c32, cb = np.zeros((E, A, D, B), np.float32), np.zeros((E, A, D, B), np.uint16)
    o32, ob = np.zeros((T, E, A, D, B), np.float32), np.zeros((T, E, A, D, B), np.uint16)
    assert L.madrl_frame_stack_f32(T, E, A, D, B, _p(xw), _p(done), _p(c32), _p(o32), None) == 0
    assert L.madrl_frame_stack_bf16(T, E, A, D, B, _p(xb), _p(done), _p(cb), _p(ob), None) == 0
    assert np.array_equal(bf16_bits(o32), ob) and np.array_equal(bf16_bits(c32), cb)
    # standardize (in place; float64 running estimates identical)
    n = E * A * D
    x32, x16 = xw.copy(), xb.copy()
    st = [(np.zeros(n), np.ones(n)) for _ in range(2)]
    assert L.madrl_standardize_f32(T, n, _p(x32), _p(st[0][0]), _p(st[0][1]), 0.05, 1e-8, 1, 1.0, 1, None) == 0
    assert L.madrl_standardize_bf16(T, n, _p(x16), _p(st[1][0]), _p(st[1][1]), 0.05, 1e-8, 1, 1.0, 1, None) == 0
    assert np.array_equal(bf16_bits(x32), x16)
    assert np.array_equal(st[0][0], st[1][0]) and np.array_equal(st[0][1], st[1][1])
    # with the terminal observations on the side
    tb = bf16_bits(rs.randn(T, E, A, D).astype(np.float32))
    x32, x16, t32, t16 = xw.copy(), xb.copy(), widen(tb), tb.copy()
    st = [(np.zeros(n), np.ones(n)) for _ in range(2)]
    assert L.madrl_standardize_obs_terminal_f32(T, E, A * D, _p(x32), _p(t32), _p(done), _p(st[0][0]), _p(st[0][1]),
                                                0.05, 1e-8, None) == 0
    assert L.madrl_standardize_obs_terminal_bf16(T, E, A * D, _p(x16), _p(t16), _p(done), _p(st[1][0]), _p(st[1][1]),
                                                 0.05, 1e-8, None) == 0
    assert np.array_equal(bf16_bits(x32), x16) and np.array_equal(bf16_bits(t32), t16)
    assert np.array_equal(st[0][0], st[1][0]) and np.array_equal(st[0][1], st[1][1])
    # path packing of 2-byte rows (odd D), with and without the one-step shift
    seg_s, seg_l = np.zeros((T, E), np.int32), np.zeros((T, E), np.int32)
    n_ep, ep_rec = np.zeros(E, np.int32), np.zeros((E, T, 3), np.int32)
    assert L.madrl_paths_plan(T, E, A, _p(done), _p(seg_s), _p(seg_l), _p(n_ep), _p(ep_rec), None) == 0
    first = bf16_bits(rs.randn(E, A, D).astype(np.float32))
    for f16, f32 in ((None, None), (first, widen(first))):
        p32 = np.zeros((T * E * A, D), np.float32)
        p16 = np.zeros((T * E * A, D), np.uint16)
        assert L.madrl_paths_pack_u32(T, E, A, D, _p(xw), _p(f32), _p(seg_s), _p(seg_l), _p(p32), None) == 0
        assert L.madrl_paths_pack_u16(T, E, A, D, _p(xb), _p(f16), _p(seg_s), _p(seg_l), _p(p16), None) == 0
        assert np.array_equal(bf16_bits(p32), p16)
    # narrow rows (D <= 4) take the one-thread-per-row kernel
    p32, p16 = np.zeros((T * E * A, 3), np.float32), np.zeros((T * E * A, 3), np.uint16)
    xs = np.ascontiguousarray(xb[..., :3])
    assert L.madrl_paths_pack_u32(T, E, A, 3, _p(widen(xs)), None, _p(seg_s), _p(seg_l), _p(p32), None) == 0
    assert L.madrl_paths_pack_u16(T, E, A, 3, _p(xs), None, _p(seg_s), _p(seg_l), _p(p16), None) == 0
    assert np.array_equal(bf16_bits(p32), p16)
