"""The replay pool kernels (madrl_replay_add_* / madrl_replay_sample_* in madrl_b200/csrc/replay.cu) executed on the CPU
by the warp emulator of tests/emu and compared, through the C ABI, with oracle/replay_oracle.py: float32 and bfloat16
rows in every word width the kernels pick (16, 8, 4 and 2 bytes), odd D, A = 1, T = 1, no done step, every step
done, nothing kept, more kept transitions than the pool holds, a wrap in the middle of an add, and [T, E] off the
block and warp sizes.  Every output sits in a canary-guarded buffer, and the pool starts filled with random bytes,
so a slot an add must not touch and still does, or a write outside a buffer, fails.  The launch-geometry edges of
tests/test_replay_edges_gpu.py (tests/replay_eval_edges.py) run here too, at the emulator's two SMs."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from emu import build_emu, driver
from emu.driver import Guarded
from emu.driver import ptr as _p
from oracle import replay_oracle as ro
import replay_eval_edges as RE

pytestmark = driver.needs_cxx

SCALE = 0.01


# The emulator library of tests/emu/build_emu.py is built from the kernel files listed there; the replay kernels get a
# library of their own, compiled the same way from replay.cu, common.cu and the emulator runtime.  Its shared arrays
# are block-static, as in the emulated postproc.cu and baseline.cu.
SOURCES = (os.path.join(build_emu.CSRC, "common.cu"), os.path.join(build_emu.CSRC, "replay.cu"),
           os.path.join(build_emu.HERE, "emu_runtime.cpp"))


def build_replay_emu():
    out = os.path.join(build_emu.OUT, "libmadrl_b200_emu_replay.so")
    deps = build_emu._deps() + [os.path.abspath(__file__)]
    if os.path.exists(out) and all(os.path.getmtime(d) <= os.path.getmtime(out) for d in deps):
        return out
    objdir = os.path.join(build_emu.OUT, "obj_replay")
    os.makedirs(objdir, exist_ok=True)
    cxx = os.environ.get("CXX", "g++")
    objs = []
    for src in SOURCES:
        obj = os.path.join(objdir, os.path.basename(src) + ".o")
        extra = ["-D__shared__=static"] if src.endswith("replay.cu") else []
        subprocess.check_call([cxx] + build_emu.CXXFLAGS + extra + ["-c", "-o", obj, src])
        objs.append(obj)
    tmp = out + ".%d.tmp" % os.getpid()
    subprocess.check_call([cxx, "-shared", "-o", tmp] + objs)
    os.replace(tmp, out)
    return out


@pytest.fixture(scope="module")
def lib():
    return driver.open_lib(build_replay_emu())


def rollout(rs, T, E, A, D, Ad, w, mpl, limit, p_done, pl0, ts0):
    """A rollout whose done flags follow the engine's rule: the env ends by itself at random or at the timestep limit,
    and the horizon cuts at max_path_length.  Observation words are random bits."""
    pl, ts = pl0.astype(np.int64).copy(), ts0.astype(np.int64).copy()
    done = np.zeros((T, E), np.uint8)
    for t in range(T):
        pl += 1
        ts += 1
        d = (rs.rand(E) < p_done) | (ts >= limit) | ((mpl > 0) & (pl >= mpl))
        done[t] = d
        pl[d] = 0
        ts[d] = 0
    bits = lambda *s: rs.randint(0, 2 ** (8 * np.dtype(w).itemsize), size=s, dtype=np.uint64).astype(w)  # noqa: E731
    return dict(obs=bits(T, E, A, D), act=rs.randn(T, E, A, Ad).astype(np.float32),
                rew=rs.randn(T, E, A).astype(np.float32), done=done, obs_before=bits(E, A, D),
                term=bits(T, E, A, D)), pl.astype(np.int32), ts.astype(np.int32)


class EmuPool(object):
    """The pool's buffers in guarded host memory, pre-filled like the oracle's with random bytes."""

    def __init__(self, lib, M, D, Ad, w, include, rs, start=None):
        self.lib, self.M, self.D, self.Ad, self.w = lib, M, D, Ad, w
        self.sfx = "bf16" if w == np.uint16 else "f32"
        self.oracle = ro.ReplayOracle(M, D, Ad, obs_dtype=w, scale_reward=SCALE,
                                      include_horizon_terminal_transitions=include)
        self.include = include
        self.bufs = {}
        for name, shape, dt in (("observations", (M, D), w), ("next_observations", (M, D), w),
                                ("actions", (M, Ad), np.float32), ("rewards", (M,), np.float32),
                                ("terminals", (M,), np.uint8)):
            g = Guarded(shape, dt, 0)
            g.arr.view(np.uint8)[...] = rs.randint(0, 256, size=g.arr.view(np.uint8).shape)
            getattr(self.oracle, name)[...] = g.arr
            self.bufs[name] = g
        self.ctl = Guarded((4,), np.int64, 0)
        if start is not None:      # (top, bottom, size, draws) of a pool part-way through its life
            o = self.oracle
            o.top, o.bottom, o.size, o.draws = start
            self.ctl.arr[...] = start

    def add(self, r, pl0, ts0, mpl, limit):
        T, E, A, D = r["obs"].shape
        n = C.c_size_t()
        assert self.lib.madrl_replay_workspace_size(T, E, C.byref(n)) == 0
        ws = Guarded((n.value,), np.uint8, 0x77)
        b = self.bufs
        fn = getattr(self.lib, "madrl_replay_add_" + self.sfx)
        assert fn(T, E, A, D, self.Ad, self.M, _p(r["obs"]), _p(r["act"]), _p(r["rew"]), _p(r["done"]),
                  _p(r["obs_before"]), _p(r["term"]), _p(pl0), _p(ts0), mpl, limit, int(self.include), SCALE,
                  _p(b["observations"].arr), _p(b["next_observations"].arr), _p(b["actions"].arr),
                  _p(b["rewards"].arr), _p(b["terminals"].arr), _p(self.ctl.arr), _p(ws.arr), None) == 0
        ws.check("workspace")
        K = self.oracle.add(r["obs"], r["act"], r["rew"], r["done"], r["obs_before"], r["term"], pl0, ts0, mpl, limit)
        self.compare()
        return K

    def compare(self):
        for name, g in self.bufs.items():
            assert np.array_equal(g.check(name).view(np.uint8), getattr(self.oracle, name).view(np.uint8)), name
        o = self.oracle
        assert self.ctl.check("ctl").tolist() == [o.top, o.bottom, o.size, o.draws]

    def sample(self, seed, n, B):
        b, D, Ad, w = self.bufs, self.D, self.Ad, self.w
        out = dict(indices=Guarded((n, B), np.int64, -7), observations=Guarded((n, B, D), w, 0x3C3C),
                   next_observations=Guarded((n, B, D), w, 0x3C3C), actions=Guarded((n, B, Ad), np.float32, np.nan),
                   rewards=Guarded((n, B), np.float32, np.nan), terminals=Guarded((n, B), np.uint8, 9))
        fn = getattr(self.lib, "madrl_replay_sample_" + self.sfx)
        assert fn(n, B, D, Ad, self.M, seed, _p(b["observations"].arr), _p(b["next_observations"].arr),
                  _p(b["actions"].arr), _p(b["rewards"].arr), _p(b["terminals"].arr), _p(self.ctl.arr),
                  _p(out["indices"].arr), _p(out["observations"].arr), _p(out["next_observations"].arr),
                  _p(out["actions"].arr), _p(out["rewards"].arr), _p(out["terminals"].arr), None) == 0
        idx, want = self.oracle.random_batches(seed, n, B)
        assert np.array_equal(out["indices"].check("indices"), idx)
        for k, v in want.items():
            assert np.array_equal(out[k].check(k).view(np.uint8), v.view(np.uint8)), k
        self.compare()
        return idx


# (T, E, A, D, Ad, dtype, M, max_path_length, p_done, adds): word widths 16 / 8 / 4 / 2 bytes, odd D, A = 1, T = 1,
# E off the warp and block sizes, pools that wrap inside an add and that one add overfills
CASES = (
    (9, 37, 3, 4, 2, np.float32, 50, 4, 0.1, 4),       # 16-byte words; wraps inside adds
    (6, 133, 2, 2, 2, np.float32, 3000, 5, 0.05, 3),   # 8-byte words; E over a 128-thread block
    (7, 5, 1, 3, 1, np.float32, 16, 3, 0.2, 3),        # 4-byte words, A = 1, K > M
    (1, 70, 5, 5, 2, np.uint16, 40, 2, 0.3, 5),        # 2-byte words (odd bf16 row), T = 1
    (11, 33, 2, 8, 3, np.uint16, 1000, 6, 0.0, 2),     # 16-byte bf16 rows
    (5, 3, 4, 13, 2, np.uint16, 7, 0, 0.5, 3),         # no horizon; pool of 7
)


@pytest.mark.parametrize("include", [False, True], ids=["drop_cuts", "keep_cuts"])
@pytest.mark.parametrize("case", range(len(CASES)))
def test_add_and_sample_equal_the_oracle(lib, case, include):
    T, E, A, D, Ad, w, M, mpl, p_done, adds = CASES[case]
    rs = np.random.RandomState(10 + case)
    pool = EmuPool(lib, M, D, Ad, w, include, rs)
    limit = 3 * T + 2
    pl = rs.randint(0, max(mpl, 1), size=E).astype(np.int32)
    ts = (pl + rs.randint(0, T + 1, size=E)).astype(np.int32)
    for k in range(adds):
        r, pl_next, ts_next = rollout(rs, T, E, A, D, Ad, w, mpl, limit, p_done, pl, ts)
        pool.add(r, pl, ts, mpl, limit)
        pl, ts = pl_next, ts_next
        pool.sample(seed=1000 + k, n=2, B=3 + k)


def test_no_done_every_step_done_and_nothing_kept(lib):
    T, E, A, D, Ad, M = 4, 40, 2, 6, 2, 300
    rs = np.random.RandomState(5)
    zeros = np.zeros(E, np.int32)
    pool = EmuPool(lib, M, D, Ad, np.float32, False, rs)
    r, _, _ = rollout(rs, T, E, A, D, Ad, np.float32, 0, 10 ** 6, 0.0, zeros, zeros)
    assert not r["done"].any()
    assert pool.add(r, zeros, zeros, 0, 10 ** 6) == T * E * A
    # every step done by the env itself (timestep limit 1): all kept, next observations from term
    r["done"][...] = 1
    assert pool.add(r, zeros, zeros, 5, 1) == T * E * A
    # every step a horizon cut (max_path_length 1): nothing kept, and the pool is untouched
    before = pool.ctl.arr.copy()
    assert pool.add(r, zeros, zeros, 1, 10 ** 6) == 0
    assert np.array_equal(pool.ctl.arr, before)
    pool.sample(seed=3, n=1, B=5)


def test_sampling_an_empty_or_single_slot_pool_stays_inside(lib):
    """size 0 or 1: every draw is slot 0 (the kernel never reads past the pool, whatever size is)."""
    rs = np.random.RandomState(6)
    pool = EmuPool(lib, 1, 3, 1, np.float32, False, rs)
    assert (pool.sample(seed=1, n=2, B=4) == 0).all()
    zeros = np.zeros(2, np.int32)
    r, _, _ = rollout(rs, 3, 2, 1, 3, 1, np.float32, 0, 100, 0.0, zeros, zeros)
    pool.add(r, zeros, zeros, 0, 100)
    assert (pool.sample(seed=2, n=1, B=9) == 0).all()


def test_argument_errors(lib):
    """MADRL_EINVAL (no launch) for sizes below 1, a pool of 0 slots, NULL buffers and a misaligned workspace."""
    x = np.zeros(4096, np.float32)
    c = np.zeros(4, np.int64)
    i = np.zeros(64, np.int32)
    u = np.zeros(64, np.uint8)
    base = [2, 2, 1, 2, 1, 8] + [_p(x)] * 3 + [_p(u)] + [_p(x)] * 2 + [_p(i)] * 2 + [0, 10, 0, 0.1] + \
        [_p(x)] * 4 + [_p(u), _p(c), _p(x)]
    assert lib.madrl_replay_add_f32(*base, None) == 0
    for k, bad in ((0, 0), (3, 0), (4, 0), (5, 0), (6, None), (11, None), (22, None), (24, _p(u[1:]))):
        args = list(base)
        args[k] = bad
        assert lib.madrl_replay_add_f32(*args, None) != 0, k
    s = [1, 2, 2, 1, 8, 0] + [_p(x)] * 4 + [_p(u), _p(c), _p(c)] + [_p(x)] * 4 + [_p(u)]
    assert lib.madrl_replay_sample_f32(*s, None) == 0
    for k, bad in ((0, 0), (1, 0), (4, 0), (6, None), (11, None), (12, None)):
        args = list(s)
        args[k] = bad
        assert lib.madrl_replay_sample_f32(*args, None) != 0, k


# ------------------------------------------------------------------ the edge cases of tests/test_replay_edges_gpu.py
# at the emulator's geometry: two SMs, so the insert grid G is 128 warps; the scan block is kScanThreads as on the
# device, reached here with one warp of envs (T = cells)

@pytest.mark.parametrize("which", range(4), ids=["G-1", "G", "G+1", "2G+1"])
def test_insert_grid_edges(lib, which):
    rows = RE.insert_grid_rows(2)[which]
    T, E, A = RE.grid_shape(rows)
    rs = np.random.RandomState(100 + which)
    pl, ts = RE.start_counters(rs, E, 5)
    r, _, _ = RE.rollout(rs, T, E, A, 3, 2, np.float32, 5, 10 ** 6, 0.05, pl, ts)
    K = int(ro.keep_flags(r["done"], pl, ts, 5, 10 ** 6, False).sum()) * A
    M = K + 37
    pool = EmuPool(lib, M, 3, 2, np.float32, False, rs, start=(M - 20, 0, M - 20, 0))
    assert pool.add(r, pl, ts, 5, 10 ** 6) == K > 0
    if which != 2:
        return
    # G + 1 rows and K >> M: the grid-stride loop starts at a step past 0
    M = max(K // 7, 1) + 1
    assert RE.landing_step(r["done"], pl, ts, 5, 10 ** 6, False, A, K - M) > 0
    EmuPool(lib, M, 3, 2, np.float32, False, rs).add(r, pl, ts, 5, 10 ** 6)


@pytest.mark.parametrize("cut", RE.CUTS)
@pytest.mark.parametrize("which", range(4), ids=["S-1", "S", "S+1", "2S+1"])
def test_scan_cuts(lib, which, cut):
    T, E, A, mpl = RE.scan_cells()[which], 20, 3, 6
    rs = np.random.RandomState(1000 * which + RE.CUTS.index(cut))
    pl, ts = RE.start_counters(rs, E, mpl)
    r, _, _ = RE.rollout(rs, T, E, A, 2, 1, np.float32, mpl, 10 ** 6, 0.02, pl, ts)
    M, first, K = RE.cut_pool_size(cut, r["done"], pl, ts, mpl, 10 ** 6, False, A)
    top = int(rs.randint(0, M))
    pool = EmuPool(lib, M, 2, 1, np.float32, False, rs, start=(top, top, M, 0) if first % 2 else (top, 0, top, 0))
    assert pool.add(r, pl, ts, mpl, 10 ** 6) == K


@pytest.mark.parametrize("E", RE.PLAN_ENVS)
def test_plan_warps(lib, E):
    T, A, mpl = 7, 2, 3
    rs = np.random.RandomState(E)
    z = np.zeros(E, np.int32)
    pool = EmuPool(lib, 5 * T * E * A, 5, 2, np.float32, False, rs)
    r, _, _ = RE.rollout(rs, T, E, A, 5, 2, np.float32, mpl, 10 ** 6, 0.0, z, z)
    pool.add(r, z, z, mpl, 10 ** 6)
    pl, ts = RE.start_counters(rs, E, mpl)
    r, _, _ = RE.rollout(rs, T, E, A, 5, 2, np.float32, mpl, 10 ** 6, 0.1, pl, ts)
    pool.add(r, pl, ts, mpl, 10 ** 6)
    pool.sample(E, 1, 3 * E)


@pytest.mark.parametrize("row", RE.WORD_ROWS, ids=["%s_D%d_%dB" % ("bf16" if w == np.uint16 else "f32", D, b)
                                                   for w, D, b in RE.WORD_ROWS])
def test_word_widths_and_sample_rows(lib, row):
    w, D, _ = row
    rs = np.random.RandomState(D)
    pool = EmuPool(lib, 500, D, 33, w, True, rs)
    pl, ts = RE.start_counters(rs, 45, 3)
    for _ in range(2):
        r, pl1, ts1 = RE.rollout(rs, 5, 45, 3, D, 33, w, 3, 9, 0.1, pl, ts)
        pool.add(r, pl, ts, 3, 9)
        pl, ts = pl1, ts1
    for n, B in RE.SAMPLE_ROWS:
        pool.sample(5 + B, n, B)
