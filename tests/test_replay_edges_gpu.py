"""The replay pool kernels (madrl_replay_add_* / madrl_replay_sample_*, csrc/replay.cu) on the GPU at the edges of
their launch geometry, through the C ABI, against oracle/replay_oracle.py (cases in tests/replay_eval_edges.py):

* the insert grid: (T + 1) E A source rows at G - 1, G, G + 1 and 2 G + 1 with G the warps of the largest grid
  (8 blocks of 8 warps per SM of this device), and at G + 1 with K >> M, where the grid-stride loop starts at a
  step past 0;
* the one-block scan: T W cells at kScanThreads - 1, kScanThreads, kScanThreads + 1 and 2 kScanThreads + 1, with
  the landing cut on a warp-cell edge, inside the last cell of a step, between two agents of one env, so that only
  the last step lands, at K = M and K = M + 1, and an add of horizon cuts only;
* the plan kernel at E = 1, 31, 33, 127, 129 with whole warps of kept envs;
* every word width the rows move in, each with one pointer one element off its allocation;
* samples of 1, 7, 8, 9 and more than 2^20 rows, rows of fewer and more than 32 words, 1 and 33 actions, and
  pools holding 0, 1 and 2 transitions.

Every add is compared byte for byte on all five pool arrays and the counters; the pool starts filled with random
bytes, so a slot an add must not touch fails the comparison if it is written."""
import ctypes as C

import numpy as np
import pytest
import torch

import replay_eval_edges as RE
from madrl_b200 import _lib
from oracle import replay_oracle as ro

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SCALE = 0.01
POOL_ARRAYS = ("observations", "next_observations", "actions", "rewards", "terminals")


@pytest.fixture(scope="module")
def lib():
    return _lib.lib()


@pytest.fixture(scope="module")
def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


class Dev(object):
    """A host array copied to a fresh device allocation, `off` elements past its start (256-byte aligned)."""

    def __init__(self, a, off=0):
        a = np.ascontiguousarray(a)
        self.shape, self.dtype, self.off = a.shape, a.dtype, off * a.dtype.itemsize
        self.buf = torch.empty(a.nbytes + self.off, dtype=torch.uint8, device=DEV)
        self.buf[self.off:].copy_(torch.from_numpy(a.reshape(-1).view(np.uint8)))

    @property
    def ptr(self):
        return C.c_void_p(self.buf.data_ptr() + self.off)

    def host(self):
        return self.buf[self.off:].cpu().numpy().view(self.dtype).reshape(self.shape)


def random_bytes(rs, shape, dtype):
    a = np.empty(shape, dtype)
    a.view(np.uint8)[...] = rs.randint(0, 256, size=a.view(np.uint8).shape)
    return a


class DevPool(object):
    """The pool's five arrays and counters in device memory, pre-filled with random bytes like the oracle's;
    `offsets` names the pool arrays placed one element off their allocation."""

    def __init__(self, lib, M, D, Ad, w, include, rs, offsets=(), start=None):
        self.lib, self.M, self.D, self.Ad, self.w, self.include = lib, M, D, Ad, w, include
        self.sfx = "bf16" if w == np.uint16 else "f32"
        self.oracle = ro.ReplayOracle(M, D, Ad, obs_dtype=w, scale_reward=SCALE,
                                      include_horizon_terminal_transitions=include)
        self.bufs = {}
        for name, shape, dt in (("observations", (M, D), w), ("next_observations", (M, D), w),
                                ("actions", (M, Ad), np.float32), ("rewards", (M,), np.float32),
                                ("terminals", (M,), np.uint8)):
            a = random_bytes(rs, shape, dt)
            getattr(self.oracle, name)[...] = a
            self.bufs[name] = Dev(a, 1 if name in offsets else 0)
        o = self.oracle
        if start is not None:
            o.top, o.bottom, o.size, o.draws = start
        self.ctl = Dev(np.array([o.top, o.bottom, o.size, o.draws], np.int64))

    def add(self, r, pl0, ts0, mpl, limit, offset=None):
        """One add of rollout `r` (host arrays), with the input named `offset` one element off its allocation."""
        T, E, A, D = r["obs"].shape
        n = C.c_size_t()
        _lib.check(self.lib.madrl_replay_workspace_size(T, E, C.byref(n)))
        ws = torch.full((n.value,), 0x77, dtype=torch.uint8, device=DEV)
        d = {k: Dev(v, 1 if k == offset else 0) for k, v in r.items()}
        dpl, dts = Dev(pl0), Dev(ts0)
        b = self.bufs
        fn = getattr(self.lib, "madrl_replay_add_" + self.sfx)
        _lib.check(fn(T, E, A, D, self.Ad, self.M, d["obs"].ptr, d["act"].ptr, d["rew"].ptr, d["done"].ptr,
                      d["obs_before"].ptr, d["term"].ptr, dpl.ptr, dts.ptr, mpl, limit, int(self.include), SCALE,
                      *[b[k].ptr for k in POOL_ARRAYS], self.ctl.ptr, C.c_void_p(ws.data_ptr()), _lib.stream(DEV)))
        for k, v in d.items():     # the inputs are read only
            assert np.array_equal(v.host().view(np.uint8), r[k].view(np.uint8)), k
        K = self.oracle.add(r["obs"], r["act"], r["rew"], r["done"], r["obs_before"], r["term"], pl0, ts0, mpl, limit)
        self.compare()
        return K

    def compare(self):
        for name in POOL_ARRAYS:
            got = self.bufs[name].host()
            assert np.array_equal(got.view(np.uint8), getattr(self.oracle, name).view(np.uint8)), name
        o = self.oracle
        assert self.ctl.host().tolist() == [o.top, o.bottom, o.size, o.draws]

    def sample(self, seed, n, B, offset=None):
        """n x B draws with the output named `offset` one element off its allocation; indices and rows against
        the oracle, and the pool unchanged."""
        D, Ad, w = self.D, self.Ad, self.w
        out = dict(indices=np.full((n, B), -7, np.int64), observations=np.full((n, B, D), 0x3C3C, w),
                   next_observations=np.full((n, B, D), 0x3C3C, w), actions=np.full((n, B, Ad), np.nan, np.float32),
                   rewards=np.full((n, B), np.nan, np.float32), terminals=np.full((n, B), 9, np.uint8))
        d = {k: Dev(v, 1 if k == offset else 0) for k, v in out.items()}
        b = self.bufs
        fn = getattr(self.lib, "madrl_replay_sample_" + self.sfx)
        _lib.check(fn(n, B, D, Ad, self.M, seed, *[b[k].ptr for k in POOL_ARRAYS], self.ctl.ptr, d["indices"].ptr,
                      d["observations"].ptr, d["next_observations"].ptr, d["actions"].ptr, d["rewards"].ptr,
                      d["terminals"].ptr, _lib.stream(DEV)))
        idx, want = self.oracle.random_batches(seed, n, B)
        got_idx = d["indices"].host()
        assert np.array_equal(got_idx, idx)
        for k, v in want.items():
            assert np.array_equal(d[k].host().view(np.uint8), v.view(np.uint8)), k
        self.compare()
        return got_idx


# ------------------------------------------------------------------------------------------------ insert grid

@pytest.mark.parametrize("which", range(4), ids=["G-1", "G", "G+1", "2G+1"])
def test_insert_grid_edges(lib, sms, which):
    """Every transition lands (M > K) in a pool whose top starts near its end, so the add wraps."""
    rows = RE.insert_grid_rows(sms)[which]
    T, E, A = RE.grid_shape(rows)
    assert (T + 1) * E * A == rows
    rs = np.random.RandomState(100 + which)
    mpl = 5
    pl, ts = RE.start_counters(rs, E, mpl)
    r, _, _ = RE.rollout(rs, T, E, A, 3, 2, np.float32, mpl, 10 ** 6, 0.05, pl, ts)
    K = int(ro.keep_flags(r["done"], pl, ts, mpl, 10 ** 6, False).sum()) * A
    M = K + 37
    pool = DevPool(lib, M, 3, 2, np.float32, False, rs, start=(M - 20, 0, M - 20, 0))
    assert pool.add(r, pl, ts, mpl, 10 ** 6) == K > 0


@pytest.mark.parametrize("include", [False, True], ids=["drop_cuts", "keep_cuts"])
def test_insert_grid_starts_past_the_first_step(lib, sms, include):
    """G + 1 source rows and K >> M: only the last M transitions land, the first of them several steps in, so the
    grid-stride loop starts mid-tensor; then a second add into the full pool."""
    T, E, A = RE.grid_shape(RE.insert_grid_rows(sms)[2])
    rs = np.random.RandomState(7)
    mpl = 4
    pl, ts = RE.start_counters(rs, E, mpl)
    r, pl1, ts1 = RE.rollout(rs, T, E, A, 4, 1, np.float32, mpl, 10 ** 6, 0.1, pl, ts)
    K = int(ro.keep_flags(r["done"], pl, ts, mpl, 10 ** 6, include).sum()) * A
    M = max(K // 7, 1) + 1
    assert RE.landing_step(r["done"], pl, ts, mpl, 10 ** 6, include, A, K - M) > 0
    pool = DevPool(lib, M, 4, 1, np.float32, include, rs)
    assert pool.add(r, pl, ts, mpl, 10 ** 6) == K
    r, _, _ = RE.rollout(rs, T, E, A, 4, 1, np.float32, mpl, 10 ** 6, 0.1, pl1, ts1)
    pool.add(r, pl1, ts1, mpl, 10 ** 6)
    pool.sample(3, 2, 50)


# ------------------------------------------------------------------------------------------------ scan

def scan_shapes(cells):
    """(T, E): one warp of envs (W = 1, T = cells) and many warps (W a divisor of cells near its square root)."""
    W = max(w for w in range(1, int(cells ** 0.5) + 2) if cells % w == 0)
    T = cells // W
    return ((cells, 20), (T, 32 * W - 5))


@pytest.mark.parametrize("cut", RE.CUTS)
@pytest.mark.parametrize("wide", [False, True], ids=["W1", "Wmany"])
@pytest.mark.parametrize("which", range(4), ids=["S-1", "S", "S+1", "2S+1"])
def test_scan_cuts(lib, which, wide, cut):
    cells = RE.scan_cells()[which]
    T, E = scan_shapes(cells)[int(wide)]
    W = (E + 31) // 32
    assert T * W == cells
    A, mpl, limit = 3, 6, 10 ** 6
    rs = np.random.RandomState(1000 * which + 10 * wide + RE.CUTS.index(cut))
    pl, ts = RE.start_counters(rs, E, mpl)
    r, _, _ = RE.rollout(rs, T, E, A, 2, 1, np.float32, mpl, limit, 0.02, pl, ts)
    M, first, K = RE.cut_pool_size(cut, r["done"], pl, ts, mpl, limit, False, A)
    top = int(rs.randint(0, M))
    pool = DevPool(lib, M, 2, 1, np.float32, False, rs, start=(top, top, M, 0) if first % 2 else (top, 0, top, 0))
    assert pool.add(r, pl, ts, mpl, limit) == K
    if cut == "last_step":
        assert RE.landing_step(r["done"], pl, ts, mpl, limit, False, A, first) == T - 1


@pytest.mark.parametrize("which", range(4), ids=["S-1", "S", "S+1", "2S+1"])
def test_scan_with_every_step_a_horizon_cut(lib, which):
    """max_path_length 1: nothing is kept, K = 0, and neither the pool nor its counters change."""
    T, E = scan_shapes(RE.scan_cells()[which])[1]
    rs = np.random.RandomState(50 + which)
    z = np.zeros(E, np.int32)
    r, _, _ = RE.rollout(rs, T, E, 2, 2, 1, np.float32, 1, 10 ** 6, 0.0, z, z)
    pool = DevPool(lib, 999, 2, 1, np.float32, False, rs, start=(17, 0, 17, 5))
    assert pool.add(r, z, z, 1, 10 ** 6) == 0
    assert pool.ctl.host().tolist() == [17, 0, 17, 5]


# ------------------------------------------------------------------------------------------------ plan

@pytest.mark.parametrize("E", RE.PLAN_ENVS)
def test_plan_warps(lib, E):
    """Paths in step: whole warps of kept envs (ranks up to 31), and steps where every env is a horizon cut.  Then
    paths out of step: every rank pattern."""
    T, A, mpl = 7, 2, 3
    rs = np.random.RandomState(E)
    pl, ts = np.zeros(E, np.int32), np.zeros(E, np.int32)
    pool = DevPool(lib, 5 * T * E * A, 5, 2, np.float32, False, rs)
    r, _, _ = RE.rollout(rs, T, E, A, 5, 2, np.float32, mpl, 10 ** 6, 0.0, pl, ts)
    keep = ro.keep_flags(r["done"], pl, ts, mpl, 10 ** 6, False)
    assert keep.all(axis=1).any() and not keep.any(axis=1).all()
    pool.add(r, pl, ts, mpl, 10 ** 6)
    pl, ts = RE.start_counters(rs, E, mpl)
    r, _, _ = RE.rollout(rs, T, E, A, 5, 2, np.float32, mpl, 10 ** 6, 0.1, pl, ts)
    pool.add(r, pl, ts, mpl, 10 ** 6)
    pool.sample(E, 1, 3 * E)


# ------------------------------------------------------------------------------------------------ word widths

@pytest.mark.parametrize("offset", RE.ADD_OFFSETS, ids=[str(o) for o in RE.ADD_OFFSETS])
@pytest.mark.parametrize("row", RE.WORD_ROWS, ids=["%s_D%d_%dB" % ("bf16" if w == np.uint16 else "f32", D, b)
                                                   for w, D, b in RE.WORD_ROWS])
def test_word_widths(lib, row, offset):
    w, D, word = row
    isz = np.dtype(w).itemsize
    assert RE.row_word(D * isz, ()) == word
    T, E, A, Ad, mpl, limit = 5, 45, 3, 2, 3, 9
    rs = np.random.RandomState(D * 7 + RE.ADD_OFFSETS.index(offset))
    pool_off = (offset,) if offset in ("observations", "next_observations") else ()
    pool = DevPool(lib, 500, D, Ad, w, True, rs, offsets=pool_off)
    pl, ts = RE.start_counters(rs, E, mpl)
    for _ in range(2):           # the second add wraps the pool of 500
        r, pl1, ts1 = RE.rollout(rs, T, E, A, D, Ad, w, mpl, limit, 0.1, pl, ts)
        pool.add(r, pl, ts, mpl, limit, offset=None if pool_off else offset)
        pl, ts = pl1, ts1
    pool.sample(5, 3, 41)
    if offset is None:
        pool.sample(6, 2, 9, offset="observations")
        pool.sample(7, 1, 9, offset="next_observations")


# ------------------------------------------------------------------------------------------------ sample

SAMPLE_SHAPE_IDS = ["f32_D8_Ad1", "f32_D150_Ad33", "bf16_D7_Ad33", "bf16_D88_Ad1"]


@pytest.mark.parametrize("rows", RE.SAMPLE_ROWS, ids=["1", "7", "8", "9"])
@pytest.mark.parametrize("shape", RE.SAMPLE_ROW_SHAPES, ids=SAMPLE_SHAPE_IDS)
def test_sample_rows(lib, shape, rows):
    sample_case(lib, shape, rows)


@pytest.mark.parametrize("shape", (RE.SAMPLE_ROW_SHAPES[0], RE.SAMPLE_ROW_SHAPES[2]), ids=SAMPLE_SHAPE_IDS[::2])
def test_sample_past_2_20_rows(lib, shape):
    sample_case(lib, shape, (3, (1 << 20) // 3 + 1))


def sample_case(lib, shape, rows):
    w, D, Ad = shape
    n, B = rows
    rs = np.random.RandomState(D + Ad)
    E, A, T = 37, 2, 6
    pool = DevPool(lib, 300, D, Ad, w, False, rs)
    pl, ts = RE.start_counters(rs, E, 4)
    r, _, _ = RE.rollout(rs, T, E, A, D, Ad, w, 4, 10 ** 6, 0.1, pl, ts)
    pool.add(r, pl, ts, 4, 10 ** 6)
    idx = pool.sample(11 + n, n, B)
    assert idx.min() >= 0 and idx.max() < pool.oracle.size - 1


@pytest.mark.parametrize("size", [0, 1, 2])
@pytest.mark.parametrize("shape", RE.SAMPLE_ROW_SHAPES[:3], ids=["f32_D8_Ad1", "f32_D150_Ad33", "bf16_D7_Ad33"])
def test_sample_tiny_pools(lib, shape, size):
    """A pool of 0, 1 or 2 transitions (of 5 slots): every draw is slot 0."""
    w, D, Ad = shape
    rs = np.random.RandomState(size)
    pool = DevPool(lib, 5, D, Ad, w, False, rs, start=(size, 0, size, 3))
    for n, B in RE.SAMPLE_ROWS:
        assert (pool.sample(20 + B, n, B) == 0).all()
