"""The entry points that split a statistic where the shards of a batch are pooled, executed on the CPU by the warp
emulator of tests/emu through the C ABI: the bins of madrl_time_baseline_bins_f32 over env shards, summed, give the
whole batch's counts exactly and its simplev (madrl_time_baseline_apply_f32) within one float32 ulp;
madrl_moments_pass_f32 over row shards, pooled, gives the float64 moments of the union, and madrl_center_apply_f32 on
each shard with them NumPy's centring of the union.  Outputs sit in canary-guarded buffers; the argument checks
(MADRL_EINVAL, no launch) are exercised."""
import ctypes as C

import numpy as np
import pytest

import postproc_edges as pe
import sharded_edges as se
from emu import build_emu, driver
from emu.driver import Guarded
from emu.driver import ptr as _p

pytestmark = driver.needs_cxx

EMU_MOM_BLOCKS = build_emu.GRID["MADRL_MOM_BLOCKS"]
# (T, E, done probability): slices of one and several envs, L off and past the 128-thread bin block
TB_SHAPES = ((5, 2, 0.3), (9, 7, 0.2), (140, 4, 0.0), (33, 11, 0.1))


@pytest.fixture(scope="module")
def lib():
    return driver.load(())


def _ws(lib, G, L):
    nbytes = C.c_size_t()
    assert lib.madrl_time_baseline_workspace_size(G, L, C.byref(nbytes)) == 0
    return np.zeros(nbytes.value, np.uint8)


def _bins(lib, q, done, t0, per_agent, L):
    T, E, A = q.shape
    G = A if per_agent else 1
    _, _, n_ep, ep_rec = driver.paths_plan(lib, done, A)
    s, c = Guarded((G, L), np.float64, np.nan), Guarded((G, L), np.int32, -1)
    assert lib.madrl_time_baseline_bins_f32(T, E, A, per_agent, L, _p(q), _p(n_ep), _p(ep_rec), _p(t0), _p(s.arr),
                                            _p(c.arr), _p(_ws(lib, G, L)), None) == 0, lib.madrl_last_error()
    return s.check("sums").copy(), c.check("counts").copy()


def _apply(lib, done, t0, per_agent, A, L, s, c):
    T, E = done.shape
    seg_s = driver.paths_plan(lib, done, A)[0]
    v = Guarded((T, E, A), np.float32, np.nan)
    assert lib.madrl_time_baseline_apply_f32(T, E, A, per_agent, L, _p(seg_s), _p(t0), _p(s), _p(c), _p(v.arr),
                                             None) == 0, lib.madrl_last_error()
    return v.check("simplev").copy()


def _whole(lib, q, done, t0, per_agent, L):
    """The whole batch's bins and simplev, from one rank's calls."""
    s, c = _bins(lib, q, done, t0, per_agent, L)
    return s, c, _apply(lib, done, t0, per_agent, q.shape[2], L, s, c)


def _case(A, k):
    T, E, p = TB_SHAPES[k]
    rs = np.random.RandomState(100 * A + k)
    done = (rs.rand(T, E) < p).astype(np.uint8)
    if T > 2:
        done[0, 0] = done[T - 1, E - 1] = 1
    q = rs.randn(T, E, A).astype(np.float32)
    return q, done, (None, rs.randint(0, 6, E).astype(np.int32))


def _last_index(done, t0):
    """The largest time index of a rollout's rows (lfb_index), + 1."""
    T, E = done.shape
    L = 0
    for e in range(E):
        s = 0
        for t in range(T):
            L = max(L, t - s + (t0[e] if (t0 is not None and s == 0) else 0) + 1)
            if done[t, e]:
                s = t + 1
    return L


@pytest.mark.parametrize("A", (1, 3))
def test_time_baseline_bins_of_two_env_halves_sum_to_the_whole_batch(lib, A):
    """Each half's bins over the pooled L (a larger L than the half's own: zero bins past its paths), summed: the
    whole batch's counts exactly, its sums to rounding, and each half's simplev within one float32 ulp of the
    whole batch's rows."""
    for k in range(len(TB_SHAPES)):
        q, done, t0s = _case(A, k)
        E = done.shape[1]
        if E < 2:
            continue
        h = E // 2
        for t0 in t0s:
            L = _last_index(done, t0)
            halves = [(slice(0, h), None if t0 is None else t0[:h].copy()),
                      (slice(h, E), None if t0 is None else t0[h:].copy())]
            for per_agent in (0, 1):
                s, c, v = _whole(lib, q, done, t0, per_agent, L)
                parts = [_bins(lib, np.ascontiguousarray(q[:, sl]), np.ascontiguousarray(done[:, sl]), t, per_agent,
                               L) for sl, t in halves]
                ps, pc = parts[0][0] + parts[1][0], parts[0][1] + parts[1][1]
                assert np.array_equal(pc, c)
                np.testing.assert_allclose(ps, s, rtol=1e-13, atol=1e-13)
                for sl, t in halves:
                    got = _apply(lib, np.ascontiguousarray(done[:, sl]), t, per_agent, A, L, ps, pc)
                    d = np.abs(got.view(np.int32).astype(np.int64) - v[:, sl].view(np.int32).astype(np.int64))
                    assert d.max() <= 1


@pytest.mark.parametrize("W", (3, 4))
@pytest.mark.parametrize("A", (1, 3))
def test_time_baseline_bins_of_uneven_shards_sum_to_the_whole_batch(lib, W, A):
    """Shards of one env (rank 0 never done, holding the largest index; rank 1 done on every step, its own L far
    below the pooled L), bins over the pooled L summed in rank order: the whole batch's counts exactly, its sums at
    1e-13, each shard's simplev within one float32 ulp of the whole batch's rows, and the bins of the float64
    reference of postproc_edges.time_index."""
    sizes = se.TB_SIZES[W]
    for L in (127, 129):
        for with_t0 in (False, True):
            q, done, t0 = se.tb_case(sizes, A, L, with_t0, 7 + L)
            shards = [(np.ascontiguousarray(q[:, lo:hi]), np.ascontiguousarray(done[:, lo:hi]),
                       None if t0 is None else t0[lo:hi].copy()) for lo, hi in se.bounds(sizes)]
            for per_agent in (0, 1):
                s, c, v = _whole(lib, q, done, t0, per_agent, L)
                parts = [_bins(lib, qs, ds, ts, per_agent, L) for qs, ds, ts in shards]
                ps, pc = parts[0][0].copy(), parts[0][1].copy()
                for bs, bc in parts[1:]:                 # rank order, as dist.pool_sum adds them
                    ps, pc = ps + bs, pc + bc
                assert np.array_equal(pc, c)
                np.testing.assert_allclose(ps, s, rtol=1e-13, atol=1e-13)
                got = [_apply(lib, ds, ts, per_agent, A, L, ps, pc) for _, ds, ts in shards]
                for g, (lo, hi) in zip(got, se.bounds(sizes)):
                    assert se.ulps(g, v[:, lo:hi]) <= 1
                pe.check_time_baseline(np.concatenate(got, axis=1), ps, pc, q, done, t0, per_agent)


def test_split_entry_points_reject_bad_arguments(lib):
    x, st, ws = np.zeros(8, np.float32), np.zeros(9), np.zeros(4096)
    mp = lib.madrl_moments_pass_f32
    assert mp(0, 1, _p(x), None, 0, _p(st), _p(ws), None) != 0
    assert mp(8, 0, _p(x), None, 0, _p(st), _p(ws), None) != 0
    assert mp(8, 1025, _p(x), None, 0, _p(st), _p(ws), None) != 0
    assert mp(8, 1, _p(x), None, 2, _p(st), _p(ws), None) != 0
    assert mp(8, 1, None, None, 0, _p(st), _p(ws), None) != 0
    assert mp(8, 1, _p(x), None, 0, None, _p(ws), None) != 0
    ca = lib.madrl_center_apply_f32
    assert ca(0, 1, _p(x), _p(st), 1, 0, None) != 0
    assert ca(8, 1025, _p(x), _p(st), 1, 0, None) != 0
    assert ca(8, 1, None, _p(st), 1, 0, None) != 0
    assert ca(8, 1, _p(x), None, 1, 0, None) != 0
    q, i32, f64 = np.zeros(8, np.float32), np.zeros(64, np.int32), np.zeros(8)
    tb, ta = lib.madrl_time_baseline_bins_f32, lib.madrl_time_baseline_apply_f32
    good_b = [2, 2, 2, 0, 2, _p(q), _p(i32), _p(i32), None, _p(f64), _p(i32), _p(i32), None]
    good_a = [2, 2, 2, 0, 2, _p(i32), None, _p(f64), _p(i32), _p(q), None]
    for k in (0, 1, 2, 4):                  # T, E, A, L (3 is per_agent)
        for fn, good in ((tb, good_b), (ta, good_a)):
            bad = list(good)
            bad[k] = 0
            assert fn(*bad) != 0, (fn, k)
    for k in (5, 6, 7, 9, 10, 11):
        bad = list(good_b)
        bad[k] = None
        assert tb(*bad) != 0, k
    for k in (5, 7, 8, 9):
        bad = list(good_a)
        bad[k] = None
        assert ta(*bad) != 0, k
    assert tb(2, 2, 1025, 1, 2, *good_b[5:]) != 0 and ta(2, 2, 1025, 1, 2, *good_a[5:]) != 0


@pytest.mark.parametrize("W", (2, 3, 4))
def test_moment_passes_over_shards_pool_to_the_union(lib, W):
    """madrl_moments_pass_f32 over W shards at the emulator's grid-stride edges, pooled as postproc._moments
    pools them (sums and rows added in rank order, minima by minimum, the second pass about the pooled means): the
    float64 moments of the union; madrl_center_apply_f32 on each shard with the pooled statistics: NumPy's centring
    and shift of the union within one float32 ulp."""
    s = EMU_MOM_BLOCKS * 256
    rows = {2: (s - 1, s + 1), 3: (s - 1, 1, s + 1), 4: (255, 1, 3 * s + 5, 256)}[W]
    A = 3
    parts = [se.moment_shard(n, A, r, 11) for r, n in enumerate(rows)]
    st = [np.full((A, 9), np.nan) for _ in rows]
    ws = np.empty((A, 4096))
    for (x, y), n, t in zip(parts, rows, st):
        assert lib.madrl_moments_pass_f32(n, A, _p(x), _p(y), 0, _p(t), _p(ws), None) == 0
    sums, mins = sum(np.concatenate([t[:, 0:3], np.full((A, 1), float(n))], 1) for t, n in zip(st, rows)), st[0][:, 6:9]
    for t in st[1:]:
        mins = np.minimum(mins, t[:, 6:9])
    pooled = np.full((A, 9), np.nan)
    pooled[:, 0:3], pooled[:, 6:9] = sums[:, 0:3] / sums[:, 3:4], mins
    sq = np.zeros((A, 3))
    for (x, y), n, t in zip(parts, rows, st):
        t[:, 0:3] = pooled[:, 0:3]
        assert lib.madrl_moments_pass_f32(n, A, _p(x), _p(y), 1, _p(t), _p(ws), None) == 0
        sq = sq + t[:, 3:6]
    pooled[:, 3:6] = sq / sums[:, 3:4]
    x, y = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
    want = se.moments_of(x, y)
    np.testing.assert_allclose(pooled, want, rtol=1e-10, atol=1e-12 * np.abs(want).max())
    assert np.array_equal(pooled[:, 6:9], want[:, 6:9])
    for center, positive in pe.CENTRE_MODES:
        got = []
        for (xs, _), n in zip(parts, rows):
            g = Guarded(xs.shape, np.float32, xs)
            assert lib.madrl_center_apply_f32(n, A, _p(g.arr), _p(pooled), center, positive, None) == 0
            got.append(g.check("adv").copy())
        want_c = np.stack([se.centred_want(x[:, a], center, positive) for a in range(A)], 1)
        assert se.ulps(np.concatenate(got), want_c.astype(np.float32)) <= 1, (center, positive)
