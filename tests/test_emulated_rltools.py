"""rltools' sample-processing kernels executed on the CPU by the warp emulator of tests/emu, through the C ABI, against
NumPy and oracle/rltools_oracle.py: madrl_running_moments_{f32,bf16} (column sums of x and x^2, pooled and per agent,
with and without the one-step observation shift), madrl_time_baseline_f32 (bins, counts and simplev, pooled and per
agent, with t0), and rltools' feature map of the linear-baseline kernels (madrl_lfbr_*), with and without an obsnorm.
The shapes cross the row-slice, warp-stride and 32-column edges of the kernels; A runs from 1 to 8.  Outputs sit in
canary-guarded buffers, and every new entry point's argument checks (MADRL_EINVAL, no launch) are exercised."""
import ctypes as C

import numpy as np
import pytest
import torch

import postproc_edges as pe
from emu import driver
from emu.driver import Guarded
from emu.driver import ptr as _p
from oracle import rltools_oracle as ro

pytestmark = driver.needs_cxx


@pytest.fixture(scope="module")
def lib():
    """The emulator build, whose few row slices (build_emu.GRID) put the slice edges inside these tests' shapes."""
    return driver.load(())


def _index(done, t0):
    """lfb_index of every (t, e): the position in the path, plus t0[e] on env e's first path."""
    T, E = done.shape
    idx = np.zeros((T, E), np.int64)
    for e in range(E):
        s = 0
        for t in range(T):
            idx[t, e] = t - s + (t0[e] if (t0 is not None and s == 0) else 0)
            if done[t, e]:
                s = t + 1
    return idx


def _moments(lib, x, G, first=None, bf16=False):
    """madrl_running_moments_* over x [R*G, D] (rows k G + g of group g), first [shift, D] or None."""
    D = x.shape[-1]
    R = x.size // (D * G)
    nbytes = C.c_size_t()
    assert lib.madrl_running_moments_workspace_size(G, D, C.byref(nbytes)) == 0
    ws = np.full(nbytes.value // 8, np.nan)
    out = Guarded((G, 2, D), np.float64, np.nan)
    fn = lib.madrl_running_moments_bf16 if bf16 else lib.madrl_running_moments_f32
    shift = 0 if first is None else first.size // D
    assert fn(R, G, D, shift, _p(x), _p(first), _p(out.arr), _p(ws), None) == 0, lib.madrl_last_error()
    return out.check("sums").copy()


# (rows per group, D): slices of fewer and more rows than the 8 warps, 1 and 32 columns, 33 and 70 (cb > 0)
MOMENT_SHAPES = ((1, 1), (7, 3), (50, 1), (61, 32), (45, 33), (26, 70))


@pytest.mark.parametrize("bf16", (False, True), ids=("f32", "bf16"))
@pytest.mark.parametrize("G", (1, 2, 3, 5, 8))
def test_running_moments_equal_numpy_sums(lib, G, bf16):
    rs = np.random.RandomState(10 * G + bf16)
    for R, D in MOMENT_SHAPES:
        x = (rs.randn(R * G, D) * 3 + 1).astype(np.float32)
        bits, x = pe.bf16_bits(x) if bf16 else (x, x)
        got = _moments(lib, bits, G, bf16=bf16)
        x64 = x.astype(np.float64).reshape(R, G, D)
        want = np.stack([x64.sum(0), (x64 * x64).sum(0)], 1)
        np.testing.assert_allclose(got, want, rtol=1e-13, atol=1e-12, err_msg=str((R, D)))
        assert np.array_equal(got, _moments(lib, bits, G, bf16=bf16))        # re-run: same bits


@pytest.mark.parametrize("A", (1, 2, 4, 8))
def test_running_moments_read_the_action_rows(lib, A):
    """With `first` (obs_before) the rows are the observations the actions were taken in, per agent and pooled."""
    T, E, D = 9, 5, 35
    rs = np.random.RandomState(A)
    obs = rs.randn(T, E, A, D).astype(np.float32)
    ob = rs.randn(E, A, D).astype(np.float32)
    seen = np.concatenate([ob[None], obs[:-1]]).astype(np.float64)
    for G in (1, A):
        got = _moments(lib, obs, G, first=ob)
        rows = seen.reshape(-1, G, D)
        np.testing.assert_allclose(got, np.stack([rows.sum(0), (rows * rows).sum(0)], 1), rtol=1e-13, atol=1e-12)


def test_standardiser_update_matches_the_reference_arithmetic(lib):
    """The float32 state update of RunningStandardizer (torch on the host here) fed with the emulated sums equals
    nn.Standardizer's restatement within one float32 ulp (the batch mean sums in another order), over three
    updates of different batch sizes; per agent and sequentially per agent (the concurrent reward normaliser)."""
    from madrl_b200.rltools_sampler import RunningStandardizer
    rs = np.random.RandomState(3)
    A, D = 3, 6
    st = RunningStandardizer(D, "cpu", n_agents=A)
    seq = RunningStandardizer(1, "cpu")
    refs = [ro.Standardizer(D) for _ in range(A)]
    ref_seq = ro.Standardizer(1)
    for N in (40, 7, 130):
        x = (rs.randn(N, A, D) * 2 + 0.7).astype(np.float32)
        sums = torch.from_numpy(_moments(lib, x, A))
        st.count, st.mean, st.meansq = st._mix(st.count, st.mean, st.meansq, sums, N)
        r = x[..., :1]
        rsum = torch.from_numpy(_moments(lib, np.ascontiguousarray(r), A))
        for a in range(A):
            refs[a].update(x[:, a].astype(np.float64))
            seq.count, seq.mean, seq.meansq = seq._mix(seq.count, seq.mean, seq.meansq, rsum[a], N)
            ref_seq.update(r[:, a].astype(np.float64))
    for a in range(A):
        assert float(st.count[a]) == refs[a].count[0]
        for got, want in ((st.mean[a], refs[a].mean[0]), (st.meansq[a], refs[a].meansq[0])):
            d = np.abs(got.numpy().view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
            assert d.max() <= 1
    assert float(seq.count) == ref_seq.count[0]
    assert abs(int(seq.mean.numpy().view(np.int32)[0]) - int(ref_seq.mean.view(np.int32)[0, 0])) <= 1


# (T, E, done probability): slices of one and several envs, L off and past the 128-thread bin block
TB_SHAPES = ((5, 2, 0.3), (9, 7, 0.2), (140, 4, 0.0), (33, 11, 0.1))


@pytest.mark.parametrize("A", (1, 2, 3, 5, 8))
def test_time_baseline_against_numpy(lib, A):
    for k, (T, E, p) in enumerate(TB_SHAPES):
        rs = np.random.RandomState(100 * A + k)
        done = (rs.rand(T, E) < p).astype(np.uint8)
        if T > 2:
            done[0, 0] = done[T - 1, E - 1] = 1            # length-1 paths at t = 0 and t = T-1
        q = rs.randn(T, E, A).astype(np.float32)
        for t0 in (None, rs.randint(0, 6, E).astype(np.int32)):
            seg_s, _, n_ep, ep_rec = driver.paths_plan(lib, done, A)
            idx = _index(done, t0)
            L = int(idx.max()) + 1
            for per_agent in (0, 1):
                G = A if per_agent else 1
                nbytes = C.c_size_t()
                assert lib.madrl_time_baseline_workspace_size(G, L, C.byref(nbytes)) == 0
                ws = np.zeros(nbytes.value, np.uint8)
                s, c = Guarded((G, L), np.float64, np.nan), Guarded((G, L), np.int32, -1)
                v = Guarded((T, E, A), np.float32, np.nan)
                assert lib.madrl_time_baseline_f32(T, E, A, per_agent, L, _p(q), _p(seg_s), _p(n_ep), _p(ep_rec),
                                                   _p(t0), _p(s.arr), _p(c.arr), _p(v.arr), _p(ws), None) == 0
                ws_, wc = np.zeros((G, L)), np.zeros((G, L), np.int64)
                for a in range(A):
                    np.add.at(ws_[a if per_agent else 0], idx, q[..., a].astype(np.float64))
                    np.add.at(wc[a if per_agent else 0], idx, 1)
                assert np.array_equal(c.check("counts"), wc)
                np.testing.assert_allclose(s.check("sums"), ws_, rtol=1e-13, atol=1e-13)
                mean = ws_ / np.maximum(wc, 1)
                want = np.stack([mean[a if per_agent else 0][idx] for a in range(A)], -1).astype(np.float32)
                got = v.check("simplev")
                np.testing.assert_allclose(got, want, rtol=2e-7, atol=1e-7)


def test_time_baseline_is_the_reference_nanmean(lib):
    """simplev of a rollout's paths equals Sampler.process's nanmean over the padded q (the oracle's)."""
    rs = np.random.RandomState(4)
    T, E, A = 12, 5, 3
    done = (rs.rand(T, E) < 0.25).astype(np.uint8)
    q = rs.randn(T, E, A).astype(np.float32)
    seg_s, _, n_ep, ep_rec = driver.paths_plan(lib, done, A)
    L = int(_index(done, None).max()) + 1
    nbytes = C.c_size_t()
    assert lib.madrl_time_baseline_workspace_size(1, L, C.byref(nbytes)) == 0
    ws = np.zeros(nbytes.value, np.uint8)
    s, c, v = np.zeros((1, L)), np.zeros((1, L), np.int32), np.zeros((T, E, A), np.float32)
    assert lib.madrl_time_baseline_f32(T, E, A, 0, L, _p(q), _p(seg_s), _p(n_ep), _p(ep_rec), None, _p(s), _p(c),
                                       _p(v), _p(ws), None) == 0
    paths = ro.batches(np.zeros((T, E, A, 1), np.float32), q.astype(np.float64), done, None, "decentralized")[0]
    rows = ro._padded([p["rewards"] for p in paths], np.nan)
    np.testing.assert_allclose(s[0] / c[0], np.nanmean(rows, axis=0), rtol=1e-13)


def _lfbr(lib, obs, obs_before, done, q, norm, coef, A_groups, bf16):
    """madrl_lfbr normal equations and predictions of the emulator build."""
    T, E, A, D = obs.shape
    seg_s = driver.paths_plan(lib, done, A)[0]
    nbytes = C.c_size_t()
    if A_groups:
        assert lib.madrl_lfbr_agents_workspace_size(D, A, C.byref(nbytes)) == 0
    else:
        assert lib.madrl_lfbr_workspace_size(D, C.byref(nbytes)) == 0
    ws = np.zeros(nbytes.value // 8)
    Dc = D + 4
    G = Guarded(((A,) if A_groups else ()) + (Dc, Dc), np.float64, np.nan)
    sfx = ("_agents" if A_groups else "") + ("_bf16" if bf16 else "_f32")
    src, first = (pe.bf16_bits(obs)[0], None if obs_before is None else pe.bf16_bits(obs_before)[0]) if bf16 \
        else (obs, obs_before)
    assert getattr(lib, "madrl_lfbr_normal_eq" + sfx)(T, E, A, D, _p(src), _p(first), _p(seg_s), None, _p(q),
                                                      _p(norm), _p(G.arr), _p(ws), None) == 0
    vals = Guarded((T, E, A), np.float32, np.nan)
    assert getattr(lib, "madrl_lfbr_predict" + sfx)(T, E, A, D, _p(src), _p(first), _p(seg_s), None, _p(norm),
                                                    _p(coef), _p(vals.arr), None) == 0
    return G.check("G"), vals.check("values")


@pytest.mark.parametrize("bf16", (False, True), ids=("f32", "bf16"))
@pytest.mark.parametrize("A,D,obsnorm,shifted", ((1, 5, True, True), (2, 61, True, False), (3, 70, False, True),
                                                  (8, 3, True, True)))
def test_rltools_feature_map_against_numpy(lib, A, D, obsnorm, shifted, bf16):
    """Gram within 1e-12 sqrt(G_ii G_jj) of the float64 product of the rltools features, predictions within float32
    rounding, pooled and per agent; D = 61 and 70 put the time, constant and return columns on and across the
    64-column tile edge, and rows past the last slice chunk must add nothing."""
    T, E = 11, 6
    rs = np.random.RandomState(A * 100 + D)
    obs = (rs.randn(T, E, A, D) * 2 + 0.5).astype(np.float32)
    ob = (rs.randn(E, A, D) * 2 + 0.5).astype(np.float32) if shifted else None
    if bf16:
        obs = pe.bf16_bits(obs)[1]
        ob = None if ob is None else pe.bf16_bits(ob)[1]
    done = (rs.rand(T, E) < 0.2).astype(np.uint8)
    q = rs.randn(T, E, A).astype(np.float32)
    seen = (np.concatenate([ob[None], obs[:-1]]) if shifted else obs).astype(np.float64)
    i = _index(done, None)[..., None].repeat(A, 2).astype(np.float64) / 100.
    for per_agent in (False, True):
        G_ = A if per_agent else 1
        mu = rs.randn(G_, D) * 0.3
        s = np.abs(rs.randn(G_, D)) + 0.5
        norm = np.ascontiguousarray(np.stack([mu, s], 1)) if obsnorm else None
        coef = rs.randn(G_, D + 3)
        G, vals = _lfbr(lib, obs, ob, done, q, None if norm is None else (norm if per_agent else norm[0]),
                        coef if per_agent else coef[0], per_agent, bf16)
        grp = np.arange(A) if per_agent else np.zeros(A, int)
        o = (seen - mu[grp]) / s[grp] if obsnorm else seen
        F = np.concatenate([o, i[..., None], (i * i)[..., None], np.ones((T, E, A, 1)), q[..., None]], -1)
        pred = (F[..., :-1] * coef[grp]).sum(-1)
        np.testing.assert_allclose(vals, pred.astype(np.float32), rtol=1e-6, atol=1e-6 * np.abs(pred).max())
        Gs = G if per_agent else G[None]
        for g in range(G_):
            rows = F[:, :, g] if per_agent else F.reshape(-1, D + 4)
            want = rows.reshape(-1, D + 4).T @ rows.reshape(-1, D + 4)
            d = np.sqrt(np.diag(want))
            assert np.all(np.abs(Gs[g] - want) <= 1e-12 * np.outer(d, d)), (per_agent, g)
    assert int(lib.madrl_emu_race_count()) == 0


def test_argument_errors(lib):
    """MADRL_EINVAL, and no launch, for sizes below 1, group counts past MADRL_AGENTS_MAX, a shift outside the rows
    and NULL buffers, at every new entry point."""
    x, d, i32 = np.zeros(64, np.float32), np.zeros(64), np.zeros(64, np.int32)
    n = C.c_size_t()
    for G, D in ((0, 1), (1, 0), (1025, 1)):
        assert lib.madrl_running_moments_workspace_size(G, D, C.byref(n)) != 0
    assert lib.madrl_running_moments_workspace_size(1, 1, None) != 0
    for fn in (lib.madrl_running_moments_f32, lib.madrl_running_moments_bf16):
        for R, G, D, shift, first in ((0, 1, 1, 0, None), (4, 0, 1, 0, None), (4, 1025, 1, 0, None),
                                      (4, 1, 0, 0, None), (4, 1, 1, 0, x), (4, 1, 1, 5, x)):
            assert fn(R, G, D, shift, _p(x), _p(first), _p(d), _p(d), None) != 0, (R, G, D, shift)
        assert fn(4, 1, 1, 0, None, None, _p(d), _p(d), None) != 0
        assert fn(4, 1, 1, 0, _p(x), None, None, _p(d), None) != 0
        assert fn(4, 1, 1, 0, _p(x), None, _p(d), None, None) != 0
    for G, L in ((0, 1), (1, 0), (1025, 1)):
        assert lib.madrl_time_baseline_workspace_size(G, L, C.byref(n)) != 0
    assert lib.madrl_time_baseline_workspace_size(1, 1, None) != 0
    ok = [_p(x), _p(i32), _p(i32), _p(i32), None, _p(d), _p(i32), _p(x), _p(d)]
    tb = lib.madrl_time_baseline_f32
    for sizes in ((0, 1, 1, 0, 1), (1, 0, 1, 0, 1), (1, 1, 0, 0, 1), (1, 1, 1, 0, 0), (1, 1, 1025, 1, 1)):
        assert tb(*sizes, *ok, None) != 0, sizes
    for k in (0, 1, 2, 3, 5, 6, 7, 8):
        args = list(ok)
        args[k] = None
        assert tb(1, 1, 1, 0, 1, *args, None) != 0, k
    for D in (0, 8193):
        assert lib.madrl_lfbr_workspace_size(D, C.byref(n)) != 0
        assert lib.madrl_lfbr_agents_workspace_size(D, 2, C.byref(n)) != 0
    assert lib.madrl_lfbr_agents_workspace_size(4, 0, C.byref(n)) != 0
    assert lib.madrl_lfbr_agents_workspace_size(4, 1025, C.byref(n)) != 0
    for ag in ("", "_agents"):
        for dt in ("f32", "bf16"):
            ne = getattr(lib, "madrl_lfbr_normal_eq%s_%s" % (ag, dt))
            pr = getattr(lib, "madrl_lfbr_predict%s_%s" % (ag, dt))
            for sizes in ((0, 1, 1, 1), (1, 1, 1, 0), (1, 1, 1, 8193), (1, 0, 1, 1)):
                assert ne(*sizes, _p(x), None, _p(i32), None, _p(x), None, _p(d), _p(d), None) != 0
                assert pr(*sizes, _p(x), None, _p(i32), None, None, _p(d), _p(x), None) != 0
            assert ne(1, 1, 1, 1, None, None, _p(i32), None, _p(x), None, _p(d), _p(d), None) != 0
            assert ne(1, 1, 1, 1, _p(x), None, _p(i32), None, None, None, _p(d), _p(d), None) != 0
            assert ne(1, 1, 1, 1, _p(x), None, _p(i32), None, _p(x), None, _p(d), None, None) != 0
            assert pr(1, 1, 1, 1, _p(x), None, None, None, None, _p(d), _p(x), None) != 0
            assert pr(1, 1, 1, 1, _p(x), None, _p(i32), None, None, None, _p(x), None) != 0
            if ag:
                assert ne(1, 1, 1025, 1, _p(x), None, _p(i32), None, _p(x), None, _p(d), _p(d), None) != 0
                assert pr(1, 1, 1025, 1, _p(x), None, _p(i32), None, None, _p(d), _p(x), None) != 0
