"""rltools' sample kernels (madrl_running_moments_*, madrl_time_baseline_*_f32, madrl_lfbr_*), the padded-path kernels
(madrl_paths_pad_*, madrl_path_sums_f32) and the closed loop's per-step wrapper (madrl_obs_wrap_step_*) on the GPU,
at the edges of the product build's grids: the row slices of each group (ceil(S / G) of them, S read from the
sources), the 8-warp row stride and 32-column blocks of the running moments, the 128-bin blocks of the time
baseline, the 64-column tiles, chunk tail and flush of the rltools Gram, the one-thread / one-warp row copies, and
both exact paths of the standardiser's reciprocal square root.  The expected values come from float64 NumPy and the
oracles of oracle/; the bit-identity contracts (bfloat16 against float32 on widened input, one agent against
pooled, the fused step against the passes it fuses, re-runs) compare two device passes by design.  Cases and checks
are shared with the emulated tests through tests/postproc_edges.py."""
import ctypes as C

import numpy as np
import pytest
import torch

import postproc_edges as pe
from oracle import recurrent_oracle as rco
from oracle import rltools_oracle as ro

pytestmark = pytest.mark.gpu
DEV = "cuda"

RM_SLICES = pe.csrc_default("MADRL_RM_SLICES", "postproc.cu")       # running-moment row slices per launch
TB_SLICES = pe.csrc_default("MADRL_TB_SLICES", "postproc.cu")       # time-baseline env slices
LFB_SLICES = pe.csrc_default("MADRL_LFB_SLICES", "baseline.cu")     # Gram row slices
LFB_FLUSH = 2048                                                    # Gram rows between accumulator flushes


def cu(x):
    return None if x is None else torch.as_tensor(np.ascontiguousarray(x), device=DEV)


def obs_dev(x, bf16):
    """float32 values (bfloat16-representable when bf16) as a device tensor of the observation dtype."""
    t = cu(x)
    return None if t is None else (t.to(torch.bfloat16) if bf16 else t)


def bits(t):
    """The tensor's raw words (so that NaNs and signed zeros compare bit for bit)."""
    return None if t is None else t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def same_bits(a, b):
    return (a is None and b is None) or (a is not None and b is not None and torch.equal(bits(a), bits(b)))


def slices(S, G):
    return -(-S // G)


# ---------------------------------------------------------------- running moments (rltools' nn.Standardizer)

def _sums(x, groups, first=None):
    from madrl_b200.rltools_sampler import RunningStandardizer
    return RunningStandardizer(x.shape[-1], DEV)._sums(x, first, groups)[0]


@pytest.mark.parametrize("G", (1, 2, 3, 5, RM_SLICES - 1, RM_SLICES, RM_SLICES + 1, 1024))
def test_running_moments_at_the_slice_edges(G):
    """ceil(64 / G) slices per group (64, 32, 22, 13, 2, 1, 1, 1), R rows per group around them (one row; empty
    slices; one row per slice; the 8-warp stride), D across the 32-column blocks; per group (G = A agents) and
    pooled over the agents, without and with the one-step shift.  Sums within n 2^-52 sum|x| of NumPy's float64
    sums; bfloat16 equals the float32 call on the widened values and a re-run equals the first, bit for bit."""
    S = slices(RM_SLICES, G)
    rs = np.random.RandomState(G)
    for R in pe.slice_rows(S):
        E = 2 if R % 2 == 0 else 1
        for D in (1, 31, 32, 33, 213):
            x = pe.mixed_scale(rs, R // E, E, G, D)
            ob = pe.mixed_scale(rs, E, G, D)
            xt, obt = cu(x), cu(ob)
            for first in (False, True):
                rows = np.concatenate([ob[None], x[:-1]]) if first else x
                rows = rows.astype(np.float64).reshape(-1, G, D)
                calls = [(G, rows)] + ([(1, rows.reshape(-1, 1, D))] if first and G > 1 else [])
                for groups, want_rows in calls:
                    got = _sums(xt, groups, obt if first else None)
                    pe.check_column_sums(got.cpu().numpy(), want_rows)
                    assert same_bits(got, _sums(xt, groups, obt if first else None)), (R, D, first, groups)
                    x16, ob16 = xt.to(torch.bfloat16), obt.to(torch.bfloat16) if first else None
                    assert same_bits(_sums(x16, groups, ob16),
                                     _sums(x16.float(), groups, None if ob16 is None else ob16.float())), \
                        (R, D, first, groups)


def _ulps(got, want):
    g = np.asarray(got, np.float32).view(np.int32).astype(np.int64)
    return np.abs(g - np.asarray(want, np.float32).view(np.int32).astype(np.int64)).max()


def test_running_standardizer_c2_update_against_the_reference():
    """One update of the C2 size (T 256, E 4096, A 5, D 32, with obs_before: 5.2M rows) after a small one, pooled
    and per agent, against nn.Standardizer's restatement fed the same rows: count exact, mean and meansq within one
    float32 ulp (the batch sums are taken in another order)."""
    from madrl_b200.rltools_sampler import RunningStandardizer
    T, E, A, D = 256, 4096, 5, 32
    g = torch.Generator(device=DEV).manual_seed(21)
    scale = torch.linspace(0.5, 4.0, D, device=DEV)
    x = torch.randn((T, E, A, D), generator=g, device=DEV) * scale + torch.linspace(-3.0, 2.0, D, device=DEV)
    ob = torch.randn((E, A, D), generator=g, device=DEV) * scale
    small = torch.randn((7, 13, A, D), generator=g, device=DEV) * 2 + 1
    seen = np.empty((T * E * A, D))
    seen[:E * A] = ob.cpu().numpy().reshape(-1, D)
    seen[E * A:] = x[:-1].cpu().numpy().reshape(-1, D)
    small_np = small.cpu().numpy().astype(np.float64)
    pooled, per = RunningStandardizer(D, DEV), RunningStandardizer(D, DEV, n_agents=A)
    for st in (pooled, per):
        st.update(small)
        st.update(x, ob)
    ref = ro.Standardizer(D)
    ref.update(small_np.reshape(-1, D))
    ref.update(seen)
    assert float(pooled.count) == ref.count[0]
    assert _ulps(pooled.mean.cpu().numpy(), ref.mean[0]) <= 1 and _ulps(pooled.meansq.cpu().numpy(), ref.meansq[0]) <= 1
    seen = seen.reshape(-1, A, D)
    for a in range(A):
        ra = ro.Standardizer(D)
        ra.update(small_np[:, :, a].reshape(-1, D))
        ra.update(seen[:, a])
        assert float(per.count[a]) == ra.count[0]
        assert _ulps(per.mean[a].cpu().numpy(), ra.mean[0]) <= 1, a
        assert _ulps(per.meansq[a].cpu().numpy(), ra.meansq[0]) <= 1, a


# ---------------------------------------------------------------- time-dependent baseline

TB_LENGTHS = (1, 127, 128, 129, 256, 257)       # bins around the 128-thread bin blocks


def _time_baseline(q, done, t0, per_agent):
    from madrl_b200.rltools_sampler import time_baseline
    args = (cu(q), cu(done), cu(t0), per_agent)
    out = time_baseline(*args)
    assert all(same_bits(a, b) for a, b in zip(out, time_baseline(*args)))        # re-run: same bits
    return [t.cpu().numpy() for t in out]


@pytest.mark.parametrize("E", (1, TB_SLICES - 1, TB_SLICES, TB_SLICES + 1, 301))
def test_time_baseline_pooled_at_the_slice_and_bin_edges(E):
    """E envs around the 32 env slices, 3 agents pooled; L bins reached through T (env 0 runs the whole horizon,
    env 1 ends a path on every step) and through env 0's t0 with T = 5."""
    for k, L in enumerate(TB_LENGTHS):
        for T in sorted({L, min(L, 5)}):
            q, done, t0 = pe.time_baseline_case(T, E, 3, L, 100 * E + 10 * k + T)
            pe.check_time_baseline(*_time_baseline(q, done, t0, False), q, done, t0, False)


@pytest.mark.parametrize("A", (2, TB_SLICES - 1, TB_SLICES, TB_SLICES + 1, 1024))
def test_time_baseline_per_agent_at_the_slice_and_bin_edges(A):
    """ceil(32 / A) env slices per agent (16, 2, 1, 1, 1), one set of bins per agent."""
    E = 17 if A == 2 else 3
    for k, L in enumerate(TB_LENGTHS):
        for T in sorted({L, min(L, 5)}):
            q, done, t0 = pe.time_baseline_case(T, E, A, L, 7 * A + 10 * k + T)
            pe.check_time_baseline(*_time_baseline(q, done, t0, True), q, done, t0, True)


@pytest.mark.parametrize("T", (257, 64), ids=("through_T", "through_t0"))
def test_time_baseline_bins_and_apply_with_fewer_bins_than_indices(T):
    """madrl_time_baseline_bins_f32 then _apply_f32 given an L below the largest time index (257 bins' worth of rows): the rows whose
    index is L or more get NaN, and the bins below L are those of the full call, bit for bit."""
    from madrl_b200 import _lib
    from madrl_b200._lib import _ptr
    from madrl_b200.postproc import _paths_plan
    E, A, L_full = 33, 3, 257
    q, done, t0 = pe.time_baseline_case(T, E, A, L_full, T)
    idx = pe.time_index(done, t0)[0]
    assert idx.max() == L_full - 1
    qt, dt, t0t = cu(q), cu(done), cu(t0)
    seg_s, _, n_ep, ep_rec = _paths_plan(dt, A)
    lib = _lib.lib()

    def run(L, per_agent):
        G = A if per_agent else 1
        nbytes = C.c_size_t()
        _lib.check(lib.madrl_time_baseline_workspace_size(G, L, C.byref(nbytes)))
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=DEV)
        s = torch.full((G, L), float("nan"), dtype=torch.float64, device=DEV)
        c = torch.full((G, L), -1, dtype=torch.int32, device=DEV)
        v = torch.zeros_like(qt)
        _lib.check(lib.madrl_time_baseline_bins_f32(T, E, A, int(per_agent), L, _ptr(qt), _ptr(n_ep), _ptr(ep_rec),
                                                    _ptr(t0t), _ptr(s), _ptr(c), _ptr(ws), _lib.stream(qt.device)))
        _lib.check(lib.madrl_time_baseline_apply_f32(T, E, A, int(per_agent), L, _ptr(seg_s), _ptr(t0t), _ptr(s),
                                                     _ptr(c), _ptr(v), _lib.stream(qt.device)))
        return v.cpu().numpy(), s.cpu().numpy(), c.cpu().numpy()

    for per_agent in (False, True):
        full = run(L_full, per_agent)
        pe.check_time_baseline(*full, q, done, t0, per_agent)
        for L in (1, 127, 128, 129, 256):
            v, s, c = run(L, per_agent)
            assert np.array_equal(c, full[2][:, :L]) and np.array_equal(s, full[1][:, :L]), (L, per_agent)
            past = np.broadcast_to((idx >= L)[..., None], q.shape)
            assert past.any() and np.isnan(v[past]).all(), (L, per_agent)
            assert np.array_equal(v[~past], full[0][~past]), (L, per_agent)


# ---------------------------------------------------------------- rltools' linear feature baseline

LFBR_DIMS = (1, 2, 59, 60, 61, 62, 63, 64, 123, 124, 125)     # D + 4 columns on and across the 64 / 128 tile edges


def _obsnorm_state(rs, D, lead=()):
    """(count, mean, meansq) float32 of an obsnorm with mean != 0 and a stdev that is not a power of two."""
    mean = (rs.randn(*lead, D) * 0.7 + 0.3).astype(np.float32)
    meansq = (mean.astype(np.float64) ** 2 + rs.rand(*lead, D) * 3 + 0.1).astype(np.float32)
    return np.full(lead, 10.0, np.float32), mean, meansq


def _rltools_baseline(D, state, n_agents=None):
    """A rltools LinearFeatureBaseline with the obsnorm state given (None: no obsnorm) and the kernels' obsnorm
    table ([2, D] or [A, 2, D] float64: mean, f32(stdev + eps)) as NumPy."""
    from madrl_b200.rltools_sampler import LinearFeatureBaseline
    b = LinearFeatureBaseline(D, DEV, state is not None, n_agents=n_agents)
    if state is None:
        return b, None
    if n_agents is not None and state[1].ndim == 1:         # the same obsnorm for every agent
        state = tuple(np.broadcast_to(s, (n_agents,) + s.shape).copy() for s in state)
    b.obsnorm.set_param_values(*state)
    return b, b.obsnorm.norm_table.cpu().numpy()


def _set_coef(b, coef):
    b.set_param_values((coef, None if b.obsnorm is None else b.obsnorm.get_param_values()))


@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
@pytest.mark.parametrize("obsnorm", [False, True], ids=["raw", "obsnorm"])
def test_rltools_single_row_normal_equations_and_predictions_are_the_exact_features(obsnorm, bf16):
    """One row (T = E = A = 1): G = outer(f, f) bit for bit, f = [(o - mu) / s, a, a * a, 1, y] with a = i / 100
    correctly rounded and the quotient one float64 division.  With an obsnorm the rows past the single row in its
    32-row chunk must store an explicit 0 ((0 - mu) / s is not 0), and the other 47 slices add nothing.  Predict
    with unit coefficient vectors returns float32(f_j): every column at once through a baseline with one agent
    per column, the time and constant columns through the pooled one."""
    rs = np.random.RandomState(31 + 2 * obsnorm + bf16)
    done = torch.zeros((1, 1), dtype=torch.uint8, device=DEV)
    for D in LFBR_DIMS:
        Df = D + 3
        state = _obsnorm_state(rs, D) if obsnorm else None
        pooled, norm = _rltools_baseline(D, state)
        per, _ = _rltools_baseline(D, state, n_agents=Df)
        _set_coef(per, np.eye(Df))
        for before in (False, True):
            for k, t0 in enumerate(pe.LFB_T0):
                o = pe.lfbr_single_row_obs(D, k, bf16, rs)
                y = np.float32(rs.randn() * 4)
                f = np.append(pe.lfbr_features(o, t0, norm), y)
                row = obs_dev(o.reshape(1, 1, 1, D), bf16)
                ob = None
                if before:                       # the row is obs_before's; obs[0] is never read
                    ob, row = row.reshape(1, 1, D), torch.full_like(row, float("nan"))
                t0_t = torch.tensor([t0], dtype=torch.int32, device=DEV)
                ret = torch.tensor([[[float(y)]]], device=DEV)
                G = pooled.normal_equations(row, done, ret, ob, t0_t).cpu().numpy()
                assert np.array_equal(G, np.outer(f, f)), (D, before, t0)
                rows = row.expand(1, 1, Df, D).contiguous()
                obs_b = None if ob is None else ob.expand(1, Df, D).contiguous()
                vals = per.predict(rows, done, obs_b, t0_t).cpu().numpy().reshape(-1)
                assert np.array_equal(vals, f[:Df].astype(np.float32)), (D, before, t0)
                if k % 4 == 0:
                    for j in range(D, Df):
                        _set_coef(pooled, np.eye(Df)[j])
                        assert pooled.predict(row, done, ob, t0_t).item() == np.float32(f[j]), (D, before, t0, j)
                    GA = per.normal_equations(rows, done, ret.expand(1, 1, Df).contiguous(), obs_b, t0_t)
                    assert np.array_equal(GA.cpu().numpy(), np.broadcast_to(np.outer(f, f), GA.shape)), (D, t0)


def _rltools_reference(c, norm, per_agent):
    """float64 features F [T,E,A,Df] of the rollout case c (rows with the one-step shift, t0) and [F | y]."""
    obs, ob = c["obs"], c["obs_before"]
    seen = np.concatenate([ob[None], obs[:-1]]) if ob is not None else obs
    idx = pe.time_index(c["done"], c["t0"])[0][..., None]
    idx = np.broadcast_to(idx, obs.shape[:3])
    F = pe.lfbr_features(seen, idx, None if norm is None else (norm[None, None] if per_agent else norm))
    return F, np.concatenate([F, c["ret"][..., None].astype(np.float64)], axis=-1)


def _rltools_calls(b, c):
    """G and its bit-identity contracts: a re-run, and bfloat16 observations against the call on obs.float()."""
    obs, ob, done, ret, t0 = cu(c["obs"]), cu(c["obs_before"]), cu(c["done"]), cu(c["ret"]), cu(c["t0"])
    G = b.normal_equations(obs, done, ret, ob, t0)
    assert same_bits(G, b.normal_equations(obs, done, ret, ob, t0))
    o16, ob16 = obs.to(torch.bfloat16), None if ob is None else ob.to(torch.bfloat16)
    assert same_bits(b.normal_equations(o16, done, ret, ob16, t0),
                     b.normal_equations(o16.float(), done, ret, None if ob16 is None else ob16.float(), t0))
    return G


@pytest.mark.parametrize("obsnorm", [False, True], ids=["raw", "obsnorm"])
@pytest.mark.parametrize("T,E,A,D", [
    (1, 1, 1, 60),                                   # one row
    (5, 3, 3, 61),                                   # fewer rows than slices
    (LFB_SLICES * LFB_FLUSH - 1, 1, 1, 62),
    (32, LFB_SLICES * LFB_FLUSH // 96, 3, 125),      # every slice exactly one flush
    (LFB_SLICES * LFB_FLUSH + 1, 1, 1, 124),
], ids=["N1", "N45", "N=S*2048-1", "N=S*2048", "N=S*2048+1"])
def test_rltools_gram_and_predict_at_the_row_count_edges(T, E, A, D, obsnorm):
    """The pooled Gram within pe.check_gram's bound of the float64 NumPy product, predictions within
    pe.check_predict's; with one agent, a baseline with n_agents=1 gives the pooled bits."""
    rs = np.random.RandomState(T + D + obsnorm)
    c = pe.lfb_case(T, E, A, D, 0.02 if T > 100 else 0.2, T + D)
    state = _obsnorm_state(rs, D) if obsnorm else None
    b, norm = _rltools_baseline(D, state)
    G = _rltools_calls(b, c)
    F, Fy = _rltools_reference(c, norm, False)
    Fy = Fy.reshape(-1, D + 4)
    pe.check_gram(G.cpu().numpy(), Fy.T @ Fy)
    coef = rs.randn(D + 3)
    _set_coef(b, coef)
    args = [cu(c[k]) for k in ("obs", "done", "obs_before", "t0")]
    vals = b.predict(*args)
    pe.check_predict(vals.cpu().numpy(), F.reshape(-1, D + 3), coef)
    if A == 1:
        b1, _ = _rltools_baseline(D, state, n_agents=1)
        assert same_bits(_rltools_calls(b1, c)[0], G)
        _set_coef(b1, coef[None])
        assert same_bits(b1.predict(*args), vals)


@pytest.mark.parametrize("A,D", [(2, 61), (LFB_SLICES - 1, 60), (LFB_SLICES, 64), (LFB_SLICES + 1, 62), (1024, 59)])
def test_rltools_per_agent_gram_and_predict_at_the_slice_edges(A, D):
    """ceil(48 / A) slices per agent (24, 2, 1, 1, 1), each agent with its own obsnorm; each agent's system
    against NumPy on its own rows, predictions per agent."""
    rs = np.random.RandomState(A + D)
    c = pe.lfb_case(4, 3, A, D, 0.3, A)
    b, norm = _rltools_baseline(D, _obsnorm_state(rs, D, (A,)), n_agents=A)
    G = _rltools_calls(b, c).cpu().numpy()
    F, Fy = _rltools_reference(c, norm, True)
    coef = rs.randn(A, D + 3)
    _set_coef(b, coef)
    vals = b.predict(*[cu(c[k]) for k in ("obs", "done", "obs_before", "t0")]).cpu().numpy()
    for a in range(A):
        rows = Fy[:, :, a].reshape(-1, D + 4)
        pe.check_gram(G[a], rows.T @ rows)
        pe.check_predict(vals[:, :, a], F[:, :, a].reshape(-1, D + 3), coef[a])


# ---------------------------------------------------------------- the closed loop's per-step wrapper

def _wrap_done(T, E, rs):
    """done [T, E]: env e % 5 == 0 never, 1 at t = 0, 2 on every step, 3 at random, 4 at t = T - 1."""
    done = np.zeros((T, E), np.uint8)
    done[0, 1::5] = 1
    done[:, 2::5] = 1
    done[:, 3::5] = rs.rand(T, len(range(3, E, 5))) < 0.4
    done[T - 1, 4::5] = 1
    return done


def _wrap_fused(B, obsnorm, obs0, obs, term, done, mean, var, alpha=pe.STD_ALPHA):
    """T single-step calls of madrl_obs_wrap_step_*: (obs, term, stacks [T,E,A,D,B], mean, var) after them."""
    from madrl_b200 import _lib
    from madrl_b200._lib import _ptr
    T, E, A, D = obs.shape
    fn = getattr(_lib.lib(), "madrl_obs_wrap_step_" + ("bf16" if obs.dtype == torch.bfloat16 else "f32"))
    x, tm = obs.clone(), term.clone()
    m, v = (mean.clone(), var.clone()) if obsnorm else (None, None)
    out = torch.empty(tuple(obs.shape) + (B,), dtype=obs.dtype, device=DEV)
    prev = obs0.unsqueeze(-1).expand(E, A, D, B).contiguous()
    for t in range(T):
        _lib.check(fn(E, A, D, B, _ptr(x[t]), _ptr(tm[t] if obsnorm else None), _ptr(done[t]),
                      _ptr(prev if B > 1 else None), _ptr(out[t]), _ptr(m), _ptr(v), alpha, pe.STD_EPS,
                      _lib.stream(x.device)))
        prev = out[t]
    return x, tm, out, m, v


def _wrap_composed(B, obsnorm, obs0, obs, term, done, mean, var, alpha=pe.STD_ALPHA):
    """The same steps through the whole-trajectory passes: Standardizer.obs with the terminal observations over
    T, then FrameStack."""
    from madrl_b200.postproc import FrameStack, Standardizer
    T, E, A, D = obs.shape
    x, tm = obs.clone(), term.clone()
    m = v = None
    if obsnorm:
        st = Standardizer(E, A, D, DEV, enable_obsnorm=True, obs_alpha=alpha, eps=pe.STD_EPS)
        st.obs_mean.copy_(mean)
        st.obs_var.copy_(var)
        st.obs(x, done, tm)
        m, v = st.obs_mean, st.obs_var
    fs = FrameStack(E, A, D, B, DEV, dtype=obs.dtype)
    fs.reset(obs0)
    return x, tm, fs.rollout(x, done), m, v


NAMES = ("obs", "term", "stack", "mean", "var")


@pytest.mark.parametrize("obsnorm", [False, True], ids=["stack", "obsnorm"])
def test_obs_wrap_step_across_both_inv_std_paths(obsnorm):
    """E*A*D = 480 (two blocks, the last partial), T = 5, B = 1..8, float32 and bfloat16, done never / at t = 0 /
    every step / at random / at t = T-1.  The running estimates are seeded from pe.std_obs_case, so that the first
    update (with the terminal observation where done is set at t = 0) lands the variance on 0, subnormals, 1e-300,
    both float32 boundaries of inv_std with their neighbours, 1 and 1e300.  T single steps equal the composed
    passes bit for bit; bfloat16 steps give the float32 steps' values rounded to nearest even and the same
    estimates; the first step's standardised values are within pe.check_standardized of the float64 oracle;
    without obsnorm obs and term are left as they are."""
    x_case, m, v, m1, v1 = pe.std_obs_case(reps=5)
    assert all(pe.std_target_classes(v1).values()), pe.std_target_classes(v1)
    E, A, D, T = 10, 3, 16, 5
    rs = np.random.RandomState(3)
    done = _wrap_done(T, E, rs)
    r16 = lambda a: pe.bf16_bits(a.astype(np.float32))[1]           # noqa: E731  (every input fits bfloat16)
    obs0, obs, term = r16(rs.randn(E, A, D)), r16(rs.randn(T, E, A, D) * 2 + 0.5), r16(rs.randn(T, E, A, D) * 3 - 1)
    reset0 = np.broadcast_to(done[0].astype(bool)[:, None, None], (E, A, D))
    xc = x_case.reshape(E, A, D)
    term[0] = np.where(reset0, xc, term[0])           # the first update of every element sees x_case
    obs[0] = np.where(reset0, obs[0], xc)
    est = (cu(m.reshape(E, A, D)), cu(v.reshape(E, A, D)))
    for B in range(1, 9):
        res = {}
        for bf16 in (False, True):
            args = (obs_dev(obs0, bf16), obs_dev(obs, bf16), obs_dev(term, bf16), cu(done)) + est
            got, want = _wrap_fused(B, obsnorm, *args), _wrap_composed(B, obsnorm, *args)
            for name, g, w in zip(NAMES, got, want):
                assert same_bits(g, w), (B, bf16, name)
            if not obsnorm:
                assert same_bits(got[0], args[1]) and same_bits(got[1], args[2]), (B, bf16)
            res[bf16] = got
        for name, f32, b16 in zip(NAMES, res[False], res[True]):
            assert same_bits(b16, f32 if f32 is None or f32.dtype == torch.float64 else f32.to(torch.bfloat16)), \
                (B, name)
    if obsnorm:
        x_out, tm_out = res[False][0][0].cpu().numpy(), res[False][1][0].cpu().numpy()
        first = np.where(reset0, tm_out, x_out)
        off = pe.check_standardized(first, (x_case.astype(np.float64) - m1) / (np.sqrt(v1) + pe.STD_EPS))
        print("obs_wrap_step: %d of %d first-step values are the other float32 neighbour of the float64 value"
              % (off, x_case.size))


@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
def test_obs_wrap_step_at_the_c2_element_count(bf16):
    """E 4096, A 5, D 213 (4 362 240 elements, 17 040 full blocks), B = 4, obsnorm with StandardizedEnv's default
    alpha = 0.001 (not a power of two, so the running update's roundings depend on how its multiply-adds are
    fused): three single steps equal the composed passes bit for bit."""
    E, A, D, T, B = 4096, 5, 213, 3, 4
    g = torch.Generator(device=DEV).manual_seed(17)
    dt = torch.bfloat16 if bf16 else torch.float32
    obs0 = torch.randn((E, A, D), generator=g, device=DEV).to(dt)
    obs = (torch.randn((T, E, A, D), generator=g, device=DEV) * 2 + 0.5).to(dt)
    term = (torch.randn((T, E, A, D), generator=g, device=DEV) * 3 - 1).to(dt)
    mean = torch.randn((E, A, D), generator=g, device=DEV, dtype=torch.float64) * 0.1
    var = 1 + torch.rand((E, A, D), generator=g, device=DEV, dtype=torch.float64)
    done = cu(_wrap_done(T, E, np.random.RandomState(5)))
    args = (obs0, obs, term, done, mean, var)
    got, want = _wrap_fused(B, True, *args, alpha=0.001), _wrap_composed(B, True, *args, alpha=0.001)
    for name, a, b in zip(NAMES, got, want):
        assert same_bits(a, b), name


# ---------------------------------------------------------------- padded paths (rllab's recurrent batch)

def _poison_allocator():
    """Return blocks of every size class to torch's caching allocator filled with 0xFF bytes, so that an output
    word a kernel leaves unwritten does not read as 0 by chance."""
    held = [torch.full((n,), -1, dtype=torch.int32, device=DEV) for n in (1 << 8, 1 << 12, 1 << 16, 1 << 18) * 8]
    held += [torch.full((1 << 24,), -1, dtype=torch.int32, device=DEV) for _ in range(2)]
    torch.cuda.synchronize()
    del held


def _words(x, itemsize):
    """NumPy words as a device tensor of the padded dtype: int32 (4-byte words) or bfloat16 (2-byte words)."""
    return cu(x.view(np.int32)) if itemsize == 4 else cu(x.view(np.int16)).view(torch.bfloat16)


PAD_SHAPES = pe.PACK_SHAPES + ((4, 133, 1, 0.4),)       # and one agent: the rows of the per-env record rule


@pytest.mark.parametrize("itemsize", [4, 2], ids=["u32", "bf16"])
def test_padded_paths_at_the_word_count_edges(itemsize):
    """Observation and per-env info rows of D in {1..5, 31, 32, 33} words (one thread per row up to 4, one warp
    beyond), 4-byte and bfloat16 words, with and without the obs_before shift, at T = 1 and with every path one
    step long (Lmax = 1) over E > 128 envs, and with one agent: bit for bit recurrent_oracle.torch_pad over the
    records of the host's path cut, every padded word 0; path_returns' sums bit for bit a float64 sum in time
    order and its first returns the paths' first returns, in both path orders."""
    from madrl_b200.postproc import pad_paths, path_returns
    for k, D in enumerate(pe.PACK_WORDS):
        for shifted in (False, True):
            for T, E, A, p_done in PAD_SHAPES:
                c = pe.pack_case(T, E, A, D, p_done, itemsize, 100 * D + 10 * shifted + A)
                obs, ob = _words(c["obs"], itemsize), _words(c["obs_before"], itemsize)
                info = _words(np.ascontiguousarray(c["obs"][:, :, 0]), itemsize)      # [T, E, D] per env
                act, rew, done = cu(c["act"]), cu(c["rew"]), cu(c["done"])
                _poison_allocator()
                pp = pad_paths(obs, act, rew, done, dict(k=info), obs_before=ob if shifted else None)
                rec = pe.path_records(c["done"], A)
                got_rec = torch.stack([pp.env, pp.agent, pp.start, pp.length], 1).cpu().numpy()
                assert np.array_equal(got_rec, rec), (D, shifted, T, E, A)
                L = int(rec[:, 3].max())
                if T == 1 or p_done == 1:
                    assert L == 1
                rec_t = cu(rec)
                valid = torch.arange(L, device=DEV)[None] < rec_t[:, 3:4]
                for name, got, want in (
                        ("obs", pp.observations, rco.torch_pad(obs, rec_t, L, first=ob if shifted else None)),
                        ("info", pp.env_infos["k"], rco.torch_pad(info, rec_t, L, per_agent=False)),
                        ("act", pp.actions, rco.torch_pad(act, rec_t, L)),
                        ("rew", pp.rewards, rco.torch_pad(rew, rec_t, L))):
                    assert same_bits(got, want), (name, D, shifted, T, E, A)
                    assert not bits(got)[~valid].any(), (name, D, shifted, T, E, A)
            if k == 0 and not shifted:
                for T, E, A, p_done in PAD_SHAPES:
                    c = pe.pack_case(T, E, A, 1, p_done, 4, 7 + A)
                    ret = np.random.RandomState(A).randn(T, E, A).astype(np.float32)
                    for per_agent in (False, True):
                        sums, first = path_returns(cu(c["rew"]), cu(ret), cu(c["done"]), per_agent)
                        rec = pe.path_records(c["done"], A, agent_major=per_agent)
                        want = [pe.sequential_sum(c["rew"][s:s + n, e, a]) for e, a, s, n in rec]
                        assert np.array_equal(sums.cpu().numpy().reshape(-1), np.array(want)), (T, E, A, per_agent)
                        assert np.array_equal(first.cpu().numpy().reshape(-1),
                                              np.array([ret[s, e, a] for e, a, s, _ in rec], np.float64))
