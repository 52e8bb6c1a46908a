"""Per-agent (concurrent-mode) LinearFeatureBaseline without a GPU: the oracle (oracle/concurrent_baseline_oracle.py)
against the real rllab pieces (tests/golden/linear_baseline_concurrent_ref.npz, written by
oracle/make_concurrent_baseline_golden.py), the per-agent kernels of csrc/baseline.cu and csrc/postproc.cu in the
warp emulator of tests/emu against the oracle, and the argument validation and host fallback of
madrl_b200.postproc."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import postproc_edges as pe
from emu import driver
from emu.driver import needs_cxx
from emu.driver import ptr as _p
from oracle import baseline_oracle as bo
from oracle import concurrent_baseline_oracle as cbo
from oracle import postproc_oracle as po

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "linear_baseline_concurrent_ref.npz")
CASES = ("ragged", "beyond_clip")
FLAVOURS = ("independent", "shared")


def _golden():
    return np.load(GOLDEN)


def _case(z, name):
    its = []
    n = 0
    while "%s/it%d/obs" % (name, n) in z.files:
        its.append({k: z["%s/it%d/%s" % (name, n, k)] for k in ("obs", "obs_before", "done", "rew")})
        n += 1
    d, gl, center, positive = z[name + "/settings"]
    return its, dict(discount=float(d), gae_lambda=float(gl), center_adv=bool(center), positive_adv=bool(positive))


def _close(got, want, rel=1e-10):
    return np.abs(got - want).max() <= rel * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("name", CASES)
def test_oracle_agent_features_bit_identical_to_reference(name):
    z = _golden()
    its, _ = _case(z, name)
    rows, _ = cbo.agent_path_rows(its[0]["done"])
    for n, it in enumerate(its):
        F = cbo.agent_features(it["obs"], it["done"], it["obs_before"])
        rows, _ = cbo.agent_path_rows(it["done"])
        for a in range(F.shape[0]):
            assert np.array_equal(F[a][rows], z["%s/it%d/featmat%d" % (name, n, a)])


@pytest.mark.parametrize("flavour", FLAVOURS)
@pytest.mark.parametrize("name", CASES)
def test_oracle_chain_matches_reference(name, flavour):
    """Two iterations: coefficients and predictions within 1e-10 relative of the real rllab baseline; the
    per-agent returns, processed advantages and explained variances of the real discount_cumsum /
    center_advantages / shift_advantages_to_positive / explained_variance_1d."""
    z = _golden()
    its, st = _case(z, name)
    res = cbo.concurrent_chain(its, flavour == "shared", **st)
    for n, (it, r) in enumerate(zip(its, res)):
        rows, _ = cbo.agent_path_rows(it["done"])
        key = "%s/%s/it%d/" % (name, flavour, n)
        assert _close(r["coeffs_fit"], z[key + "coeffs"])
        A = it["obs"].shape[2]
        for a in range(A):
            assert _close(r["values"][:, :, a].reshape(-1)[rows], z[key + "pred%d" % a])
            assert _close(r["returns"][:, :, a].reshape(-1)[rows], z[key + "ret%d" % a], 1e-12)
            assert _close(r["advantages"][:, :, a].reshape(-1)[rows], z[key + "adv%d" % a], 1e-8)
        assert np.abs(r["ev"] - z[key + "ev"]).max() <= 1e-8


@pytest.mark.parametrize("name", CASES)
def test_shared_flavour_agent0_uses_previous_last_agent_fit(name):
    """The runner's single object: agent 0 is predicted with zeros in iteration 1 and with iteration 1's fit on
    agent A-1 in iteration 2; agent a >= 1 with the fit just made on agent a-1."""
    z = _golden()
    its, _ = _case(z, name)
    A = its[0]["obs"].shape[2]
    assert not np.any(z["%s/shared/it0/pred0" % name])
    c0 = z["%s/shared/it0/coeffs" % name]
    F = z["%s/it1/featmat0" % name]
    assert _close(z["%s/shared/it1/pred0" % name], F.dot(c0[A - 1]))
    c1 = z["%s/shared/it1/coeffs" % name]
    for a in range(1, A):
        assert _close(z["%s/shared/it1/pred%d" % (name, a)], z["%s/it1/featmat%d" % (name, a)].dot(c1[a - 1]))
    # the independent flavour differs from it (the quirk is visible in the data)
    assert not np.allclose(z["%s/shared/it1/pred1" % name], z["%s/independent/it1/pred1" % name])


def test_golden_cases_cover_agents_ragged_paths_constants_and_clipping():
    z = _golden()
    its, _ = _case(z, "ragged")
    assert its[0]["obs"].shape[2] >= 3 and its[0]["obs_before"] is not None
    _, lens = cbo.agent_path_rows(its[0]["done"])
    assert len(set(lens.tolist())) >= 4
    F1 = z["ragged/it0/featmat1"]
    assert np.linalg.matrix_rank(F1.T.dot(F1)) < F1.shape[1]
    b, _ = _case(z, "beyond_clip")
    assert b[0]["obs"].shape[2] >= 3 and np.abs(b[0]["obs"]).max() > 20
    assert np.abs(z["beyond_clip/it0/featmat0"][:, :3]).max() == 10.0


# ---------------------------------------------------------------- the kernels in the warp emulator

@pytest.fixture(scope="module")
def lib():
    return driver.load(())


def _run(lib, obs, obs_before, done, ret, t0, coef, bf16, per_agent):
    T, E, A, D = obs.shape
    seg_s = driver.paths_plan(lib, done, A)[0]
    nbytes = C.c_size_t()
    if per_agent:
        assert lib.madrl_lfb_agents_workspace_size(D, A, C.byref(nbytes)) == 0
    else:
        assert lib.madrl_lfb_workspace_size(D, C.byref(nbytes)) == 0
    ws = np.empty(nbytes.value // 8)
    G = np.full(((A,) if per_agent else ()) + (2 * D + 5, 2 * D + 5), np.nan)
    vals = np.full((T, E, A), np.nan, np.float32)
    sfx = ("agents_" if per_agent else "") + ("bf16" if bf16 else "f32")
    assert getattr(lib, "madrl_lfb_normal_eq_" + sfx)(T, E, A, D, _p(obs), _p(obs_before), _p(seg_s), _p(t0), _p(ret),
                                                      _p(G), _p(ws), None) == 0
    assert getattr(lib, "madrl_lfb_predict_" + sfx)(T, E, A, D, _p(obs), _p(obs_before), _p(seg_s), _p(t0), _p(coef),
                                                    _p(vals), None) == 0
    return G, vals


EMU_SHAPES = [  # T, E, A, D, p_done, obs_before, t0
    (9, 3, 3, 7, 0.25, True, True),
    (11, 2, 5, 5, 0.3, False, False),
    (5, 2, 3, 70, 0.2, True, True),        # 145 columns: three tiles, pairs off the diagonal
    (13, 2, 20, 3, 0.15, True, False),     # 20 agents: 3 slices per agent (1 in this 3-slice build)
    (6, 2, 3, 30, 0.2, True, True),        # 65 columns: y alone in the second tile
    (5, 3, 4, 31, 0.25, False, True),      # 67 columns: the time, constant and return columns cross the tile edge
]


@needs_cxx
@pytest.mark.parametrize("shape", EMU_SHAPES, ids=lambda s: "T%dE%dA%dD%d%s%s" % (s[:4] + ("_before" if s[5] else "",
                                                                                          "_t0" if s[6] else "")))
def test_emulated_agent_kernels_match_oracle(lib, shape):
    T, E, A, D, p_done, with_before, with_t0 = shape
    rs = np.random.RandomState(D + 11 * A)
    obs = (rs.randn(T, E, A, D) * 6).astype(np.float32)
    obs[:, :, 1, 0] = 0.0                                                # a constant column on agent 1
    obs_before = (rs.randn(E, A, D) * 6).astype(np.float32) if with_before else None
    done = (rs.rand(T, E) < p_done).astype(np.uint8)
    done[T // 2, 0] = 1
    ret = rs.randn(T, E, A).astype(np.float32)
    t0 = rs.randint(0, 300, size=E).astype(np.int32) if with_t0 else None
    coef = rs.randn(A, 2 * D + 4)
    driver.races()
    G, vals = _run(lib, obs, obs_before, done, ret, t0, coef, False, True)
    F = cbo.agent_features(obs, done, obs_before, t0)
    for a in range(A):
        G_ref = bo.normal_equations(F[a], ret[:, :, a].reshape(-1))
        bound = 1e-12 * np.sqrt(np.outer(np.diag(G_ref), np.diag(G_ref)))
        assert np.all(np.abs(G[a] - G_ref) <= bound), (a, np.abs(G[a] - G_ref).max())
        assert np.array_equal(G[a], G[a].T)
        want = F[a].dot(coef[a])
        tol = np.spacing(np.abs(want.astype(np.float32))) + 1e-12 * np.abs(F[a] * coef[a]).sum(axis=1)
        assert np.all(np.abs(vals[:, :, a].reshape(-1).astype(np.float64) - want) <= tol)
    # bfloat16 observations: the call on the widened float32 input, bit for bit
    o, o_w = pe.bf16_bits(obs)
    ob, ob_w = pe.bf16_bits(obs_before) if with_before else (None, None)
    for x, y in zip(_run(lib, o, ob, done, ret, t0, coef, True, True), _run(lib, o_w, ob_w, done, ret, t0, coef,
                                                                            False, True)):
        assert np.array_equal(x, y)
    assert driver.races() == 0


@needs_cxx
@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
def test_emulated_one_agent_equals_pooled_bitwise(lib, bf16):
    rs = np.random.RandomState(5)
    T, E, D = 37, 3, 9
    obs = (rs.randn(T, E, 1, D) * 6).astype(np.float32)
    obs_before = (rs.randn(E, 1, D) * 6).astype(np.float32)
    if bf16:
        obs, obs_before = pe.bf16_bits(obs)[0], pe.bf16_bits(obs_before)[0]
    done = (rs.rand(T, E) < 0.2).astype(np.uint8)
    ret = rs.randn(T, E, 1).astype(np.float32)
    t0 = rs.randint(0, 50, size=E).astype(np.int32)
    coef = rs.randn(1, 2 * D + 4)
    nb1, nbA = C.c_size_t(), C.c_size_t()
    assert lib.madrl_lfb_workspace_size(D, C.byref(nb1)) == 0
    assert lib.madrl_lfb_agents_workspace_size(D, 1, C.byref(nbA)) == 0
    assert nb1.value == nbA.value
    Gp, vp = _run(lib, obs, obs_before, done, ret, t0, coef[0], bf16, False)
    Ga, va = _run(lib, obs, obs_before, done, ret, t0, coef, bf16, True)
    assert np.array_equal(Ga[0], Gp) and np.array_equal(va, vp)
    adv = (rs.randn(T, E, 1) * 3 + 1).astype(np.float32)
    stats_p, stats_a = np.empty(9), np.empty((1, 9))
    ws = np.empty(4096)
    assert lib.madrl_moments_f32(adv.size, _p(adv), _p(ret), _p(stats_p), _p(ws), None) == 0
    assert lib.madrl_moments_agents_f32(adv.size, 1, _p(adv), _p(ret), _p(stats_a), _p(ws), None) == 0
    assert np.array_equal(stats_a[0], stats_p)
    for center, positive in ((1, 0), (1, 1), (0, 1)):
        x_p, x_a = adv.copy(), adv.copy()
        assert lib.madrl_center_advantages_f32(x_p.size, _p(x_p), center, positive, _p(stats_p), _p(ws), None) == 0
        assert lib.madrl_center_advantages_agents_f32(x_a.size, 1, _p(x_a), center, positive, _p(stats_a), _p(ws),
                                                      None) == 0
        assert np.array_equal(x_a, x_p)
    assert driver.races() == 0


@needs_cxx
@pytest.mark.parametrize("A", [1, 3, 7])
def test_emulated_agent_moments_and_centring(lib, A):
    rs = np.random.RandomState(A)
    rows = 997
    a = (rs.randn(rows, A) * np.arange(1, A + 1) + np.arange(A) * 3).astype(np.float32)
    b = (a + rs.randn(rows, A)).astype(np.float32)
    stats, ws = np.empty((A, 9)), np.empty(4096 * A)
    driver.races()
    assert lib.madrl_moments_agents_f32(rows, A, _p(a), _p(b), _p(stats), _p(ws), None) == 0
    for c in range(A):
        s = [a[:, c].astype(np.float64), b[:, c].astype(np.float64)]
        s.append(s[1] - s[0])
        want = [x.mean() for x in s] + [x.var() for x in s] + [x.min() for x in s]
        assert np.allclose(stats[c], want, rtol=1e-12, atol=1e-12)
        ev = po.explained_variance_1d(s[0], s[1])
        got = 1 - stats[c, 5] / (stats[c, 4] + 1e-8)
        assert abs(got - ev) <= 1e-12
    for center, positive in ((1, 0), (1, 1), (0, 1)):
        x = a.copy()
        assert lib.madrl_center_advantages_agents_f32(rows, A, _p(x), center, positive, _p(stats), _p(ws), None) == 0
        for c in range(A):
            want = a[:, c].astype(np.float64)
            if center:
                want = po.center_advantages(want)
            if positive:
                want = po.shift_advantages_to_positive(want)
            assert np.all(np.abs(x[:, c] - want) <= np.spacing(np.abs(want).astype(np.float32)) + 1e-12), c
    assert driver.races() == 0


@needs_cxx
def test_emulated_agent_workspace_and_bad_sizes(lib):
    nbytes = C.c_size_t()
    assert lib.madrl_lfb_agents_workspace_size(213, 5, C.byref(nbytes)) == 0
    assert nbytes.value == 5 * 1 * 28 * 64 * 64 * 8                    # emulator build: 3 slices -> 1 per agent
    assert lib.madrl_lfb_agents_workspace_size(213, 2, C.byref(nbytes)) == 0
    assert nbytes.value == 2 * 2 * 28 * 64 * 64 * 8
    assert lib.madrl_lfb_agents_workspace_size(213, 0, C.byref(nbytes)) != 0
    assert lib.madrl_lfb_agents_workspace_size(213, 64, C.byref(nbytes)) == 0       # at least 64 agents
    assert lib.madrl_lfb_agents_workspace_size(213, 1025, C.byref(nbytes)) != 0
    assert lib.madrl_lfb_agents_workspace_size(0, 3, C.byref(nbytes)) != 0
    assert lib.madrl_lfb_agents_workspace_size(8193, 3, C.byref(nbytes)) != 0
    x = np.zeros(64, np.float32)
    seg = np.zeros(4, np.int32)
    f = lib.madrl_lfb_normal_eq_agents_f32
    assert f(1, 1, 1025, 4, _p(x), None, _p(seg), None, _p(x), _p(x), _p(x), None) != 0
    assert f(1, 1, 0, 4, _p(x), None, _p(seg), None, _p(x), _p(x), _p(x), None) != 0
    assert f(1, 1, 2, 0, _p(x), None, _p(seg), None, _p(x), _p(x), _p(x), None) != 0
    assert f(1 << 16, 1 << 10, 32, 4, _p(x), None, _p(seg), None, _p(x), _p(x), _p(x), None) != 0   # T*E*A = 2^31
    assert f(1, 1, 2, 4, _p(x), None, _p(seg), None, _p(x), None, _p(x), None) != 0                # NULL G
    p = lib.madrl_lfb_predict_agents_f32
    assert p(1, 1, 1025, 4, _p(x), None, _p(seg), None, _p(x), _p(x), None) != 0
    assert p(1, 1, 2, 4, _p(x), None, _p(seg), None, None, _p(x), None) != 0                       # NULL coef
    s = np.zeros(9 * 4)
    assert lib.madrl_moments_agents_f32(0, 2, _p(x), None, _p(s), _p(s), None) != 0
    assert lib.madrl_moments_agents_f32(4, 0, _p(x), None, _p(s), _p(s), None) != 0
    assert lib.madrl_moments_agents_f32(4, 1025, _p(x), None, _p(s), _p(s), None) != 0
    assert lib.madrl_moments_agents_f32(4, 2, None, None, _p(s), _p(s), None) != 0
    assert lib.madrl_center_advantages_agents_f32(4, 2, _p(x), 1, 0, None, _p(s), None) != 0
    assert lib.madrl_center_advantages_agents_f32(4, 1025, _p(x), 1, 0, _p(s), _p(s), None) != 0


# ---------------------------------------------------------------- argument validation (no library call)

@pytest.fixture
def no_library(monkeypatch):
    from madrl_b200 import _lib

    def refuse():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_validation_raises_before_any_library_call(no_library):
    from madrl_b200.postproc import (LinearFeatureBaseline, center_advantages, explained_variance,
                                     process_samples_concurrent)
    with pytest.raises(ValueError):
        LinearFeatureBaseline(5, "cuda:0", shared=True)                   # shared needs n_agents
    with pytest.raises(ValueError):
        LinearFeatureBaseline(5, "cuda:0", n_agents=0)
    with pytest.raises(ValueError):
        LinearFeatureBaseline(5, "cuda:0", n_agents=1025)
    T, E, A, D = 4, 3, 3, 5
    b = LinearFeatureBaseline(D, "cpu", n_agents=A)
    obs = torch.zeros((T, E, A + 1, D))
    done = torch.zeros((T, E), dtype=torch.uint8)
    with pytest.raises(ValueError):
        b.predict(obs, done)                                               # 4 agents, built for 3
    with pytest.raises(ValueError):
        b.fit(obs, done, torch.zeros((T, E, A + 1)))
    with pytest.raises(ValueError):
        b.set_param_values(np.zeros(2 * D + 4))                            # [Df], not [A, Df]
    with pytest.raises(ValueError):
        b.set_param_values(np.zeros((A, 2 * D + 4)), carry=np.zeros(2 * D + 4))   # carry only when shared
    with pytest.raises(TypeError):
        b.set_param_values(torch.zeros((A, 2 * D + 4), dtype=torch.float32))
    bs = LinearFeatureBaseline(D, "cpu", n_agents=A, shared=True)
    with pytest.raises(ValueError):
        process_samples_concurrent(bs, obs, done, torch.zeros((T, E, A + 1)), 0.99, 0.97)
    with pytest.raises(ValueError):
        process_samples_concurrent(LinearFeatureBaseline(D, "cpu"), obs[:, :, :A], done, torch.zeros((T, E, A)),
                                   0.99, 0.97)                             # a pooled baseline
    with pytest.raises(ValueError):
        process_samples_concurrent(bs, obs[:, :, :A], done, torch.zeros((T, E, A + 1)), 0.99, 0.97)
    with pytest.raises(TypeError):
        center_advantages(torch.zeros((T, E, A), dtype=torch.float64), per_agent=True)
    with pytest.raises(ValueError):
        center_advantages(torch.zeros((T, E, 0)), per_agent=True)
    with pytest.raises(ValueError):
        center_advantages(torch.zeros((2, 1025)), per_agent=True)
    with pytest.raises(ValueError):
        explained_variance(torch.zeros((T, E, A)), torch.zeros((T, E, A + 1)), per_agent=True)


def test_param_values_round_trip_per_agent(no_library):
    from madrl_b200.postproc import LinearFeatureBaseline
    b = LinearFeatureBaseline(3, "cpu", n_agents=4, shared=True)
    c = np.arange(40, dtype=np.float64).reshape(4, 10)
    assert b.get_param_values() is None and b.carry is None
    b.set_param_values(c, carry=np.ones(10))
    assert np.array_equal(b.get_param_values(), c) and np.array_equal(b.carry, np.ones(10))
    b.set_param_values(None)
    assert b.get_param_values() is None and b.carry is None


def test_batched_solve_falls_back_per_agent():
    """A stack where agent 1's system is not positive definite: agent 1 takes rllab's host lstsq loop, agents 0 and
    2 keep their Cholesky solutions (equal to the single-system solve)."""
    from madrl_b200.postproc import LinearFeatureBaseline
    z = _golden()
    its, _ = _case(z, "ragged")
    it = its[0]
    F = cbo.agent_features(it["obs"], it["done"], it["obs_before"])
    rows, _ = cbo.agent_path_rows(it["done"])
    A, Df = F.shape[0], F.shape[2]
    y = it["rew"].astype(np.float64).reshape(-1, A).T                       # any right-hand side
    G = np.stack([bo.normal_equations(F[a][rows], y[a][rows]) for a in range(A)])
    G[1, :Df, :Df] = -np.identity(Df)
    G[1, :Df, Df] = G[1, Df, :Df] = np.arange(Df)
    b = LinearFeatureBaseline(it["obs"].shape[3], "cpu", n_agents=A)
    c = b.solve(torch.from_numpy(G)).numpy()
    want1 = np.linalg.lstsq(-np.identity(Df) + 1e-5 * np.identity(Df), np.arange(Df, dtype=np.float64),
                            rcond=None)[0]
    assert np.array_equal(c[1], want1)
    pooled = LinearFeatureBaseline(it["obs"].shape[3], "cpu")
    for a in (0, 2):
        single = pooled.solve(torch.from_numpy(G[a])).numpy()
        assert np.allclose(c[a], single, rtol=1e-9, atol=1e-9 * np.abs(single).max())
        Fa, ya = F[a][rows], y[a][rows]
        assert bo.objective(Fa, ya, c[a]) <= bo.objective(Fa, ya, bo.fit(Fa, ya)) * (1 + 1e-8)
