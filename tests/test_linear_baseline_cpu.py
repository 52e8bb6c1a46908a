"""LinearFeatureBaseline without a GPU: the oracle (oracle/baseline_oracle.py) against the real rllab class
(tests/golden/linear_baseline_ref.npz, written by oracle/make_baseline_golden.py), the madrl_lfb_* kernels of
csrc/baseline.cu executed by the warp emulator of tests/emu against the oracle, and the argument validation of
madrl_b200.postproc.LinearFeatureBaseline."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import postproc_edges as pe
from emu import build_emu, driver
from emu.driver import needs_cxx
from emu.driver import ptr as _p
from oracle import baseline_oracle as bo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "linear_baseline_ref.npz")
CASES = ("ragged", "rank_deficient", "beyond_clip")


def _case(name):
    z = np.load(GOLDEN)
    get = lambda k: z[name + "/" + k] if name + "/" + k in z.files else None   # noqa: E731
    return {k: get(k) for k in ("obs", "obs_before", "done", "returns", "featmat", "coeffs", "pred")}


@pytest.mark.parametrize("name", CASES)
def test_oracle_matches_reference_golden(name):
    """Features bit-identical to the reference's _features (in path order); normal equations bit-identical when
    formed the same way from them (one BLAS call on identical inputs); coefficients and predictions within
    1e-10 relative (LAPACK gelsd, so not bitwise across BLAS builds)."""
    c = _case(name)
    A = c["obs"].shape[2]
    F = bo.features(c["obs"], c["done"], c["obs_before"])
    rows, _ = bo.path_rows(c["done"], A)
    Fp, yp = F[rows], c["returns"].reshape(-1)[rows].astype(np.float64)
    assert Fp.dtype == np.float64 and np.array_equal(Fp, c["featmat"])
    G = bo.normal_equations(Fp, yp)
    ref = c["featmat"]
    assert np.array_equal(G[:-1, :-1], ref.T.dot(ref))
    assert np.array_equal(G[:-1, -1], ref.T.dot(yp)) and G[-1, -1] == yp.dot(yp)
    coef = bo.fit(Fp, yp)
    assert np.abs(coef - c["coeffs"]).max() <= 1e-10 * np.abs(c["coeffs"]).max()
    pred = F.dot(coef)[rows]
    assert np.abs(pred - c["pred"]).max() <= 1e-10 * max(1.0, np.abs(c["pred"]).max())


def test_golden_cases_cover_clipping_and_rank_deficiency():
    c = _case("beyond_clip")
    assert np.abs(c["obs"]).max() > 20 and np.abs(c["featmat"][:, :4]).max() == 10.0
    r = _case("rank_deficient")
    F = r["featmat"]
    assert np.linalg.matrix_rank(F.T.dot(F)) < F.shape[1]
    rg = _case("ragged")
    _, lens = bo.path_rows(rg["done"], rg["obs"].shape[2])
    assert len(set(lens.tolist())) >= 4


def test_chained_launches_with_t0_equal_one_long_launch():
    """t0 = the env's path length before the launch continues the time index of a path begun earlier."""
    rs = np.random.RandomState(3)
    T, E, A, D = 30, 4, 2, 3
    obs = rs.randn(T, E, A, D).astype(np.float32)
    obs0 = rs.randn(E, A, D).astype(np.float32)
    done = (rs.rand(T, E) < 0.1).astype(np.uint8)
    long = bo.features(obs, done, obs0)
    h = 13
    first = bo.features(obs[:h], done[:h], obs0)
    path_len = bo.time_index(done[:h])[-1] + 1
    path_len[done[h - 1].astype(bool)] = 0
    second = bo.features(obs[h:], done[h:], obs[h - 1], t0=path_len)
    assert np.array_equal(np.concatenate([first, second]), long)


# ---------------------------------------------------------------- the kernels in the warp emulator

@pytest.fixture(scope="module")
def lib():
    return driver.load(())


def _run(lib, obs, obs_before, done, ret, t0, coef, bf16):
    T, E, A, D = obs.shape
    seg_s = driver.paths_plan(lib, done, A)[0]
    nbytes = C.c_size_t()
    assert lib.madrl_lfb_workspace_size(D, C.byref(nbytes)) == 0
    ws = np.empty(nbytes.value // 8)
    G = np.full((2 * D + 5, 2 * D + 5), np.nan)
    vals = np.full((T, E, A), np.nan, np.float32)
    dt = "bf16" if bf16 else "f32"
    assert getattr(lib, "madrl_lfb_normal_eq_" + dt)(T, E, A, D, _p(obs), _p(obs_before), _p(seg_s), _p(t0), _p(ret),
                                                     _p(G), _p(ws), None) == 0
    assert getattr(lib, "madrl_lfb_predict_" + dt)(T, E, A, D, _p(obs), _p(obs_before), _p(seg_s), _p(t0), _p(coef),
                                                   _p(vals), None) == 0
    return G, vals


EMU_SHAPES = [  # T, E, A, D, p_done, obs_before, t0
    (9, 3, 2, 7, 0.25, True, True),
    (11, 2, 3, 5, 0.3, False, False),
    (6, 2, 3, 213, 0.2, True, True),
    (40, 3, 1, 1, 0.15, False, True),
    (7, 3, 2, 30, 0.25, True, True),       # 65 columns: y alone in the second tile
    (5, 2, 3, 31, 0.3, False, True),       # 67 columns: the time, constant and return columns cross the tile edge
]


@needs_cxx
@pytest.mark.parametrize("shape", EMU_SHAPES, ids=lambda s: "T%dE%dA%dD%d%s%s" % (s[:4] + ("_before" if s[5] else "",
                                                                                          "_t0" if s[6] else "")))
def test_emulated_kernels_match_oracle(lib, shape):
    T, E, A, D, p_done, with_before, with_t0 = shape
    rs = np.random.RandomState(D + 7 * T)
    obs = (rs.randn(T, E, A, D) * 6).astype(np.float32)               # |o| > 10 on some entries
    obs_before = (rs.randn(E, A, D) * 6).astype(np.float32) if with_before else None
    done = (rs.rand(T, E) < p_done).astype(np.uint8)
    done[T // 2, 0] = done[T // 2 + 2, 0] = 1                           # several paths in env 0
    ret = rs.randn(T, E, A).astype(np.float32)
    t0 = rs.randint(0, 300, size=E).astype(np.int32) if with_t0 else None
    coef = rs.randn(2 * D + 4)
    driver.races()
    results = {}
    for bf16 in (False, True):
        if bf16:
            o, o_w = pe.bf16_bits(obs)
            ob, ob_w = pe.bf16_bits(obs_before) if with_before else (None, None)
            results["bf16"] = _run(lib, o, ob, done, ret, t0, coef, True)
            results["f32_widened"] = _run(lib, o_w, ob_w, done, ret, t0, coef, False)
            o_ref, ob_ref = o_w, ob_w
        else:
            results["f32"] = _run(lib, obs, obs_before, done, ret, t0, coef, False)
            o_ref, ob_ref = obs, obs_before
        F = bo.features(o_ref, done, ob_ref, t0)
        G_ref = bo.normal_equations(F, ret.reshape(-1))
        G, vals = results["bf16" if bf16 else "f32"]
        bound = 1e-12 * np.sqrt(np.outer(np.diag(G_ref), np.diag(G_ref)))
        assert np.all(np.abs(G - G_ref) <= bound), np.abs(G - G_ref).max()
        assert np.array_equal(G, G.T)
        want = F.dot(coef)
        tol = np.spacing(np.abs(want.astype(np.float32))) + 1e-12 * np.abs(F * coef).sum(axis=1)
        assert np.all(np.abs(vals.reshape(-1).astype(np.float64) - want) <= tol)
    for a, b in zip(results["bf16"], results["f32_widened"]):                 # bf16 == the call on obs.float()
        assert np.array_equal(a, b)
    assert driver.races() == 0


@needs_cxx
@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
def test_emulated_single_row_reads_out_the_exact_features(lib, bf16):
    """One row: G = outer(f, f) bit for bit, f = [clip(o), clip(o)^2, a, a^2, a^3, 1, y] with the correctly rounded
    a^3 (not NumPy's al ** 3, which is an ulp off at some of these indices), at the obs_dims whose time columns sit
    at a tile edge; predict with a unit coefficient on a time column returns that feature rounded to float32
    (tests/test_postproc_edges_gpu.py sweeps more obs_dims and indices on the device)."""
    rs = np.random.RandomState(3 + bf16)
    done = np.zeros((1, 1), np.uint8)
    driver.races()
    for D in (30, 31, 32):
        for before in (False, True):
            for k, t0 in enumerate((1, 99, 767, 50004)):
                o = pe.single_row_obs(D, k, bf16, rs)
                y = np.float32(rs.randn())
                f = pe.single_row_features(o, y, t0)
                row = (pe.bf16_bits(o)[0] if bf16 else o).reshape(1, 1, 1, D)
                obs, ob = (np.full_like(row, 0x7FC0 if bf16 else np.nan), row.reshape(1, 1, D)) if before else (row, None)
                for j in (2 * D, 2 * D + 1, 2 * D + 2):
                    G, vals = _run(lib, obs, ob, done, np.array([[[y]]], np.float32), np.array([t0], np.int32),
                                   np.eye(2 * D + 4)[j], bf16)
                    assert np.array_equal(G, np.outer(f, f)), (D, before, t0)
                    assert vals.item() == np.float32(f[j]), (D, before, t0, j)
    assert driver.races() == 0


@needs_cxx
def test_emulated_workspace_and_bad_sizes(lib):
    nbytes = C.c_size_t()
    assert lib.madrl_lfb_workspace_size(213, C.byref(nbytes)) == 0
    assert nbytes.value == build_emu.GRID["MADRL_LFB_SLICES"] * 28 * 64 * 64 * 8        # 431 columns -> 7 tiles
    assert lib.madrl_lfb_workspace_size(0, C.byref(nbytes)) != 0
    assert lib.madrl_lfb_workspace_size(8193, C.byref(nbytes)) != 0
    x = np.zeros(64, np.float32)
    seg = np.zeros(4, np.int32)
    assert lib.madrl_lfb_predict_f32(0, 1, 1, 4, _p(x), None, _p(seg), None, _p(x), _p(x), None) != 0
    assert lib.madrl_lfb_predict_f32(1, 1, 1, 4, _p(x), None, None, None, _p(x), _p(x), None) != 0
    assert lib.madrl_lfb_normal_eq_f32(1, 1, 1, 0, _p(x), None, _p(seg), None, _p(x), _p(x), _p(x), None) != 0


# ---------------------------------------------------------------- argument validation (no library call)

@pytest.fixture
def no_library(monkeypatch):
    from madrl_b200 import _lib

    def refuse():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "lib", refuse)


def test_validation_raises_before_any_library_call(no_library):
    from madrl_b200.postproc import LinearFeatureBaseline
    b = LinearFeatureBaseline(5, "cuda:0")
    T, E, A, D = 4, 3, 2, 5
    obs = torch.zeros((T, E, A, D))
    done = torch.zeros((T, E), dtype=torch.uint8)
    ret = torch.zeros((T, E, A))
    with pytest.raises(TypeError):
        b.predict(obs.double(), done)
    with pytest.raises(TypeError):
        b.predict(obs.half(), done)
    with pytest.raises(TypeError):
        b.predict(obs, done.bool())
    with pytest.raises(TypeError):
        b.fit(obs, done, ret.double())
    with pytest.raises(TypeError):
        b.predict(obs, done, obs_before=torch.zeros((E, A, D), dtype=torch.bfloat16))
    with pytest.raises(TypeError):
        b.predict(obs, done, t0=torch.zeros(E, dtype=torch.int64))
    with pytest.raises(TypeError):
        b.predict(obs.numpy(), done)
    with pytest.raises(ValueError):
        b.predict(obs.reshape(T, E, A * D), done)                        # not [T,E,A,D]
    with pytest.raises(ValueError):
        b.predict(torch.zeros((T, E, A, D + 1)), done)                   # wrong obs_dim
    with pytest.raises(ValueError):
        b.predict(obs, done[:-1])
    with pytest.raises(ValueError):
        b.fit(obs, done, ret[:, :, :1])
    with pytest.raises(ValueError):
        b.predict(obs, done, obs_before=torch.zeros((E, A, D + 1)))
    with pytest.raises(ValueError):
        b.predict(obs, done, t0=torch.zeros(E + 1, dtype=torch.int32))
    with pytest.raises(ValueError):
        b.predict(obs, done)                                               # host tensors, device baseline
    with pytest.raises(ValueError):
        b.set_param_values(np.zeros(2 * D + 3))
    with pytest.raises(TypeError):
        b.set_param_values(torch.zeros(2 * D + 4, dtype=torch.float32))
    assert b.get_param_values() is None


def test_param_values_round_trip_on_host(no_library):
    from madrl_b200.postproc import LinearFeatureBaseline
    b = LinearFeatureBaseline(3, "cpu")
    c = np.arange(10, dtype=np.float64)
    b.set_param_values(c)
    assert np.array_equal(b.get_param_values(), c) and b.get_param_values().dtype == np.float64
    b.set_param_values(None)
    assert b.get_param_values() is None


def test_host_solve_fallback_follows_rllab_retry():
    """`solve` on a well-posed system minimises rllab's objective as the oracle's fit does; on normal equations
    whose Cholesky factorisation fails (not positive definite) it takes rllab's host lstsq."""
    from madrl_b200.postproc import LinearFeatureBaseline
    c = _case("ragged")
    F = bo.features(c["obs"], c["done"], c["obs_before"])
    y = c["returns"].reshape(-1)
    b = LinearFeatureBaseline(c["obs"].shape[3], "cpu")
    got = b.solve(torch.from_numpy(bo.normal_equations(F, y))).numpy()
    want = bo.fit(F, y)
    assert bo.objective(F, y, got) <= bo.objective(F, y, want) * (1 + 1e-8)
    Df = F.shape[1]
    G = torch.zeros((Df + 1, Df + 1), dtype=torch.float64)
    G[:Df, :Df] = -torch.eye(Df, dtype=torch.float64)
    G[:Df, Df] = torch.arange(Df, dtype=torch.float64)
    want = np.linalg.lstsq(-np.identity(Df) + 1e-5 * np.identity(Df), np.arange(Df, dtype=np.float64), rcond=None)[0]
    assert np.array_equal(b.solve(G).numpy(), want)
