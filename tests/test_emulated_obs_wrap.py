"""The closed loop's per-step observation wrapper (madrl_obs_wrap_step_*, csrc/postproc.cu) in the warp emulator of
tests/emu: T single-step calls against the whole-trajectory passes it fuses (madrl_standardize_obs_terminal_* then
madrl_frame_stack_*), bit for bit, and against StandardizedEnv / ObservationBuffer of oracle/postproc_oracle.py;
then every argument error."""
import numpy as np
import pytest

import postproc_edges as pe
from emu import driver
from emu.driver import Guarded
from emu.driver import ptr as _p

pytestmark = driver.needs_cxx

ALPHA, EPS = 0.05, 1e-8
E, A, D, T = 37, 3, 29, 6          # E*A*D = 3219 elements: 13 blocks of 256 threads, the last one partial


@pytest.fixture(scope="module")
def lib():
    return driver.load(())


def _case(bf16, seed=11):
    """Reset observations, T steps of observations and terminal observations, and done per env:
    e % 5 == 0 never, 1 at t = 0 only, 2 on every step, 3 at random, 4 at t = T - 1."""
    rs = np.random.RandomState(seed)
    cvt = (lambda x: pe.bf16_bits(x)[1]) if bf16 else (lambda x: x)            # noqa: E731
    obs0 = cvt((rs.randn(E, A, D) * 2 + 0.5).astype(np.float32))
    obs = cvt((rs.randn(T, E, A, D) * 2 + 0.5).astype(np.float32))
    term = cvt((rs.randn(T, E, A, D) * 3 - 1).astype(np.float32))
    done = np.zeros((T, E), np.uint8)
    done[0, 1::5] = 1
    done[:, 2::5] = 1
    done[:, 3::5] = rs.rand(T, len(range(3, E, 5))) < 0.3
    done[T - 1, 4::5] = 1
    mean = rs.randn(E, A, D) * 0.1
    var = 1 + rs.rand(E, A, D)
    return obs0, obs, term, done, mean, var


def _enc(bf16):
    return (lambda v: pe.bf16_bits(v)[0]) if bf16 else (lambda v: np.array(v, np.float32))   # noqa: E731


def _dec(bf16):
    return (lambda v: (v.astype(np.uint32) << 16).view(np.float32)) if bf16 else np.copy     # noqa: E731


def fused(lib, bf16, B, obsnorm, obs0, obs, term, done, mean, var):
    """T calls of madrl_obs_wrap_step_*: -> (obs, term, stacks [T,E,A,D,B], mean, var) as stored (bf16 bits)."""
    enc = _enc(bf16)
    dt = np.uint16 if bf16 else np.float32
    fn = lib.madrl_obs_wrap_step_bf16 if bf16 else lib.madrl_obs_wrap_step_f32
    m = Guarded((E, A, D), np.float64, mean) if obsnorm else None
    v = Guarded((E, A, D), np.float64, var) if obsnorm else None
    prev = np.ascontiguousarray(np.repeat(enc(obs0)[..., None], B, axis=-1))
    xs, ts, outs = [], [], []
    for t in range(T):
        x = Guarded((E, A, D), dt, enc(obs[t]))
        tm = Guarded((E, A, D), dt, enc(term[t]))
        out = Guarded((E, A, D, B), dt, 0)
        dn = np.ascontiguousarray(done[t])
        assert fn(E, A, D, B, _p(x.arr), _p(tm.arr) if obsnorm else None, _p(dn), _p(prev), _p(out.arr),
                  _p(m.arr) if obsnorm else None, _p(v.arr) if obsnorm else None, ALPHA, EPS, None) == 0
        xs.append(x.check("obs").copy())
        ts.append(tm.check("term").copy())
        prev = out.check("out").copy()
        outs.append(prev)
    return (np.stack(xs), np.stack(ts), np.stack(outs), m.check("mean") if obsnorm else None,
            v.check("var") if obsnorm else None)


def composed(lib, bf16, B, obsnorm, obs0, obs, term, done, mean, var):
    """The same steps through the whole-trajectory passes: standardize_obs_terminal over T, then frame_stack."""
    enc = _enc(bf16)
    sfx = "bf16" if bf16 else "f32"
    x, tm = np.ascontiguousarray(enc(obs)), np.ascontiguousarray(enc(term))
    m, v = mean.copy(), var.copy()
    if obsnorm:
        assert getattr(lib, "madrl_standardize_obs_terminal_" + sfx)(T, E, A * D, _p(x), _p(tm), _p(done), _p(m),
                                                                    _p(v), ALPHA, EPS, None) == 0
    carry = np.ascontiguousarray(np.repeat(enc(obs0)[..., None], B, axis=-1))
    out = np.empty((T, E, A, D, B), x.dtype)
    assert getattr(lib, "madrl_frame_stack_" + sfx)(T, E, A, D, B, _p(x), _p(done), _p(carry), _p(out), None) == 0
    return x, tm, out, m if obsnorm else None, v if obsnorm else None


@pytest.mark.parametrize("obsnorm", [False, True], ids=["stack", "obsnorm"])
@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
def test_single_steps_equal_the_whole_trajectory_passes(lib, bf16, obsnorm):
    """Every B in 1..8: observations, terminal observations, stacks and running estimates bit for bit; without
    obsnorm the observations and terminal observations are left as they are."""
    case = _case(bf16)
    enc = _enc(bf16)
    for B in range(1, 9):
        got = fused(lib, bf16, B, obsnorm, *case)
        want = composed(lib, bf16, B, obsnorm, *case)
        for name, g, w in zip(("obs", "term", "out", "mean", "var"), got, want):
            assert (g is None) == (w is None) and (g is None or np.array_equal(g.view(np.uint8), w.view(np.uint8))), \
                (B, name)
        if not obsnorm:
            assert np.array_equal(got[0], enc(case[1])) and np.array_equal(got[1], enc(case[2]))
        assert case[3].any(0).any() and not case[3].all(0).all()


@pytest.mark.parametrize("obsnorm", [False, True], ids=["stack", "obsnorm"])
def test_single_steps_follow_the_reference_wrappers(lib, obsnorm):
    """StandardizedEnv (terminal observation first at a done step) within a float32 ulp of its float64 values, and
    ObservationBuffer over the standardised observations exactly."""
    obs0, obs, term, done, mean, var = _case(False)
    B = 4
    x, tm, out, m, _ = fused(lib, False, B, obsnorm, obs0, obs, term, done, np.zeros((E, A, D)), np.ones((E, A, D)))
    if obsnorm:
        # the oracle starts from zero mean / unit variance, as the reference does
        pe.check_terminal(x.reshape(T, E, -1), tm.reshape(T, E, -1), obs.reshape(T, E, -1), term.reshape(T, E, -1),
                          done, ALPHA, m.reshape(E, -1))
    else:
        assert np.array_equal(x, obs)
    pe.check_frame_stack(obs0, [(x, done)], [out], B)


def test_argument_errors(lib):
    """MADRL_EINVAL for every bad argument, and nothing written."""
    x = np.zeros((2, 2, 3), np.float32)
    tm, done = x.copy(), np.zeros(2, np.uint8)
    prev, out = np.zeros((2, 2, 3, 4), np.float32), Guarded((2, 2, 3, 4), np.float32, 5.0)
    m, v = np.zeros((2, 2, 3)), np.ones((2, 2, 3))
    good = dict(E=2, A=2, D=3, B=4, obs=x, term=tm, done=done, prev=prev, out=out.arr, mean=m, var=v)

    def call(fn, **kw):
        a = dict(good, **kw)
        return fn(a["E"], a["A"], a["D"], a["B"], _p(a["obs"]), _p(a["term"]), _p(a["done"]), _p(a["prev"]),
                  _p(a["out"]), _p(a["mean"]), _p(a["var"]), ALPHA, EPS, None)

    for fn in (lib.madrl_obs_wrap_step_f32, lib.madrl_obs_wrap_step_bf16):
        for bad in (dict(E=0), dict(A=0), dict(D=0), dict(E=-1), dict(B=0), dict(B=9), dict(mean=None),
                    dict(var=None), dict(term=None), dict(prev=None), dict(out=None), dict(obs=None),
                    dict(done=None)):
            assert call(fn, **bad) == -1, bad
            assert b"" != lib.madrl_last_error()
        assert np.all(out.check("out") == 5.0)
        assert np.all(m == 0) and np.all(v == 1)
    # accepted: no obsnorm at all (term then unused); B = 1 without prev / out
    assert call(lib.madrl_obs_wrap_step_f32, mean=None, var=None, term=None) == 0
    assert call(lib.madrl_obs_wrap_step_f32, B=1, prev=None, out=None) == 0
