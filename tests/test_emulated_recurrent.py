"""The padded-path kernels of the recurrent sample batch (madrl_paths_pad_u32 / _u16, madrl_path_sums_f32 in
madrl_b200/csrc/postproc.cu) executed on the CPU by the warp emulator of tests/emu and compared, through the C ABI,
with rllab's padding as oracle/recurrent_oracle.py restates it: wide and narrow rows, 4- and 2-byte words, odd
widths, with and without the one-step observation shift, per-env rows (A = 1), record tables in every control
mode's order and in a shuffled one, and P * L off the block size.  Every output sits in a canary-guarded buffer
pre-filled with non-zero words, so a padding word the kernel fails to write, or a write outside the buffer, fails."""
import ctypes as C
import os
import shutil

import numpy as np
import pytest

from emu.driver import Guarded
from oracle import recurrent_oracle as ro

pytestmark = pytest.mark.skipif(shutil.which(os.environ.get("CXX", "g++")) is None, reason="no host C++ compiler")


def _p(a):
    return C.c_void_p(a.ctypes.data) if a is not None else C.c_void_p(0)


@pytest.fixture(scope="module")
def lib():
    from emu import driver
    L = driver.load(())
    vp, i32 = C.c_void_p, C.c_int
    L.madrl_paths_pad_u32.argtypes = [i32] * 6 + [vp] * 5
    L.madrl_paths_pad_u16.argtypes = [i32] * 6 + [vp] * 5
    L.madrl_path_sums_f32.argtypes = [i32] * 4 + [vp] * 6
    return L


def episodes(done):
    """(env, start, length) of every episode in (env, episode) order (cut at done and at the end)."""
    T, E = done.shape
    out = []
    for e in range(E):
        ends = list(np.nonzero(done[:, e])[0] + 1)
        if not ends or ends[-1] != T:
            ends.append(T)
        s = 0
        for end in ends:
            out.append((e, s, end - s))
            s = end
    return out


def records(done, A, order, seed=0):
    """int32 [P, 4] record table: (env, episode, agent) order, agent-major, or a random permutation."""
    eps = episodes(done)
    if order == "agent_major":
        rec = [(e, a, s, L) for a in range(A) for e, s, L in eps]
    else:
        rec = [(e, a, s, L) for e, s, L in eps for a in range(A)]
    rec = np.array(rec, np.int32)
    if order == "shuffled":
        rec = rec[np.random.RandomState(seed).permutation(len(rec))]
    return np.ascontiguousarray(rec)


def padded_want(src, first, rec, Lmax, per_agent):
    """rllab's pad_tensor_n of each record's rows; src [T,E,A,D] ([T,E,D] per env), first [E,A,D] or None."""
    if first is not None:
        src = np.concatenate([first[None], src[:-1]])
    rows = [src[s:s + L, e, a] if per_agent else src[s:s + L, e] for e, a, s, L in rec]
    return ro.pad_tensor_n(rows, Lmax)


# (T, E, A, done probability): a tail of P * L off every block size; one-step episodes everywhere; T = 1
SHAPES = ((9, 5, 3, 0.25), (6, 7, 2, 1.0), (1, 11, 3, 0.0), (13, 3, 1, 0.3))
WORDS = (1, 2, 3, 4, 5, 33)        # one thread per row up to 4 words, one warp beyond; odd widths


@pytest.mark.parametrize("itemsize", [4, 2], ids=["u32", "u16"])
def test_padding_equals_rllab_pad_tensor_n(lib, itemsize):
    pad = lib.madrl_paths_pad_u32 if itemsize == 4 else lib.madrl_paths_pad_u16
    w = np.uint32 if itemsize == 4 else np.uint16
    fill = w(0x5A5A5A5A & (2 ** (8 * itemsize) - 1))
    for k, D in enumerate(WORDS):
        T, E, A, p_done = SHAPES[k % len(SHAPES)]
        rs = np.random.RandomState(100 + k)
        done = (rs.rand(T, E) < p_done).astype(np.uint8)
        src = rs.randint(1, 2 ** (8 * itemsize), size=(T, E, A, D), dtype=np.uint64).astype(w)
        first = rs.randint(1, 2 ** (8 * itemsize), size=(E, A, D), dtype=np.uint64).astype(w)
        env_rows = rs.randint(1, 2 ** (8 * itemsize), size=(T, E, D), dtype=np.uint64).astype(w)
        for order in ("env_major", "agent_major", "shuffled"):
            rec = records(done, A, order, seed=k)
            P = len(rec)
            Lmax = int(rec[:, 3].max())
            for shifted in (False, True):
                out = Guarded((P, Lmax, D), w, fill)
                assert pad(T, E, A, D, P, Lmax, _p(src), _p(first if shifted else None), _p(rec), _p(out.arr),
                           None) == 0
                got = out.check("padded")
                assert np.array_equal(got, padded_want(src, first if shifted else None, rec, Lmax, True)), \
                    (D, order, shifted)
            # per-env rows (A = 1): every agent's path reads its env's row, whatever its agent field
            out = Guarded((P, Lmax, D), w, fill)
            assert pad(T, E, 1, D, P, Lmax, _p(env_rows), None, _p(rec), _p(out.arr), None) == 0
            assert np.array_equal(out.check("padded infos"), padded_want(env_rows, None, rec, Lmax, False)), (D, order)


def test_padding_to_a_longer_length_than_any_path(lib):
    """Lmax beyond the longest path (a batch padded to a common length): the extra rows are zeros as well."""
    T, E, A, D = 5, 4, 2, 7
    rs = np.random.RandomState(3)
    done = np.zeros((T, E), np.uint8)
    done[1, 0] = done[3, 2] = 1
    src = rs.randn(T, E, A, D).astype(np.float32)
    rec = records(done, A, "env_major")
    for Lmax in (T, T + 3):
        out = Guarded((len(rec), Lmax, D), np.float32, np.nan)
        assert lib.madrl_paths_pad_u32(T, E, A, D, len(rec), Lmax, _p(src), None, _p(rec), _p(out.arr), None) == 0
        assert np.array_equal(out.check("padded"), padded_want(src, None, rec, Lmax, True))


def test_path_sums_are_pythons_sum_and_first_return(lib):
    """Per path: the float64 sum of the float32 rewards in time order, bit for bit Python's sum() over the widened
    rewards, and the path's first return; every order of the table, A = 1."""
    for k, (T, E, A, p_done) in enumerate(SHAPES + ((40, 3, 2, 0.02),)):
        rs = np.random.RandomState(200 + k)
        done = (rs.rand(T, E) < p_done).astype(np.uint8)
        rew = (rs.randn(T, E, A) * np.exp(rs.randn(T, E, A) * 3)).astype(np.float32)
        ret = rs.randn(T, E, A).astype(np.float32)
        for order in ("env_major", "agent_major", "shuffled"):
            rec = records(done, A, order, seed=k)
            P = len(rec)
            sums, first = Guarded((P,), np.float64, np.nan), Guarded((P,), np.float64, np.nan)
            assert lib.madrl_path_sums_f32(T, E, A, P, _p(rew), _p(ret), _p(rec), _p(sums.arr), _p(first.arr),
                                           None) == 0
            want = [sum(rew[s:s + L, e, a].astype(np.float64)) for e, a, s, L in rec]
            assert np.array_equal(sums.check("sums"), np.array(want)), (k, order)
            assert np.array_equal(first.check("first_ret"), np.array([ret[s, e, a] for e, a, s, L in rec], np.float64))


def test_argument_errors(lib):
    """MADRL_EINVAL (no launch) for sizes below 1 and NULL buffers."""
    x = np.zeros(16, np.uint32)
    rec = np.array([[0, 0, 0, 1]], np.int32)
    d = np.zeros(1)
    for args in ((0, 1, 1, 1, 1, 1), (1, 1, 1, 0, 1, 1), (1, 1, 1, 1, 0, 1), (1, 1, 1, 1, 1, 0), (1, 1, 0, 1, 1, 1)):
        assert lib.madrl_paths_pad_u32(*args, _p(x), None, _p(rec), _p(x), None) != 0, args
    assert lib.madrl_paths_pad_u16(1, 1, 1, 1, 1, 1, None, None, _p(rec), _p(x), None) != 0
    assert lib.madrl_paths_pad_u32(1, 1, 1, 1, 1, 1, _p(x), None, None, _p(x), None) != 0
    assert lib.madrl_path_sums_f32(1, 1, 1, 0, _p(x), _p(x), _p(rec), _p(d), _p(d), None) != 0
    assert lib.madrl_path_sums_f32(1, 1, 1, 1, _p(x), None, _p(rec), _p(d), _p(d), None) != 0
