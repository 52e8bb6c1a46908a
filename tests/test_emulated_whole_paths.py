"""The whole-path sampling kernels (madrl_b200/csrc/postproc.cu: madrl_whole_paths_fold / _finish / _gather) and the
flat batch's path-parallel passes (madrl_paths_plan_flat, madrl_gae_paths_f32) executed on the CPU by the warp
emulator of tests/emu, against oracle/whole_paths_oracle.py and the serial kernels on the [N, 1] view, bit for bit.
The selection must not depend on the launch length."""
import numpy as np
import pytest

from emu import driver
from emu.driver import ptr as _p
from oracle import whole_paths_oracle as wo

pytestmark = driver.needs_cxx


@pytest.fixture(scope="module")
def lib():
    return driver.load(())


def stream(seed, S, E, mpl, p_end):
    """A done stream from reset: each env's paths end at random (probability p_end per step) or at mpl steps."""
    rs = np.random.RandomState(seed)
    done = np.zeros((S, E), np.uint8)
    for e in range(E):
        n = 0
        for t in range(S):
            n += 1
            if n == mpl or rs.rand() < p_end:
                done[t, e], n = 1, 0
    return done


def _cases():
    # (name, done, batch_size): ragged paths; length-1 paths; the threshold crossed exactly at a path end; envs
    # still running long after t*
    S, E, mpl = 40, 5, 9
    ragged = stream(1, S, E, mpl, 0.2)
    ones = ragged.copy()
    ones[3:6, 1] = 1                                 # three paths of length 1 in env 1
    ones[0, 4] = 1                                   # a length-1 path at the start
    exact = np.zeros((S, E), np.uint8)
    exact[[2, 5, 9, 12, 20, 29], 0] = 1
    exact[[8, 16, 24, 32], 1] = 1
    exact[[3, 11, 19, 27, 35], 2] = 1
    exact[[7, 15, 23, 31, 39], 3] = 1
    exact[[1, 4, 13, 22, 30, 38], 4] = 1
    wo_exact = wo.select(exact, 1)
    late = np.zeros((S, E), np.uint8)                # envs 0-3 end often, env 4 runs to the horizon
    late[:, :4] = stream(2, S, 4, 3, 0.0)
    late[[mpl - 1, 2 * mpl - 1, 3 * mpl - 1], 4] = 1
    out = [("ragged", ragged, 31), ("ones", ones, 23), ("late", late, 20), ("first", ragged, 1)]
    # the count after each step of `exact`: batch_size equal to one of them is crossed exactly at a path end
    last, count, counts = np.full(E, -1), 0, []
    for t in range(S):
        d = exact[t].astype(bool)
        count += int(np.sum(t - last[d]))
        last[d] = t
        counts.append(count)
    assert wo_exact is not None
    out.append(("exact", exact, counts[12]))
    return out


CASES = _cases()


def run(lib, done, batch_size, T, tensors):
    """Fold the stream in launches of T steps, finish and gather each tensor of `tensors` (name -> (x [S, E, ...],
    first or None)).  Returns (acc, path_start, done_flat, env_off, gathered dict)."""
    S, E = done.shape
    S_run = -(-S // T) * T
    stage = np.zeros((S_run, E), np.uint8)
    stage[:S] = done
    carry = np.concatenate([np.full(E, -1), np.full(E, -1), np.zeros(E)]).astype(np.int32)
    acc = np.array([0, -1, 0, 0, 0], np.int64)
    launches = 0
    for t in range(0, S_run, T):
        chunk = np.ascontiguousarray(stage[t:t + T])
        assert lib.madrl_whole_paths_fold(T, E, t, batch_size, _p(chunk), _p(carry), _p(acc), None) == 0
        launches += 1
        if acc[2]:
            break
    assert acc[2] == 1
    N, P = int(acc[3]), int(acc[4])
    env_off = np.zeros(2 * E, np.int32)
    ps = np.zeros(P + 1, np.int32)
    flat = np.zeros(N, np.uint8)
    assert lib.madrl_whole_paths_finish(E, S_run, _p(stage), _p(carry), _p(env_off), _p(ps), _p(flat), None) == 0
    out = {}
    for name, (x, first) in tensors.items():
        pad = np.zeros((S_run,) + x.shape[1:], x.dtype)
        pad[:S] = x
        dst = np.full((N,) + x.shape[2:], 0x5A, np.uint8).view(x.dtype) if x.dtype == np.uint8 else \
            np.zeros((N,) + x.shape[2:], x.dtype)
        for j in range(launches):
            src = np.ascontiguousarray(pad[j * T:(j + 1) * T])
            fst = first if j == 0 else (None if first is None else np.ascontiguousarray(pad[j * T - 1]))
            slab = int(np.prod(x.shape[2:], dtype=np.int64)) * x.itemsize
            assert lib.madrl_whole_paths_gather(T, E, slab, j * T, _p(src), _p(fst), _p(carry), _p(env_off), _p(dst),
                                                None) == 0
        out[name] = dst
    return acc, ps, flat, env_off, out


def _tensors(done, seed):
    S, E = done.shape
    rs = np.random.RandomState(seed)
    A = 3
    return {"obs": (rs.randn(S, E, A, 8).astype(np.float32), rs.randn(E, A, 8).astype(np.float32)),
            "obs_bf16": (rs.randint(0, 2 ** 16, (S, E, A, 5)).astype(np.uint16),
                         rs.randint(0, 2 ** 16, (E, A, 5)).astype(np.uint16)),
            "rew": (rs.randn(S, E, A).astype(np.float32), None),
            "act_i32": (rs.randint(0, 5, (S, E, A)).astype(np.int32), None),
            "info_odd": (rs.randint(0, 255, (S, E, 3)).astype(np.uint8), None)}


@pytest.mark.parametrize("T", [1, 7, "all"])
@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_selection_and_gather_match_oracle(lib, case, T):
    name, done, bs = CASES[case]
    T = done.shape[0] if T == "all" else T
    sel = wo.select(done, bs)
    assert sel is not None
    t_star, end = sel
    tensors = _tensors(done, case)
    acc, ps, flat, env_off, out = run(lib, done, bs, T, tensors)
    assert acc[1] == t_star
    assert acc[3] == int(np.sum(end + 1))
    np.testing.assert_array_equal(ps, wo.path_start(done, end))
    np.testing.assert_array_equal(flat, wo.gather(done, end))
    np.testing.assert_array_equal(env_off[:len(end)], np.concatenate([[0], np.cumsum(end + 1)[:-1]]))
    assert flat[-1] == 1 and flat.sum() == len(ps) - 1
    for k, (x, first) in tensors.items():
        np.testing.assert_array_equal(out[k], wo.gather(x, end, first), err_msg=k)


def test_threshold_at_path_end(lib):
    """At t* an env whose path ends there keeps only the paths up to t*."""
    name, done, bs = CASES[[c[0] for c in CASES].index("exact")]
    t_star, end = wo.select(done, bs)
    assert done[t_star].any()
    for e in np.nonzero(done[t_star])[0]:
        assert end[e] == t_star


@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_flat_plan_and_gae_equal_serial_kernels(lib, case):
    name, done, bs = CASES[case]
    t_star, end = wo.select(done, bs)
    ps = wo.path_start(done, end)
    flat = np.ascontiguousarray(wo.gather(done, end))
    N, P, A = len(flat), len(ps) - 1, 3
    want = [np.zeros((N, 1), np.int32), np.zeros((N, 1), np.int32), np.zeros(1, np.int32),
            np.zeros((1, N, 3), np.int32)]
    assert lib.madrl_paths_plan(N, 1, A, _p(flat), *map(_p, want), None) == 0
    got = [np.zeros((N, 1), np.int32), np.zeros((N, 1), np.int32), np.zeros(1, np.int32),
           np.zeros((1, N, 3), np.int32)]
    assert lib.madrl_paths_plan_flat(N, P, _p(ps), *map(_p, got), None) == 0
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)
    rs = np.random.RandomState(case)
    rew, val = rs.randn(N, 1, A).astype(np.float32), rs.randn(N, 1, A).astype(np.float32)
    adv_s, ret_s, adv_p, ret_p = (np.zeros_like(rew) for _ in range(4))
    assert lib.madrl_gae_f32(N, 1, A, _p(rew), _p(val), _p(flat), None, 0.99, 0.95, _p(adv_s), _p(ret_s), None) == 0
    assert lib.madrl_gae_paths_f32(P, A, _p(ps), _p(rew), _p(val), 0.99, 0.95, _p(adv_p), _p(ret_p), None) == 0
    assert adv_p.tobytes() == adv_s.tobytes() and ret_p.tobytes() == ret_s.tobytes()


def test_abi_rejects_bad_arguments(lib):
    d = np.zeros((2, 2), np.uint8)
    carry, acc = np.zeros(6, np.int32), np.zeros(5, np.int64)
    assert lib.madrl_whole_paths_fold(2, 2, 0, 0, _p(d), _p(carry), _p(acc), None) != 0
    assert lib.madrl_whole_paths_fold(0, 2, 0, 4, _p(d), _p(carry), _p(acc), None) != 0
    assert lib.madrl_whole_paths_fold(2, 2, 0, 4, None, _p(carry), _p(acc), None) != 0
    assert lib.madrl_paths_plan_flat(4, 5, _p(carry), _p(carry), _p(carry), _p(carry), _p(carry), None) != 0
