"""The whole-path sampling kernels (madrl_b200/csrc/postproc.cu: madrl_whole_paths_fold / _finish / _gather) and the
flat batch's path-parallel passes (madrl_paths_plan_flat, madrl_gae_paths_f32) executed on the CPU by the warp
emulator of tests/emu, against oracle/whole_paths_oracle.py and the serial kernels on the [N, 1] view, bit for bit,
and against a float64 GAE per path.  The selection must not depend on the launch length.  The edge streams, gather
cells and path tables of tests/whole_paths_edges.py up to EMU_MAX_E envs run here as extra cases, and the stream that
needs the most steps runs at exactly the capacity max_steps() gives it."""
import numpy as np
import pytest

import whole_paths_edges as wpe
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
    # (name, done, batch_size, the case's own launch length)
    return [c + (5,) for c in out] + [(s.name, s.done, s.batch_size, s.T) for s in wpe.STREAMS
                                       if s.done.shape[1] <= wpe.EMU_MAX_E]


CASES = _cases()
CELLS = set()                  # the gather cells the runs below reached


def run(lib, done, batch_size, T, tensors, S_run=None):
    """Fold the stream in launches of T steps, finish and gather each tensor of `tensors` (name -> (x [S, E, ...],
    first or None)) into a destination filled with a sentinel; every launch's `first` sits at the same offset from a
    16-byte boundary as the given one.  S_run: the rows of the done stage (the selection's capacity; the stream
    rounded up to whole launches by default).  Returns (acc, path_start, done_flat, env_off, gathered dict), or
    the acc of an incomplete selection."""
    S, E = done.shape
    S_run = -(-S // T) * T if S_run is None else S_run
    stage = np.zeros((S_run, E), np.uint8)
    stage[:min(S, S_run)] = done[:S_run]
    carry = np.concatenate([np.full(E, -1), np.full(E, -1), np.zeros(E)]).astype(np.int32)
    acc = np.array([0, -1, 0, 0, 0], np.int64)
    launches = 0
    for t in range(0, S_run, T):
        chunk = np.ascontiguousarray(stage[t:t + T])
        assert lib.madrl_whole_paths_fold(T, E, t, batch_size, _p(chunk), _p(carry), _p(acc), None) == 0
        launches += 1
        if acc[2]:
            break
    if not acc[2]:
        return acc
    N, P = int(acc[3]), int(acc[4])
    env_off = np.zeros(2 * E, np.int32)
    ps = np.zeros(P + 1, np.int32)
    flat = np.zeros(N, np.uint8)
    assert lib.madrl_whole_paths_finish(E, S_run, _p(stage), _p(carry), _p(env_off), _p(ps), _p(flat), None) == 0
    out = {}
    for name, (x, first) in tensors.items():
        pad = np.zeros((S_run,) + x.shape[1:], x.dtype)
        pad[:S] = x[:S_run]
        dst = np.full(N * x[0, 0].nbytes, wpe.SENTINEL, np.uint8).view(x.dtype).reshape((N,) + x.shape[2:])
        off = None if first is None else first.ctypes.data % 16
        for j in range(launches):
            src = np.ascontiguousarray(pad[j * T:(j + 1) * T])
            fst = first if j == 0 else (None if first is None else wpe.at_offset(pad[j * T - 1], off))
            slab = int(np.prod(x.shape[2:], dtype=np.int64)) * x.itemsize
            CELLS.add(wpe.gather_cell(slab, [src.ctypes.data, dst.ctypes.data] +
                                      ([] if fst is None else [fst.ctypes.data])))
            assert lib.madrl_whole_paths_gather(T, E, slab, j * T, _p(src), _p(fst), _p(carry), _p(env_off), _p(dst),
                                                None) == 0
        out[name] = dst
    return acc, ps, flat, env_off, out


def _tensors(done, seed):
    S, E = done.shape
    rs = np.random.RandomState(seed)
    A = 3
    out = {"obs": (rs.randn(S, E, A, 8).astype(np.float32), rs.randn(E, A, 8).astype(np.float32)),
           "obs_bf16": (rs.randint(0, 2 ** 16, (S, E, A, 5)).astype(np.uint16),
                        rs.randint(0, 2 ** 16, (E, A, 5)).astype(np.uint16)),
           "rew": (rs.randn(S, E, A).astype(np.float32), None),
           "act_i32": (rs.randint(0, 5, (S, E, A)).astype(np.int32), None),
           "info_odd": (rs.randint(0, 255, (S, E, 3)).astype(np.uint8), None)}
    for k, (x, first, off) in wpe.gather_inputs(S, E, seed + 1).items():
        out[k] = (x, None if first is None else wpe.at_offset(first, off))
    return out


# the scripted streams at T = 1, 7, one launch and their own T; the edge streams beyond 129 envs at 1 and their own T
# only (the emulator's time goes with E * launches)
GATHER_RUNS = [(i, T) for i, c in enumerate(CASES) for T in ([1, 7, "all", "own"] if c[1].shape[1] <= 129 else
                                                               [1, "own"])]


@pytest.mark.parametrize("case,T", GATHER_RUNS, ids=["%s-%s" % (CASES[i][0], T) for i, T in GATHER_RUNS])
def test_selection_and_gather_match_oracle(lib, case, T):
    name, done, bs, T_own = CASES[case]
    T = done.shape[0] if T == "all" else T_own if T == "own" else T
    sel = wo.select(done, bs)
    assert sel is not None
    t_star, end = sel
    tensors = _tensors(done, case)
    acc, ps, flat, env_off, out = run(lib, done, bs, T, tensors)
    assert acc[1] == t_star
    assert acc[3] == int(np.sum(end + 1)) and acc[4] == len(ps) - 1
    np.testing.assert_array_equal(ps, wo.path_start_np(done, end))
    np.testing.assert_array_equal(flat, wo.take(done, end))
    np.testing.assert_array_equal(env_off[:len(end)], wo.env_rows(end))
    assert flat[-1] == 1 and flat.sum() == len(ps) - 1
    for k, (x, first) in tensors.items():
        wpe.check_gathered(out[k], x, end, first)


def test_threshold_at_path_end(lib):
    """At t* an env whose path ends there keeps only the paths up to t*."""
    name, done, bs, _ = CASES[[c[0] for c in CASES].index("exact")]
    t_star, end = wo.select(done, bs)
    assert done[t_star].any()
    for e in np.nonzero(done[t_star])[0]:
        assert end[e] == t_star


def test_gather_cells_all_reached(lib):
    """Run after the gather tests (file order): the table reaches every (word, thread / warp) cell of the dispatch,
    and the shifted tensors with a 4- or 2-byte aligned `first` fall back on its account."""
    if not CELLS:
        pytest.skip("run with test_selection_and_gather_match_oracle")
    assert CELLS == wpe.ALL_CELLS
    for k, (dt, sh, off) in wpe.GATHER_FIRST.items():
        slab = int(np.prod(sh)) * np.dtype(dt).itemsize
        assert slab % 16 == 0 and wpe.gather_cell(slab, [0, 16, off])[0] == off, k


def test_vectorised_oracle_equals_loops():
    for name, done, bs, _ in CASES:
        t_star, end = wo.select(done, bs)
        x = np.random.RandomState(1).randn(*done.shape, 2)
        first = np.random.RandomState(2).randn(done.shape[1], 2)
        t, e = wo.rows_index(end)
        assert list(zip(t.tolist(), e.tolist())) == wo.rows(end), name
        for f in (None, first):
            np.testing.assert_array_equal(wo.take(x, end, f), wo.gather(x, end, f), err_msg=name)
        np.testing.assert_array_equal(wo.path_start_np(done, end), wo.path_start(done, end), err_msg=name)
        np.testing.assert_array_equal(wo.env_rows(end), np.concatenate([[0], np.cumsum(end + 1)[:-1]]))


def test_edge_table_reaches_its_reasons():
    wpe.check_table()
    Es = {s.done.shape[1] for s in wpe.STREAMS if s.done.shape[1] <= wpe.EMU_MAX_E}
    assert {129, 257, 300} <= Es         # a second rows block, a second fold stride, two envs per scan thread


@pytest.mark.parametrize("T", [1, 4])
def test_worst_stream_completes_within_max_steps(lib, T):
    """The stream that needs the most steps completes within max_steps() rows of done stage; a path lengthened to
    the capacity's last step still completes, one step more does not (the sampler raises before the next fold)."""
    done, bs, cap, tight, over = wpe.worst_case(T=T)
    t_star, end = wo.select(done, bs)
    assert cap % T == 0
    acc, ps, flat, env_off, _ = run(lib, done, bs, T, {}, S_run=cap)
    assert acc[1] == t_star and acc[3] == int(np.sum(end + 1))
    np.testing.assert_array_equal(ps, wo.path_start(done, end))
    acc, ps, flat, env_off, _ = run(lib, tight, bs, T, {}, S_run=cap)
    assert wo.select(tight, bs)[1].max() == cap - 1 and acc[3] == int(np.sum(wo.select(tight, bs)[1] + 1))
    acc = run(lib, over, bs, T, {}, S_run=cap)
    assert len(acc) == 5 and acc[2] == 0 and acc[1] == t_star


def _plan_inputs():
    """(name, path_start, done_flat, rew, val, discount, gae_lambda): the streams' batches and the path tables."""
    out = []
    for i, (name, done, bs, _) in enumerate(CASES):
        t_star, end = wo.select(done, bs)
        rs = np.random.RandomState(i)
        N = int(np.sum(end + 1))
        out.append((name, wo.path_start(done, end), np.ascontiguousarray(wo.gather(done, end)),
                    rs.randn(N, 1, 3).astype(np.float32), rs.randn(N, 1, 3).astype(np.float32), 0.99, 0.95))
    for i, c in enumerate(wpe.PLAN_CASES):
        ps, flat, rew, val = wpe.plan_inputs(c, 100 + i)
        out.append(("plan_" + c.name, ps, flat, rew, val, c.discount, c.gae_lambda))
    return out


PLAN_INPUTS = _plan_inputs()


@pytest.mark.parametrize("case", range(len(PLAN_INPUTS)), ids=[c[0] for c in PLAN_INPUTS])
def test_flat_plan_and_gae_equal_serial_kernels(lib, case):
    name, ps, flat, rew, val, discount, gae_lambda = PLAN_INPUTS[case]
    N, P, A = len(flat), len(ps) - 1, rew.shape[2]
    want = [np.zeros((N, 1), np.int32), np.zeros((N, 1), np.int32), np.zeros(1, np.int32),
            np.zeros((1, N, 3), np.int32)]
    assert lib.madrl_paths_plan(N, 1, A, _p(flat), *map(_p, want), None) == 0
    got = [np.zeros((N, 1), np.int32), np.zeros((N, 1), np.int32), np.zeros(1, np.int32),
           np.zeros((1, N, 3), np.int32)]
    assert lib.madrl_paths_plan_flat(N, P, _p(ps), *map(_p, got), None) == 0
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g, w)
    adv_s, ret_s, adv_p, ret_p = (np.zeros_like(rew) for _ in range(4))
    assert lib.madrl_gae_f32(N, 1, A, _p(rew), _p(val), _p(flat), None, discount, gae_lambda, _p(adv_s), _p(ret_s),
                             None) == 0
    assert lib.madrl_gae_paths_f32(P, A, _p(ps), _p(rew), _p(val), discount, gae_lambda, _p(adv_p), _p(ret_p),
                                   None) == 0
    assert adv_p.tobytes() == adv_s.tobytes() and ret_p.tobytes() == ret_s.tobytes()
    wpe.check_gae_float64(adv_p, ret_p, rew, val, flat, discount, gae_lambda)


def test_abi_rejects_bad_arguments(lib):
    d = np.zeros((2, 2), np.uint8)
    carry, acc = np.zeros(6, np.int32), np.zeros(5, np.int64)
    assert lib.madrl_whole_paths_fold(2, 2, 0, 0, _p(d), _p(carry), _p(acc), None) != 0
    assert lib.madrl_whole_paths_fold(0, 2, 0, 4, _p(d), _p(carry), _p(acc), None) != 0
    assert lib.madrl_whole_paths_fold(2, 2, 0, 4, None, _p(carry), _p(acc), None) != 0
    assert lib.madrl_paths_plan_flat(4, 5, _p(carry), _p(carry), _p(carry), _p(carry), _p(carry), None) != 0
