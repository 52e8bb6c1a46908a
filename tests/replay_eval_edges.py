"""Inputs shared by the edge-case tests of the replay pool kernels (csrc/replay.cu) and the episode-record kernel
(eval_episodes_kernel, csrc/postproc.cu): tests/test_replay_edges_gpu.py and tests/test_evaluate_edges_gpu.py run
them on the device, tests/test_emulated_replay.py and tests/test_evaluate_cpu.py in the warp emulator of tests/emu.
The geometry-dependent cases take the launch geometry as an argument: the emulator reports two SMs, an H100 132.
Every expected value comes from oracle/replay_oracle.py or oracle/eval_oracle.py."""
import os
import re

import numpy as np

from oracle import eval_oracle as eo
from oracle import replay_oracle as ro

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "madrl_b200", "csrc")


def csrc_constexpr(name, source):
    """The value of a `constexpr int name = <int>;` of a kernel source."""
    with open(os.path.join(CSRC, source)) as f:
        return int(re.search(r"constexpr int %s = (\d+);" % name, f.read()).group(1))


# ---------------------------------------------------------------- replay pool (csrc/replay.cu)

SCAN_THREADS = csrc_constexpr("kScanThreads", "replay.cu")   # threads of the one-block scan
INSERT_WARPS_PER_SM = 8 * 8                                  # insert grid: 8 blocks of 8 warps per SM, grid-stride


def insert_grid_warps(sms):
    """Warps of the largest insert grid: min(ceil(rows / 8), 8 SMs) blocks of 8 warps."""
    return INSERT_WARPS_PER_SM * sms


def grid_shape(rows):
    """(T, E, A) with (T + 1) E A == rows exactly: A = 3, 2 or 1, E the largest divisor up to 400 leaving T >= 1."""
    for A in (3, 2, 1):
        if rows % A:
            continue
        m = rows // A
        for E in range(min(m // 2, 400), 0, -1):
            if m % E == 0:
                return m // E - 1, E, A
    raise AssertionError(rows)


def insert_grid_rows(sms):
    """Source rows (T + 1) E A around the insert grid G: G - 1, G, G + 1 and 2 G + 1."""
    G = insert_grid_warps(sms)
    return (G - 1, G, G + 1, 2 * G + 1)


def scan_cells():
    """T W (steps x warps of envs) around the scan block: one cell per thread, and one cell more or less."""
    S = SCAN_THREADS
    return (S - 1, S, S + 1, 2 * S + 1)


def rollout(rs, T, E, A, D, Ad, w, mpl, limit, p_done, pl0, ts0):
    """A rollout whose done flags follow the engine's rule: the env ends by itself at random or at the timestep limit,
    and the horizon cuts at max_path_length.  Observation words are random bits.  Returns the rollout and the
    counters after it."""
    pl, ts = pl0.astype(np.int64).copy(), ts0.astype(np.int64).copy()
    done = np.zeros((T, E), np.uint8)
    for t in range(T):
        pl += 1
        ts += 1
        d = (rs.rand(E) < p_done) | (ts >= limit) | ((mpl > 0) & (pl >= mpl))
        done[t] = d
        pl[d] = 0
        ts[d] = 0
    bits = lambda *s: rs.randint(0, 2 ** (8 * np.dtype(w).itemsize), size=s, dtype=np.uint64).astype(w)  # noqa: E731
    return dict(obs=bits(T, E, A, D), act=rs.randn(T, E, A, Ad).astype(np.float32),
                rew=rs.randn(T, E, A).astype(np.float32), done=done, obs_before=bits(E, A, D),
                term=bits(T, E, A, D)), pl.astype(np.int32), ts.astype(np.int32)


def start_counters(rs, E, mpl):
    """Path-length and timestep counters of envs part-way through their paths."""
    pl = rs.randint(0, max(mpl, 1), size=E).astype(np.int32)
    return pl, (pl + rs.randint(0, 5, size=E)).astype(np.int32)


def cell_prefix(done, pl0, ts0, mpl, limit, include):
    """(kept transitions per (t, warp) cell in step-major order, their exclusive prefix, W)."""
    keep = ro.keep_flags(done, pl0, ts0, mpl, limit, include)
    T, E = keep.shape
    W = (E + 31) // 32
    pad = np.zeros((T, W * 32), np.int64)
    pad[:, :E] = keep
    cnt = pad.reshape(T, W, 32).sum(-1).reshape(-1)
    return cnt, np.concatenate([[0], np.cumsum(cnt)[:-1]]), W


CUTS = ("cell_edge", "in_cell", "in_env", "last_step", "k_eq_m", "k_eq_m_plus_1")


def cut_pool_size(kind, done, pl0, ts0, mpl, limit, include, A):
    """max_pool_size M that puts the first landing transition (first = K - M) where `kind` says:
    cell_edge      on the first transition of a warp cell, in the middle of the rollout;
    in_cell        inside the last warp cell of a step (the next cell is the next step's);
    in_env         between two agents of one (t, env) (needs A > 1: A does not divide M);
    last_step      on the first transition of step T - 1 (only the last step lands);
    k_eq_m, k_eq_m_plus_1  K = M and K = M + 1.
    Returns (M, first, K)."""
    T = done.shape[0]
    cnt, pre, W = cell_prefix(done, pl0, ts0, mpl, limit, include)
    K = int(cnt.sum()) * A
    mid = [c for c in range(len(cnt)) if cnt[c] >= 2 and pre[c] > 0 and c // W < T - 1]
    if kind == "cell_edge":
        first = int(pre[mid[len(mid) // 2]]) * A
    elif kind in ("in_cell", "in_env"):
        last = [c for c in mid if c % W == W - 1]
        c = last[len(last) // 2]
        first = int(pre[c] + cnt[c] // 2) * A + (A // 2 if kind == "in_env" else 0)
        assert kind == "in_cell" or first % A
    elif kind == "last_step":
        first = int(pre[(T - 1) * W]) * A
        assert first < K
    elif kind == "k_eq_m":
        first = 0
    else:
        first = 1
    return K - first, first, K


def landing_step(done, pl0, ts0, mpl, limit, include, A, first):
    """The step of kept transition `first` (the insert kernel's first step)."""
    keep = ro.keep_flags(done, pl0, ts0, mpl, limit, include)
    per_step = np.cumsum(keep.sum(1) * A)
    return int(np.searchsorted(per_step, first, side="right"))


PLAN_ENVS = (1, 31, 33, 127, 129)      # a plan warp of one env, of 31 and 33 envs, and the plan block of 128 threads

# (obs dtype, D): float32 rows of 16, 8 and 4 bytes, bfloat16 rows of 16, 8, 4 and 2 bytes (the word row_word picks
# for aligned pointers)
WORD_ROWS = ((np.float32, 8, 16), (np.float32, 6, 8), (np.float32, 5, 4),
             (np.uint16, 16, 16), (np.uint16, 12, 8), (np.uint16, 6, 4), (np.uint16, 7, 2))
# the one pointer placed one element off its allocation (None: every pointer aligned)
ADD_OFFSETS = (None, "obs", "obs_before", "term", "observations", "next_observations")


def row_word(row_bytes, offsets_bytes):
    """The word the kernels move rows in (replay.cu's row_word) for pointers at these byte offsets from 256-byte
    aligned allocations."""
    for w in (16, 8, 4):
        if row_bytes % w == 0 and all(o % w == 0 for o in offsets_bytes):
            return w
    return 2


# (n, B) of a sample: 1, 7, 8 and 9 rows (one launch block holds 8 row warps)
SAMPLE_ROWS = ((1, 1), (1, 7), (2, 4), (3, 3))
# (obs dtype, D, Ad): rows of fewer and more than 32 words, one action and 33 (the action loop runs twice)
SAMPLE_ROW_SHAPES = ((np.float32, 8, 1), (np.float32, 150, 33), (np.uint16, 7, 33), (np.uint16, 88, 1))


# ---------------------------------------------------------------- episode records (eval_episodes_kernel)

RECORD_SENTINEL_F64 = np.array([0x7FF4DEAD5EA1F00D], np.int64).view(np.float64)[0]   # a signalling-NaN pattern
RECORD_SENTINEL_INT = -0x5A5A5A5B


def record_sentinels(E, A, C, K):
    """Record arrays (ret, qsum, len, info_sum) filled with sentinels: a record the kernel must not write keeps them."""
    ret, qsum, ln, isum = eo.new_records(E, A, C, K)
    ret[...] = qsum[...] = RECORD_SENTINEL_F64
    ln[...] = RECORD_SENTINEL_INT
    isum[...] = RECORD_SENTINEL_INT
    return [ret, qsum, ln, isum]


def records_equal(got, want):
    """Bit identity of (ret, qsum, len, info_sum) record arrays, NaN sentinels included."""
    return all(np.array_equal(np.ascontiguousarray(g).view(np.uint8), np.ascontiguousarray(w).view(np.uint8))
               for g, w in zip(got, want))


# (E, A): E A at 127, 128 and 129 threads (one 128-thread block and one more), 128 k + 1; with A = 5 and A = 32
# an env's agents straddle a block edge
RECORD_SHAPES = ((127, 1), (128, 1), (129, 1), (1025, 1), (25, 5), (26, 5), (77, 5), (4, 32), (5, 32), (33, 32))
INFO_BIG = 2 ** 31 - 1


def record_case(T, E, A, C, K, seed, f64, launch_len=5):
    """rew [T,E,A], done [T,E], info [T,E,C] and the launch cuts of one record case; env e % 6 ==
    0  done on every step: episodes of length 1, more than K of them (the records past K are dropped);
    1  never done: no record, its K slots keep their sentinels;
    2  done at random (p = 0.2);
    3  done on the first step of every launch;
    4  done on the last step of every launch;
    5  one episode of T - 1 steps, ending at T - 2: fewer than K records, and a carry left running.
    Info values lie within 8 of 2^31 - 1, so the int64 sums leave the int32 range after two steps.  Launches
    alternate between 1 step and `launch_len` steps."""
    rs = np.random.RandomState(seed)
    rew = (rs.randn(T, E, A) * 3 + 0.25).astype(np.float64 if f64 else np.float32)
    cuts, t = [], 0
    while t < T:
        t += 1 if len(cuts) % 2 == 0 else launch_len
        if t < T:
            cuts.append(t)
    starts, ends = [0] + cuts, [c - 1 for c in cuts] + [T - 1]
    done = np.zeros((T, E), np.uint8)
    kind = np.arange(E) % 6
    done[:, kind == 0] = 1
    done[:, kind == 2] = rs.rand(T, int((kind == 2).sum())) < 0.2
    done[np.ix_(starts, np.nonzero(kind == 3)[0])] = 1
    done[np.ix_(ends, np.nonzero(kind == 4)[0])] = 1
    done[T - 2, kind == 5] = 1
    info = (INFO_BIG - rs.randint(0, 8, size=(T, E, C))).astype(np.int32)
    return rew, done, info, tuple(cuts)


# (T, K, discount, launch_len): discount 0, 1, and 0.5 over an episode of 1 199 steps (0.5^t goes subnormal at
# t = 1 023 and to 0 at t = 1 075, after which G stops growing)
RECORD_RUNS = ((24, 3, 0.99, 5), (24, 2, 0.0, 4), (24, 1, 1.0, 3), (1200, 2, 0.5, 150))


def run_records_oracle(rew, done, info, discount, K, cuts, records):
    """eo.eval_episodes launch by launch from a zeroed carry: yields (carry, records) after every launch."""
    T, E, A = rew.shape
    carry = eo.new_carry(E, A)
    for t0, t1 in zip((0,) + tuple(cuts), tuple(cuts) + (T,)):
        eo.eval_episodes(rew[t0:t1], done[t0:t1], info[t0:t1], discount, K, carry, records)
        yield t0, t1, carry, records
