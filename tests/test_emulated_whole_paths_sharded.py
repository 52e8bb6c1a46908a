"""The whole-path selection over the ranks of a sharded batch (madrl_whole_paths_steps and
madrl_whole_paths_fold_pooled of madrl_b200/csrc/postproc.cu) executed on the CPU by the warp emulator of tests/emu.
Each stream's env columns are split into W = 2, 3 and 4 shards (one-env shards, very uneven shards, a shard across
the fold's 256-env stride); the shards fold in lockstep, their increments summed in rank order between the two
calls, as WholePathSampler does with a group.  Against the whole stream folded by madrl_whole_paths_fold: the summed
increments are the steps of the running count, the steps kernel leaves carry alone, every shard ends with the whole
fold's count, t* and carry slice, the shards' N and P add up, and each shard's finish and gather, concatenated with
its row and path offsets, are the whole stream's outputs.  Launch lengths 1, 7 and the stream's own."""
import numpy as np
import pytest

import whole_paths_edges as wpe
from emu import driver
from emu.driver import ptr as _p
from oracle import whole_paths_oracle as wo
from test_emulated_whole_paths import CASES

pytestmark = driver.needs_cxx

STRIDE = wpe.FOLD_THREADS


@pytest.fixture(scope="module")
def lib():
    return driver.load(())


def splits(E, W):
    """Shard sizes (rank order) of E envs over W ranks: balanced, one-env shards first, one-env shards last, and,
    where E allows, a shard that spans the 256-env stride of the fold."""
    if E < W:
        return []
    out = [tuple((E * (r + 1)) // W - (E * r) // W for r in range(W)),
           (1,) * (W - 1) + (E - W + 1,),
           (E - W + 1,) + (1,) * (W - 1)]
    if E > STRIDE + W:
        lo = STRIDE - 3                                   # shard 1 holds envs 253 .. 258 (or more): across 256
        out.append((lo, 6) + (1,) * (W - 3) + (E - lo - 6 - (W - 3),) if W > 2 else (lo, E - lo))
    return list(dict.fromkeys(s for s in out if min(s) >= 1))


def bounds(sizes):
    c = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    return [(int(c[r]), int(c[r + 1])) for r in range(len(sizes))]


def new_carry(E):
    return np.concatenate([np.full(E, -1), np.full(E, -1), np.zeros(E)]).astype(np.int32)


def new_acc():
    return np.array([0, -1, 0, 0, 0], np.int64)


def staged(done, T):
    S, E = done.shape
    stage = np.zeros((-(-S // T) * T, E), np.uint8)
    stage[:S] = done
    return stage


def fold_whole(lib, stage, bs, T):
    """The unsharded fold: (carry, acc, launches)."""
    E = stage.shape[1]
    carry, acc = new_carry(E), new_acc()
    for j in range(stage.shape[0] // T):
        chunk = np.ascontiguousarray(stage[j * T:(j + 1) * T])
        assert lib.madrl_whole_paths_fold(T, E, j * T, bs, _p(chunk), _p(carry), _p(acc), None) == 0
        if acc[2]:
            return carry, acc, j + 1
    raise AssertionError("the stream did not complete")


def fold_shards(lib, stage, bs, T, sizes):
    """The shards' lockstep folds: ([carry], [acc], launches, pooled increments of the launches that pooled)."""
    cuts = bounds(sizes)
    carry, acc = [new_carry(hi - lo) for lo, hi in cuts], [new_acc() for _ in cuts]
    pooled = []
    for j in range(stage.shape[0] // T):
        chunks = [np.ascontiguousarray(stage[j * T:(j + 1) * T, lo:hi]) for lo, hi in cuts]
        inc = np.zeros(T, np.int64)
        if acc[0][1] < 0:                                 # t* not known yet on any rank (it is one value on all)
            total = np.zeros(T, np.int64)
            for r, (lo, hi) in enumerate(cuts):
                before = carry[r].copy()
                mine = np.full(T, -7, np.int64)
                assert lib.madrl_whole_paths_steps(T, hi - lo, j * T, _p(chunks[r]), _p(carry[r]), _p(mine),
                                                   None) == 0
                assert np.array_equal(carry[r], before), "steps wrote carry"
                total += mine                             # int64: the order of the sum does not matter
            inc = total
            pooled.append((j, inc.copy()))
        for r, (lo, hi) in enumerate(cuts):
            assert lib.madrl_whole_paths_fold_pooled(T, hi - lo, j * T, bs, _p(chunks[r]), _p(inc), _p(carry[r]),
                                                     _p(acc[r]), None) == 0
        if min(a[2] for a in acc):
            return carry, acc, j + 1, pooled
    raise AssertionError("the shards did not complete")


def finish_gather(lib, stage, carry, acc, T, launches, tensors):
    """One shard's (or the whole stream's) finish and gathers: (path_start, done_flat, env_off, {name: rows})."""
    S, E = stage.shape
    N, P = int(acc[3]), int(acc[4])
    env_off, ps, flat = np.zeros(2 * E, np.int32), np.zeros(P + 1, np.int32), np.zeros(N, np.uint8)
    assert lib.madrl_whole_paths_finish(E, S, _p(stage), _p(carry), _p(env_off), _p(ps), _p(flat), None) == 0
    out = {}
    for name, (x, first) in tensors.items():
        dst = np.full(N * x[0, 0].nbytes, wpe.SENTINEL, np.uint8).view(x.dtype).reshape((N,) + x.shape[2:])
        slab = x[0, 0].nbytes
        for j in range(launches):
            src = np.ascontiguousarray(x[j * T:(j + 1) * T])
            fst = None if first is None else (first if j == 0 else np.ascontiguousarray(x[j * T - 1]))
            assert lib.madrl_whole_paths_gather(T, E, slab, j * T, _p(src), _p(fst), _p(carry), _p(env_off),
                                                _p(dst), None) == 0
        out[name] = dst
    return ps, flat, env_off[:E], out


def tensors_of(S, E, seed):
    rs = np.random.RandomState(seed)
    return {"obs": (rs.randn(S, E, 2, 4).astype(np.float32), rs.randn(E, 2, 4).astype(np.float32)),
            "rew": (rs.randn(S, E, 2).astype(np.float32), None),
            "info_odd": (rs.randint(0, 255, (S, E, 3)).astype(np.uint8), None)}


def _runs():
    out = []
    for i, (name, done, bs, T_own) in enumerate(CASES):
        E = done.shape[1]
        for W in (2, 3, 4):
            for k, sizes in enumerate(splits(E, W)):
                # every split at T = 7; the balanced split also at T = 1 and the stream's own T (at most 129 envs
                # at T = 1: the emulator's time goes with E * launches)
                Ts = [7] + ([1, "own"] if k == 0 else []) if E <= 129 else [7] + (["own"] if k == 0 else [])
                out += [(i, sizes, T) for T in Ts]
    return out


RUNS = _runs()


def test_splits_reach_their_reasons():
    seen = set()
    for i, sizes, T in RUNS:
        E = CASES[i][1].shape[1]
        seen.add(len(sizes))
        if min(sizes) == 1:
            seen.add("one-env")
        if max(sizes) >= 10 * min(sizes):
            seen.add("uneven")
        if any(lo < STRIDE < hi for lo, hi in bounds(sizes)[1:]):
            seen.add("across-stride")
        seen.add(T)
    assert {2, 3, 4, "one-env", "uneven", "across-stride", 1, 7, "own"} <= seen


@pytest.mark.parametrize("case,sizes,T", RUNS, ids=["%s-%s-T%s" % (CASES[i][0], "_".join(map(str, s)), T)
                                                     for i, s, T in RUNS])
def test_shards_select_the_whole_streams_batch(lib, case, sizes, T):
    name, done, bs, T_own = CASES[case]
    T = T_own if T == "own" else T
    stage = staged(done, T)
    S, E = stage.shape
    carry, acc, launches = fold_whole(lib, stage, bs, T)
    t_star, end = wo.select(done, bs)
    assert acc[1] == t_star
    s_carry, s_acc, s_launches, pooled = fold_shards(lib, stage, bs, T, sizes)
    assert s_launches == launches
    # the pooled increments are the running count's steps, for every launch that pooled (those up to t*'s)
    steps = np.diff(np.concatenate([[0], wpe.counts(stage)]))
    assert [j for j, _ in pooled] == list(range(t_star // T + 1))
    for j, inc in pooled:
        assert np.array_equal(inc, steps[j * T:(j + 1) * T]), j
    cuts = bounds(sizes)
    whole = carry.reshape(3, E)
    for r, (lo, hi) in enumerate(cuts):
        assert np.array_equal(s_carry[r].reshape(3, hi - lo), whole[:, lo:hi]), r
        assert s_acc[r][0] == acc[0] and s_acc[r][1] == acc[1] and s_acc[r][2] == 1, r
    assert sum(a[3] for a in s_acc) == acc[3] and sum(a[4] for a in s_acc) == acc[4]
    # finish and gather: each shard's outputs, shifted by the rows and paths of the lower shards, are the whole's
    x = tensors_of(S, E, case)
    ps, flat, env_off, out = finish_gather(lib, stage, carry, acc, T, launches, x)
    got_ps, got_flat, got_off, got = [], [], [], {k: [] for k in x}
    row = 0
    for r, (lo, hi) in enumerate(cuts):
        part = {k: (np.ascontiguousarray(v[:, lo:hi]), None if f is None else np.ascontiguousarray(f[lo:hi]))
                for k, (v, f) in x.items()}
        sps, sflat, soff, sout = finish_gather(lib, np.ascontiguousarray(stage[:, lo:hi]), s_carry[r], s_acc[r], T,
                                               s_launches, part)
        got_ps.append(sps[:-1] + row)
        got_flat.append(sflat)
        got_off.append(soff + row)
        for k in x:
            got[k].append(sout[k])
        row += int(s_acc[r][3])
    assert np.array_equal(np.concatenate(got_ps + [[row]]), ps)
    assert np.array_equal(np.concatenate(got_flat), flat)
    assert np.array_equal(np.concatenate(got_off), env_off)
    for k in x:
        assert np.concatenate(got[k]).tobytes() == out[k].tobytes(), k
    np.testing.assert_array_equal(ps, wo.path_start_np(done, end))


def test_steps_reads_the_carry_of_earlier_launches(lib):
    """An env whose last done was in an earlier launch adds the steps since then; one with none, since reset."""
    done = np.zeros((3, 3), np.uint8)
    done[:, 0] = 1                                        # last done at step 9: adds 1 per step
    done[1, 1] = 1                                        # no done yet: adds 10 + 1 at step 11
    done[2, 2] = 1                                        # last done at step 4: adds 8 at step 12
    carry = np.array([9, -1, 4, -1, -1, -1, 3, 0, 1], np.int32)
    inc = np.zeros(3, np.int64)
    assert lib.madrl_whole_paths_steps(3, 3, 10, _p(done), _p(carry), _p(inc), None) == 0
    assert inc.tolist() == [1, 1 + 12, 1 + 8]


def test_abi_rejects_bad_arguments(lib):
    d = np.zeros((2, 2), np.uint8)
    carry, acc, inc = np.zeros(6, np.int32), np.zeros(5, np.int64), np.zeros(2, np.int64)
    st = lib.madrl_whole_paths_steps
    assert st(2, 2, 0, _p(d), _p(carry), _p(inc), None) == 0
    for args in ((0, 2, 0, _p(d), _p(carry), _p(inc)), (2, 0, 0, _p(d), _p(carry), _p(inc)),
                 (2, 2, -1, _p(d), _p(carry), _p(inc)), (2, 2, 0, None, _p(carry), _p(inc)),
                 (2, 2, 0, _p(d), None, _p(inc)), (2, 2, 0, _p(d), _p(carry), None)):
        assert st(*args, None) != 0, args
    fp = lib.madrl_whole_paths_fold_pooled
    assert fp(2, 2, 0, 4, _p(d), _p(inc), _p(carry), _p(acc), None) == 0
    for args in ((2, 2, 0, 0, _p(d), _p(inc), _p(carry), _p(acc)), (2, 2, 0, 1 << 62, _p(d), _p(inc), _p(carry), _p(acc)),
                 (0, 2, 0, 4, _p(d), _p(inc), _p(carry), _p(acc)), (2, 0, 0, 4, _p(d), _p(inc), _p(carry), _p(acc)),
                 (2, 2, -1, 4, _p(d), _p(inc), _p(carry), _p(acc)), (2, 2, 0, 4, None, _p(inc), _p(carry), _p(acc)),
                 (2, 2, 0, 4, _p(d), None, _p(carry), _p(acc)), (2, 2, 0, 4, _p(d), _p(inc), None, _p(acc)),
                 (2, 2, 0, 4, _p(d), _p(inc), _p(carry), None)):
        assert fp(*args, None) != 0, args
