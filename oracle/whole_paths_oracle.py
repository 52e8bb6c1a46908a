"""CPU oracle (TEST INFRASTRUCTURE) of the whole-path selection of madrl_b200.whole_paths (DESIGN §4.9): rllab's
``BatchMASampler.obtain_samples`` with ``whole_paths=True`` (batch_ma_sampler.py:40-57, ma_sampler.py:52-100,
stateful_pool.py:102-190) restated for E lockstep envs over a scripted continuing auto-reset stream.

Every env is reset at step 0.  After each step the paths that ended there (``done``) add their env-steps to one
count; t* is the first step at which it reaches ``batch_size``.  Env e keeps its steps 0 .. end_e, end_e = its first
done at or after t*.  The batch is env-major: env 0's rows, then env 1's, ...
"""
import numpy as np


def select(done, batch_size):
    """done [S, E] (a stream from reset) -> (t_star, end [E]), or None if the stream ends before the batch does."""
    done = np.asarray(done).astype(bool)
    S, E = done.shape
    last = np.full(E, -1, np.int64)
    count, t_star = 0, -1
    for t in range(S):
        d = done[t]
        count += int(np.sum(t - last[d]))
        last[d] = t
        if count >= batch_size:
            t_star = t
            break
    if t_star < 0:
        return None
    end = np.full(E, -1, np.int64)
    for e in range(E):
        hits = np.nonzero(done[t_star:, e])[0]
        if len(hits) == 0:
            return None
        end[e] = t_star + hits[0]
    return t_star, end


def rows(end):
    """(step, env) of every kept row, in batch order."""
    return [(t, e) for e in range(len(end)) for t in range(int(end[e]) + 1)]


def gather(x, end, first=None):
    """x [S, E, ...] -> its kept rows [N, ...]; `first` [E, ...]: the rows are shifted by one step (row (t, e) reads
    x[t-1, e], first[e] at t = 0), as the policy's observations are."""
    x = np.asarray(x)
    out = []
    for t, e in rows(end):
        out.append(x[t - 1, e] if (first is not None and t > 0) else (first[e] if first is not None else x[t, e]))
    return np.stack(out)


def path_start(done, end):
    """int32 [P + 1]: the first row of each kept path, then N."""
    flat = gather(np.asarray(done).astype(bool), end)
    return np.concatenate([[0], np.nonzero(flat)[0] + 1]).astype(np.int32)


# ---- the same selection as NumPy fancy indexing, for batches of millions of rows (the loops above take minutes)

def rows_index(end):
    """(t, e) int64 [N]: `rows(end)` as two index arrays."""
    n = np.asarray(end, np.int64) + 1
    e = np.repeat(np.arange(len(n)), n)
    t = np.arange(int(n.sum())) - np.repeat(np.cumsum(n) - n, n)
    return t, e


def take(x, end, first=None):
    """`gather(x, end, first)` by fancy indexing."""
    t, e = rows_index(end)
    x = np.asarray(x)
    if first is None:
        return x[t, e]
    out = x[np.maximum(t - 1, 0), e]
    out[t == 0] = np.asarray(first)[e[t == 0]]
    return out


def path_start_np(done, end):
    """`path_start(done, end)` by fancy indexing."""
    flat = take(np.asarray(done).astype(bool), end)
    return np.concatenate([[0], np.nonzero(flat)[0] + 1]).astype(np.int32)


def env_rows(end):
    """int32 [E]: the first row of each env's paths."""
    n = np.asarray(end, np.int64) + 1
    return (np.cumsum(n) - n).astype(np.int32)
