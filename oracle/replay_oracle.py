"""rllab's DDPG replay pool restated in NumPy (TEST INFRASTRUCTURE).

``MAReplayPool`` (rllab/rllab/algos/ddpg.py:85-145) as ``DDPG.train`` fills it in decentralized mode
(:285-353), for a batch of envs stepped in lockstep: the transitions of a rollout are added in (t, env, agent)
order, each env continuing its own path; a horizon cut (a done step at path length >= max_path_length of an env
that did not terminate by itself, :310) is dropped unless ``include_horizon_terminal_transitions``, and stored with
terminal = 1 otherwise.  The ring keeps ``top`` / ``bottom`` / ``size`` as ``add_sample`` does (:106-116).

Deliberate differences from the reference, shared with madrl_b200.replay.ReplayPool:
  * rewards are float32(float64(r) * scale_reward), rounded once; the reference keeps float64;
  * sampled rows return the stored next observations (the reference returns the observations, :140);
  * indices are drawn uniformly over [0, size - 1) -- the set the reference's rejection loop accepts, which
    tests/golden/replay_pool_ref.npz pins on the reference's own code -- from the Philox stream below, not from
    np.random.randint.

The sampler's stream: draw c (c = the pool's draw counter + row) is Philox4x32-10 of counter (c & 0xffffffff,
c >> 32, 0, TAG) under key (seed & 0xffffffff, seed >> 32); its words 1:0 form a 64-bit u, and the slot is the high
64 bits of u * max(size - 1, 1).
"""
import numpy as np

from oracle.philox import philox_block_numpy

TAG = 2
M32 = np.uint64(0xFFFFFFFF)


def check_mode(mode):
    """The reference's DDPG raises for concurrent mode (ddpg.py:307-308), and its centralized branch stores the
    summed reward of one joint action (:338), which these envs' per-agent reward vectors cannot feed."""
    if mode != "decentralized":
        raise NotImplementedError("the replay pool supports decentralized mode only, got %r" % (mode,))


def keep_flags(done, path_len0, timestep0, max_path_length, timestep_limit, include_horizon):
    """uint8 [T, E]: which (t, e) transitions DDPG.train adds; the paths continue from the engine's counters."""
    T, E = done.shape
    pl = np.array(path_len0, np.int64).copy()
    ts = np.array(timestep0, np.int64).copy()
    keep = np.zeros((T, E), np.uint8)
    for t in range(T):
        d = done[t] != 0
        pl += 1
        ts += 1
        cut = d & (max_path_length > 0) & (pl >= max_path_length) & (ts < timestep_limit)
        keep[t] = ~cut | bool(include_horizon)
        pl[d] = 0
        ts[d] = 0
    return keep


def scaled_reward(r, scale_reward):
    return (np.asarray(r, np.float32).astype(np.float64) * scale_reward).astype(np.float32)


def mulhi64(u, n):
    """High 64 bits of u * n for uint64 arrays (32-bit partial products, as the kernel computes them)."""
    u = np.asarray(u, np.uint64)
    n = np.uint64(n)
    s = np.uint64(32)
    a_lo, a_hi, b_lo, b_hi = u & M32, u >> s, n & M32, n >> s
    lo_lo, hi_lo, lo_hi, hi_hi = a_lo * b_lo, a_hi * b_lo, a_lo * b_hi, a_hi * b_hi
    mid = (lo_lo >> s) + (hi_lo & M32) + lo_hi
    return hi_hi + (hi_lo >> s) + (mid >> s)


def sample_indices(seed, counter, rows, size):
    """int64 [rows]: the slots of draws counter .. counter + rows - 1 of a pool of `size` transitions."""
    c = np.arange(counter, counter + rows, dtype=np.uint64)
    w = philox_block_numpy(c, 0, TAG, int(seed)).astype(np.uint64)
    u = (w[..., 1] << np.uint64(32)) | w[..., 0]
    return mulhi64(u, max(int(size) - 1, 1)).astype(np.int64)


def accepted_candidates(bottom, size, max_pool_size):
    """The indices MAReplayPool.random_batch keeps (:122-128): every candidate of randint(bottom, bottom + size),
    taken mod max_pool_size, but index == size - 1."""
    cand = np.arange(bottom, bottom + size) % max_pool_size
    return np.unique(cand[cand != size - 1])


class ReplayOracle(object):
    """MAReplayPool with float32 rewards and actions; `obs_dtype` np.float32, or np.uint16 for bfloat16 bits."""

    def __init__(self, max_pool_size, obs_dim, action_dim, obs_dtype=np.float32, scale_reward=0.1,
                 include_horizon_terminal_transitions=False, mode="decentralized"):
        check_mode(mode)
        M = int(max_pool_size)
        self.max_pool_size, self.scale_reward = M, scale_reward
        self.include_horizon = bool(include_horizon_terminal_transitions)
        self.observations = np.zeros((M, obs_dim), obs_dtype)
        self.next_observations = np.zeros((M, obs_dim), obs_dtype)
        self.actions = np.zeros((M, action_dim), np.float32)
        self.rewards = np.zeros(M, np.float32)
        self.terminals = np.zeros(M, np.uint8)
        self.top = self.bottom = self.size = 0
        self.draws = 0

    def add_sample(self, observation, action, reward, next_observation, terminal):
        """ddpg.py:106-116."""
        self.observations[self.top] = observation
        self.next_observations[self.top] = next_observation
        self.actions[self.top] = action
        self.rewards[self.top] = reward
        self.terminals[self.top] = terminal
        self.top = (self.top + 1) % self.max_pool_size
        if self.size >= self.max_pool_size:
            self.bottom = (self.bottom + 1) % self.max_pool_size
        else:
            self.size += 1

    def add(self, obs, act, rew, done, obs_before, term, path_len0, timestep0, max_path_length, timestep_limit):
        """Every kept transition of one rollout: obs [T, E, A, D], act [T, E, A, Ad], rew [T, E, A], done [T, E],
        obs_before [E, A, D], term [T, E, A, D].  Only the transitions that land in the ring are gathered (the last
        max_pool_size), so the result is K add_sample calls without building all K rows."""
        T, E, A = rew.shape
        keep = keep_flags(done, path_len0, timestep0, max_path_length, timestep_limit, self.include_horizon)
        t, e = np.nonzero(keep)                      # step-major, then env
        t = np.repeat(t, A)
        e = np.repeat(e, A)
        a = np.tile(np.arange(A), len(t) // A if A else 0)
        K, M = len(t), self.max_pool_size
        first = max(K - M, 0)
        t, e, a = t[first:], e[first:], a[first:]
        slots = (self.top + np.arange(first, K)) % M
        d = done[t, e] != 0
        prev = np.where((t == 0)[:, None], obs_before[e, a], obs[np.maximum(t - 1, 0), e, a])
        nxt = np.where(d[:, None], term[t, e, a], obs[t, e, a])
        self.observations[slots] = prev
        self.next_observations[slots] = nxt
        self.actions[slots] = act[t, e, a]
        self.rewards[slots] = scaled_reward(rew[t, e, a], self.scale_reward)
        self.terminals[slots] = d
        over = max(self.size + K - M, 0)
        self.top = (self.top + K) % M
        self.bottom = (self.bottom + over) % M
        self.size = min(self.size + K, M)
        return K

    def random_batches(self, seed, n, batch_size):
        """int64 [n, batch_size] slots of the next n minibatches, and the rows gathered from them."""
        idx = sample_indices(seed, self.draws, n * batch_size, self.size).reshape(n, batch_size)
        self.draws += n * batch_size
        return idx, dict(observations=self.observations[idx], actions=self.actions[idx], rewards=self.rewards[idx],
                         terminals=self.terminals[idx], next_observations=self.next_observations[idx])
