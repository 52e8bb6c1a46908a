"""ReplayPool (madrl_b200/replay.py, csrc/replay.cu) on the GPU against oracle/replay_oracle.py.

* Pools filled from real rollouts equal the oracle's host pool built from the same tensors, bit for bit: ring
  contents, counters and rewards.  Waterworld at C2's shape (4096 envs x 5 pursuers) and Hostage at C5's agent
  counts, with a max_path_length that cuts several paths inside each rollout and set_terminal_obs, in float32 and
  bfloat16, both values of include_horizon_terminal_transitions, a pool that one rollout overfills; one case runs
  through PolicyRollout.
* random_batch / random_batches indices equal the oracle's Philox indices and the rows are the pool's rows there.
* Uniformity: chi-square over the slots of a small pool before and after it fills (fixed seeds, fixed threshold).
* add + random_batches captured in a CUDA graph and replayed three times equal the eager sequence.
* A bfloat16 pool of more than 2^31 elements, inserted across its wrap and sampled at its far end (64-bit offsets).
"""
import numpy as np
import pytest
import torch

from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, PolicyRollout, ReplayPool
from oracle import replay_oracle as ro

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
WW = dict(n_pursuers=5, n_evaders=5, n_poison=10, n_sensors=30)
HW = (10, 16, 16, 4, 2)


def host(x):
    """A device tensor as NumPy; bfloat16 as its uint16 bits."""
    if x.dtype == torch.bfloat16:
        x = x.view(torch.int16)
        return x.cpu().numpy().view(np.uint16)
    return x.cpu().numpy()


def oracle_for(pool):
    w = np.uint16 if pool.obs_dtype == torch.bfloat16 else np.float32
    return ro.ReplayOracle(pool.max_pool_size, pool.obs_dim, pool.action_dim, obs_dtype=w,
                           scale_reward=pool.scale_reward,
                           include_horizon_terminal_transitions=pool.include_horizon_terminal_transitions)


def assert_pool_equal(pool, orc):
    for name in ("observations", "next_observations", "actions", "rewards", "terminals"):
        got = host(getattr(pool, name))
        assert np.array_equal(got.view(np.uint8), getattr(orc, name).view(np.uint8)), name
    st = pool.get_state()
    assert (st["top"], st["bottom"], st["size"], st["draws"]) == (orc.top, orc.bottom, orc.size, orc.draws)


def open_loop_adds(eng, pool, orc, T, rounds, seed, timestep0=None):
    """`rounds` auto-reset rollouts with random actions, each added to the pool and to the oracle; `timestep0`: the
    envs' timestep counter after the reset."""
    E, A, D = eng.n_envs, eng._n_acting, eng.obs_dim
    g = torch.Generator(device=DEV).manual_seed(seed)
    prev = eng.reset()
    if timestep0 is not None:
        eng.state["timestep"].fill_(timestep0)
    term = torch.zeros((T, E, A, D), dtype=eng.obs_dtype, device=DEV)
    eng.set_terminal_obs(term)
    cuts = 0
    for _ in range(rounds):
        pl0 = eng.state["path_len"].clone()
        ts0 = eng.state["timestep"].clone()
        act = torch.randn((T, E, A, 2), generator=g, device=DEV)
        obs, rew, done, _ = eng.rollout(act)
        pool.add(obs, act, rew, done, prev, term, pl0, ts0, eng.cfg.max_path_length, eng.timestep_limit)
        args = [host(x) for x in (obs, act, rew, done, prev, term, pl0, ts0)]
        orc.add(*args, eng.cfg.max_path_length, eng.timestep_limit)
        keep = ro.keep_flags(args[3], args[6], args[7], eng.cfg.max_path_length, eng.timestep_limit, False)
        cuts += int((keep == 0).sum())
        prev = obs[-1].clone()
        torch.cuda.synchronize()
        assert_pool_equal(pool, orc)
    return cuts


@pytest.mark.parametrize("include", [False, True], ids=["drop_cuts", "keep_cuts"])
@pytest.mark.parametrize("obs_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_waterworld_c2_rollouts_equal_the_oracle(obs_dtype, include):
    eng = BatchedMAWaterWorld(4096, device=DEV, seed=3, max_path_length=7, obs_dtype=obs_dtype, **WW)
    # 24 x 4096 x 5 = 491 520 transitions a rollout: the pool of 150 000 wraps inside every add
    pool = ReplayPool(150000, 5, eng.obs_dim, 2, DEV, obs_dtype=obs_dtype, scale_reward=0.01,
                      include_horizon_terminal_transitions=include, seed=11)
    orc = oracle_for(pool)
    assert open_loop_adds(eng, pool, orc, 24, 2, seed=5) > 4096 * 4   # several horizon cuts per env
    idx, want = orc.random_batches(11, 3, 12000)
    got = pool.random_batches(3, 12000)
    assert np.array_equal(host(got["indices"]), idx)
    for k, v in want.items():
        assert np.array_equal(host(got[k]).view(np.uint8), v.view(np.uint8)), k


def test_waterworld_small_pool_and_timestep_limit():
    """A pool smaller than one step's transitions, and paths that end at the env's own timestep limit (reset
    counters near it), where the horizon rule must not cut."""
    eng = BatchedMAWaterWorld(300, device=DEV, seed=8, max_path_length=5, **WW)
    pool = ReplayPool(777, 5, eng.obs_dim, 2, DEV, scale_reward=0.5)
    orc = oracle_for(pool)
    open_loop_adds(eng, pool, orc, 9, 3, seed=9, timestep0=eng.timestep_limit - 3)


@pytest.mark.parametrize("obs_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
def test_hostage_rollouts_equal_the_oracle(obs_dtype):
    eng = BatchedHostageWorld(2048, *HW, device=DEV, seed=4, max_path_length=6, obs_dtype=obs_dtype)
    pool = ReplayPool(200000, 10, eng.obs_dim, 2, DEV, obs_dtype=obs_dtype, seed=2)
    orc = oracle_for(pool)
    assert open_loop_adds(eng, pool, orc, 16, 2, seed=6) > 0
    for B in (1000, 4097):
        idx, want = orc.random_batches(2, 1, B)
        got = pool.random_batch(B)
        assert np.array_equal(host(got["indices"]), idx[0])
        for k, v in want.items():
            assert np.array_equal(host(got[k]).view(np.uint8), v[0].view(np.uint8)), k


def test_policy_rollout_feeds_the_pool():
    E, T = 512, 20
    eng = BatchedMAWaterWorld(E, device=DEV, seed=1, max_path_length=6, **WW)
    D = eng.obs_dim
    term = torch.zeros((T, E, 5, D), device=DEV)
    eng.set_terminal_obs(term)
    W = torch.randn(D, 2, generator=torch.Generator().manual_seed(0)).to(DEV) * 0.1
    ro_ = PolicyRollout(eng, lambda o, s: (torch.tanh(o @ W), {}, s), T)
    pool = ReplayPool(30000, 5, D, 2, DEV)
    orc = oracle_for(pool)
    prev = eng.reset()
    for _ in range(2):
        pl0, ts0 = eng.state["path_len"].clone(), eng.state["timestep"].clone()
        r = ro_(prev)
        pool.add(r.obs, r.actions, r.rew, r.done, prev, term, pl0, ts0, 6, eng.timestep_limit)
        orc.add(*[host(x) for x in (r.obs, r.actions, r.rew, r.done, prev, term, pl0, ts0)], 6, eng.timestep_limit)
        prev = r.obs[-1].clone()
        torch.cuda.synchronize()
        assert_pool_equal(pool, orc)
    assert host(r.done).any()


def filled_pool(M, n, seed=0, D=3):
    """A pool of M slots holding n transitions of distinct rows (one env, one agent, no done)."""
    pool = ReplayPool(M, 1, D, 1, DEV, seed=seed)
    obs = torch.arange(n * D, dtype=torch.float32, device=DEV).view(n, 1, 1, D)
    z = torch.zeros(1, dtype=torch.int32, device=DEV)
    pool.add(obs, torch.zeros(n, 1, 1, 1, device=DEV), torch.ones(n, 1, 1, device=DEV),
             torch.zeros(n, 1, dtype=torch.uint8, device=DEV), torch.zeros(1, 1, D, device=DEV), torch.zeros_like(obs),
             z, z, 0, 10 ** 9)
    return pool


def test_uniform_over_all_but_the_newest_slot():
    """Chi-square of 400 000 draws over the slots [0, size - 1), on a pool of 64 before (size 40) and after it
    fills; no draw outside that range."""
    from scipy.stats import chisquare
    for n, seed in ((40, 1), (100, 2)):
        pool = filled_pool(64, n, seed=seed)
        size = pool.size
        idx = host(pool.random_batches(40, 10000)["indices"]).reshape(-1)
        assert idx.min() >= 0 and idx.max() < size - 1
        counts = np.bincount(idx, minlength=size - 1)
        assert chisquare(counts).pvalue > 1e-3, (n, counts)
        assert np.array_equal(idx, ro.sample_indices(seed, 0, idx.size, size))


def test_random_batch_needs_more_than_batch_size():
    pool = filled_pool(64, 10)
    with pytest.raises(ValueError):
        pool.random_batch(10)
    assert pool.random_batch(9)["observations"].shape == (9, 3)
    with pytest.raises(NotImplementedError):
        ReplayPool(10, 1, 1, 1, DEV, mode="centralized")


def test_graph_capture_replays_equal_the_eager_sequence():
    E, A, D, T = 256, 5, 37, 6
    rs = np.random.RandomState(0)
    rounds = []
    for _ in range(3):
        done = (rs.rand(T, E) < 0.2).astype(np.uint8)
        rounds.append([torch.as_tensor(x, device=DEV) for x in (
            rs.randn(T, E, A, D).astype(np.float32), rs.randn(T, E, A, 2).astype(np.float32),
            rs.randn(T, E, A).astype(np.float32), done, rs.randn(E, A, D).astype(np.float32),
            rs.randn(T, E, A, D).astype(np.float32), rs.randint(0, 5, E).astype(np.int32),
            rs.randint(0, 50, E).astype(np.int32))])

    def make():
        return ReplayPool(3000, A, D, 2, DEV, seed=77)

    eager, outs = make(), []
    for r in rounds:
        eager.add(*r, 5, 60)
        outs.append({k: v.clone() for k, v in eager.random_batches(4, 500).items()})
    pool = make()
    static = [torch.zeros_like(x) for x in rounds[0]]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        pool.add(*static, 5, 60)
        batch = pool.random_batches(4, 500)
    assert pool.get_state() == dict(top=0, bottom=0, size=0, draws=0)   # capture ran nothing
    for r, want in zip(rounds, outs):
        for d, x in zip(static, r):
            d.copy_(x)
        g.replay()
        for k, v in want.items():
            assert torch.equal(batch[k], v), k
    assert pool.get_state() == eager.get_state()
    for name in ("observations", "next_observations", "actions", "rewards", "terminals"):
        assert torch.equal(getattr(pool, name), getattr(eager, name)), name


def test_far_end_of_a_pool_beyond_2_31_elements():
    """bfloat16, D = 4, M = 2^29 + 1000 slots: M * D > 2^31.  An add starting 300 slots before the end wraps; the
    rows land at (top + j) mod M, and draws reach the far end."""
    M, D, E, A, T = (1 << 29) + 1000, 4, 64, 2, 5
    pool = ReplayPool(M, A, D, 1, DEV, obs_dtype=torch.bfloat16, seed=5)
    top = M - 300
    pool.set_state(dict(top=top, bottom=top, size=M, draws=0))
    rs = np.random.RandomState(1)
    bits = lambda *s: torch.as_tensor(rs.randint(0, 1 << 15, size=s).astype(np.int16), device=DEV).view(  # noqa
        torch.bfloat16)
    r = [bits(T, E, A, D), torch.as_tensor(rs.randn(T, E, A, 1).astype(np.float32), device=DEV),
         torch.as_tensor(rs.randn(T, E, A).astype(np.float32), device=DEV),
         torch.as_tensor((rs.rand(T, E) < 0.3).astype(np.uint8), device=DEV), bits(E, A, D), bits(T, E, A, D),
         torch.zeros(E, dtype=torch.int32, device=DEV), torch.zeros(E, dtype=torch.int32, device=DEV)]
    pool.add(*r, 0, 1000)
    K = T * E * A
    orc = ro.ReplayOracle(K, D, 1, obs_dtype=np.uint16, scale_reward=pool.scale_reward)
    orc.add(*[host(x) for x in r], 0, 1000)
    slots = torch.as_tensor((top + np.arange(K)) % M, device=DEV)
    for name in ("observations", "next_observations", "actions", "rewards", "terminals"):
        got = host(getattr(pool, name).index_select(0, slots))
        assert np.array_equal(got.view(np.uint8), getattr(orc, name).view(np.uint8)), name
    assert pool.get_state() == dict(top=(top + K) % M, bottom=(top + K) % M, size=M, draws=0)
    b = pool.random_batches(2, 50000)
    idx = host(b["indices"]).reshape(-1)
    assert np.array_equal(idx, ro.sample_indices(5, 0, idx.size, M))
    assert idx.max() > M - M // 1000
    i = b["indices"].reshape(-1)
    assert torch.equal(b["observations"].reshape(-1, D), pool.observations.index_select(0, i))
    assert torch.equal(b["next_observations"].reshape(-1, D), pool.next_observations.index_select(0, i))
    assert torch.equal(b["rewards"].reshape(-1), pool.rewards.index_select(0, i))
