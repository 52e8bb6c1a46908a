"""Whole-episode evaluation on the GPU (madrl_b200.evaluate, madrl_eval_episodes_*, Waterworld's heuristic with one
norm per env):

  * an fp64 Waterworld evaluate_heuristic reproduces rltools' evaluate_policy run by the reference's own code on
    the same streams (tests/golden/eval_ww_heuristic.npz, oracle/make_eval_golden.py);
  * the float32 joint-norm decisions are the reference's; norm="agent" leaves rollout_heuristic bit-identical;
  * the kernel equals the NumPy oracle at the C2, C3 and C5 shapes;
  * evaluate_policy equals an eager step loop plus the NumPy statistics, and neither graph capture nor the chunk
    size changes the records;
  * Pursuit's heuristic and policies, and Hostage's refusal and policies.
"""
import json
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, ROOT
from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade, evaluate_heuristic, evaluate_policy
from madrl_b200 import evaluate as ev
from oracle import eval_oracle as eo

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def same(a, b):
    return sorted(a) == sorted(b) and all(np.array_equal(np.asarray(a[k]), np.asarray(b[k])) for k in a)


def test_fp64_heuristic_evaluation_reproduces_the_reference():
    g = np.load(os.path.join(GOLDEN_DIR, "eval_ww_heuristic.npz"))
    c = json.loads(str(g["case"]))
    def engine():       # a fresh engine per run: reset() continues each env's stream, it does not re-seed
        return BatchedMAWaterWorld(c["E"], device=DEV, seed=c["seed"], env_id_base=c["env_id_base"],
                                   max_path_length=c["max_traj_len"], dtype=torch.float64, **c["config"])
    for chunk in (64, 17):
        got = evaluate_heuristic(engine(), c["n_trajs"], c["discount"], "decentralized", chunk=chunk)
        for k in ("ret", "retstd", "disc_ret"):
            assert np.abs(got[k] - g[k]).max() < 1e-9, k
        for j, k in enumerate(g["info_keys"]):
            assert np.array_equal(got[str(k)], g["info"][:, j]), k
    # the records themselves: lengths and info sums exactly, returns within 1e-9
    eng = engine()
    mpl, K = ev._plan(eng, c["n_trajs"], c["discount"], "decentralized", 64)
    rec = ev.EpisodeRecords(eng, K, c["discount"])
    o0 = eng.reset()
    _, obs, rew, done, info = eng.rollout_heuristic(K * mpl, o0, record_actions=False, norm="env")
    rec.add(rew, done, info)
    ret, qsum, ln, isum = rec.read(c["n_trajs"])
    assert np.array_equal(ln, g["ep_len"]) and np.array_equal(isum, g["ep_info"])
    assert np.abs(ret - g["ep_ret"]).max() < 1e-9


def test_fp32_env_norm_decisions_are_the_reference():
    cfg, E, T = dict(n_pursuers=5, n_evaders=5), 256, 40
    eng = BatchedMAWaterWorld(E, device=DEV, seed=9, max_path_length=25, **cfg)
    obs0 = eng.reset()
    act, obs = [x.cpu().numpy() for x in eng.rollout_heuristic(T, obs0, norm="env")[:2]]
    prev = np.concatenate([obs0.cpu().numpy()[None], obs[:-1]]).astype(np.float64)
    checked = 0
    for t in range(T):
        for e in range(E):
            want, n = eo.waterworld_env_action(prev[t, e])
            if n == 0:
                assert not act[t, e].any()
            elif n > 1e-2:
                checked += 1
                assert np.abs(want - act[t, e]).max() < 1e-5, (t, e)
    assert checked > 0.9 * T * E


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_agent_norm_leaves_rollout_heuristic_unchanged(dtype):
    cfg, E, T = dict(n_pursuers=5, n_evaders=5), 512, 48
    a = BatchedMAWaterWorld(E, device=DEV, seed=4, max_path_length=20, dtype=dtype, **cfg)
    b = BatchedMAWaterWorld(E, device=DEV, seed=4, max_path_length=20, dtype=dtype, **cfg)
    ra = a.rollout_heuristic(T, a.reset())
    n0 = b.launch_settings
    b.rollout_heuristic(3, b.reset(), norm="env")
    assert b.launch_settings == n0 + 1
    b.seed(4)
    rb = b.rollout_heuristic(T, b.reset(), norm="agent")
    assert all(torch.equal(x, y) for x, y in zip(ra, rb))
    env_run = b.rollout_heuristic(T, b.reset(), norm="env")
    assert not torch.equal(env_run[0], ra[0])


def rollout_rows(eng, T, seed):
    """rew, done, info of a T-step random-action rollout with auto-reset (horizon cuts from max_path_length)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    eng.reset()
    if eng._abi == "pursuit":
        act = torch.randint(0, 5, (T, eng.n_envs, eng._n_acting), generator=g, device=DEV, dtype=torch.int32)
    else:
        act = torch.randn((T, eng.n_envs, eng._n_acting, 2), generator=g, device=DEV, dtype=eng.dtype)
    return eng.rollout(act)[1:]


@pytest.mark.parametrize("shape", ["c2", "c3", "c5"])
def test_kernel_matches_the_oracle_at_product_shapes(shape):
    # T = 3 max_path_length + a few steps, so that every env completes K = 3 episodes; cut into launches of `ch`
    if shape == "c2":
        eng = BatchedMAWaterWorld(4096, n_pursuers=5, n_evaders=5, device=DEV, seed=1, max_path_length=37)
        T, ch = 120, 40
    elif shape == "c3":
        eng = pursuit(65536, seed=2, max_path_length=9)
        T, ch = 30, 11
    else:
        eng = BatchedHostageWorld(8192, 10, 16, 16, 4, 2, device=DEV, seed=3, max_path_length=39)
        T, ch = 120, 40
    K, disc = 3, 0.99
    rew, done, info = rollout_rows(eng, T, 5)
    rec = ev.EpisodeRecords(eng, K, disc)
    for t0 in range(0, T, ch):
        rec.add(rew[t0:t0 + ch], done[t0:t0 + ch], info[t0:t0 + ch])
    got = rec.read(K * eng.n_envs)
    E, A, C = eng.n_envs, eng._n_acting, rec.C
    r, d, i = rew.cpu().numpy(), done.cpu().numpy(), info.cpu().numpy().reshape(T, E, C)
    carry, want = eo.new_carry(E, A), eo.new_records(E, A, C, K)
    eo.eval_episodes(r, d, i, disc, K, carry, want)
    assert np.array_equal(got[2], want[2]) and np.array_equal(got[3], want[3])
    assert (want[2] > 0).all(), "every env must complete K episodes"
    # every float64 operation is rounded on its own, in the oracle's order: the records are its bits
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


class Linear(object):
    """A fixed deterministic policy: tanh of a linear map of the observation."""

    def __init__(self, D, seed):
        self.W = torch.randn(D, 2, generator=torch.Generator().manual_seed(seed)).to(DEV) * 0.1

    def __call__(self, obs, state):
        return torch.tanh(obs @ self.W.to(obs.dtype)), {}, state


def eager_statistics(eng, policy, n_trajs, disc, mode):
    """An eager step loop over the same K * max_path_length steps and the NumPy statistics of its episodes."""
    mpl, K = ev._plan(eng, n_trajs, disc, mode, 64)
    obs = eng.reset()
    rews, dones, infos = [], [], []
    for _ in range(K * mpl):
        a = policy(obs, None)[0]
        obs, r, d, info = eng.step(a, auto_reset=True)
        rews.append(r.cpu().numpy()); dones.append(d.cpu().numpy())
        infos.append(np.stack([info[k].cpu().numpy() for k in eng._info_keys], -1))
    rew, done, info = np.array(rews), np.array(dones), np.array(infos)
    E = eng.n_envs
    per_env = [[] for _ in range(E)]
    for e in range(E):
        s = 0
        for t in range(len(done)):
            if done[t, e]:
                per_env[e].append((rew[s:t + 1, e].astype(np.float64), info[s:t + 1, e].sum(0)))
                s = t + 1
    eps = [per_env[e][k] for k in range(K) for e in range(E)][:n_trajs]
    return eo.reference_statistics(eps, disc, mode, eng._info_keys)


@pytest.mark.parametrize("mode", ["decentralized", "centralized"])
def test_evaluate_policy_equals_an_eager_loop(mode):
    kw = dict(n_pursuers=3, n_evaders=4, max_path_length=23, reward_mech="global" if mode == "centralized" else "local")
    pol = Linear(BatchedMAWaterWorld(1, device=DEV, **kw).obs_dim, 0)
    got = evaluate_policy(BatchedMAWaterWorld(6, device=DEV, seed=8, **kw), pol, 10, 0.97, mode, chunk=16)
    want = eager_statistics(BatchedMAWaterWorld(6, device=DEV, seed=8, **kw), pol, 10, 0.97, mode)
    assert sorted(got) == sorted(want)
    for k in want:
        assert np.allclose(got[k], want[k], rtol=1e-9, atol=1e-12), (k, got[k], want[k])


def test_graph_eager_and_chunk_sizes_give_the_same_records():
    kw = dict(n_pursuers=5, n_evaders=5, max_path_length=30)
    pol = Linear(BatchedMAWaterWorld(1, device=DEV, **kw).obs_dim, 1)
    runs = []
    for graph, chunk in ((True, 64), (False, 64), (True, 7), (True, 90)):
        eng = BatchedMAWaterWorld(64, device=DEV, seed=12, **kw)
        runs.append(evaluate_policy(eng, pol, 100, 0.99, "decentralized", chunk=chunk, graph=graph))
    assert all(same(runs[0], r) for r in runs[1:])
    # the same through the wrappers: frame stack and standardiser, started as PolicyRollout describes
    from madrl_b200.postproc import Standardizer
    pol4 = Linear(BatchedMAWaterWorld(1, device=DEV, **kw).obs_dim * 3, 2)
    wrapped = lambda o, s: pol4(o.reshape(o.shape[0], o.shape[1], -1), s)  # noqa: E731
    outs = []
    for chunk in (64, 11):
        eng = BatchedMAWaterWorld(64, device=DEV, seed=12, **kw)
        std = Standardizer(64, 5, eng.obs_dim, DEV, enable_obsnorm=True)
        outs.append(evaluate_policy(eng, wrapped, 100, 0.99, "decentralized", chunk=chunk, frame_stack=3,
                                    standardizer=std))
    assert same(*outs)


def pursuit(E, **kw):
    return BatchedPursuitEvade(E, np.load(os.path.join(ROOT, "maps", "map_pool16.npy")), n_evaders=30, n_pursuers=8,
                               obs_range=7, surround=True, sample_maps=True, device=DEV, **kw)


def test_pursuit_heuristic_and_policy():
    got = evaluate_heuristic(pursuit(32, seed=6, max_path_length=40), 50, 0.99, "decentralized", chunk=24)
    eng = pursuit(32, seed=6, max_path_length=40)
    _, obs, rew, done, info = eng.rollout_heuristic(2 * 40, eng.reset(), record_actions=False)
    r, d, i = rew.cpu().numpy(), done.cpu().numpy(), info.cpu().numpy()[..., None]
    recs = eo.new_records(32, 8, 1, 2)
    eo.eval_episodes(r, d, i, 0.99, 2, eo.new_carry(32, 8), recs)
    want = ev.statistics(recs[0][:50], recs[1][:50], recs[2][:50], recs[3][:50], "decentralized", ("removed",))
    assert sorted(got) == sorted(want)
    for k in want:
        assert np.allclose(got[k], want[k], rtol=1e-12, atol=0), k
    W = torch.randn(pursuit(1).obs_dim, 5, generator=torch.Generator().manual_seed(3)).to(DEV)
    pol = lambda o, s: ((o.reshape(o.shape[0], o.shape[1], -1) @ W).argmax(-1), {}, s)  # noqa: E731
    a = evaluate_policy(pursuit(16, seed=2, max_path_length=25), pol, 40, 0.95, "decentralized", chunk=16)
    b = evaluate_policy(pursuit(16, seed=2, max_path_length=25), pol, 40, 0.95, "decentralized", chunk=64, graph=False)
    assert same(a, b) and np.all(a["removed"] >= 0)


def test_hostage_has_no_heuristic_but_evaluates_policies():
    eng = BatchedHostageWorld(8, 10, 16, 16, 4, 2, device=DEV, seed=1, max_path_length=15, dtype=torch.float64)
    with pytest.raises(ValueError, match="Hostage"):
        evaluate_heuristic(eng, 8, 0.99, "decentralized")
    pol = Linear(eng.obs_dim, 4)
    got = evaluate_policy(eng, pol, 12, 0.99, "centralized", chunk=8)
    want = eager_statistics(BatchedHostageWorld(8, 10, 16, 16, 4, 2, device=DEV, seed=1, max_path_length=15,
                                                dtype=torch.float64), pol, 12, 0.99, "centralized")
    for k in want:
        assert np.allclose(got[k], want[k], rtol=1e-9, atol=1e-12), k
