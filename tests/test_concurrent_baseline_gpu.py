"""Per-agent (concurrent-mode) LinearFeatureBaseline on the GPU: real auto-reset rollouts of the three families
against the NumPy oracle (oracle/concurrent_baseline_oracle.py), process_samples_concurrent in both flavours
against the oracle chain, the full C4 launch against the chunked PyTorch float64 Gram of each agent,
determinism, memory, bfloat16, A = 1 against the pooled path and the distributed fit."""
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import baseline_oracle as bo
from oracle import concurrent_baseline_oracle as cbo

pytestmark = pytest.mark.gpu

PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
DISCOUNT, GAE_LAMBDA = 0.99, 0.97


def make(family, E, **kw):
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    kw = dict(dict(seed=13, device="cuda"), **kw)
    if family == "ww":
        return BatchedMAWaterWorld(E, 5, 5, n_poison=10, n_sensors=30, **kw)
    if family == "pe":
        return BatchedPursuitEvade(E, np.load(os.path.join(ROOT, "maps", "map_pool16.npy")), **PE_C3, **kw)
    return BatchedHostageWorld(E, 10, 16, 16, 4, 2, **kw)


def actions(eng, T, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    shape = (T, eng.n_envs, eng._n_acting) + eng._act_tail
    if eng._act_dtype == torch.int32:
        return torch.randint(0, 5, shape, dtype=torch.int32, device="cuda", generator=g)
    return torch.randn(shape, device="cuda", generator=g) * 0.5


def returns_of(rew, done):
    from madrl_b200.postproc import gae
    return gae(rew.float(), torch.zeros_like(rew, dtype=torch.float32), done, DISCOUNT, 1.0)[1]


def check_gram(G, G_ref):
    d = np.sqrt(np.outer(np.diag(G_ref), np.diag(G_ref)))
    err = np.abs(G - G_ref)
    assert np.all(err <= 1e-12 * d), (err / np.maximum(d, 1e-300)).max()


def check_predict(vals, F, c):
    want = F.dot(c)
    tol = np.spacing(np.abs(want.astype(np.float32))) + 1e-12 * np.abs(F * c).sum(axis=1)
    assert np.all(np.abs(vals.reshape(-1).astype(np.float64) - want) <= tol)


def chained_launches(family, E, T, n=2):
    """n consecutive auto-reset launches (max_path_length 7): obs_before = the previous launch's last observations,
    t0 = state['path_len'] read before each launch."""
    eng = make(family, E, max_path_length=7)
    obs_before = eng.reset()
    out = []
    for launch in range(n):
        t0 = eng.state["path_len"].clone()
        obs, rew, done, _ = eng.rollout(actions(eng, T, launch))
        assert done.any() and (launch == 0 or t0.any())
        out.append(dict(obs=obs, obs_before=obs_before, done=done, rew=rew.float(), t0=t0))
        obs_before = obs[-1].clone()
    return out


def host(it):
    return {k: v.cpu().numpy() for k, v in it.items()}


FAMILIES = [("ww", 400, 30), ("pe", 600, 16), ("hw", 400, 20)]       # 5, 8 and 10 agents


@pytest.mark.parametrize("family,E,T", FAMILIES)
def test_real_rollouts_per_agent_fit_and_predict_match_oracle(family, E, T):
    from madrl_b200.postproc import LinearFeatureBaseline
    its = chained_launches(family, E, T)
    A, D = its[0]["obs"].shape[2], its[0]["obs"].shape[3]
    assert A in (5, 8, 10)
    b = LinearFeatureBaseline(D, "cuda", n_agents=A)
    for it in its:
        ret = returns_of(it["rew"], it["done"])
        kw = dict(obs_before=it["obs_before"], t0=it["t0"])
        G = b.normal_equations(it["obs"], it["done"], ret, **kw).cpu().numpy()
        h = host(it)
        F = cbo.agent_features(h["obs"], h["done"], h["obs_before"], h["t0"])
        y = ret.cpu().numpy().astype(np.float64)
        b.fit(it["obs"], it["done"], ret, **kw)
        c = b.get_param_values()
        assert c.shape == (A, 2 * D + 4)
        vals = b.predict(it["obs"], it["done"], **kw).cpu().numpy()
        for a in range(A):
            ya = y[:, :, a].reshape(-1)
            check_gram(G[a], bo.normal_equations(F[a], ya))
            obj, obj_np = bo.objective(F[a], ya, c[a]), bo.objective(F[a], ya, bo.fit(F[a], ya))
            assert obj <= obj_np * (1 + 1e-8), (a, obj, obj_np)
            check_predict(vals[:, :, a], F[a], c[a])


def _device_fits(b):
    """The coefficients this call's fit produced, [A, Df]: the held rows (independent), or the held rows 1..A-1
    plus the carried row A-1 (shared)."""
    held = b.get_param_values()
    return np.concatenate([held[1:], b.carry[None]]) if b.shared else held


@pytest.mark.parametrize("shared", [False, True], ids=["independent", "shared"])
@pytest.mark.parametrize("family,E,T", FAMILIES)
def test_process_samples_concurrent_matches_oracle_chain(family, E, T, shared):
    """Values, returns, per-agent centred advantages and explained variances against the oracle chain run with the
    device's own fits (its Cholesky solution differs from lstsq in the last digits); each fit minimises rllab's
    objective as well as NumPy's."""
    from madrl_b200.postproc import LinearFeatureBaseline, process_samples_concurrent
    its = chained_launches(family, E, T)
    A, D = its[0]["obs"].shape[2], its[0]["obs"].shape[3]
    b = LinearFeatureBaseline(D, "cuda", n_agents=A, shared=shared)
    got, fits = [], []
    for it in its:
        values, adv, ret, ev = process_samples_concurrent(b, it["obs"], it["done"], it["rew"], DISCOUNT, GAE_LAMBDA,
                                                          obs_before=it["obs_before"], t0=it["t0"],
                                                          positive_adv=True)
        got.append((values.cpu().numpy(), adv.cpu().numpy(), ret.cpu().numpy(), np.array(ev)))
        fits.append(_device_fits(b))
    hs = [host(it) for it in its]
    chain = cbo.concurrent_chain(hs, shared, DISCOUNT, GAE_LAMBDA, positive_adv=True, fits=fits)
    for n, (h, res) in enumerate(zip(hs, chain)):
        values, adv, ret, ev = got[n]
        F = cbo.agent_features(h["obs"], h["done"], h["obs_before"], h["t0"])
        rows, _ = cbo.agent_path_rows(h["done"])
        for a in range(A):
            if res["coeffs_used"][a].any():
                check_predict(values[:, :, a], F[a], res["coeffs_used"][a])
            else:
                assert not values[:, :, a].any()
            Fa, ya = F[a][rows], ret[:, :, a].astype(np.float64).reshape(-1)[rows]     # what the fit saw
            assert bo.objective(Fa, ya, fits[n][a]) <= bo.objective(Fa, ya, bo.fit(Fa, ya)) * (1 + 1e-8)
        assert np.allclose(ret, res["returns"], rtol=1e-5, atol=1e-5 * np.abs(res["returns"]).max())
        assert np.allclose(adv, res["advantages"], rtol=1e-4, atol=1e-4 * np.abs(res["advantages"]).max())
        assert np.allclose(ev, res["ev"], rtol=1e-4, atol=1e-4)
    if shared:                                    # agent 0: zeros first, then the previous call's agent A-1 fit
        assert not got[0][0][:, :, 0].any()
        assert np.array_equal(chain[1]["coeffs_used"][0], fits[0][A - 1])


@pytest.fixture(scope="module")
def c4_launch():
    from madrl_b200 import BatchedMAWaterWorld
    eng = BatchedMAWaterWorld(4096, 20, 50, n_poison=50, n_sensors=30, seed=4, device="cuda", max_path_length=40)
    obs0 = eng.reset()
    t0 = eng.state["path_len"].clone()
    obs, rew, done, _ = eng.rollout(actions(eng, 64, 9))
    return obs, obs0, done, returns_of(rew, done), t0


def test_full_c4_per_agent_gram_deterministic_and_small(c4_launch):
    from madrl_b200.postproc import LinearFeatureBaseline
    obs, obs0, done, ret, t0 = c4_launch
    T, E, A, D = obs.shape
    assert (T, E, A) == (64, 4096, 20)
    b = LinearFeatureBaseline(D, "cuda", n_agents=A)
    G = b.normal_equations(obs, done, ret, obs0, t0)
    for a in range(A):
        G_ref = bo.torch_normal_equations(obs[:, :, a:a + 1], done, ret[:, :, a:a + 1].contiguous(),
                                          obs0[:, a:a + 1], t0, chunk=8192, pairwise=True)
        check_gram(G[a].cpu().numpy(), G_ref.cpu().numpy())
    assert torch.equal(G, b.normal_equations(obs, done, ret, obs0, t0))            # same bits, run to run
    # the fit's extra device memory: the per-agent workspace (A * ceil(48/A) * 28 tile pairs * 32 KiB = 55.1 MB at
    # D = 213, A = 20), the [A, Df+1, Df+1] stack and the solver's copies of it (3.7 MB each): under 100 MB
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    b.fit(obs, done, ret, obs0, t0)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    assert extra < 100 * 2 ** 20, extra
    c1 = b.get_param_values()
    b.fit(obs, done, ret, obs0, t0)
    assert np.array_equal(c1, b.get_param_values())
    v = b.predict(obs, done, obs0, t0)
    assert torch.equal(v, b.predict(obs, done, obs0, t0))
    for a in (0, A - 1):
        v_ref = bo.torch_predict(obs[:, :, a:a + 1], done, torch.from_numpy(c1[a]).cuda(), obs0[:, a:a + 1], t0)
        assert torch.allclose(v[:, :, a:a + 1], v_ref, rtol=1e-5, atol=1e-5 * float(v_ref.abs().max()))


def test_full_c4_bf16_equals_the_call_on_widened_obs(c4_launch):
    from madrl_b200.postproc import LinearFeatureBaseline
    obs, obs0, done, ret, t0 = c4_launch
    A, D = obs.shape[2], obs.shape[3]
    o16, ob16 = obs.to(torch.bfloat16), obs0.to(torch.bfloat16)
    b = LinearFeatureBaseline(D, "cuda", n_agents=A)
    G16 = b.normal_equations(o16, done, ret, ob16, t0)
    o32 = o16.float()
    assert torch.equal(G16, b.normal_equations(o32, done, ret, ob16.float(), t0))
    b.fit(o16, done, ret, ob16, t0)
    assert torch.equal(b.predict(o16, done, ob16, t0), b.predict(o32, done, ob16.float(), t0))


def test_one_agent_per_agent_equals_pooled_bitwise():
    from madrl_b200.postproc import (LinearFeatureBaseline, center_advantages, explained_variance,
                                     process_samples_concurrent)
    its = chained_launches("ww", 300, 24, n=1)
    it = its[0]
    # agent 2 of a Waterworld launch as a one-agent rollout
    obs, obs0 = it["obs"][:, :, 2:3].contiguous(), it["obs_before"][:, 2:3].contiguous()
    rew, done, t0 = it["rew"][:, :, 2:3].contiguous(), it["done"], it["t0"]
    ret = returns_of(rew, done)
    D = obs.shape[3]
    pooled, per = LinearFeatureBaseline(D, "cuda"), LinearFeatureBaseline(D, "cuda", n_agents=1)
    assert torch.equal(per.normal_equations(obs, done, ret, obs0, t0)[0],
                       pooled.normal_equations(obs, done, ret, obs0, t0))
    pooled.fit(obs, done, ret, obs0, t0)
    per.fit(obs, done, ret, obs0, t0)
    assert np.array_equal(per.get_param_values()[0], pooled.get_param_values())
    assert torch.equal(per.predict(obs, done, obs0, t0), pooled.predict(obs, done, obs0, t0))
    adv = torch.randn_like(ret) * 3 + 1
    for center, positive in ((True, False), (True, True)):
        assert torch.equal(center_advantages(adv, center, positive, per_agent=True),
                           center_advantages(adv, center, positive))
    assert explained_variance(adv, ret, per_agent=True) == [explained_variance(adv, ret)]
    v, a_, r, ev = process_samples_concurrent(LinearFeatureBaseline(D, "cuda", n_agents=1), obs, done, rew, DISCOUNT,
                                              GAE_LAMBDA, obs0, t0)
    assert len(ev) == 1 and not v.any()


def _group_worker(rank, world, init_file, shards, result_file):
    import torch.distributed as dist
    from madrl_b200.postproc import LinearFeatureBaseline
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="file://" + init_file, rank=rank, world_size=world)
    try:
        obs, done, ret = [x.cuda(rank) for x in shards[rank]]
        b = LinearFeatureBaseline(obs.shape[3], "cuda:%d" % rank, n_agents=obs.shape[2])
        b.fit(obs, done, ret, group=dist.group.WORLD)
        np.save(result_file % rank, b.get_param_values())
    finally:
        dist.destroy_process_group()


def _shards(world):
    eng = make("ww", 256 * world, max_path_length=9)
    eng.reset()
    obs, rew, done, _ = eng.rollout(actions(eng, 24, 5))
    ret = returns_of(rew, done)
    E = eng.n_envs // world
    return [(obs[:, r * E:(r + 1) * E].cpu(), done[:, r * E:(r + 1) * E].cpu(), ret[:, r * E:(r + 1) * E].cpu())
            for r in range(world)]


def test_group_fit_with_one_rank_equals_ungrouped_fit():
    from madrl_b200.postproc import LinearFeatureBaseline
    with tempfile.TemporaryDirectory() as d:
        shards = _shards(1)
        _group_worker(0, 1, os.path.join(d, "init"), shards, os.path.join(d, "c%d.npy"))
        obs, done, ret = [x.cuda() for x in shards[0]]
        b = LinearFeatureBaseline(obs.shape[3], "cuda", n_agents=obs.shape[2])
        b.fit(obs, done, ret)
        assert np.array_equal(np.load(os.path.join(d, "c0.npy")), b.get_param_values())


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_group_fit_two_ranks_solves_the_summed_stacks():
    import torch.multiprocessing as mp
    from madrl_b200.postproc import LinearFeatureBaseline
    with tempfile.TemporaryDirectory() as d:
        shards = _shards(2)
        out = os.path.join(d, "c%d.npy")
        mp.spawn(_group_worker, args=(2, os.path.join(d, "init"), shards, out), nprocs=2, join=True)
        c0, c1 = np.load(out % 0), np.load(out % 1)
        assert np.array_equal(c0, c1)
        b = LinearFeatureBaseline(shards[0][0].shape[3], "cuda", n_agents=shards[0][0].shape[2])
        G = sum(b.normal_equations(*[x.cuda() for x in s]) for s in shards)
        assert np.array_equal(b.solve(G).cpu().numpy(), c0)
