"""LinearFeatureBaseline on the GPU (csrc/baseline.cu): real auto-reset rollouts of the three families against
the NumPy oracle, the full C2 launch against the chunked PyTorch float64 Gram, determinism, bfloat16, memory and
the distributed fit."""
import os
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT
from oracle import baseline_oracle as bo

pytestmark = pytest.mark.gpu

PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)


def make(family, E, **kw):
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    kw = dict(dict(seed=11, device="cuda"), **kw)
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
    return gae(rew.float(), torch.zeros_like(rew, dtype=torch.float32), done, 0.99, 1.0)[1]


def check_gram(G, G_ref):
    d = np.sqrt(np.outer(np.diag(G_ref), np.diag(G_ref)))
    err = np.abs(G - G_ref)
    assert np.all(err <= 1e-12 * d), (err / np.maximum(d, 1e-300)).max()


def check_predict(vals, F, c):
    want = F.dot(c)
    tol = np.spacing(np.abs(want.astype(np.float32))) + 1e-12 * np.abs(F * c).sum(axis=1)
    assert np.all(np.abs(vals.reshape(-1).astype(np.float64) - want) <= tol)


@pytest.mark.parametrize("family,E,T", [("ww", 500, 40), ("pe", 800, 16), ("hw", 500, 20)])
def test_real_rollouts_two_chained_launches_match_oracle(family, E, T):
    """About 10^5 rows per launch, auto-reset with max_path_length 7; the second launch continues with
    obs_before = the first launch's last observations and t0 = state['path_len'] read before it."""
    from madrl_b200.postproc import LinearFeatureBaseline
    eng = make(family, E, max_path_length=7)
    obs_before = eng.reset()
    b = LinearFeatureBaseline(eng.obs_dim, "cuda")
    for launch in range(2):
        t0 = eng.state["path_len"].clone()
        obs, rew, done, _ = eng.rollout(actions(eng, T, launch))
        assert done.any() and (launch == 0 or t0.any())
        ret = returns_of(rew, done)
        G = b.normal_equations(obs, done, ret, obs_before=obs_before, t0=t0).cpu().numpy()
        o, ob, d, tt = obs.cpu().numpy(), obs_before.cpu().numpy(), done.cpu().numpy(), t0.cpu().numpy()
        F = bo.features(o, d, ob, tt)
        y = ret.cpu().numpy().reshape(-1).astype(np.float64)
        check_gram(G, bo.normal_equations(F, y))
        b.fit(obs, done, ret, obs_before=obs_before, t0=t0)
        c = b.get_param_values()
        # the device solution minimises rllab's objective at least as well as NumPy's lstsq (within 1e-8); on these
        # ill-conditioned systems the Cholesky solve can land lower than gelsd, whose rcond cut drops directions
        obj, obj_np = bo.objective(F, y, c), bo.objective(F, y, bo.fit(F, y))
        assert obj <= obj_np * (1 + 1e-8), (obj, obj_np)
        check_predict(b.predict(obs, done, obs_before=obs_before, t0=t0).cpu().numpy(), F, c)
        obs_before = obs[-1].clone()


def test_predict_before_fit_is_zero_and_param_values_round_trip():
    from madrl_b200.postproc import LinearFeatureBaseline
    eng = make("ww", 64)
    obs0 = eng.reset()
    obs, rew, done, _ = eng.rollout(actions(eng, 8, 0))
    b = LinearFeatureBaseline(eng.obs_dim, "cuda")
    assert torch.equal(b.predict(obs, done, obs0), torch.zeros(obs.shape[:3], device="cuda"))
    b.fit(obs, done, returns_of(rew, done), obs0)
    c = b.get_param_values()
    b2 = LinearFeatureBaseline(eng.obs_dim, "cuda")
    b2.set_param_values(c)
    assert torch.equal(b.predict(obs, done, obs0), b2.predict(obs, done, obs0))
    # centralized mode: the view [T, E, 1, A*D] with no other change
    T, E, A, D = obs.shape
    bc = LinearFeatureBaseline(A * D, "cuda")
    ret_c = returns_of(rew.sum(-1, keepdim=True), done)
    Gc = bc.normal_equations(obs.view(T, E, 1, A * D), done, ret_c, obs0.view(E, 1, A * D)).cpu().numpy()
    F = bo.features(obs.view(T, E, 1, A * D).cpu().numpy(), done.cpu().numpy(), obs0.view(E, 1, A * D).cpu().numpy())
    check_gram(Gc, bo.normal_equations(F, ret_c.cpu().numpy().reshape(-1)))


@pytest.fixture(scope="module")
def c2_launch():
    eng = make("ww", 4096, max_path_length=100)
    obs0 = eng.reset()
    t0 = eng.state["path_len"].clone()
    obs, rew, done, _ = eng.rollout(actions(eng, 256, 3))
    return obs, obs0, done, returns_of(rew, done), t0


def test_full_c2_against_chunked_pytorch_gram_deterministic_and_small(c2_launch):
    from madrl_b200.postproc import LinearFeatureBaseline
    obs, obs0, done, ret, t0 = c2_launch
    assert tuple(obs.shape) == (256, 4096, 5, 213)
    b = LinearFeatureBaseline(213, "cuda")
    G = b.normal_equations(obs, done, ret, obs0, t0)
    G_ref = bo.torch_normal_equations(obs, done, ret, obs0, t0, chunk=8192, pairwise=True)
    check_gram(G.cpu().numpy(), G_ref.cpu().numpy())
    assert torch.equal(G, b.normal_equations(obs, done, ret, obs0, t0))          # same bits, run to run
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
    v_ref = bo.torch_predict(obs, done, torch.from_numpy(c1).cuda(), obs0, t0)
    assert torch.allclose(v, v_ref, rtol=1e-5, atol=1e-5 * float(v_ref.abs().max()))


def test_full_c2_bf16_equals_the_call_on_widened_obs(c2_launch):
    from madrl_b200.postproc import LinearFeatureBaseline
    obs, obs0, done, ret, t0 = c2_launch
    o16, ob16 = obs.to(torch.bfloat16), obs0.to(torch.bfloat16)
    b = LinearFeatureBaseline(213, "cuda")
    G16 = b.normal_equations(o16, done, ret, ob16, t0)
    o32 = o16.float()
    G32 = b.normal_equations(o32, done, ret, ob16.float(), t0)
    assert torch.equal(G16, G32)
    b.fit(o16, done, ret, ob16, t0)
    assert torch.equal(b.predict(o16, done, ob16, t0), b.predict(o32, done, ob16.float(), t0))


def _group_worker(rank, world, init_file, shards, result_file):
    import torch.distributed as dist
    from madrl_b200.postproc import LinearFeatureBaseline
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", init_method="file://" + init_file, rank=rank, world_size=world)
    try:
        obs, done, ret = [x.cuda(rank) for x in shards[rank]]
        b = LinearFeatureBaseline(obs.shape[3], "cuda:%d" % rank)
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
        b = LinearFeatureBaseline(obs.shape[3], "cuda")
        b.fit(obs, done, ret)
        assert np.array_equal(np.load(os.path.join(d, "c0.npy")), b.get_param_values())


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two visible GPUs")
def test_group_fit_two_ranks_pools_the_shards():
    import torch.multiprocessing as mp
    from madrl_b200.postproc import LinearFeatureBaseline
    with tempfile.TemporaryDirectory() as d:
        shards = _shards(2)
        out = os.path.join(d, "c%d.npy")
        mp.spawn(_group_worker, args=(2, os.path.join(d, "init"), shards, out), nprocs=2, join=True)
        c0, c1 = np.load(out % 0), np.load(out % 1)
        assert np.array_equal(c0, c1)
        b = LinearFeatureBaseline(shards[0][0].shape[3], "cuda")
        G = sum(b.normal_equations(*[x.cuda() for x in s]) for s in shards)
        assert np.array_equal(b.solve(G).cpu().numpy(), c0)
