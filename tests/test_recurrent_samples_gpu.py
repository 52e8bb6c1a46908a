"""The recurrent branch of rllab's process_samples on the GPU (madrl_b200.postproc.pad_paths, path_returns,
path_statistics, process_samples_recurrent): against the real rllab run stored in tests/golden/recurrent_samples_ref.npz
in all three control modes, against a PyTorch gather into zeros, and at the full C2 shape on a real auto-reset
Waterworld rollout in float32 and bfloat16."""
import os

import numpy as np
import pytest
import torch

from oracle import recurrent_oracle as ro

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recurrent_samples_ref.npz")
CASES = ("ragged", "bf16_int")
RUNS = ("decentralized", "concurrent_independent", "concurrent_shared", "centralized")
STATS = ("AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "StdReturn", "MaxReturn",
         "MinReturn")
BF16 = dict(ragged=(False,), bf16_int=(False, True))   # bfloat16 runs where the observations are representable
EXACT_STATS = ("AverageReturn", "StdReturn", "MaxReturn", "MinReturn", "NumTrajs")   # functions of the rewards only


def load(case):
    z = np.load(GOLDEN)
    its = []
    for n in range(2):
        pre = "%s/it%d/" % (case, n)
        its.append({k[len(pre):]: z[k] for k in z.files if k.startswith(pre) and k.count("/") == 2})
    info_key = next(k.split(".")[-1] for k in z.files if k.startswith(case + "/decentralized/it0/env_infos."))
    ai_key = next(k.split(".")[-1] for k in z.files if k.startswith(case + "/decentralized/it0/agent_infos."))
    return z, its, info_key, ai_key


def device_inputs(it, info_key, ai_key, bf16=False, centralized=False):
    cuda = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()      # noqa: E731
    obs = cuda(it["obs"])
    ob = cuda(it["obs_before"]) if "obs_before" in it else None
    if bf16:
        obs, ob = obs.bfloat16(), (None if ob is None else ob.bfloat16())
    return dict(obs=obs, obs_before=ob, actions=cuda(it["actions"]), done=cuda(it["done"]),
                rew=cuda(it["rew_cent"] if centralized else it["rew"]), infos={info_key: cuda(it["info"])},
                agent_infos={ai_key: cuda(it["agent_info"])})


def golden_keys(case, run, n, A):
    """(golden key prefix, index into the device result) per path list of a run."""
    pre = "%s/%s/it%d/" % (case, run, n)
    if run.startswith("concurrent"):
        return [(pre + "a%d/" % a, a) for a in range(A)]
    return [(pre, None)]


def pick(x, a):
    return x if a is None else x[a]


def as_np(x):
    return x.double().cpu().numpy() if x.dtype in (torch.float32, torch.bfloat16) else x.cpu().numpy()


@pytest.mark.parametrize("case", CASES)
def test_pad_paths_equals_the_reference_padding_bitwise(case):
    """Observations, actions, rewards, valids, env_infos and agent_infos of every mode bit for bit the reference's
    padded arrays (float32 / bfloat16 values widened), and a PyTorch gather into zeros; the padding is exactly 0."""
    from madrl_b200.postproc import pad_paths
    z, its, ik, ak = load(case)
    for n, it in enumerate(its):
        A = it["obs"].shape[2]
        for run in ("decentralized", "concurrent_independent", "centralized"):
            mode = run.split("_")[0]
            for bf16 in BF16[case]:
                inp = device_inputs(it, ik, ak, bf16, mode == "centralized")
                pp = pad_paths(mode=mode, **inp)
                for key, a in golden_keys(case, run, n, A):
                    for k, got in (("observations", pp.observations), ("actions", pp.actions),
                                   ("rewards", pp.rewards), ("valids", pp.valids),
                                   ("env_infos." + ik, pp.env_infos[ik]), ("agent_infos." + ak, pp.agent_infos[ak])):
                        want = z[key + k]
                        if k == "observations" and bf16:
                            assert pick(got, a).dtype == torch.bfloat16
                        assert np.array_equal(as_np(pick(got, a)), want), (run, n, bf16, k)
                    v = pick(pp.valids, a)
                    assert torch.equal(pick(pp.length, a), v.sum(1).long())
                    assert not pick(pp.observations, a)[v == 0].any() and not pick(pp.agent_infos[ak], a)[v == 0].any()
                rec = torch.stack([pp.env, pp.agent, pp.start, pp.length], dim=-1).reshape(-1, 4)
                L = pp.valids.shape[-1]
                o, ob = inp["obs"], inp["obs_before"]
                if mode == "centralized":
                    T, E = o.shape[:2]
                    o, ob = o.reshape(T, E, 1, -1), None if ob is None else ob.reshape(E, 1, -1)
                assert torch.equal(pp.observations.reshape(rec.shape[0], L, -1),
                                   ro.torch_pad(o, rec, L, first=ob).reshape(rec.shape[0], L, -1))
                assert torch.equal(pp.env_infos[ik].reshape(rec.shape[0], L, -1),
                                   ro.torch_pad(inp["infos"][ik], rec, L, per_agent=False).reshape(rec.shape[0], L, -1))


@pytest.mark.parametrize("run", RUNS)
@pytest.mark.parametrize("case", CASES)
def test_process_samples_recurrent_matches_the_reference(case, run):
    """Two iterations with one baseline (the second predicts with the first's fit), float32 and bfloat16
    observations; tolerances of the existing GAE / centring / baseline tests."""
    from madrl_b200.postproc import LinearFeatureBaseline, process_samples_recurrent
    z, its, ik, ak = load(case)
    settings = z[case + "/settings"]
    mode = run.split("_")[0]
    T, E, A, D = its[0]["obs"].shape
    for bf16 in BF16[case]:
        if mode == "concurrent":
            bl = LinearFeatureBaseline(D, "cuda", n_agents=A, shared=run.endswith("shared"))
        else:
            bl = LinearFeatureBaseline(A * D if mode == "centralized" else D, "cuda")
        for n, it in enumerate(its):
            inp = device_inputs(it, ik, ak, bf16, mode == "centralized")
            res = process_samples_recurrent(bl, discount=settings[0], gae_lambda=settings[1], mode=mode,
                                            center_adv=bool(settings[2]), **inp)
            for key, a in golden_keys(case, run, n, A):
                for k in ("observations", "actions", "rewards", "valids"):
                    assert np.array_equal(as_np(pick(res[k], a)), z[key + k]), (k, n, bf16)
                assert np.array_equal(as_np(pick(res["env_infos"][ik], a)), z[key + "env_infos." + ik])
                assert np.array_equal(as_np(pick(res["agent_infos"][ak], a)), z[key + "agent_infos." + ak])
                ret, adv = as_np(pick(res["returns"], a)), as_np(pick(res["advantages"], a))
                gret, gadv = z[key + "returns"], z[key + "advantages"]
                assert np.allclose(ret, gret, rtol=1e-5, atol=1e-5 * np.abs(gret).max()), (n, bf16)
                assert np.allclose(adv, gadv, rtol=1e-4, atol=1e-4 * np.abs(gadv).max()), (n, bf16)
                valid = z[key + "valids"] == 1
                assert not ret[~valid].any() and not adv[~valid].any()                 # padded entries exactly 0
                stats = {k: pick(res[k], a) for k in STATS}
                want = dict(zip(STATS, z[key + "stats"]))
                for k in EXACT_STATS:
                    assert np.isclose(stats[k], want[k], rtol=1e-12, atol=0), (k, n)
                assert np.isclose(stats["AverageDiscountedReturn"], want["AverageDiscountedReturn"], rtol=1e-5,
                                  atol=1e-5 * np.abs(gret).max())
                assert np.isclose(stats["ExplainedVariance"], want["ExplainedVariance"], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("case", CASES)
def test_path_returns_and_statistics(case):
    """Per-path undiscounted returns bit for bit Python's sum() over the float64 rewards; the summary values at
    rtol 1e-12 of NumPy's over the same per-path values (AverageDiscountedReturn over the device's returns)."""
    from madrl_b200.postproc import gae, path_returns, path_statistics
    z, its, ik, ak = load(case)
    discount = z[case + "/settings"][0]
    for n, it in enumerate(its):
        A = it["obs"].shape[2]
        for run, per_agent in (("decentralized", False), ("concurrent_independent", True), ("centralized", False)):
            inp = device_inputs(it, ik, ak, centralized=run == "centralized")
            rew, done = inp["rew"], inp["done"]
            if run == "centralized":
                rew = rew[..., :1]
            _, ret = gae(rew, torch.zeros_like(rew), done, discount, 1.0)
            sums, first = path_returns(rew, ret, done, per_agent=per_agent)
            stats = path_statistics(rew, ret, done, per_agent=per_agent)
            for key, a in golden_keys(case, run, n, A):
                s, f = pick(sums, a).cpu().numpy(), pick(first, a).cpu().numpy()
                st = pick(stats, a)
                assert np.array_equal(s, z[key + "undisc"]), (run, n)
                assert st["NumTrajs"] == len(s)
                for k, v in (("AverageReturn", np.mean(s)), ("StdReturn", np.std(s)), ("MaxReturn", np.max(s)),
                             ("MinReturn", np.min(s)), ("AverageDiscountedReturn", np.mean(f))):
                    assert np.isclose(st[k], v, rtol=1e-12, atol=0), (run, n, k)
                g = z[key + "returns"][:, 0]
                assert np.allclose(f, g, rtol=1e-5, atol=1e-5 * np.abs(g).max())


@pytest.fixture(scope="module")
def c2_rollout():
    from madrl_b200 import BatchedMAWaterWorld
    eng = BatchedMAWaterWorld(4096, 5, 5, n_poison=10, n_sensors=30, seed=5, device="cuda", max_path_length=100)
    obs0 = eng.reset()
    g = torch.Generator(device="cuda")
    g.manual_seed(7)
    act = torch.randn((256, 4096, 5, 2), device="cuda", generator=g) * 0.5
    obs, rew, done, _ = eng.rollout(act)
    return obs, obs0, act, rew, done


@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
def test_full_c2_shape_equals_a_pytorch_gather(c2_rollout, bf16):
    """4096 envs x 5 agents x 256 steps x 213 observations (padded tensor past 2^31 bytes) with auto-reset cuts:
    decentralized and concurrent padding bit for bit a PyTorch gather into zeros; the records agree with
    pack_paths, and the per-path sums with a float64 PyTorch sum."""
    from madrl_b200.postproc import gae, pack_paths, pad_paths, path_returns
    obs, obs0, act, rew, done = c2_rollout
    assert tuple(obs.shape) == (256, 4096, 5, 213) and done.any()
    if bf16:
        obs, obs0 = obs.bfloat16(), obs0.bfloat16()
    for mode in ("decentralized", "concurrent"):
        pp = pad_paths(obs, act, rew, done, obs_before=obs0, mode=mode)
        rec = torch.stack([pp.env, pp.agent, pp.start, pp.length], dim=-1).reshape(-1, 4)
        P, L = rec.shape[0], pp.valids.shape[-1]
        assert P * L * 213 * obs.element_size() >= 2 ** 31 and L == 100
        assert int(pp.length.sum()) == 256 * 4096 * 5
        got = pp.observations.reshape(P, L, 213)
        assert got.dtype == obs.dtype
        want = ro.torch_pad(obs, rec, L, first=obs0)
        assert torch.equal(got, want)
        del want
        assert torch.equal(pp.actions.reshape(P, L, 2), ro.torch_pad(act, rec, L))
        assert torch.equal(pp.rewards.reshape(P, L), ro.torch_pad(rew, rec, L))
        if mode == "decentralized":
            pk = pack_paths(obs, act, rew, done, obs_before=obs0)
            for k in ("env", "agent", "length", "terminated"):
                assert torch.equal(getattr(pp, k), getattr(pk, k)), k
        del pp, got
    _, ret = gae(rew, torch.zeros_like(rew), done, 0.99, 1.0)
    sums, first = path_returns(rew, ret, done)
    pk = pack_paths(rew.unsqueeze(-1), act, ret, done)           # packed rewards as 'observations', returns as rewards
    off, n = pk.offset.long(), pk.length.long()
    csum = torch.cat([torch.zeros(1, dtype=torch.float64, device="cuda"), pk.observations[:, 0].double().cumsum(0)])
    assert torch.allclose(sums, csum[off + n] - csum[off], rtol=1e-9, atol=1e-6)
    assert torch.equal(first, pk.rewards[off].double())
