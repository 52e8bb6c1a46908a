"""Whole-path sampling on the GPU (madrl_b200.whole_paths.WholePathSampler): the batch against the selection rule of
oracle/whole_paths_oracle.py applied to one long PolicyRollout of the same seed, at the C2 (Waterworld), C3 (Pursuit)
and C5 (Hostage) shapes in float32 and bfloat16; Waterworld at its horizon; and every sample-processing pass on the
batch (path-parallel kernels) against the same pass through the serial kernels on the [N, 1, A] view, bit for bit;
and rllab's processing of scripted streams (tests/golden/whole_paths_ref.npz) through the fold and gather kernels."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from madrl_b200 import WholePathSampler, postproc, rltools_sampler
from madrl_b200.closed_loop import PolicyRollout
from madrl_b200.whole_paths import _Selection
from oracle import whole_paths_oracle as wo

pytestmark = pytest.mark.gpu

WW_C2 = dict(n_pursuers=5, n_evaders=5, n_poison=10, n_sensors=30)
PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
HW_C5 = (10, 16, 16, 4, 2)


def engine(fam, E, mpl, seed=11, obs_dtype=None):
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    if fam == "ww_c2":
        return BatchedMAWaterWorld(E, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **WW_C2)
    if fam == "pe_c3":
        maps = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
        return BatchedPursuitEvade(E, maps, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **PE_C3)
    return BatchedHostageWorld(E, *HW_C5, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype)


class Policy(object):
    """A capture-safe deterministic MLP: the mean (continuous families) or the argmax of the logits (Pursuit)."""

    def __init__(self, eng, seed=0):
        D, self.categorical = eng.obs_dim, eng._act_dtype == torch.int32
        n_out = 5 if self.categorical else 2
        g = torch.Generator().manual_seed(seed)
        self.W1 = (torch.randn(D, 32, generator=g) / D ** 0.5).cuda()
        self.W2 = (torch.randn(32, n_out, generator=g) * 0.5).cuda()

    def __call__(self, obs, state):
        out = torch.tanh(obs.float() @ self.W1) @ self.W2
        if self.categorical:
            return out.argmax(-1), {"logits": out}, state
        return out, {"mean": out}, state


def _long_rollout(fam, E, mpl, steps, obs_dtype):
    eng = engine(fam, E, mpl, obs_dtype=obs_dtype)
    obs0 = eng.reset()
    r = PolicyRollout(eng, Policy(eng), steps)(obs0)
    return obs0.cpu().numpy() if obs_dtype is None else obs0.view(torch.int16).cpu().numpy(), r


def _np(x):
    return x.view(torch.int16).cpu().numpy() if x.dtype == torch.bfloat16 else x.cpu().numpy()


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("fam", ["ww_c2", "pe_c3", "hw_c5"])
def test_batch_equals_selection_of_one_long_rollout(fam, dtype):
    E, mpl, chunk = 24, 9, 5
    obs_dtype = torch.bfloat16 if dtype == "bf16" else None
    eng = engine(fam, E, mpl, obs_dtype=obs_dtype)
    bs = 3 * E + 7
    batch = WholePathSampler(eng, Policy(eng), bs, mpl, chunk=chunk)()
    obs0, r = _long_rollout(fam, E, mpl, batch.n_steps, obs_dtype)
    done = r.done.cpu().numpy()
    t_star, end = wo.select(done, bs)
    assert batch.t_star == t_star and batch.n_steps < t_star + mpl + chunk
    np.testing.assert_array_equal(batch.path_start.cpu().numpy(), wo.path_start(done, end))
    np.testing.assert_array_equal(batch.done.cpu().numpy(), wo.gather(done, end))
    np.testing.assert_array_equal(batch.env_rows.cpu().numpy(), np.concatenate([[0], np.cumsum(end + 1)[:-1]]))
    np.testing.assert_array_equal(_np(batch.obs), wo.gather(_np(r.policy_obs), end, obs0))
    for got, want in ((batch.actions, r.actions), (batch.rew, r.rew), (batch.infos, r.info)):
        np.testing.assert_array_equal(_np(got), wo.gather(_np(want), end))
    for k, v in r.extras.items():
        np.testing.assert_array_equal(_np(batch.extras[k]), wo.gather(_np(v), end))
    # the rollout view: obs shifted as the auto-reset convention has it
    obs, dn, rew, before = batch.as_rollout()
    assert torch.equal(before[0], batch.obs[0]) and torch.equal(obs[:-1, 0], batch.obs[1:])
    assert torch.equal(dn[:, 0], batch.done) and torch.equal(rew[:, 0], batch.rew)


def test_waterworld_at_the_horizon_is_the_rollout_env_major():
    E, mpl = 32, 12
    eng = engine("ww_c2", E, mpl)
    batch = WholePathSampler(eng, Policy(eng), E * mpl, mpl, chunk=mpl)()
    obs0, r = _long_rollout("ww_c2", E, mpl, mpl, None)
    assert bool(r.done[-1].all()) and not bool(r.done[:-1].any())
    ps = batch.path_start.cpu().numpy()
    assert len(ps) == E + 1 and (np.diff(ps) == mpl).all() and batch.t_star == mpl - 1
    np.testing.assert_array_equal(_np(batch.rew), _np(r.rew).transpose(1, 0, 2).reshape(E * mpl, -1))
    np.testing.assert_array_equal(_np(batch.actions), _np(r.actions).transpose(1, 0, 2, 3).reshape(E * mpl, -1, 2))
    shifted = np.concatenate([obs0[None], _np(r.obs)[:-1]])
    np.testing.assert_array_equal(_np(batch.obs), shifted.transpose(1, 0, 2, 3).reshape(E * mpl, *obs0.shape[1:]))


def test_sampler_refuses_another_max_path_length():
    eng = engine("hw_c5", 4, 9)
    with pytest.raises(ValueError):
        WholePathSampler(eng, Policy(eng), 10, 10)


def _serial(view):
    """The same tensors without the batch's path table: the passes run their serial kernels."""
    obs, done, rew, before = view
    return obs.clone(), done.clone(), rew.clone(), before.clone()


def _same(a, b):
    if isinstance(a, dict):
        assert a.keys() == b.keys()
        for k in a:
            _same(a[k], b[k])
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b)
        for x, y in zip(a, b):
            _same(x, y)
    elif torch.is_tensor(a):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    elif isinstance(a, np.ndarray):
        np.testing.assert_array_equal(a, b)
    elif isinstance(a, postproc.PaddedPaths):
        _same(vars(a), vars(b))
    else:
        assert a == b or (a != a and b != b), (a, b)


@pytest.fixture(scope="module")
def pe_batch():
    E, mpl = 64, 13
    eng = engine("pe_c3", E, mpl)
    batch = WholePathSampler(eng, Policy(eng), 3 * E * mpl, mpl, chunk=6)()
    assert batch.n_paths >= 3 * E   # several paths per env, so the batch's paths cross env boundaries
    return batch


def test_gae_and_baseline_equal_serial_kernels(pe_batch):
    b = pe_batch
    fast, slow = b.as_rollout(), _serial(b.as_rollout())
    N, _, A, D = fast[0].shape
    vals = torch.randn(N, 1, A, device=b.rew.device)
    _same(postproc.gae(fast[2], vals, fast[1], 0.99, 0.95), postproc.gae(slow[2], vals, slow[1], 0.99, 0.95))
    _same(postproc._paths_plan(fast[1], A), postproc._paths_plan(slow[1], A))
    for kw in (dict(), dict(n_agents=A)):
        bl = [postproc.LinearFeatureBaseline(D, b.rew.device, **kw) for _ in range(2)]
        ret = postproc.gae(fast[2], vals, fast[1], 0.99, 1.0)[1]
        for base, (o, d, _, ob) in zip(bl, (fast, slow)):
            base.fit(o, d, ret, obs_before=ob)
        _same(bl[0].get_param_values(), bl[1].get_param_values())
        _same(bl[0].predict(fast[0], fast[1], fast[3]), bl[1].predict(slow[0], slow[1], slow[3]))


def test_process_samples_equal_serial_kernels(pe_batch):
    b = pe_batch
    fast, slow = b.as_rollout(), _serial(b.as_rollout())
    N, _, A, D = fast[0].shape
    dev = b.rew.device
    act = b.actions.unsqueeze(1)
    infos, agent_infos = {"info": b.infos.unsqueeze(1)}, {"logits": b.extras["logits"].unsqueeze(1)}
    outs = []
    for o, d, r, ob in (fast, slow):
        res = {}
        bl = postproc.LinearFeatureBaseline(D, dev, n_agents=A)
        for _ in range(2):
            res.setdefault("conc", []).append(postproc.process_samples_concurrent(bl, o, d, r, 0.99, 0.97,
                                                                                  obs_before=ob))
        for mode in ("decentralized", "concurrent"):
            bl = postproc.LinearFeatureBaseline(D, dev, n_agents=A if mode == "concurrent" else None)
            out = postproc.process_samples_recurrent(bl, o, act, r, d, 0.99, 0.97, mode, obs_before=ob, infos=infos,
                                                     agent_infos=agent_infos)
            out.pop("paths")
            res[mode] = out
        res["pad"] = vars(postproc.pad_paths(o, act, r, d, infos, ob, agent_infos))
        ret = postproc.gae(r, torch.zeros_like(r), d, 0.99, 1.0)[1]
        res["stats"] = postproc.path_statistics(r, ret, d, per_agent=True)
        rb = rltools_sampler.LinearFeatureBaseline(D, dev, enable_obsnorm=True, n_agents=A)
        res["rltools"] = rltools_sampler.process_samples(rb, o, d, r, 0.99, 0.97, mode="concurrent", obs_before=ob)
        res["tb"] = rltools_sampler.time_baseline(ret, d)
        outs.append(res)
    _same(outs[0], outs[1])


GOLDEN = os.path.join(ROOT, "tests", "golden", "whole_paths_ref.npz")
STATS = ("AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "StdReturn", "MaxReturn",
         "MinReturn")


@pytest.mark.parametrize("case", ["ragged", "exact", "late"])
def test_rllab_golden(case):
    g = np.load(GOLDEN)
    c = {k: g[case + "/" + k] for k in ("done", "policy_obs", "obs0", "rew", "actions", "mean")}
    bs, T = int(g[case + "/batch_size"]), int(g[case + "/chunk"])
    S, E = c["done"].shape
    dev = torch.device("cuda", 0)
    S_run = -(-S // T) * T

    def pad(x):
        return torch.as_tensor(np.concatenate([x, np.zeros((S_run - S,) + x.shape[1:], x.dtype)])).to(dev)
    full = {k: pad(c[k]) for k in ("done", "policy_obs", "rew", "actions", "mean")}
    info = torch.zeros((S_run, E), dtype=torch.int32, device=dev)
    sel = _Selection(E, T, bs, S_run, dev)
    first = torch.as_tensor(c["obs0"]).to(dev)
    for j in range(S_run // T):
        sl = slice(j * T, (j + 1) * T)
        if sel.add(first, full["policy_obs"][sl].clone(), full["actions"][sl].clone(), full["rew"][sl].clone(),
                   full["done"][sl].contiguous(), info[sl].clone(), {"mean": full["mean"][sl].clone()}):
            break
        first = full["policy_obs"][(j + 1) * T - 1].clone()
    batch = sel.batch()
    assert batch.t_star == int(g[case + "/t_star"])
    np.testing.assert_array_equal(batch.path_start.cpu().numpy(), g[case + "/path_start"])
    obs, done, rew, ob = batch.as_rollout()
    bl = postproc.LinearFeatureBaseline(obs.shape[3], dev)
    for it in range(2):
        out = postproc.process_samples_recurrent(bl, obs, batch.actions.unsqueeze(1), rew, done, 0.99, 0.95,
                                                 "decentralized", obs_before=ob,
                                                 agent_infos={"mean": batch.extras["mean"].unsqueeze(1)})
        key = "%s/recurrent/it%d/" % (case, it)
        np.testing.assert_array_equal(out["observations"].cpu().numpy(), g[key + "observations"].astype(np.float32))
        np.testing.assert_array_equal(out["valids"].cpu().numpy(), g[key + "valids"])
        ret, adv = out["returns"].cpu().numpy(), out["advantages"].cpu().numpy()
        gret, gadv = g[key + "returns"], g[key + "advantages"]
        assert np.allclose(ret, gret, rtol=1e-5, atol=1e-5 * np.abs(gret).max()), it
        assert np.allclose(adv, gadv, rtol=1e-4, atol=1e-4 * np.abs(gadv).max()), it
        fadv = g["%s/flat/it%d/advantages" % (case, it)]
        valid = out["valids"].cpu().numpy().astype(bool)
        assert np.allclose(adv[valid], fadv, rtol=1e-4, atol=1e-4 * np.abs(fadv).max()), it
        want = dict(zip(STATS, g[key + "stats"]))
        for k in ("AverageReturn", "StdReturn", "MaxReturn", "MinReturn", "NumTrajs"):
            assert np.isclose(out[k], want[k], rtol=1e-12, atol=0), (k, it)
        assert np.isclose(out["AverageDiscountedReturn"], want["AverageDiscountedReturn"], rtol=1e-5,
                          atol=1e-5 * np.abs(gret).max())
        assert np.isclose(out["ExplainedVariance"], want["ExplainedVariance"], rtol=1e-4, atol=1e-4)
