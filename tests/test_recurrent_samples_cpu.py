"""The recurrent branch of rllab's process_samples without a GPU: the NumPy oracle (oracle/recurrent_oracle.py)
against the real rllab run stored in tests/golden/recurrent_samples_ref.npz, and every argument refusal of
madrl_b200.postproc.pad_paths / path_returns / path_statistics / process_samples_recurrent on host tensors, each
raised before the library is reached."""
import os
import re

import numpy as np
import pytest
import torch

from madrl_b200 import _lib
from madrl_b200 import postproc as P
from oracle import recurrent_oracle as ro

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "recurrent_samples_ref.npz")
CASES = ("ragged", "bf16_int")
RUNS = ("decentralized", "concurrent_independent", "concurrent_shared", "centralized")
STATS = ("AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "StdReturn", "MaxReturn",
         "MinReturn")


def golden_case(z, name):
    """(settings, info key, agent_info key, iterations as dicts of inputs)."""
    its = []
    for n in range(2):
        pre = "%s/it%d/" % (name, n)
        its.append({k[len(pre):]: z[k] for k in z.files if k.startswith(pre) and k.count("/") == 2})
    info_key = next(k.split("/")[-1].split(".")[1] for k in z.files if k.startswith(name + "/decentralized/it0/env"))
    ai_key = next(k.split("/")[-1].split(".")[1] for k in z.files if k.startswith(name + "/decentralized/it0/agent"))
    return z[name + "/settings"], info_key, ai_key, its


def oracle_run(its, run, settings, info_key, ai_key):
    """The oracle over both iterations of one run: per iteration, a list of (samples_data, stats, undisc, coeffs)
    per path list (one per agent for the concurrent runs)."""
    discount, lam, center = settings[0], settings[1], bool(settings[2])
    mode = run.split("_")[0]
    A = its[0]["obs"].shape[2]
    if run == "concurrent_shared":
        one = ro.PathBaseline()
        baselines = [one] * A
    else:
        baselines = [ro.PathBaseline() for _ in range(A if mode == "concurrent" else 1)]
    out = []
    for it in its:
        paths = ro.rollout_paths(it["obs"], it["actions"], it["rew_cent"] if mode == "centralized" else it["rew"],
                                 it["done"], {info_key: it["info"]}, {ai_key: it["agent_info"]}, it.get("obs_before"),
                                 mode)
        groups = paths if mode == "concurrent" else [paths]
        res = []
        for ps, bl in zip(groups, baselines):
            data, stats = ro.process_samples_recurrent(ps, bl, discount, lam, center)
            res.append((data, stats, np.array([sum(p["rewards"]) for p in ps]), bl.coeffs.copy()))
        out.append(res)
    return out


@pytest.mark.parametrize("run", RUNS)
@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference_recurrent_branch(case, run):
    z = np.load(GOLDEN)
    settings, info_key, ai_key, its = golden_case(z, case)
    for n, res in enumerate(oracle_run(its, run, settings, info_key, ai_key)):
        for a, (data, stats, undisc, coeffs) in enumerate(res):
            key = "%s/%s/it%d/" % (case, run, n) + ("a%d/" % a if run.startswith("concurrent") else "")
            for k in ("observations", "actions", "rewards", "valids", "returns"):
                assert np.array_equal(data[k], z[key + k]), (key, k)
                assert data[k].dtype == z[key + k].dtype, (key, k)
            assert np.array_equal(data["env_infos"][info_key], z[key + "env_infos." + info_key])
            assert np.array_equal(data["agent_infos"][ai_key], z[key + "agent_infos." + ai_key])
            assert np.allclose(data["advantages"], z[key + "advantages"], rtol=1e-9, atol=1e-12), key
            assert np.array_equal(undisc, z[key + "undisc"]), key
            assert np.allclose([stats[k] for k in STATS], z[key + "stats"], rtol=1e-9, atol=1e-12), key
            assert np.allclose(coeffs, z[key + "coeffs"], rtol=1e-7, atol=1e-9), key
            assert not data["advantages"][data["valids"] == 0].any()


def test_golden_covers_the_listed_edges():
    z = np.load(GOLDEN)
    its = golden_case(z, "ragged")[3]
    done = np.concatenate([it["done"] for it in its], axis=1).astype(bool)
    T = done.shape[0]
    assert done[0].any() and done[T - 1].any() and (~done.any(axis=0)).any()
    assert (z["ragged/decentralized/it0/valids"].sum(axis=1) == 1).any()                  # a length-1 path
    assert "obs_before" in its[0] and "obs_before" not in golden_case(z, "bf16_int")[3][0]
    obs = golden_case(z, "bf16_int")[3][0]["obs"]
    assert np.array_equal(obs, torch.from_numpy(obs).bfloat16().float().numpy()) and obs.shape[3] % 2 == 1
    assert golden_case(z, "bf16_int")[3][0]["actions"].dtype == np.int32
    assert z["ragged/settings"][3] == 1 and z["ragged/settings"][2] == 1 and z["bf16_int/settings"][2] == 0


# --------------------------------------------------------------------------------------------- refusals

T, E, A, D = 4, 3, 2, 5
F32, U8 = torch.float32, torch.uint8


@pytest.fixture
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "lib", refuse)


def z(*shape, dtype=F32, device="cpu"):
    return torch.zeros(shape, dtype=dtype, device=device)


def refused(exc, name, fn):
    with pytest.raises(exc, match="^" + re.escape(name) + " "):
        fn()


def _pad(**kw):
    args = dict(obs=z(T, E, A, D), actions=z(T, E, A, 2), rew=z(T, E, A), done=z(T, E, dtype=U8))
    args.update(kw)
    return lambda: P.pad_paths(**args)


def _returns(fn=P.path_returns, **kw):
    args = dict(rew=z(T, E, A), ret=z(T, E, A), done=z(T, E, dtype=U8))
    args.update(kw)
    return lambda: fn(**args)


def _recurrent(baseline=None, **kw):
    args = dict(obs=z(T, E, A, D), actions=z(T, E, A, 2), rew=z(T, E, A), done=z(T, E, dtype=U8), discount=0.99,
                gae_lambda=0.95, mode="decentralized")
    args.update(kw)
    bl = baseline if baseline is not None else P.LinearFeatureBaseline(D, "cpu")
    return lambda: P.process_samples_recurrent(bl, **args)


def test_pad_paths_refusals(no_library):
    refused(TypeError, "obs", _pad(obs=z(T, E, A, D, dtype=torch.float64)))
    refused(TypeError, "obs", _pad(obs=np.zeros((T, E, A, D), np.float32)))
    refused(ValueError, "obs", _pad(obs=z(T, E)))
    refused(TypeError, "actions", _pad(actions=z(T, E, A, dtype=torch.int64)))
    refused(ValueError, "actions", _pad(actions=z(T, E + 1, A)))
    refused(TypeError, "rew", _pad(rew=z(T, E, A, dtype=torch.float16)))
    refused(ValueError, "rew", _pad(rew=z(T, E, A, 1)))
    refused(TypeError, "done", _pad(done=z(T, E)))
    refused(ValueError, "done", _pad(done=z(T + 1, E, dtype=U8)))
    refused(ValueError, "obs_before", _pad(obs_before=z(E, A, D + 1)))
    refused(TypeError, "obs_before", _pad(obs_before=z(E, A, D, dtype=torch.bfloat16)))
    refused(ValueError, "infos['k']", _pad(infos=dict(k=z(T, E + 1))))
    refused(TypeError, "infos['k']", _pad(infos=dict(k=z(T, E, dtype=torch.int8))))
    refused(ValueError, "agent_infos['mean']", _pad(agent_infos=dict(mean=z(T, E, A + 1, 2))))
    refused(TypeError, "agent_infos['mean']", _pad(agent_infos=dict(mean=z(T, E, A, 2, dtype=torch.float64))))
    refused(ValueError, "obs", _pad())                                       # host tensors: the device comes last
    for mode in P.MODES:
        refused(ValueError, "obs", _pad(mode=mode))
    refused(ValueError, "mode", _pad(mode="recurrent"))
    rew = z(T, E, A)
    rew[2, 1, 1] = 1.0
    refused(ValueError, "centralized", _pad(rew=rew, mode="centralized"))
    refused(ValueError, "obs", _pad(rew=rew, mode="concurrent"))           # unequal rewards only matter centralized


def test_path_statistics_refusals(no_library):
    for fn in (P.path_returns, P.path_statistics):
        refused(TypeError, "rew", _returns(fn, rew=z(T, E, A, dtype=torch.int32)))
        refused(ValueError, "rew", _returns(fn, rew=z(T, E)))
        refused(TypeError, "ret", _returns(fn, ret=z(T, E, A, dtype=torch.float64)))
        refused(ValueError, "ret", _returns(fn, ret=z(T, E, A + 1)))
        refused(ValueError, "done", _returns(fn, done=z(T, E + 1, dtype=U8)))
        refused(ValueError, "rew", _returns(fn))


def test_process_samples_recurrent_refusals(no_library):
    refused(ValueError, "mode", _recurrent(mode="rnn"))
    refused(ValueError, "process_samples_recurrent", _recurrent(baseline=object()))
    refused(ValueError, "mode", _recurrent(mode="concurrent"))                           # pooled baseline
    refused(ValueError, "mode", _recurrent(baseline=P.LinearFeatureBaseline(D, "cpu", n_agents=A)))
    refused(TypeError, "obs", _recurrent(obs=z(T, E, A, D, dtype=torch.int32)))
    refused(ValueError, "obs", _recurrent(obs=z(T, E, A * D)))
    refused(TypeError, "rew", _recurrent(rew=z(T, E, A, dtype=torch.bfloat16)))
    refused(ValueError, "actions", _recurrent(actions=z(T - 1, E, A)))
    refused(TypeError, "t0", _recurrent(t0=z(E)))
    refused(ValueError, "t0", _recurrent(t0=z(E + 1, dtype=torch.int32)))
    refused(ValueError, "agent_infos['m']", _recurrent(agent_infos=dict(m=z(T, E, 1, 2))))
    rew = z(T, E, A)
    rew[0, 0, 0] = 0.5
    refused(ValueError, "centralized", _recurrent(rew=rew, mode="centralized",
                                                  baseline=P.LinearFeatureBaseline(A * D, "cpu")))
    refused(ValueError, "obs", _recurrent())                                            # host tensors
