"""The Python wrappers check every tensor before its data_ptr() crosses the C ABI (_lib.require_tensor): one
malformed argument per case, each refused with an error that names it and before the library is reached.
Shapes are checked before devices, so host tensors exercise the shape checks without a GPU; the CUDA-only
cases (mixed devices) are at the end."""
import re

import pytest
import torch

from madrl_b200 import EngineError, _lib
from madrl_b200 import postproc as P
from madrl_b200.heuristics import pursuit_heuristic, waterworld_heuristic

T, E, A, D = 4, 3, 2, 5
F32, U8 = torch.float32, torch.uint8


@pytest.fixture(autouse=True)
def no_library(monkeypatch):
    def refuse():
        raise AssertionError("the library was reached")
    monkeypatch.setattr(_lib, "lib", refuse)


def z(*shape, dtype=F32, device="cpu"):
    return torch.zeros(shape, dtype=dtype, device=device)


def refused(exc, name, fn):
    with pytest.raises(exc, match="^" + re.escape(name) + " "):
        fn()


def test_require_tensor_options():
    req = _lib.require_tensor
    x = z(T, E, A)
    assert req(x, "x", (torch.bfloat16, F32), (None, E, ...), "cpu") is x
    assert req(x, "x", F32, (...,), None) is x and req(None, "x", F32, (T,), "cpu", optional=True) is None
    assert req(x.transpose(0, 1), "x", F32, (E, T, A), "cpu", contiguous=False) is not None
    refused(TypeError, "x", lambda: req(None, "x", F32, (T,), "cpu"))
    refused(TypeError, "x", lambda: req(x.double(), "x", (torch.bfloat16, F32), (T, E, A), "cpu"))
    assert req(x, "x", F32, (T, E, A, ...), "cpu") is x                                 # ... may match no dim
    refused(ValueError, "x", lambda: req(x, "x", F32, (None, E), "cpu"))                 # rank
    refused(ValueError, "x", lambda: req(x, "x", F32, (T, E + 1, ...), "cpu"))
    refused(ValueError, "x", lambda: req(x, "x", F32, (T, E, A, D, ...), "cpu"))        # fewer dims than the head
    refused(ValueError, "x", lambda: req(x, "x", F32, (T, E, A), "cuda"))                # host tensor, any CUDA device
    refused(ValueError, "x", lambda: req(x[:, :2], "x", F32, (T, 2, A), "cpu"))          # strided view
    with pytest.raises(ValueError, match="^x must have shape"):                          # shape before device
        req(x, "x", F32, (T + 1, E, A), "cuda")


# --------------------------------------------------------------------------------------------- postproc

def _gae(**kw):
    args = dict(rew=z(T, E, A), values=z(T, E, A), done=z(T, E, dtype=U8), discount=0.99, gae_lambda=0.95)
    args.update(kw)
    return lambda: P.gae(**args)


def _frame_stack(obs=None, done=None):
    fs = P.FrameStack(E, A, D, 3, "cpu")
    return lambda: fs.rollout(z(T, E, A, D) if obs is None else obs, z(T, E, dtype=U8) if done is None else done)


def _std_obs(obs=None, done=None, terminal=None):
    st = P.Standardizer(E, A, D, "cpu", enable_obsnorm=True)
    return lambda: st.obs(z(T, E, A, D) if obs is None else obs, done, terminal)


def _std_rew(rew):
    return lambda: P.Standardizer(E, A, D, "cpu").rew(rew)


def _episode_stats(rew=None, done=None):
    es = P.EpisodeStats(E, A, "cpu")
    return lambda: es.rollout(z(T, E, A) if rew is None else rew, z(T, E, dtype=U8) if done is None else done)


def _pack(**kw):
    args = dict(obs=z(T, E, A, D), actions=z(T, E, A, 2), rew=z(T, E, A), done=z(T, E, dtype=U8),
                infos=dict(evcatches=z(T, E, dtype=torch.int32)), obs_before=z(E, A, D))
    args.update(kw)
    return lambda: P.pack_paths(**args)


def _baseline(method, n_agents=None, **kw):
    b = P.LinearFeatureBaseline(D, "cpu", n_agents=n_agents)
    args = dict(obs=z(T, E, A, D), done=z(T, E, dtype=U8))
    if method == "normal_equations":
        args["returns"] = z(T, E, A)
    args.update(kw)
    return lambda: getattr(b, method)(**args)


POSTPROC = {
    "gae-values-short": (ValueError, "values", _gae(values=z(1))),
    "gae-done-short": (ValueError, "done", _gae(done=z(1, 1, dtype=U8))),
    "gae-last_value-short": (ValueError, "last_value", _gae(last_value=z(1))),
    "gae-host": (ValueError, "rew", _gae()),
    "center_advantages-host": (ValueError, "adv", lambda: P.center_advantages(z(T, E, A))),
    "center_advantages-per_agent-host": (ValueError, "adv", lambda: P.center_advantages(z(T, E, A), per_agent=True)),
    "moments-b-short": (ValueError, "b", lambda: P.moments(z(T, E, A), z(T * E * A - 1))),
    "moments-host": (ValueError, "a", lambda: P.moments(z(T, E, A), z(T, E, A))),
    "moments_agents-host": (ValueError, "a", lambda: P.moments_agents(z(T, E, A))),
    "frame_stack-obs-agents": (ValueError, "obs", _frame_stack(obs=z(T, E, A + 1, D))),
    "frame_stack-done-short": (ValueError, "done", _frame_stack(done=z(T - 1, E, dtype=U8))),
    "frame_stack-host": (ValueError, "FrameStack.carry", _frame_stack()),
    "standardizer-obs-envs": (ValueError, "obs", _std_obs(obs=z(T, 2 * E, A, D))),
    "standardizer-obs-strided": (ValueError, "obs", _std_obs(obs=z(T, E, A, 2 * D)[..., :D])),
    "standardizer-terminal-short": (ValueError, "terminal_obs",
                                    _std_obs(done=z(T, E, dtype=U8), terminal=z(T - 1, E, A, D))),
    "standardizer-terminal-no-done": (TypeError, "done", _std_obs(terminal=z(T, E, A, D))),
    "standardizer-terminal-done-short": (ValueError, "done",
                                         _std_obs(done=z(T, E - 1, dtype=U8), terminal=z(T, E, A, D))),
    "standardizer-obs-host": (ValueError, "Standardizer.obs_mean", _std_obs()),
    "standardizer-rew-envs": (ValueError, "rew", _std_rew(z(T, 2 * E, A))),
    "standardizer-rew-strided": (ValueError, "rew", _std_rew(z(T, E, 2 * A)[..., :A])),
    "standardizer-rew-host": (ValueError, "Standardizer.rew_mean", _std_rew(z(T, E, A))),
    "episode_stats-rew-envs": (ValueError, "rew", _episode_stats(rew=z(T, 2 * E, A))),
    "episode_stats-rew-agents": (ValueError, "rew", _episode_stats(rew=z(T, E, A + 1))),
    "episode_stats-done-short": (ValueError, "done", _episode_stats(done=z(T, E - 1, dtype=U8))),
    "episode_stats-host": (ValueError, "EpisodeStats.carry", _episode_stats()),
    "pack_paths-done-short": (ValueError, "done", _pack(done=z(T, E - 1, dtype=U8))),
    "pack_paths-actions-envs": (ValueError, "actions", _pack(actions=z(T, 2 * E, A, 2))),
    "pack_paths-rew-agents": (ValueError, "rew", _pack(rew=z(T, E, A + 1))),
    "pack_paths-infos-short": (ValueError, "infos['evcatches']", _pack(infos=dict(evcatches=z(T - 1, E)))),
    "pack_paths-obs_before-short": (ValueError, "obs_before", _pack(obs_before=z(E, A, D - 1))),
    "pack_paths-host": (ValueError, "obs", _pack()),
    "baseline-predict-host": (ValueError, "this baseline", _baseline("predict")),
    "baseline-normal_equations-host": (ValueError, "this baseline", _baseline("normal_equations")),
    "baseline-agents-predict-host": (ValueError, "this baseline", _baseline("predict", n_agents=A)),
}


@pytest.mark.parametrize("case", sorted(POSTPROC))
def test_postproc_refuses_before_the_library(case):
    exc, name, call = POSTPROC[case]
    refused(exc, name, call)


# ------------------------------------------------------------------------------------------- heuristics

R = 7

HEURISTICS = {
    "waterworld-dtype": (TypeError, "obs", lambda: waterworld_heuristic(z(E, A, 213, dtype=torch.float16), 30)),
    "pursuit-channels": (ValueError, "obs", lambda: pursuit_heuristic(z(E, A, R, R, 3))),
    "pursuit-window": (ValueError, "obs", lambda: pursuit_heuristic(z(E, A, R + 1, R, 4))),
    "pursuit-fallback-short": (ValueError, "fallback",
                               lambda: pursuit_heuristic(z(E, A, R, R, 4), fallback=z(E, dtype=torch.int32))),
}


@pytest.mark.parametrize("case", sorted(HEURISTICS))
def test_heuristics_refuse_before_the_library(case):
    exc, name, call = HEURISTICS[case]
    refused(exc, name, call)


def test_heuristics_keep_engine_error_for_host_tensors():
    for call in (lambda: waterworld_heuristic(z(E, A, 213), 30), lambda: pursuit_heuristic(z(E, A, R, R, 4)),
                 lambda: pursuit_heuristic(z(E, A, R, R, 4), fallback=z(E, A, dtype=torch.int32))):
        with pytest.raises(EngineError, match="needs a CUDA tensor"):
            call()


# ---------------------------------------------------------------------------------------------- engines

class _OnlySetTerminalObs(object):
    """The engine's library handle: setting the terminal-observation tensor succeeds, anything else fails."""

    def madrl_ww_set_terminal_obs(self, h, ptr):
        return 0

    def __getattr__(self, name):
        raise AssertionError("the library was reached: " + name)


def _engine():
    """A Waterworld engine on the host (no handle, no state): what the wrappers check before a launch."""
    from madrl_b200 import BatchedMAWaterWorld
    eng = BatchedMAWaterWorld.__new__(BatchedMAWaterWorld)
    eng._L, eng._h, eng._term_obs = _OnlySetTerminalObs(), None, None
    eng.n_envs, eng._n_acting, eng.obs_dim, eng.device = E, A, D, torch.device("cpu")
    eng.dtype = eng.obs_dtype = eng._act_dtype = F32
    return eng


def _term_then_rollout(term, steps):
    eng = _engine()
    eng.set_terminal_obs(term)
    return eng.rollout(z(steps, E, A, 2), auto_reset=True)


ENGINE = {
    "rollout-actions-agents": (ValueError, "actions", lambda: _engine().rollout(z(T, E, A + 1, 2))),
    "rollout-actions-tail": (ValueError, "actions", lambda: _engine().rollout(z(T, E, A))),
    "reset-mask-short": (ValueError, "mask", lambda: _engine().reset(mask=z(E - 1, dtype=U8))),
    "set_terminal_obs-envs": (ValueError, "term_obs", lambda: _engine().set_terminal_obs(z(T, E - 1, A, D))),
    "set_terminal_obs-strided": (ValueError, "term_obs",
                                 lambda: _engine().set_terminal_obs(z(T, E, A, 2 * D)[..., :D])),
    "rollout-terminal-obs-shorter": (ValueError, "the set_terminal_obs tensor",
                                     lambda: _term_then_rollout(z(T - 1, E, A, D), T)),
    "rollout-terminal-obs-longer": (ValueError, "the set_terminal_obs tensor",
                                    lambda: _term_then_rollout(z(T + 1, E, A, D), T)),
}


@pytest.mark.parametrize("case", sorted(ENGINE))
def test_engine_refuses_before_the_library(case):
    exc, name, call = ENGINE[case]
    refused(exc, name, call)


# ------------------------------------------------------------------------------------------ mixed devices

@pytest.mark.gpu
def test_tensors_of_one_call_share_its_cuda_device():
    dev = "cuda"
    cuda = lambda *s, dtype=F32: z(*s, dtype=dtype, device=dev)   # noqa: E731
    done = cuda(T, E, dtype=U8)
    refused(ValueError, "values", lambda: P.gae(cuda(T, E, A), z(T, E, A), done, 0.99, 0.95))
    refused(ValueError, "last_value", lambda: P.gae(cuda(T, E, A), cuda(T, E, A), done, 0.99, 0.95, z(E, A)))
    refused(ValueError, "done", lambda: P.pack_paths(cuda(T, E, A, D), cuda(T, E, A, 2), cuda(T, E, A),
                                                     z(T, E, dtype=U8)))
    refused(ValueError, "b", lambda: P.moments(cuda(T, E, A), z(T, E, A)))
    refused(ValueError, "done", lambda: P.FrameStack(E, A, D, 3, dev).rollout(cuda(T, E, A, D), z(T, E, dtype=U8)))
    refused(ValueError, "obs", lambda: P.FrameStack(E, A, D, 3, dev).rollout(z(T, E, A, D), z(T, E, dtype=U8)))
    refused(ValueError, "obs", lambda: P.Standardizer(E, A, D, dev, enable_obsnorm=True).obs(z(T, E, A, D)))
    refused(ValueError, "done", lambda: P.EpisodeStats(E, A, dev).rollout(cuda(T, E, A), z(T, E, dtype=U8)))
    refused(ValueError, "done", lambda: P.LinearFeatureBaseline(D, dev).predict(cuda(T, E, A, D), z(T, E, dtype=U8)))
    refused(ValueError, "obs", lambda: P.LinearFeatureBaseline(D, dev).predict(z(T, E, A, D), z(T, E, dtype=U8)))
