"""PolicyRollout with the reference's observation wrappers (frame_stack=B, standardizer=) on the GPU, at the C2
(Waterworld), C3 (Pursuit) and C5 (Hostage) shapes: the CUDA-graph replay against the same loop run eagerly, and
against an open-loop rollout of the recorded actions followed by the whole-trajectory passes (Standardizer.obs with
the terminal observations, FrameStack.rollout, Standardizer.rew), bit for bit; the raw trajectory through
StandardizedEnv / ObservationBuffer of oracle/postproc_oracle.py; chained calls, re-capture, argument errors and one
C2-sized rollout."""
import os

import numpy as np
import pytest
import torch

import postproc_edges as pe
from conftest import ROOT
from madrl_b200 import _lib
from madrl_b200.closed_loop import PolicyRollout
from madrl_b200.postproc import FrameStack, Standardizer
from oracle import postproc_oracle as po

pytestmark = pytest.mark.gpu

WW_C2 = dict(n_pursuers=5, n_evaders=5, n_poison=10, n_sensors=30)
PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
HW_C5 = (10, 16, 16, 4, 2)
FAMILIES = ["ww_c2", "pe_c3", "hw_c5"]
OBS_ALPHA, REW_ALPHA, SCALE = 0.05, 0.05, 0.5


def make_engine(fam, E, seed=3, mpl=7, obs_dtype=None, **kw):
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    if fam == "ww_c2":
        return BatchedMAWaterWorld(E, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **dict(WW_C2, **kw))
    if fam == "pe_c3":
        maps = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
        return BatchedPursuitEvade(E, maps, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **dict(PE_C3, **kw))
    return BatchedHostageWorld(E, *HW_C5, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **kw)


def make_std(eng, obsnorm=True, rewnorm=True):
    return Standardizer(eng.n_envs, eng._n_acting, eng.obs_dim, eng.device, scale_reward=SCALE,
                        enable_obsnorm=obsnorm, enable_rewnorm=rewnorm, obs_alpha=OBS_ALPHA, rew_alpha=REW_ALPHA)


class MLPPolicy(object):
    """One tanh layer of 32 over the flattened stack [E, A, D * B] (the reference's buffer.flatten()); the mean
    (continuous families) or the argmax of the logits (Pursuit) as the action; its input is returned as an extra."""

    def __init__(self, eng, B, seed=0):
        self.categorical = eng._act_dtype == torch.int32
        n_in, n_out = eng.obs_dim * B, 5 if self.categorical else 2
        g = torch.Generator().manual_seed(seed)
        self.W1 = (torch.randn(n_in, 32, generator=g) / n_in ** 0.5).cuda()
        self.b1 = (torch.randn(32, generator=g) * 0.1).cuda()
        self.W2 = (torch.randn(32, n_out, generator=g) * 0.5).cuda()

    def __call__(self, obs, state):
        out = torch.tanh(obs.reshape(obs.shape[0], obs.shape[1], -1).float() @ self.W1 + self.b1) @ self.W2
        act = out.argmax(-1) if self.categorical else out
        return act, {"out": out, "input": obs}, state


def start(eng, std, B):
    """The reset recipe of the PolicyRollout docstring -> (raw reset obs, obs0)."""
    o = eng.reset()
    raw = o.clone()
    std.obs(o)
    return raw, (FrameStack(eng.n_envs, eng._n_acting, eng.obs_dim, B, eng.device, eng.obs_dtype).reset(o)
                 if B > 1 else o)


def std_state(std):
    return [t.clone() for t in (std.obs_mean, std.obs_var, std.rew_mean, std.rew_var)]


def assert_rollouts_equal(a, b):
    for name in ("actions", "obs", "rew", "done", "info", "policy_obs"):
        assert torch.equal(getattr(a, name), getattr(b, name)), name
    assert sorted(a.extras) == sorted(b.extras)
    for k in a.extras:
        assert torch.equal(a.extras[k], b.extras[k]), k


def check_oracle(raw0, obs_raw, rew_raw, term_raw, done, got, B, obsnorm, bf16):
    """The raw open-loop trajectory through StandardizedEnv and ObservationBuffer, per env: standardised
    observations and rewards within a float32 ulp (plus the float64 rounding of the running mean; a bfloat16 ulp for
    bfloat16 observations), the stack exactly over the standardised values."""
    T, E, A, D = obs_raw.shape
    g_obs = got.obs.float().cpu().numpy().astype(np.float64)
    g_rew = got.rew.cpu().numpy().astype(np.float64)
    g_pol = got.policy_obs.float().cpu().numpy().astype(np.float64)
    g_0 = got.extras["input"][0].float().cpu().numpy().astype(np.float64)
    def check_obs(got_o, want, x, m):
        if not obsnorm:
            assert np.array_equal(got_o, want)
            return
        # the float64 running mean carries rounding relative to the coordinate's scale (sqrt(var)), which shows where
        # it has cancelled to ~0 (x = 0 after values of both signs)
        sd = np.sqrt(m.obs_var)
        tol = pe.f32_ulp(want) + 1e-12 * (np.abs(x) + np.abs(m.obs_mean) + sd) / (sd + 1e-8)
        if bf16:     # the float32 result rounded once more, to bfloat16: within one bfloat16 ulp of the value
            with np.errstate(divide="ignore"):
                tol = tol + np.where(want == 0, 0.0, 2.0 ** (np.floor(np.log2(np.abs(want))) - 7))
        err = np.abs(got_o - want)
        k = np.unravel_index(np.argmax(err - tol), err.shape)
        assert np.all(err <= tol), dict(got=got_o[k], want=want[k], tol=tol[k], x=x[k], mean=m.obs_mean[k],
                                        var=m.obs_var[k])

    for e in range(E):
        m = po.StandardizeEnv(A, D, SCALE, obsnorm, True, OBS_ALPHA, REW_ALPHA)
        check_obs(g_0[e].reshape(A, D, -1)[..., -1], m.obs(raw0[e]), raw0[e], m)
        for t in range(T):
            if done[t, e]:
                m.obs(term_raw[t, e])                   # StandardizedEnv.step: the terminal observation first
            check_obs(g_obs[t, e], m.obs(obs_raw[t, e]), obs_raw[t, e], m)
            r = m.rew(rew_raw[t, e])
            assert np.all(np.abs(g_rew[t, e] - r) <= pe.f32_ulp(r) + 1e-12 * np.abs(r)), (t, e)
        if B > 1:
            _, stacked = po.frame_stack_env(g_0[e, ..., -1], g_obs[:, e], done[:, e].astype(bool), B)
            assert np.array_equal(g_pol[:, e], stacked), e


@pytest.mark.parametrize("obsnorm", [False, True], ids=["raw", "obsnorm"])
@pytest.mark.parametrize("B", [1, 2, 4])
@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("fam", FAMILIES)
def test_graph_equals_eager_open_loop_and_oracle(fam, dtype, B, obsnorm):
    E, T, mpl = 48, 20, 7
    bf16 = dtype == "bf16"
    engines = [make_engine(fam, E, mpl=mpl, obs_dtype=torch.bfloat16 if bf16 else None) for _ in range(3)]
    stds = [make_std(e, obsnorm) for e in engines]
    starts = [start(e, s, B) for e, s in zip(engines, stds)]
    raw0, obs0 = starts[0]
    assert all(torch.equal(obs0, o) for _, o in starts[1:])
    pol = MLPPolicy(engines[0], B)
    launches = _lib.launch_count()
    g = PolicyRollout(engines[0], pol, T, frame_stack=B, standardizer=stds[0])(obs0)
    wrapped = B > 1 or obsnorm
    assert _lib.launch_count() - launches == T * (2 if wrapped else 1) + 1     # + Standardizer.rew
    eager = PolicyRollout(engines[1], pol, T, frame_stack=B, standardizer=stds[1], graph=False)(starts[1][1])
    assert_rollouts_equal(g, eager)
    for a, b in zip(std_state(stds[0]), std_state(stds[1])):
        assert torch.equal(a, b)
    assert g.done.any(0).all()                         # every env resets inside the launch
    assert engines[0]._term_obs is None and engines[1]._term_obs is None     # the private buffer is unset
    if B == 1:
        assert g.policy_obs is g.obs
    else:
        assert g.policy_obs.shape == (T,) + tuple(obs0.shape)
    # the policy read the wrapped stack, not the raw rows
    assert torch.equal(g.extras["input"], torch.cat([obs0[None], g.policy_obs[:-1]]))

    # open loop: the recorded actions, then the whole-trajectory passes
    eng, std = engines[2], stds[2]
    term = torch.zeros((T, E, eng._n_acting, eng.obs_dim), dtype=eng.obs_dtype, device=eng.device)
    eng.set_terminal_obs(term)
    obs, rew, done, info = eng.rollout(g.actions.clone())
    obs_raw, rew_raw, term_raw = obs.clone(), rew.clone(), term.clone()
    std.obs(obs, done, term)
    std.rew(rew)
    for a, b in ((obs, g.obs), (rew, g.rew), (done, g.done), (info, g.info)):
        assert torch.equal(a, b)
    if B > 1:
        fs = FrameStack(E, eng._n_acting, eng.obs_dim, B, eng.device, eng.obs_dtype)
        fs.carry.copy_(starts[2][1])
        assert torch.equal(fs.rollout(obs, done), g.policy_obs)
    for a, b in zip(std_state(std), std_state(stds[0])):
        assert torch.equal(a, b)

    f64 = lambda x: x.float().cpu().numpy().astype(np.float64)    # noqa: E731
    check_oracle(f64(raw0), f64(obs_raw), f64(rew_raw), f64(term_raw), done.cpu().numpy(), g, B, obsnorm, bf16)


@pytest.mark.parametrize("fam", ["ww_c2", "pe_c3"])
def test_two_calls_equal_one_call_of_twice_the_length(fam):
    E, T, B = 32, 12, 4
    eng, ref = make_engine(fam, E, mpl=9), make_engine(fam, E, mpl=9)
    std, ref_std = make_std(eng), make_std(ref)
    pol = MLPPolicy(eng, B)
    ro = PolicyRollout(eng, pol, T, frame_stack=B, standardizer=std)
    names = ("actions", "obs", "rew", "done", "info", "policy_obs")
    out = ro(start(eng, std, B)[1])
    first = {k: getattr(out, k).clone() for k in names}
    graph = ro._graph
    second = ro(first["policy_obs"][-1])
    assert ro._graph is graph
    whole = PolicyRollout(ref, pol, 2 * T, frame_stack=B, standardizer=ref_std)(start(ref, ref_std, B)[1])
    for k in names:
        assert torch.equal(torch.cat([first[k], getattr(second, k)]), getattr(whole, k)), k
    for a, b in zip(std_state(std), std_state(ref_std)):
        assert torch.equal(a, b)


def test_recapture_and_terminal_buffers():
    """A change of obs_alpha, of the Standardizer object or of B re-captures; the caller's set_terminal_obs tensor
    is used and left set, the private one is unset after each call."""
    E, T = 32, 8
    eng = make_engine("ww_c2", E)
    std = make_std(eng)
    pol = MLPPolicy(eng, 2)
    ro = PolicyRollout(eng, pol, T, frame_stack=2, standardizer=std)
    _, obs0 = start(eng, std, 2)
    out = ro(obs0)
    graph = ro._graph
    ro(out.policy_obs[-1].clone())
    assert ro._graph is graph
    std.obs_alpha = 0.01
    ro(out.policy_obs[-1].clone())
    assert ro._graph is not graph
    graph = ro._graph
    ro.standardizer = make_std(eng)
    ro(out.policy_obs[-1].clone())
    assert ro._graph is not graph
    graph = ro._graph
    ro.frame_stack, ro.policy = 1, MLPPolicy(eng, 1)
    ro(out.obs[-1].clone())
    assert ro._graph is not graph
    assert eng._term_obs is None
    # the caller's terminal tensor: written at the done steps, standardised in place, and still set afterwards
    term = torch.full((T, E, eng._n_acting, eng.obs_dim), 7.0, device=eng.device)
    eng.set_terminal_obs(term)
    res = ro(out.obs[-1].clone())
    assert eng._term_obs is term
    assert res.done.any() and (term[res.done.bool()] != 7.0).float().mean() > 0.99
    assert (term[~res.done.bool()] == 7.0).all()


def test_argument_errors():
    from madrl_b200 import BatchedMAWaterWorld
    E, T = 8, 4
    eng = make_engine("ww_c2", E)
    pol = MLPPolicy(eng, 1)
    std = make_std(eng)
    for B in (0, 9, 2.0):
        with pytest.raises(ValueError, match="frame_stack"):
            PolicyRollout(eng, pol, T, frame_stack=B)
    with pytest.raises(ValueError, match="standardizer needs auto_reset"):
        PolicyRollout(eng, pol, T, standardizer=std, auto_reset=False)
    with pytest.raises(ValueError, match="frame_stack needs auto_reset"):
        PolicyRollout(eng, pol, T, frame_stack=2, auto_reset=False)
    f64 = BatchedMAWaterWorld(E, seed=1, dtype=torch.float64, **WW_C2)
    with pytest.raises(TypeError, match="frame_stack needs float32 or bfloat16"):
        PolicyRollout(f64, pol, T, frame_stack=2)
    with pytest.raises(TypeError, match="standardizer needs float32 or bfloat16"):
        PolicyRollout(f64, pol, T, standardizer=make_std(f64))
    pe3 = make_engine("pe_c3", E, flatten=False)
    with pytest.raises(ValueError, match="flatten=True"):
        PolicyRollout(pe3, pol, T, frame_stack=4)
    with pytest.raises(ValueError, match="standardizer.obs_mean"):
        PolicyRollout(eng, pol, T, standardizer=Standardizer(E + 1, eng._n_acting, eng.obs_dim, "cuda"))
    with pytest.raises(ValueError, match="standardizer.obs_mean must live on"):
        PolicyRollout(eng, pol, T, standardizer=Standardizer(E, eng._n_acting, eng.obs_dim, "cpu"))
    with pytest.raises(TypeError, match="standardizer must be"):
        PolicyRollout(eng, pol, T, standardizer=object())
    ro = PolicyRollout(eng, pol, T, frame_stack=2)
    with pytest.raises(ValueError, match="obs0"):
        ro(eng.reset())                                   # [E, A, D] where [E, A, D, 2] is expected


def test_c2_sized_rollout_graph_equals_eager():
    E, T, B = 4096, 16, 4
    engs = [make_engine("ww_c2", E, mpl=10) for _ in range(2)]
    stds = [make_std(e) for e in engs]
    pol = MLPPolicy(engs[0], B)
    outs = [PolicyRollout(e, pol, T, frame_stack=B, standardizer=s, graph=g)(start(e, s, B)[1])
            for e, s, g in zip(engs, stds, (True, False))]
    assert_rollouts_equal(*outs)
    for a, b in zip(std_state(stds[0]), std_state(stds[1])):
        assert torch.equal(a, b)
    assert outs[0].done.any() and torch.isfinite(outs[0].policy_obs.float()).all()
