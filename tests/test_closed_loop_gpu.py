"""Closed-loop rollouts with a PyTorch policy (madrl_b200.closed_loop.PolicyRollout) on the GPU: the CUDA-graph replay
against the same loop run eagerly and against an open-loop rollout() fed the recorded actions, bit for bit, at the
C2 (Waterworld), C3 (Pursuit) and C5 (Hostage) shapes; bfloat16 observations and terminal observations; recurrent
state resets; stochastic policies; re-capture; two engines side by side; and the stand-alone Waterworld heuristic
through the loop against the in-kernel one (rollout_heuristic)."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT
from madrl_b200 import _lib
from madrl_b200.closed_loop import PolicyRollout

pytestmark = pytest.mark.gpu

WW_C2 = dict(n_pursuers=5, n_evaders=5, n_poison=10, n_sensors=30)
PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
HW_C5 = (10, 16, 16, 4, 2)
FAMILIES = ["ww_c2", "pe_c3", "hw_c5"]


def make_engine(fam, E, seed=3, mpl=7, obs_dtype=None):
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    if fam == "ww_c2":
        return BatchedMAWaterWorld(E, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **WW_C2)
    if fam == "pe_c3":
        maps = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
        return BatchedPursuitEvade(E, maps, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, **PE_C3)
    return BatchedHostageWorld(E, *HW_C5, seed=seed, max_path_length=mpl, obs_dtype=obs_dtype)


class MLPPolicy(object):
    """rllab's GaussianMLPPolicy shape: one tanh hidden layer of 32, fixed weights; `mean` (continuous families) or
    the argmax of the logits (Pursuit) as the action, or a Gaussian sample with `stochastic`."""

    def __init__(self, D, n_out, categorical, stochastic=False, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.W1 = (torch.randn(D, 32, generator=g) / D ** 0.5).cuda()
        self.b1 = (torch.randn(32, generator=g) * 0.1).cuda()
        self.W2 = (torch.randn(32, n_out, generator=g) * 0.5).cuda()
        self.log_std = torch.full((n_out,), -0.5).cuda()
        self.categorical, self.stochastic = categorical, stochastic

    def dist(self, obs):
        return torch.tanh(obs.float() @ self.W1 + self.b1) @ self.W2

    def __call__(self, obs, state):
        out = self.dist(obs)
        if self.categorical:
            return out.argmax(-1), {"logits": out}, state
        log_std = self.log_std.expand_as(out)
        act = out + torch.randn_like(out) * log_std.exp() if self.stochastic else out
        return act, {"mean": out, "log_std": log_std}, state


def policy_for(eng, **kw):
    pe = eng._act_dtype == torch.int32
    return MLPPolicy(eng.obs_dim, 5 if pe else 2, pe, **kw)


@pytest.mark.parametrize("variant", ["f32", "bf16_term"])
@pytest.mark.parametrize("fam", FAMILIES)
def test_graph_equals_eager_and_open_loop(fam, variant):
    E, T, mpl = 48, 20, 7
    bf16 = variant == "bf16_term"
    engines = [make_engine(fam, E, mpl=mpl, obs_dtype=torch.bfloat16 if bf16 else None) for _ in range(3)]
    pol = policy_for(engines[0])
    obs0 = [e.reset() for e in engines]
    assert all(torch.equal(obs0[0], o) for o in obs0[1:])
    terms = []
    if bf16:
        for e in engines:
            terms.append(torch.full((T, E, e._n_acting, e.obs_dim), 7.0, dtype=e.obs_dtype, device=e.device))
            e.set_terminal_obs(terms[-1])
    launches = _lib.launch_count()
    g = PolicyRollout(engines[0], pol, T)(obs0[0])
    assert _lib.launch_count() - launches == T   # the captured launches; the replay adds none
    launches = _lib.launch_count()
    eager = PolicyRollout(engines[1], pol, T, graph=False)(obs0[1])
    assert _lib.launch_count() - launches == T
    open_loop = engines[2].rollout(g.actions.clone())
    for a, b in zip((g.actions,) + tuple(g[1:5]), (eager.actions,) + tuple(eager[1:5])):
        assert torch.equal(a, b)
    for a, b in zip(g[1:5], open_loop):
        assert torch.equal(a, b)
    for k in g.extras:
        assert torch.equal(g.extras[k], eager.extras[k])
    assert g.done.any(0).all()   # every env ends an episode (at the latest at max_path_length) inside the launch
    if bf16:
        assert torch.equal(terms[0], terms[1]) and torch.equal(terms[0], terms[2])
        assert (terms[0][g.done.bool()] != 7.0).any()
        assert engines[0]._term_obs is terms[0]
    assert torch.equal(engines[0]._blob, engines[1]._blob) and torch.equal(engines[0]._blob, engines[2]._blob)
    assert engines[0].obs_cache == _lib.OBS_CACHE_STREAM   # restored after the loop


class GRUPolicy(object):
    """A GRU cell over each agent's observation: state [E, A, H]."""

    def __init__(self, D, H=16, seed=1):
        torch.manual_seed(seed)
        self.cell = torch.nn.GRUCell(D, H).cuda()
        self.head = torch.nn.Linear(H, 2).cuda()

    @torch.no_grad()
    def __call__(self, obs, h):
        E, A, D = obs.shape
        h = self.cell(obs.reshape(E * A, D).float(), h.reshape(E * A, -1)).view(E, A, -1)
        return self.head(h), {"h": h}, h


def test_recurrent_state_restarts_with_each_episode():
    E, T, mpl = 32, 24, 5
    eng, ref_eng = make_engine("ww_c2", E, mpl=mpl), make_engine("ww_c2", E, mpl=mpl)
    pol = GRUPolicy(eng.obs_dim)
    h0 = torch.randn(E, eng._n_acting, 16, device="cuda")
    obs0 = eng.reset()
    ref_eng.reset()
    out = PolicyRollout(eng, pol, T)(obs0, h0)
    hs = out.extras["h"]                    # the state each step's policy call produced
    # a reference loop that resets by hand
    h, prev = h0.clone(), obs0
    for t in range(T):
        a, ex, h = pol(prev, h)
        assert torch.equal(ex["h"], hs[t]) and torch.equal(a, out.actions[t])
        prev, _, done, _ = ref_eng.step(a, auto_reset=True)
        assert torch.equal(prev, out.obs[t])
        h = torch.where(done.bool().view(E, 1, 1), torch.zeros_like(h), h)
    assert torch.equal(h, out.state)
    # every env whose done is set at step t starts step t+1 from the zero state: its h equals one cell step from 0
    done = out.done.bool()
    assert done[:-1].any()
    A = eng._n_acting
    with torch.no_grad():
        for t in range(T - 1):
            d = done[t]
            if d.any():
                fresh = pol.cell(out.obs[t].reshape(E * A, -1), torch.zeros(E * A, 16, device="cuda")).view(E, A, 16)
                assert torch.equal(fresh[d], hs[t + 1][d])


def test_stochastic_policy_and_recurrent_samples():
    from madrl_b200.postproc import LinearFeatureBaseline, process_samples_recurrent
    E, T = 64, 16
    eng = make_engine("ww_c2", E, mpl=6)
    pol = policy_for(eng, stochastic=True)
    ro = PolicyRollout(eng, pol, T)
    obs0 = eng.reset()
    a1 = ro(obs0).actions.clone()
    r2 = ro(obs0)
    assert not torch.equal(a1, r2.actions)                  # fresh noise at each replay
    prev = torch.cat([obs0[None], r2.obs[:-1]])
    assert torch.allclose(r2.extras["mean"], pol.dist(prev), rtol=0, atol=1e-6)   # recorded agent_infos = a recomputation
    assert torch.equal(r2.extras["log_std"], pol.log_std.expand(T, E, eng._n_acting, 2))
    res = process_samples_recurrent(LinearFeatureBaseline(eng.obs_dim, "cuda"), r2.obs, r2.actions, r2.rew, r2.done,
                                    0.99, 0.97, "decentralized", obs_before=obs0, agent_infos=r2.extras)
    assert res["valids"].sum() == T * E * eng._n_acting
    assert torch.isfinite(res["advantages"]).all()


@pytest.mark.parametrize("fam", FAMILIES)
def test_recapture_and_chained_calls(fam):
    E, T = 32, 12
    eng, ref = make_engine(fam, E, mpl=9), make_engine(fam, E, mpl=9)
    pol = policy_for(eng)
    ro = PolicyRollout(eng, pol, T)
    obs0 = eng.reset()
    first = [x.clone() for x in ro(obs0)[:5]]
    graph = ro._graph
    second = [x.clone() for x in ro(first[1][-1])[:5]]
    assert ro._graph is graph                                   # same settings: replayed
    whole = PolicyRollout(ref, pol, 2 * T)(ref.reset())
    for a, b, c in zip(first, second, whole[:5]):
        assert torch.equal(torch.cat([a, b]), c)
    ro.T = 5                                                    # a T change re-captures
    out = ro(second[1][-1])
    assert ro._graph is not graph and out.obs.shape[0] == 5
    tail = PolicyRollout(ref, pol, 5)(whole.obs[-1].clone())
    for a, b in zip(out[:5], tail[:5]):
        assert torch.equal(a, b)


def test_two_engines_keep_separate_graphs():
    E, T = 32, 10
    e1, e2 = make_engine("ww_c2", E, seed=1), make_engine("ww_c2", E, seed=2)
    r1, r2 = make_engine("ww_c2", E, seed=1), make_engine("ww_c2", E, seed=2)
    pol = policy_for(e1)
    ro1, ro2 = PolicyRollout(e1, pol, T), PolicyRollout(e2, pol, T)
    o1, o2 = e1.reset(), e2.reset()
    a = [x.clone() for x in ro1(o1)[:5]]
    b = [x.clone() for x in ro2(o2)[:5]]
    c = [x.clone() for x in ro1(a[1][-1])[:5]]
    ref1 = PolicyRollout(r1, pol, 2 * T, graph=False)(r1.reset())
    ref2 = PolicyRollout(r2, pol, T, graph=False)(r2.reset())
    for x, y, z in zip(a, c, ref1[:5]):
        assert torch.equal(torch.cat([x, y]), z)
    for x, z in zip(b, ref2[:5]):
        assert torch.equal(x, z)
    assert not torch.equal(a[1], b[1])


def test_waterworld_heuristic_through_the_loop_matches_rollout_heuristic():
    """The stand-alone generator closes the loop through PolicyRollout; the in-kernel policy through
    rollout_heuristic.  Both are the reference's heuristic; they differ only in float32 summation order, so actions
    agree within the generators' 1e-5 and the trajectories stay together over 64 steps."""
    from madrl_b200.heuristics import waterworld_heuristic
    E, T = 64, 64
    eng, ref = make_engine("ww_c2", E, mpl=0), make_engine("ww_c2", E, mpl=0)
    obs0 = eng.reset()
    ref.reset()
    out = PolicyRollout(eng, lambda o, s: (waterworld_heuristic(o, 30), {}, s), T)(obs0)
    act, obs, rew, done, info = ref.rollout_heuristic(T, obs0.clone())
    assert (act - out.actions).abs().max() < 1e-5
    assert (obs - out.obs).abs().max() < 1e-5
    assert (rew - out.rew).abs().max() < 1e-5
    assert torch.equal(done, out.done) and torch.equal(info, out.info)


@pytest.mark.parametrize("change", ["pursuit_set_params", "ww_seed", "pursuit_seed", "ww_set_launch"])
def test_settings_changed_between_calls_match_eager(change):
    """Host settings a launch copies into its kernel parameters (the seed, Pursuit's curriculum parameters, the
    launch geometry) changed between two calls: the graph is re-captured and follows them as the eager loop does."""
    fam = "pe_c3" if change.startswith("pursuit") else "ww_c2"
    E, T = 48, 12
    engs = [make_engine(fam, E, mpl=9) for _ in range(2)]
    pol = policy_for(engs[0])
    ros = [PolicyRollout(engs[0], pol, T), PolicyRollout(engs[1], pol, T, graph=False)]
    obs0 = [e.reset() for e in engs]
    outs = [[x.clone() for x in ro(o)[:5]] for ro, o in zip(ros, obs0)]
    graph = ros[0]._graph
    for e in engs:
        if change == "pursuit_set_params":
            e.set_params(catchr=0.7, constraint_window=0.5)
        elif change == "ww_set_launch":
            e.set_launch(0, 3)
        else:
            e.seed(99)
            e.reset()
    second = [ro(o[1][-1])[:5] for ro, o in zip(ros, outs)]
    assert ros[0]._graph is not graph
    for a, b in zip(*second):
        assert torch.equal(a, b)
    if change == "ww_seed":   # the new seed's streams: as an engine built with that seed (Pursuit keeps its never-
        # cleared window counts across reset, as the reference does, so a re-seeded Pursuit engine is not a new one)
        fresh = make_engine(fam, E, seed=99, mpl=9)
        fresh.reset()
        for a, b in zip(second[0], PolicyRollout(fresh, pol, T, graph=False)(outs[0][1][-1])[:5]):
            assert torch.equal(a, b)


@pytest.mark.parametrize("fam", FAMILIES)
def test_step_writes_into_caller_buffers(fam):
    E = 16
    a_eng, b_eng = make_engine(fam, E, mpl=3), make_engine(fam, E, mpl=3)
    a_eng.reset()
    prev = b_eng.reset()
    pol = policy_for(a_eng)
    obs, rew, done, info = [torch.full(s, 5, dtype=dt, device="cuda") for dt, s in b_eng._trajectory_shapes(1)]
    bufs = (obs[0], rew[0], done[0], info[0])
    any_done = False
    for t in range(5):   # done and auto-reset inside
        act = pol(prev, None)[0]
        want = a_eng.step(act, auto_reset=True)
        got = b_eng.step(act, auto_reset=True, out=bufs)
        for g, w, buf in zip(got[:3], want[:3], bufs[:3]):
            assert g.data_ptr() == buf.data_ptr() and torch.equal(g, w)
        assert list(got[3]) == list(want[3]) and len(got[3]) == len(b_eng._info_keys)
        for k in want[3]:
            assert torch.equal(got[3][k], want[3][k])
            assert bufs[3].data_ptr() <= got[3][k].data_ptr() < bufs[3].data_ptr() + bufs[3].nbytes
        prev = got[0]
        any_done = any_done or bool(done.any())
    assert any_done
    with pytest.raises(ValueError, match="^obs "):
        b_eng.step(act, out=(obs, rew[0], done[0], info[0]))


def test_float64_engine_streams_by_default():
    from madrl_b200 import BatchedMAWaterWorld, EngineError
    E, T = 16, 8
    engs = [BatchedMAWaterWorld(E, seed=4, max_path_length=5, dtype=torch.float64, **WW_C2) for _ in range(2)]
    pol = policy_for(engs[0])
    g = PolicyRollout(engs[0], pol, T)(engs[0].reset())
    e = PolicyRollout(engs[1], pol, T, graph=False)(engs[1].reset())
    for a, b in zip(g[:5], e[:5]):
        assert torch.equal(a, b)
    with pytest.raises(EngineError, match="fp32"):
        PolicyRollout(engs[0], pol, T, obs_cache=_lib.OBS_CACHE_KEEP)(engs[0].reset())
