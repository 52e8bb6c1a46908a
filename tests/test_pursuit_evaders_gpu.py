"""Pursuit's evaders under a caller's controller on the device: the random controller's own actions fed back reproduce
the random launch bit for bit, fixed and per-step actions and model_state follow the oracle,
PolicyRollout(evader_policy=...) replays as it runs eagerly, the drop-in takes evader_controller, and what cannot
work is refused."""
import os

import numpy as np
import pytest
import torch

import env_dispatch_edges as D
import pursuit_evaders_edges as V
from madrl_b200 import BatchedHostageWorld, BatchedPursuitEvade, PolicyRollout, PursuitEvade, SingleActionPolicy
from madrl_b200 import _lib
from madrl_b200.evaluate import evaluate_heuristic

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAPS = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
          catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
NE64 = dict(n_evaders=64, n_pursuers=16, obs_range=5, surround=False, n_catch=1, flatten=False, reward_mech='global',
            catchr=0.05, random_opponents=True, max_opponents=65)
SEED, BASE, MPL = 17, 300, 23
MODE = "decentralized"


def engine(cfg, E, obs_dtype=None, **kw):
    return BatchedPursuitEvade(E, MAPS, device="cuda", seed=SEED, env_id_base=BASE, max_path_length=MPL,
                               obs_dtype=obs_dtype, **dict(cfg, **kw))


def blob(eng):
    return eng._blob.cpu().numpy().copy()


def cfg_cases():
    return [("c3", C3, None), ("c3_bf16", C3, torch.bfloat16), ("ne64_conv", NE64, None),
            ("ne64_flat_bf16", dict(NE64, flatten=True), torch.bfloat16)]


@pytest.mark.parametrize("policy", [False, True], ids=["open", "heuristic"])
@pytest.mark.parametrize("name,cfg,odt", cfg_cases(), ids=[c[0] for c in cfg_cases()])
def test_random_actions_fed_back_equal_random_launch(name, cfg, odt, policy):
    """Random-mode equivalence: the evader actions of a random launch, read step by step off the env's stream by
    original index, fed to two chained EVC launches give the same obs, rew, done, info, actions and state blob."""
    E, T, T1 = 96, 60, 25
    Np, Ne = cfg["n_pursuers"], cfg["n_evaders"]
    act = torch.as_tensor(np.random.RandomState(2).randint(0, 5, size=(T, E, Np)).astype(np.int32), device="cuda")
    a = engine(cfg, E, odt)
    obs0 = a.reset()
    ev = np.zeros((T, E, Ne), np.int32)
    outs, prev = [], obs0
    for t in range(T):
        st = a.state
        ev[t] = V.random_evader_actions(SEED, BASE, st['rng_counter'].cpu().numpy(), st['gone'].cpu().numpy(), Ne,
                                        fill_seed=t)
        if policy:
            r = a.rollout_heuristic(1, prev)
        else:
            r = (act[t:t + 1],) + a.rollout(act[t:t + 1])
        outs.append([x.clone() for x in r])
        prev = r[1][0]
    want = [torch.cat(x) for x in zip(*outs)]
    assert want[3].any(), "no auto-reset inside the launch"

    b = engine(cfg, E, odt)
    ms = torch.zeros((E, 4, 16, 16), device="cuda")
    b.set_model_state(ms)
    assert torch.equal(b.reset(), obs0)
    evd = torch.as_tensor(ev, device="cuda")
    got = []
    for lo, hi in ((0, T1), (T1, T)):
        if policy:
            r = b.rollout_heuristic(hi - lo, obs0 if lo == 0 else got[-1][1][-1], evader_actions=evd[lo:hi])
        else:
            r = (act[lo:hi],) + b.rollout(act[lo:hi], evader_actions=evd[lo:hi])
        got.append([x.clone() for x in r])
    got = [torch.cat(x) for x in zip(*got)]
    for w, g, n in zip(want, got, ("actions", "obs", "rew", "done", "info")):
        assert torch.equal(w, g), n
    assert np.array_equal(blob(a), blob(b))


@pytest.mark.parametrize("a_fix", [4, 1])
def test_fixed_controller_forms_agree_with_oracle(a_fix):
    """set_evader_controller(a) == a stride-0 view of one row of a == an explicit [T, E, Ne] tensor of a, and equals
    the oracle under SingleActionPolicy(a)."""
    E, T = 64, 30
    cfg = C3
    act = np.random.RandomState(4).randint(0, 5, size=(T, E, cfg["n_pursuers"])).astype(np.int32)
    actd = torch.as_tensor(act, device="cuda")
    runs = []
    for kind in ("fixed", "row", "full"):
        eng = engine(cfg, E)
        obs0 = eng.reset()
        if kind == "fixed":
            eng.set_evader_controller(a_fix)
            out = eng.rollout(actd)
        elif kind == "row":
            row = torch.full((cfg["n_evaders"],), a_fix, dtype=torch.int32, device="cuda")
            out = eng.rollout(actd, evader_actions=row.expand(T, E, -1))
        else:
            out = eng.rollout(actd, evader_actions=torch.full((T, E, cfg["n_evaders"]), a_fix, dtype=torch.int32,
                                                              device="cuda"))
        runs.append([x.cpu().numpy() for x in (obs0,) + out] + [blob(eng)])
    for r in runs[1:]:
        for x, y in zip(runs[0], r):
            assert np.array_equal(x, y)
    case = D.PCase("c3", (1, 2, 7), lambda: MAPS, **C3)
    oracles = V.pe_oracles(case, MAPS, SEED, BASE, E)
    for e, o in enumerate(oracles):
        assert np.array_equal(D.f32(o.reset()), runs[0][0][e])
    w_obs, w_rew, w_done, w_rem = V.oracle_trajectory(oracles, act, np.full((T, E, cfg["n_evaders"]), a_fix), MPL)
    assert np.array_equal(runs[0][1], w_obs) and np.array_equal(runs[0][2], w_rew)
    assert np.array_equal(runs[0][3].astype(bool), w_done) and np.array_equal(runs[0][4], w_rem)


def test_model_state_matches_oracle_with_capture_at_last_step():
    """model_state after reset() and after launches, against the oracle, including an evader caught at the
    launch's last step: it is still in channel 2."""
    E, T = 256, 12
    cfg = dict(C3, surround=False, n_catch=1)   # a pursuer on an evader's cell catches it: captures are common
    eng = engine(cfg, E)
    ms = torch.full((E, 4, 16, 16), float("nan"), device="cuda")
    eng.set_model_state(ms)
    eng.reset()
    case = D.PCase("c3", (1, 2, 7), lambda: MAPS, **cfg)
    oracles = V.pe_oracles(case, MAPS, SEED, BASE, E)
    for e, o in enumerate(oracles):
        o.reset()
        assert np.array_equal(ms[e].cpu().numpy(), o.model_state), e
    rs = np.random.RandomState(8)
    caught_last = 0
    for k in range(4):
        act = rs.randint(0, 5, size=(T, E, cfg["n_pursuers"])).astype(np.int32)
        ev = rs.randint(-1, 6, size=(T, E, cfg["n_evaders"])).astype(np.int32)
        _, _, done, rem = eng.rollout(torch.as_tensor(act, device="cuda"), auto_reset=False,
                                      evader_actions=torch.as_tensor(ev, device="cuda"))
        V.oracle_trajectory(oracles, act, ev, 10 ** 9, auto_reset=False)
        m = ms.cpu().numpy()
        rem = rem.cpu().numpy()
        for e, o in enumerate(oracles):
            assert np.array_equal(m[e], o.model_state), (k, e)
            if rem[-1, e]:   # an evader caught at the last step is still counted
                caught_last += 1
                assert m[e, 2].sum() == (~o.gone).sum() + rem[-1, e]
    assert caught_last > 0


def test_policy_rollout_evader_policy_equals_manual_loop():
    """PolicyRollout(evader_policy=..., graph=False) == a hand-written loop of step() calls: the recorded evader
    actions are what the policy returned on each step's model_state."""
    E, T = 128, 20
    Ne = C3["n_evaders"]

    def policy(obs, state):
        a = (obs.float().sum(-1) * 13).long() % 5
        return a, {}, state

    def ev_policy(ms):   # [E, 4, xs, ys] -> [E, Ne]
        k = ms[:, 1].sum((1, 2)) * 3 + ms[:, 2].flatten(1).argmax(1)
        return (k.long()[:, None] + torch.arange(Ne, device=ms.device)) % 6

    results = []
    for mode in ("eager", "manual"):
        eng = engine(C3, E)
        ms = torch.zeros((E, 4, 16, 16), device="cuda")
        eng.set_model_state(ms)
        obs0 = eng.reset()
        if mode == "manual":
            acts, evs, obs_l, rew_l, done_l, info_l = [], [], [], [], [], []
            prev = obs0
            for t in range(T):
                a, _, _ = policy(prev, None)
                ev = ev_policy(ms).to(torch.int32)
                o, r, d, i = eng.step(a, auto_reset=True, evader_actions=ev)
                acts.append(a.to(torch.int32)); evs.append(ev)
                obs_l.append(o.clone()); rew_l.append(r.clone()); done_l.append(d.clone()); info_l.append(i['removed'].clone())
                prev = o
            res = [torch.stack(x) for x in (acts, obs_l, rew_l, done_l, info_l, evs)]
        else:
            out = PolicyRollout(eng, policy, T, graph=False, evader_policy=ev_policy)(obs0)
            res = [x.clone() for x in (out.actions, out.obs, out.rew, out.done, out.info, out.evader_actions)]
        results.append((res, blob(eng), ms.clone()))
    eager, manual = results
    assert eager[0][5].shape == (T, E, Ne) and eager[0][5].dtype == torch.int32
    for x, y in zip(eager[0], manual[0]):
        assert torch.equal(x, y)
    assert np.array_equal(eager[1], manual[1]) and torch.equal(eager[2], manual[2])


def test_policy_rollout_graph_replay_equals_eager():
    """Three chained calls: graph replays == eager calls, evader actions and model_state included."""
    E, T = 64, 16
    Ne = C3["n_evaders"]

    def policy(obs, state):
        return (obs.float().sum(-1) * 7).long() % 5, {}, state

    def ev_policy(ms):
        return ((ms[:, 1] * 5 + ms[:, 2]).flatten(1).sum(1).long()[:, None] + torch.arange(Ne, device=ms.device)) % 5

    outs = []
    for graph in (True, False):
        eng = engine(C3, E)
        ms = torch.zeros((E, 4, 16, 16), device="cuda")
        eng.set_model_state(ms)
        obs = eng.reset()
        pr = PolicyRollout(eng, policy, T, graph=graph, evader_policy=ev_policy)
        rec = []
        for _ in range(3):
            out = pr(obs)
            rec.append([x.clone() for x in (out.actions, out.obs, out.rew, out.done, out.info, out.evader_actions)])
            obs = out.obs[-1].clone()
        outs.append((rec, blob(eng), ms.clone()))
    for ra, rb in zip(outs[0][0], outs[1][0]):
        for x, y in zip(ra, rb):
            assert torch.equal(x, y)
    assert np.array_equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])
    assert len(out) == 8


class TableController(object):
    """Replays one action per call from a table indexed by (step, original evader index): calls come in live order,
    so the live rank is mapped back to the original index through the env's gone flags."""

    def __init__(self, table, env):
        self.table, self.env, self.t, self.k = table, env, 0, 0

    def live(self):
        g = int(self.env._engine.state['gone'][0].item())
        return [j for j in range(self.table.shape[1]) if not (g >> j) & 1]

    def act(self, state):
        assert state.shape == (4, self.env.xs, self.env.ys) and state.dtype == np.float32
        live = self.live()
        a = int(self.table[self.t, live[self.k]])
        self.k += 1
        if self.k == len(live):
            self.t, self.k = self.t + 1, 0
        return a


def test_drop_in_controllers_follow_oracle():
    """PursuitEvade(evader_controller=SingleActionPolicy(4)) and with a host controller object: step by step as the
    oracle under the same evader actions; the controller sees the model_state of the previous step."""
    kw = dict(n_evaders=6, n_pursuers=4, obs_range=5, n_catch=1, surround=False, reward_mech='local',
              random_opponents=True, max_opponents=7)
    T = 40
    rs = np.random.RandomState(11)
    table = rs.randint(0, 5, size=(T, 6)).astype(np.int32)
    act = rs.randint(0, 5, size=(T, 4)).astype(np.int32)
    for kind in ("single", "table"):
        ctl = TableController(table, None) if kind == "table" else SingleActionPolicy(4)
        env = PursuitEvade(MAPS, seed=SEED, evader_controller=ctl, **kw)
        if kind == "table":
            ctl.env = env
        case = D.PCase("small", (1, 1, 0), lambda: MAPS, **kw)
        o = V.pe_oracles(case, MAPS, SEED, 0, 1)[0]
        obs = env.reset()
        assert np.array_equal(D.f32(np.array(obs)), D.f32(np.array(o.reset())))
        for t in range(T):
            if kind == "table":
                ms_seen = o.model_state.copy()
                assert np.array_equal(env._model_state[0].cpu().numpy(), ms_seen)
            ev = table[t] if kind == "table" else 4
            oo, rr, dd, ii = o.step(act[t], ev)
            obs, rew, done, info = env.step(act[t])
            assert np.array_equal(D.f32(np.array(obs)), D.f32(np.array(oo))), (kind, t)
            assert np.array_equal(D.f32(rew), D.f32(rr)) and done == dd and info['removed'] == ii['removed']
            if done:
                break
        if kind == "table":
            assert ctl.t == t + 1


def test_stationary_evaluation_runs_against_fixed_evaders():
    """evaluate_heuristic on an engine with set_evader_controller(4): the evaders never move."""
    eng = engine(C3, 64)
    eng.set_evader_controller(4)
    obs0 = eng.reset()
    pos0 = (eng.state['evader_x'].clone(), eng.state['evader_y'].clone())
    eng.rollout_heuristic(5, obs0, auto_reset=False)
    assert torch.equal(eng.state['evader_x'], pos0[0]) and torch.equal(eng.state['evader_y'], pos0[1])
    assert evaluate_heuristic(eng, 64, 0.99, MODE, chunk=32) is not None
    eng.set_evader_controller(None)
    assert eng.evader_controller is None


def test_refusals():
    E = 8
    eng = engine(C3, E)
    eng.reset()
    act = torch.zeros((2, E, 8), dtype=torch.int32, device="cuda")
    good = torch.zeros((2, E, 30), dtype=torch.int32, device="cuda")
    for bad, err in ((good.long(), TypeError), (good[:, :, :29], ValueError), (good.cpu(), ValueError),
                     (good.transpose(0, 1).contiguous().transpose(0, 1), None),
                     (torch.zeros((2, E, 60), dtype=torch.int32, device="cuda")[:, :, ::2], ValueError)):
        if err is None:
            eng.rollout(act, evader_actions=bad)   # any step / env strides are read in place
            continue
        with pytest.raises(err):
            eng.rollout(act, evader_actions=bad)
    with pytest.raises(ValueError):
        eng.step(act[0], evader_actions=good[0, :, :5])
    with pytest.raises(ValueError):
        eng.set_model_state(torch.zeros((E, 4, 16, 15), device="cuda"))
    with pytest.raises(TypeError):
        eng.set_model_state(torch.zeros((E, 4, 16, 16), dtype=torch.float64, device="cuda"))
    with pytest.raises(TypeError):
        eng.set_evader_controller(1.5)
    with pytest.raises(TypeError):
        eng.set_evader_controller(True)
    for k in ("pursuer_controller", "ally_layer", "opponent_layer", "initial_config"):
        with pytest.raises(NotImplementedError):
            PursuitEvade(MAPS, **{k: SingleActionPolicy(4)})
    with pytest.raises(NotImplementedError):
        PursuitEvade(MAPS, train_pursuit=False)
    with pytest.raises(TypeError):
        PursuitEvade(MAPS, evader_controller=object())
    class Ctl(object):
        def act(self, model_state):
            return 1
    with pytest.raises(NotImplementedError):
        PursuitEvade(MAPS, evader_controller=Ctl()).vec_env_executor(4, 10)
    hw = BatchedHostageWorld(4, 10, 16, 16, 4, 2, device="cuda")
    with pytest.raises(ValueError):
        PolicyRollout(hw, lambda o, s: (o, {}, s), 4, evader_policy=lambda m: m)
    with pytest.raises(ValueError):   # no model_state to read
        PolicyRollout(engine(C3, E), lambda o, s: ((o.float().sum(-1)).long() % 5, {}, s), 2,
                      evader_policy=lambda m: m[:, 0, 0, :1].long().expand(-1, 30))(engine(C3, E).reset())
    assert _lib.PURSUIT_EVADERS_FIXED == 1
