"""Writes tests/golden/replay_pool_ref.npz: rllab's DDPG replay pool as the REFERENCE's own ``DDPG.train`` fills it
(rllab/rllab/algos/ddpg.py:268-366, decentralized mode) on a scripted env, and the slots its ``random_batch``
accepts.

Executed from reference source: ``DDPG.__init__`` / ``DDPG.train`` and ``MAReplayPool`` (ddpg.py, loaded from its
file with oracle.refshim's rllab stubs, plus stubs for ``pyprind`` (prog_bar = the iterable), ``lasagne.updates``
and ``rllab.plotter``).  ``start_worker``, ``init_opt``, ``do_training``, ``evaluate`` and ``get_epoch_snapshot`` are
no-ops, and the logger's calls do nothing; the policy and exploration strategy are stubs whose action is a fixed
function of the agent's observation.  The pool class is swapped for a subclass that records:
  * the pool's arrays and top / bottom / size after the run;
  * at each ``random_batch`` call of the loop, the slots the real ``MAReplayPool.random_batch`` accepts when its
    ``np.random.randint`` offers every candidate in [bottom, bottom + size) once, in descending order, with
    batch_size = size - 1 (run on a copy of the ring counters whose rewards are the slot numbers).

The scripted env (A agents, D-dim float32-representable observations, float32-representable rewards) ends an episode
by itself when its timestep reaches ``timestep_limit``, or at scripted event steps (Hostage's bomb), and DDPG cuts at
``max_path_length``.  The engine-shaped rollout of the same run is stored too (E = 1: obs, act, rew, done,
obs_before, term; the env's counters start at 0), so tests can feed oracle/replay_oracle.py the same transitions.

Cases (each 2 epochs x 40 steps, a pool of 13 slots that wraps several times):
  cuts        max_path_length 4, timestep_limit 7: horizon cuts, dropped
  cuts_kept   the same with include_horizon_terminal_transitions
  at_limit    max_path_length 5, timestep_limit 5: the env terminates exactly at the horizon (stored, terminal)
  events      max_path_length 6, timestep_limit 50, env-terminal events at path lengths 2 and 3, and cuts
Run:  python -m oracle.make_replay_golden
"""
import importlib.util
import os
import sys
import types

import numpy as np

from oracle import refshim

A, D, AD, M = 2, 5, 2, 13
CASES = {"cuts": (4, 7, False, ()), "cuts_kept": (4, 7, True, ()), "at_limit": (5, 5, False, ()),
         "events": (6, 50, False, (2, 3))}


def _module(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


def load_ddpg():
    """rllab/rllab/algos/ddpg.py, executed from its file."""
    refshim.load_rllab_callers()
    if "pyprind" not in sys.modules:
        _module("pyprind", prog_bar=lambda it, **k: it)
    if "lasagne" not in sys.modules:
        las = _module("lasagne")
        las.updates = _module("lasagne.updates", adam=lambda *a, **k: None, sgd=lambda *a, **k: None)
    if "rllab.plotter" not in sys.modules:
        _module("rllab.plotter").plotter = _module("rllab.plotter.plotter", init_plot=None, update_plot=None)
    spec = importlib.util.spec_from_file_location(
        "_ref_ddpg", os.path.join(refshim.REFERENCE_ROOT, "rllab", "rllab", "algos", "ddpg.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.logger = types.SimpleNamespace(push_prefix=lambda *a: None, pop_prefix=lambda *a: None,
                                       log=lambda *a, **k: None, dump_tabular=lambda *a, **k: None,
                                       save_itr_params=lambda *a: None)
    return mod


class _Space(object):
    def __init__(self, n):
        self.flat_dim = n

    def flatten(self, x):
        return np.asarray(x, np.float64).ravel()


class ScriptedEnv(object):
    """A agents; an episode ends by itself at timestep_limit or at the path lengths in `events`."""

    def __init__(self, timestep_limit, events, seed):
        self.agents = list(range(A))
        self.observation_space, self.action_space = _Space(D), _Space(AD)
        self.timestep_limit, self.events = timestep_limit, events
        self.rs = np.random.RandomState(seed)
        self.log = []            # ('reset', obs) / ('step', action, next_obs, reward, terminal)
        self.episode = 0

    def _obs(self):
        return [self.rs.randn(D).astype(np.float32).astype(np.float64) for _ in range(A)]

    def reset(self):
        self.t = 0
        self.episode += 1
        o = self._obs()
        self.log.append(("reset", o))
        return o

    def step(self, action):
        self.t += 1
        o = self._obs()
        r = [float(np.float32(x)) for x in self.rs.randn(A) * 3]
        # scripted events: at the given path length of every other episode
        term = self.t >= self.timestep_limit or (self.episode % 2 == 0 and self.t in self.events)
        self.log.append(("step", np.array(action, np.float64), o, r, term))
        return o, r, term, {}


class Policy(object):
    def reset(self):
        pass

    def get_param_values(self):
        return np.zeros(1)

    def set_param_values(self, v):
        pass

    def terminate(self):
        pass


class Strategy(object):
    def reset(self):
        pass

    def get_action(self, itr, observation, policy):
        return (np.asarray(observation[:AD]) * 0.5).astype(np.float32).astype(np.float64)


class _Candidates(object):
    """np.random stand-in: randint offers the candidates of [low, high) in descending order, cyclically."""

    def __init__(self):
        self.k = 0

    def randint(self, low, high):
        n = high - low
        self.k += 1
        if self.k > 3 * n:
            raise RuntimeError("random_batch did not finish on the offered candidates")
        return high - 1 - (self.k - 1) % n


def run_case(mod, max_path_length, timestep_limit, include, events, seed):
    accepted, pools = [], []
    Base = mod.MAReplayPool

    class RecordingPool(Base):
        def __init__(self, *a, **k):
            Base.__init__(self, *a, **k)
            pools.append(self)

        def random_batch(self, batch_size):
            shadow = Base(self._max_pool_size, 1, 1)
            shadow._rewards = np.arange(self._max_pool_size, dtype=np.float64)
            shadow._bottom, shadow._top, shadow._size = self._bottom, self._top, self._size
            real_np = mod.np
            mod.np = types.SimpleNamespace(random=_Candidates(), zeros=np.zeros)
            try:
                got = Base.random_batch(shadow, self._size - 1)
            finally:
                mod.np = real_np
            accepted.append((self._bottom, self._size, np.unique(got["rewards"].astype(np.int64))))
            return got

    mod.MAReplayPool = RecordingPool
    env = ScriptedEnv(timestep_limit, events, seed)
    algo = mod.DDPG(env, Policy(), None, Strategy(), batch_size=4, n_epochs=2, epoch_length=40, min_pool_size=5,
                    replay_pool_size=M, max_path_length=max_path_length, scale_reward=0.01,
                    include_horizon_terminal_transitions=include, mode="decentralized")
    algo.start_worker = algo.init_opt = lambda *a: None
    algo.do_training = algo.evaluate = lambda *a: None
    algo.get_epoch_snapshot = lambda *a: {}
    algo.train()
    pool = pools[0]
    # the engine-shaped rollout of the run: E = 1
    steps = [x for x in env.log if x[0] == "step"]
    T = len(steps)
    obs_before = np.array(env.log[0][1])[None]
    obs, term = np.zeros((T, 1, A, D)), np.zeros((T, 1, A, D))
    act, rew, done = np.zeros((T, 1, A, AD)), np.zeros((T, 1, A)), np.zeros((T, 1), np.uint8)
    resets = iter([x[1] for x in env.log[1:] if x[0] == "reset"])
    for t, (_, a, o, r, terminal) in enumerate(steps):
        act[t, 0], rew[t, 0] = a, r
        # DDPG's own horizon ends the path as the engine's max_path_length does
        done[t, 0] = 1 if terminal or _path_len(done, t) + 1 >= max_path_length else 0
        obs[t, 0] = o
        if done[t, 0]:
            term[t, 0] = o
            obs[t, 0] = next(resets, np.zeros((A, D)))   # the last step's reset is never drawn; nothing reads it
    out = dict(observations=pool._observations, next_observations=pool._next_observations, actions=pool._actions,
               rewards=pool._rewards, terminals=pool._terminals,
               ring=np.array([pool._top, pool._bottom, pool._size], np.int64),
               obs=obs, act=act, rew=rew, done=done, obs_before=obs_before, term=term,
               config=np.array([max_path_length, timestep_limit, int(include), M], np.int64),
               acc_state=np.array([(b, s) for b, s, _ in accepted], np.int64).reshape(-1, 2),
               acc_slots=np.concatenate([x for _, _, x in accepted]) if accepted else np.zeros(0, np.int64),
               acc_count=np.array([len(x) for _, _, x in accepted], np.int64))
    return out


def _path_len(done, t):
    """Steps since the last done before step t."""
    n = 0
    for u in range(t - 1, -1, -1):
        if done[u, 0]:
            break
        n += 1
    return n


def main():
    mod = load_ddpg()
    base = mod.MAReplayPool
    arrays = {}
    for k, (name, (mpl, limit, include, events)) in enumerate(CASES.items()):
        mod.MAReplayPool = base
        for key, v in run_case(mod, mpl, limit, include, events, seed=100 + k).items():
            arrays["%s__%s" % (name, key)] = v
    path = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                        "replay_pool_ref.npz")
    np.savez_compressed(path, **arrays)
    print("wrote", path, sum(v.nbytes for v in arrays.values()), "bytes")


if __name__ == "__main__":
    main()
