"""PursuitEvade on the H100 engine (integer path, bit-exact with the reference).

``BatchedPursuitEvade`` is the batched tensor API; ``PursuitEvade`` is the drop-in for
``madrl_environments.pursuit.pursuit_evade.PursuitEvade`` (constructor ``PursuitEvade(map_pool,
**kwargs)`` with the reference's keyword names, pursuit_evade.py:28-152) backed by a one-env
engine, including the curriculum attributes that survive pickling (pursuit_evade.py:397-411).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import _ptr
from .core import Agent, EzPickle
from .engine import BatchedEngine, DropInEnv
from .spaces import Box, Discrete


class DiscreteAgent(Agent):
    """Per-pursuer descriptor (utils/DiscreteAgent.py:11-62): spaces only."""

    def __init__(self, obs_range=3, n_channels=3, flatten=False):
        self._obs_range = obs_range
        if flatten:
            self._obs_shape = (n_channels * obs_range ** 2 + 1,)
        else:
            self._obs_shape = (obs_range, obs_range, 4)

    @property
    def observation_space(self):
        return Box(low=-np.inf, high=np.inf, shape=self._obs_shape)

    @property
    def action_space(self):
        return Discrete(5)


def map_pool_array(map_pool):
    """The map pool as a C-contiguous int32 [n_maps, xs, ys] array (one [xs, ys] map is a pool of one)."""
    mp = np.ascontiguousarray(np.asarray(map_pool), dtype=np.int32)
    return mp[None] if mp.ndim == 2 else mp


def pe_config(n_envs, map_pool, n_evaders=1, n_pursuers=1, obs_range=3, flatten=True, layer_norm=10, n_catch=2,
              catchr=0.01, term_pursuit=5.0, urgency_reward=0.0, include_id=True, surround=True,
              constraint_window=1.0, sample_maps=False, reward_mech='global', random_opponents=False,
              max_opponents=10, seed=0, env_id_base=0, max_path_length=0):
    """The madrl_pursuit_config of BatchedPursuitEvade's arguments; `map_pool` as map_pool_array returns it."""
    return _lib.PEConfig(
        n_envs=n_envs, env_id_base=env_id_base, n_pursuers=n_pursuers, n_evaders=n_evaders,
        xs=map_pool.shape[1], ys=map_pool.shape[2], n_maps=map_pool.shape[0], obs_range=obs_range,
        flatten=int(bool(flatten)), n_catch=n_catch, surround=int(bool(surround)),
        reward_global=int(reward_mech == 'global'), include_id=int(bool(include_id)),
        sample_maps=int(bool(sample_maps)), max_path_length=int(max_path_length or 0),
        max_opponents=int(max_opponents) if random_opponents else 0,   # pursuit_evade.py:81-82,177-181
        layer_norm=float(layer_norm), catchr=float(catchr), term_pursuit=float(term_pursuit),
        urgency_reward=float(urgency_reward), constraint_window=float(constraint_window),
        seed=int(seed))


class BatchedPursuitEvade(BatchedEngine):
    """E lockstep PursuitEvade instances resident in HBM.

    Keyword names follow pursuit_evade.py:49-148.  Evader motion uses the env's counter-based
    stream (the reference's default controller is an unseeded RandomState shared by every
    instance, utils/Controllers.py:11, so there is no reference stream to reproduce).
    ``obs_dtype`` torch.float32 (None) or torch.bfloat16: observations stored as bfloat16, bit-identical to
    the float32 ones rounded to nearest even.  The in-kernel heuristic policy only tests which cells
    hold an evader, which rounding never changes, so chained bfloat16 launches equal one long launch.
    """

    _abi, _Layout, _act_tail, _info_tail, _info_keys = "pursuit", _lib.PELayout, (), (), ("removed",)

    def __init__(self, n_envs, map_pool, n_evaders=1, n_pursuers=1, obs_range=3, flatten=True,
                 layer_norm=10, n_catch=2, catchr=0.01, term_pursuit=5.0, urgency_reward=0.0,
                 include_id=True, surround=True, constraint_window=1.0, sample_maps=False,
                 reward_mech='global', random_opponents=False, max_opponents=10, device=None, seed=0,
                 env_id_base=0, max_path_length=0, obs_dtype=None):
        mp = map_pool_array(map_pool)
        cfg = pe_config(n_envs, mp, n_evaders=n_evaders, n_pursuers=n_pursuers, obs_range=obs_range,
                        flatten=flatten, layer_norm=layer_norm, n_catch=n_catch, catchr=catchr,
                        term_pursuit=term_pursuit, urgency_reward=urgency_reward, include_id=include_id,
                        surround=surround, constraint_window=constraint_window, sample_maps=sample_maps,
                        reward_mech=reward_mech, random_opponents=random_opponents, max_opponents=max_opponents,
                        seed=seed, env_id_base=env_id_base, max_path_length=max_path_length)
        self.map_pool = mp
        self.n_envs, self.n_pursuers, self.n_evaders = n_envs, n_pursuers, n_evaders
        self.obs_range, self.reward_mech, self.flatten = obs_range, reward_mech, bool(flatten)
        super().__init__(cfg, n_pursuers, device, torch.float32, torch.int32,
                         create_args=(C.c_void_p(mp.ctypes.data),), obs_dtype=obs_dtype)
        self.n_agents = int(self.layout.n_agents)   # pursuers + evaders (the state records), not the acting agents

    @property
    def state(self):
        L, E, Np, A, RR = self.layout, self.n_envs, self.n_pursuers, self.n_agents, self.obs_range ** 2
        pos = self._view(L.pos, torch.uint8, (E, 2, A))
        return dict(pursuer_x=pos[:, 0, :Np], pursuer_y=pos[:, 1, :Np], evader_x=pos[:, 0, Np:],
                    evader_y=pos[:, 1, Np:], gone=self._view(L.gone, torch.int64, (E,)),
                    map_id=self._view(L.map_id, torch.int32, (E,)),
                    path_len=self._view(L.path_len, torch.int32, (E,)),
                    rng_counter=self._view(L.rng_counter, torch.int64, (E,)),
                    stale=self._view(L.stale, torch.int16, (E, Np, RR)))

    def render_frames(self, env_ids, cell=16, out=None):
        """Frames of the listed envs (a sequence or an int tensor; repeats allowed; a sharded engine's local ids):
        uint8 [n, ys * cell, xs * cell, 3], RGB, on the engine's device -- the picture of the reference's render
        (pursuit_evade.py:274-295) under the integer rule of DESIGN §4.10: pixel (row, col) shows cell
        (col // cell, row // cell); free cells white, buildings (64, 64, 64); each pursuer's observation window
        blended with #FF9848 as (v + o + 1) >> 1; then pursuer markers (255, 0, 0) and live evader markers
        (0, 0, 255) over the cell's [cell/4, cell - cell/4) square.  `out` as BatchedMAWaterWorld.render_frames."""
        c = int(cell)
        if c != cell or c < 1:
            raise ValueError("cell must be an int >= 1, got %r" % (cell,))
        return self._render(env_ids, (self.map_pool.shape[2] * c, self.map_pool.shape[1] * c, 3), out, c)

    def set_params(self, catchr=None, constraint_window=None):
        """Curriculum updates (pursuit_evade.py:264-272)."""
        if catchr is not None:
            self.cfg.catchr = float(catchr)
        if constraint_window is not None:
            self.cfg.constraint_window = float(constraint_window)
        _lib.check(self._L.madrl_pursuit_set_params(self._h, self.cfg.catchr, self.cfg.constraint_window))
        self._launch_settings_changed()

    def rollout_heuristic(self, T, obs0, auto_reset=True, out=None, record_actions=True, py2_division=True,
                          actions_out=None, evader_actions=None):
        """T lockstep steps in one launch with the reference's hand-written policy
        (heuristics/pursuit.py:18-50: walk towards the nearest visible evader, a random move when none is
        visible) evaluated inside the kernel: closed loop, no action tensor, no per-step launch.
        obs0 [E, Np, D] = the observation the first action is computed from (`reset()`'s, or `obs[-1]` of
        the previous rollout).  `py2_division`: the window centre `xs / 2` (heuristics/pursuit.py:23) as
        Python 2 -- the reference's language -- computes it (R // 2); False = Python 3 true division.
        `evader_actions`: as rollout()'s.
        Returns (actions int32 [T,E,Np] or None, obs, rew, done, removed)."""
        if evader_actions is None:
            return self._rollout_heuristic(T, obs0, auto_reset, out, record_actions, actions_out,
                                           int(bool(py2_division)))
        st, se = self._evader_strides(evader_actions, T)
        return self._rollout_heuristic(T, obs0, auto_reset, out, record_actions, actions_out, int(bool(py2_division)),
                                       fn="rollout_heuristic_evaders", mid=(_ptr(evader_actions), st, se))

    # ---- the evaders' controller (pursuit_evade.py:87 evader_controller, DESIGN §4.2) ----
    evader_controller = None   # set_evader_controller's argument
    model_state = None         # set_model_state's tensor

    def set_evader_controller(self, action=None):
        """The evaders' controller of every launch that is given no `evader_actions`: None = the reference's
        default RandomPolicy(5), one draw of the env's stream per live evader per step; an int `a` =
        SingleActionPolicy(a), every evader takes action a each step (4 = stay: the stationary evaluation;
        a value outside 0..3 stays too).  evaluate_heuristic / evaluate_policy on this engine then run against
        those evaders.  A launch setting: a PolicyRollout graph is re-captured after it."""
        if action is None:
            mode, a = _lib.PURSUIT_EVADERS_RANDOM, 4
        else:
            if isinstance(action, bool) or not isinstance(action, (int, np.integer)):
                raise TypeError("the evader controller must be None (random) or an int action, got %r" % (action,))
            if not -2 ** 31 <= int(action) < 2 ** 31:
                raise ValueError("the evader action must fit in int32, got %d" % action)
            mode, a = _lib.PURSUIT_EVADERS_FIXED, int(action)
        _lib.check(self._L.madrl_pursuit_set_evader_control(self._h, mode, a))
        self.evader_controller = None if action is None else a
        self._launch_settings_changed()

    def set_model_state(self, out):
        """After this call reset() and every rollout write `out`, float32 [E, 4, xs, ys] on the engine's device: the
        reference's model_state (pursuit_evade.py:152) of each env they touch as it stands after the launch's last
        step -- channel 0 the map (-1 building, 0 free), 1 pursuer counts, 2 evader counts, 3 zeros -- taken, like
        the reference, before that step's removals (an evader caught at the last step is still counted).  It is
        what the reference hands the evader controller at the next step.  None switches it off."""
        E, xs, ys = self.n_envs, self.map_pool.shape[1], self.map_pool.shape[2]
        _lib.require_tensor(out, "model_state", torch.float32, (E, 4, xs, ys), self.device, optional=True)
        _lib.check(self._L.madrl_pursuit_set_model_state(self._h, _ptr(out)))
        self.model_state = out
        self._launch_settings_changed()

    def _evader_strides(self, ev, T):
        """Check a caller's evader actions int32 [T, E, Ne] -> the element strides (step, env) the kernel indexes
        with.  Any strides >= 0 are taken as long as the evader axis is dense, so an expanded view (one row of
        Ne actions for every env and step: stride 0 and 0) is read without a copy."""
        _lib.require_tensor(ev, "evader_actions", torch.int32, (T, self.n_envs, self.n_evaders), self.device,
                            contiguous=False)
        if self.n_evaders > 1 and ev.stride(2) != 1:
            raise ValueError("evader_actions must be dense along the evader axis (stride 1), got strides %s"
                             % (ev.stride(),))
        return ev.stride(0), ev.stride(1)

    def rollout(self, actions, auto_reset=True, out=None, evader_actions=None):
        """BatchedEngine.rollout.  `evader_actions` int32 [T, E, Ne] on the engine's device moves evader j of env
        e at step t by evader_actions[t, e, j] (j its original index; entries of removed evaders and of evaders
        that do not exist this episode are not read; a value outside 0..3 stays) instead of the controller of
        set_evader_controller."""
        if evader_actions is None:
            return super().rollout(actions, auto_reset, out)
        actions = actions.to(device=self.device, dtype=self._act_dtype).contiguous()
        T = _lib.require_tensor(actions, "actions", self._act_dtype, (None, self.n_envs, self._n_acting),
                                self.device).shape[0]
        st, se = self._evader_strides(evader_actions, T)
        obs, rew, done, info = self._outputs(T, out, auto_reset)
        with torch.cuda.device(self.device):
            _lib.check(self._L.madrl_pursuit_rollout_evaders(self._h, T, _ptr(actions), _ptr(evader_actions), st, se,
                                                             _ptr(obs), _ptr(rew), _ptr(done), _ptr(info),
                                                             int(auto_reset), _lib.stream(self.device)))
        return obs, rew, done, info

    def step(self, actions, auto_reset=False, out=None, evader_actions=None):
        """BatchedEngine.step.  `evader_actions`: int32 [E, Ne], rollout()'s for one step."""
        if evader_actions is None:
            return super().step(actions, auto_reset, out)
        _lib.require_tensor(evader_actions, "evader_actions", torch.int32, (self.n_envs, self.n_evaders), self.device,
                            contiguous=False)
        return super().step(actions, auto_reset, out, evader_actions=evader_actions.unsqueeze(0))


class RandomPolicy(object):
    """The reference's default evader controller (utils/Controllers.py:8-16): a uniform action of
    `n_actions`.  PursuitEvade runs RandomPolicy(5) on the device, from the env's own stream."""

    def __init__(self, n_actions, rng=np.random.RandomState()):
        self.rng = rng
        self.n_actions = n_actions

    def act(self, state):
        return self.rng.randint(self.n_actions)


class SingleActionPolicy(object):
    """The reference's constant controller (utils/Controllers.py:19-26): SingleActionPolicy(4) keeps the evaders
    where they spawned (the stationary evaluation)."""

    def __init__(self, a):
        self.action = a

    def act(self, state):
        return self.action


def _controller_kind(c):
    """(fixed action or None, host controller?) of a drop-in's evader_controller: None and RandomPolicy(5) are the
    device's random controller; a SingleActionPolicy (this module's or any class of that name with `.action`) is
    the fixed one; any other object with act(model_state) is called on the host."""
    name = type(c).__name__
    if c is None or (name == 'RandomPolicy' and getattr(c, 'n_actions', None) == 5):
        return None, False
    if name == 'SingleActionPolicy' and hasattr(c, 'action'):
        return int(c.action), False
    if not callable(getattr(c, 'act', None)):
        raise TypeError("evader_controller must have act(model_state), got %r" % (c,))
    return None, True


class PursuitEvade(DropInEnv):
    """Drop-in for the reference class: ``PursuitEvade(map_pool, **kwargs)``."""

    def __init__(self, map_pool, **kwargs):
        EzPickle.__init__(self, map_pool, **kwargs)
        kw = dict(kwargs)
        self.sample_maps = kw.pop('sample_maps', False)
        self.map_pool = map_pool
        self.map_matrix = np.asarray(map_pool)[0]
        self.xs, self.ys = self.map_matrix.shape
        self._reward_mech = kw.pop('reward_mech', 'global')
        self.n_evaders = kw.pop('n_evaders', 1)
        self.n_pursuers = kw.pop('n_pursuers', 1)
        self.obs_range = kw.pop('obs_range', 3)
        self.obs_offset = int((self.obs_range - 1) / 2)
        self.flatten = kw.pop('flatten', True)
        self.layer_norm = kw.pop('layer_norm', 10)
        self.n_catch = kw.pop('n_catch', 2)
        self.random_opponents = kw.pop('random_opponents', False)      # pursuit_evade.py:81-82
        self.max_opponents = kw.pop('max_opponents', 10)
        self.catchr = kw.pop('catchr', 0.01)
        self.caughtr = kw.pop('caughtr', -0.01)
        self.term_pursuit = kw.pop('term_pursuit', 5.0)
        self.term_evade = kw.pop('term_evade', -5.0)
        self.urgency_reward = kw.pop('urgency_reward', 0.0)
        self.include_id = kw.pop('include_id', True)
        if not kw.pop('train_pursuit', True):   # DESIGN §8: the reference's evader-training mode does not hold together
            raise NotImplementedError("train_pursuit=False is not supported by the batched engine")
        self.surround = kw.pop('surround', True)
        self.constraint_window = kw.pop('constraint_window', 1.0)
        self.curriculum_remove_every = kw.pop('curriculum_remove_every', 500)
        self.curriculum_constrain_rate = kw.pop('curriculum_constrain_rate', 0.0)
        self.curriculum_turn_off_shaping = kw.pop('curriculum_turn_off_shaping', np.inf)
        self._engine_kwargs = dict(device=kw.pop('device', None))
        self._seed_value = kw.pop('seed', 0)
        self._env_id = kw.pop('env_id', 0)
        for k in ('ally_layer', 'opponent_layer', 'pursuer_controller', 'initial_config'):
            if kw.pop(k, None) is not None:
                raise NotImplementedError("%s cannot be injected into the batched engine" % k)
        self.evader_controller = kw.pop('evader_controller', None)
        self._ev_fixed, self._ev_host = _controller_kind(self.evader_controller)
        n = 3 * self.obs_range ** 2 + (1 if self.include_id else 0)
        self.low, self.high = np.zeros(n), np.ones(n)
        self.action_space = Discrete(5)
        if self.flatten:
            self.observation_space = Box(self.low, self.high)
        else:
            self.observation_space = Box(low=-np.inf, high=np.inf, shape=(4, self.obs_range, self.obs_range))
        self.act_dims = [5 for _ in range(self.n_pursuers)]
        self.setup()

    def _make_engine(self, n_envs, **kw):
        # looks up the module-level class at call time, so that a test double can stand in for it
        eng = BatchedPursuitEvade(n_envs, self.map_pool, n_evaders=self.n_evaders, n_pursuers=self.n_pursuers,
                                   obs_range=self.obs_range, flatten=self.flatten, layer_norm=self.layer_norm,
                                   n_catch=self.n_catch, catchr=self.catchr, term_pursuit=self.term_pursuit,
                                   urgency_reward=self.urgency_reward, include_id=self.include_id,
                                   surround=self.surround, constraint_window=self.constraint_window,
                                   sample_maps=self.sample_maps, reward_mech=self._reward_mech,
                                   random_opponents=self.random_opponents, max_opponents=self.max_opponents,
                                   seed=self._seed_value, **self._engine_kwargs, **kw)
        if self._ev_fixed is not None:
            eng.set_evader_controller(self._ev_fixed)
        return eng

    def setup(self):
        self.pursuers = [DiscreteAgent(self.obs_range, flatten=self.flatten) for _ in range(self.n_pursuers)]
        super().setup()
        self._n_live = self.n_evaders
        if self._ev_host:
            self._model_state = torch.zeros((1, 4, self.xs, self.ys), dtype=torch.float32, device=self._engine.device)
            self._engine.set_model_state(self._model_state)

    def vec_env_executor(self, n_envs, max_path_length):
        if self._ev_host:
            raise NotImplementedError("a host evader_controller steps one env at a time; the batched executor "
                                      "takes None, RandomPolicy(5) or SingleActionPolicy")
        return super().vec_env_executor(n_envs, max_path_length)

    @property
    def agents(self):
        return self.pursuers

    def n_agents(self):
        return self.n_pursuers

    def reset(self):
        self._engine.set_params(self.catchr, self.constraint_window)
        obs = self._engine.reset().cpu().numpy().astype(np.float64)
        self._n_live = self.n_evaders
        if self.random_opponents:      # this episode's evader count was drawn on the device (pursuit_evade.py:179)
            gone = int(self._engine.state['gone'][0].item()) & ((1 << self.n_evaders) - 1)
            self._n_live = self.n_evaders - bin(gone).count("1")
        return [self._shape(obs[0, i]) for i in range(self.n_pursuers)]

    def _shape(self, o):
        return o if self.flatten else o.reshape(self.obs_range, self.obs_range, 4)

    @property
    def is_terminal(self):
        return self._n_live == 0

    def step(self, actions):
        if isinstance(actions, (list, np.ndarray)):
            acts = np.asarray(actions).reshape(-1)[:self.n_pursuers]
        else:  # one joint action, pursuit_evade.py:233
            acts = np.array(np.unravel_index(actions, self.act_dims))
        kw = {}
        if self._ev_host:   # pe:237-241: act(model_state) once per live evader, in index order
            ms = self._model_state[0].cpu().numpy()
            gone = int(self._engine.state['gone'][0].item())
            a = np.full(self.n_evaders, 4, np.int32)
            for j in range(self.n_evaders):
                if not (gone >> j) & 1:
                    a[j] = self.evader_controller.act(ms)
            kw['evader_actions'] = torch.as_tensor(a[None], device=self._engine.device)
        obs, rew, done, info = self._engine.step(acts.astype(np.int32)[None], auto_reset=False, **kw)
        obs = obs.cpu().numpy().astype(np.float64)
        rew = rew[0].cpu().numpy().astype(np.float64)
        removed = int(info['removed'][0].item())
        self._n_live -= removed
        obslist = [self._shape(obs[0, i]) for i in range(self.n_pursuers)]
        if self._reward_mech == 'global':
            return obslist, [rew[0]] * self.n_pursuers, bool(done[0].item()), {'removed': removed}
        return obslist, rew, bool(done[0].item()), {'removed': removed}

    def render(self, plt_delay=1.0, cell=16):
        """Env 0's frame (BatchedPursuitEvade.render_frames) as a NumPy RGB uint8 array [ys * cell, xs * cell, 3],
        where the reference plots it with matplotlib.  No window is opened: `plt_delay` is accepted for the
        reference's signature and unused."""
        return self._frame(cell=cell)

    def update_curriculum(self, itr):
        self.constraint_window += self.curriculum_constrain_rate
        self.constraint_window = np.clip(self.constraint_window, 0.0, 1.0)
        if itr != 0 and itr % self.curriculum_remove_every == 0 and self.n_pursuers > 4:
            self.n_evaders -= 1
            self.n_pursuers -= 1
            self.setup()
        if itr > self.curriculum_turn_off_shaping:
            self.catchr = 0.0

    def __getstate__(self):
        d = EzPickle.__getstate__(self)
        d['constraint_window'] = self.constraint_window
        d['n_evaders'] = self.n_evaders
        d['n_pursuers'] = self.n_pursuers
        d['catchr'] = self.catchr
        return d

    def __setstate__(self, d):
        EzPickle.__setstate__(self, d)
        self.constraint_window = d['constraint_window']
        self.n_evaders = d['n_evaders']
        self.n_pursuers = d['n_pursuers']
        self.catchr = d['catchr']
        self.setup()
