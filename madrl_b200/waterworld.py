"""MAWaterWorld on the H100 engine.

``BatchedMAWaterWorld`` is the batched tensor API (E envs, torch CUDA tensors in and out).
``MAWaterWorld`` is the drop-in for ``madrl_environments.pursuit.waterworld.MAWaterWorld``
(same constructor, ``reset/step/seed/agents/reward_mech/timestep_limit/is_terminal/
get_param_values/set_param_values``; waterworld.py:75-436) backed by a one-env engine, and it
advertises rllab's batched plug-in hook (``vectorized`` / ``vec_env_executor``;
rllab/sandbox/rocky/tf/envs/base.py:97-103) so that ``VectorizedSampler`` gets a GPU batch.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from .core import Agent, EzPickle
from .engine import BatchedEngine, DropInEnv
from .spaces import Box


class Archea(Agent):
    """Per-pursuer descriptor (waterworld.py:10-39): spaces only; state lives on the GPU."""

    def __init__(self, idx, radius, n_sensors, sensor_range, addid=True, speed_features=True):
        self._idx = idx
        self._radius = radius
        self._n_sensors = n_sensors
        self._sensor_range = sensor_range
        self._sensor_obscoord = 4 + (3 if speed_features else 0)
        self._obs_dim = n_sensors * self._sensor_obscoord + 2 + (1 if addid else 0)

    @property
    def observation_space(self):
        return Box(low=-10, high=10, shape=(self._obs_dim,))

    @property
    def action_space(self):
        return Box(low=-1, high=1, shape=(2,))


def ww_config(n_envs, n_pursuers, n_evaders, n_coop=2, n_poison=10, radius=0.015, obstacle_radius=0.2,
              obstacle_loc=np.array([0.5, 0.5]), ev_speed=0.01, poison_speed=0.01, n_sensors=30, sensor_range=0.2,
              action_scale=0.01, poison_reward=-1., food_reward=1., encounter_reward=.05, control_penalty=-.5,
              reward_mech='local', addid=True, speed_features=True, seed=0, env_id_base=0, max_path_length=0,
              fp64=False):
    """The madrl_ww_config of BatchedMAWaterWorld's arguments (`obstacle_loc=None`: a random obstacle)."""
    rand_obst = obstacle_loc is None
    ox, oy = (0.0, 0.0) if rand_obst else (float(obstacle_loc[0]), float(obstacle_loc[1]))
    return _lib.WWConfig(
        n_envs=n_envs, env_id_base=env_id_base, n_pursuers=n_pursuers, n_evaders=n_evaders,
        n_poison=n_poison, n_sensors=n_sensors, n_coop=n_coop,
        reward_global=int(reward_mech == 'global'), addid=int(bool(addid)),
        speed_features=int(bool(speed_features)), random_obstacle=int(rand_obst),
        timestep_limit=1000, max_path_length=int(max_path_length or 0),
        fp64=int(fp64), radius=radius, obstacle_radius=obstacle_radius,
        obstacle_x=ox, obstacle_y=oy, ev_speed=ev_speed, poison_speed=poison_speed,
        sensor_range=sensor_range, action_scale=action_scale, poison_reward=poison_reward,
        food_reward=food_reward, encounter_reward=encounter_reward,
        control_penalty=control_penalty, seed=int(seed))


class BatchedMAWaterWorld(BatchedEngine):
    """E lockstep MAWaterWorld instances resident in HBM.

    Parameters mirror waterworld.py:77-81 plus the batch/engine arguments:
    ``n_envs``; ``device``; ``seed`` and ``env_id_base`` (RNG key = (seed, env_id_base + e), so a
    sharded batch reproduces the unsharded one); ``max_path_length`` (VecEnvExecutor horizon);
    ``dtype`` torch.float32 (production) or torch.float64 (verification build); ``obs_dtype``
    ``dtype`` (None) or torch.bfloat16 with float32 ``dtype``: observations stored as bfloat16,
    bit-identical to the float32 ones rounded to nearest even (madrl_ww_set_obs_format).  The
    in-kernel heuristic policy widens a bfloat16 ``obs0``, so its first decision after a launch
    boundary sees rounded features: chained launches equal one long launch in float32 only.
    """

    timestep_limit = 1000
    _abi, _Layout, _act_tail, _info_tail, _info_keys = "ww", _lib.WWLayout, (2,), (2,), ("evcatches", "pocatches")

    def __init__(self, n_envs, n_pursuers, n_evaders, n_coop=2, n_poison=10, radius=0.015,
                 obstacle_radius=0.2, obstacle_loc=np.array([0.5, 0.5]), ev_speed=0.01,
                 poison_speed=0.01, n_sensors=30, sensor_range=0.2, action_scale=0.01,
                 poison_reward=-1., food_reward=1., encounter_reward=.05, control_penalty=-.5,
                 reward_mech='local', addid=True, speed_features=True, device=None, seed=0,
                 env_id_base=0, max_path_length=0, dtype=torch.float32, obs_dtype=None):
        assert dtype in (torch.float32, torch.float64)
        cfg = ww_config(n_envs, n_pursuers, n_evaders, n_coop=n_coop, n_poison=n_poison, radius=radius,
                        obstacle_radius=obstacle_radius, obstacle_loc=obstacle_loc, ev_speed=ev_speed,
                        poison_speed=poison_speed, n_sensors=n_sensors, sensor_range=sensor_range,
                        action_scale=action_scale, poison_reward=poison_reward, food_reward=food_reward,
                        encounter_reward=encounter_reward, control_penalty=control_penalty,
                        reward_mech=reward_mech, addid=addid, speed_features=speed_features, seed=seed,
                        env_id_base=env_id_base, max_path_length=max_path_length, fp64=dtype == torch.float64)
        self.n_envs, self.n_pursuers, self.n_evaders, self.n_poison = n_envs, n_pursuers, n_evaders, n_poison
        self.n_sensors = n_sensors
        self.reward_mech = reward_mech
        super().__init__(cfg, n_pursuers, device, dtype, dtype, obs_dtype=obs_dtype)
        self.n_obj = int(self.layout.n_obj)

    @property
    def state(self):
        """Named views into the HBM state blob (one record per env)."""
        L, E, N, dt = self.layout, self.n_envs, self.n_obj, self.dtype
        objs = self._view(L.objs, dt, (E, 4, N))
        obst = self._view(L.obst, dt, (E, 2))
        return dict(
            pos_x=objs[:, 0], pos_y=objs[:, 1], vel_x=objs[:, 2], vel_y=objs[:, 3],
            obst_x=obst[:, 0], obst_y=obst[:, 1],
            timestep=self._view(L.timestep, torch.int32, (E,)),
            path_len=self._view(L.path_len, torch.int32, (E,)),
            rng_counter=self._view(L.rng_counter, torch.int64, (E,)),
            sensors=self._view(L.sensors, dt, (2, self.n_sensors)))

    def render_frames(self, env_ids, screen_size=800, out=None):
        """Frames of the listed envs (a sequence or an int tensor; repeats allowed; a sharded engine's local ids)
        as the reference's render draws them (waterworld.py:438-479, with 8-connected lines and circles in place
        of the anti-aliased ones; DESIGN §4.10): uint8 [n, screen_size, screen_size, 3], RGB, on the engine's
        device.  `out`: a tensor of that shape to draw into; with it and a CUDA tensor of ids the call makes no
        host synchronisation and no allocation after its first call, and may be captured in a CUDA graph."""
        return self._render_sensor_frames(env_ids, screen_size, out)

    def set_peers(self, rank, t_max, rew_peers, done_peers, info_peers):
        """Enable the fused exchange: `*_peers` are lists (one per DESTINATION rank) of tensors
        aliasing the destination gather buffers; this rank writes slot `rank` of each
        (see madrl_b200.dist.PeerGather).  Each destination is contiguous on the engine's device, with S > rank
        slots: rewards (S, E, t_max, Np) of the engine's dtype, dones (S, E, t_max) uint8 and infos
        (S, E, t_max, 2) int32.  Every rollout must then be one launch: rollout() or step().  rollout_host and
        PolicyRollout, which run a rollout as several launches, refuse to run while peers are set."""
        n = len(rew_peers)
        if not 1 <= n <= 8 or len(done_peers) != n or len(info_peers) != n:
            raise ValueError("set_peers needs 1 to 8 destinations and as many reward, done and info buffers, got "
                             "%d, %d and %d" % (n, len(done_peers), len(info_peers)))
        rank, t_max = int(rank), int(t_max)
        if rank < 0 or t_max < 1:
            raise ValueError("set_peers needs rank >= 0 and t_max >= 1, got %d and %d" % (rank, t_max))
        E, Np = self.n_envs, self.n_pursuers
        for d in range(n):
            for t, name, dt, tail in ((rew_peers[d], "rew_peers", self.dtype, (Np,)),
                                      (done_peers[d], "done_peers", torch.uint8, ()),
                                      (info_peers[d], "info_peers", torch.int32, (2,))):
                _lib.require_tensor(t, "%s[%d]" % (name, d), dt, (None, E, t_max) + tail, self.device)
                if t.shape[0] <= rank:
                    raise ValueError("%s[%d] has %d slots, rank %d writes slot %d" % (name, d, t.shape[0], rank, rank))
        arr = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])
        self._peer_keepalive = (rew_peers, done_peers, info_peers)
        _lib.check(self._L.madrl_ww_set_peers(self._h, n, rank, t_max, arr(rew_peers), arr(done_peers),
                                              arr(info_peers)))
        self._launch_settings_changed()

    def clear_peers(self):
        self._peer_keepalive = None
        _lib.check(self._L.madrl_ww_set_peers(self._h, 0, 0, 0, None, None, None))
        self._launch_settings_changed()

    def set_obs_writer(self, mode):
        """Observation write path of float32 open-loop rollouts (madrl_ww_set_obs_writer): _lib.WW_OBS_WRITER_AUTO
        (the default), _OFF or _ON.  The values written are the same either way."""
        _lib.check(self._L.madrl_ww_set_obs_writer(self._h, int(mode)))
        self._launch_settings_changed()

    _heuristic_norms = {"agent": _lib.HEURISTIC_NORM_AGENT, "env": _lib.HEURISTIC_NORM_ENV}
    _heuristic_norm = _lib.HEURISTIC_NORM_AGENT

    def rollout_heuristic(self, T, obs0, auto_reset=True, out=None, record_actions=True, actions_out=None,
                          norm="agent"):
        """T lockstep steps in one launch with the reference's hand-written policy
        (heuristics/waterworld.py:11-53) evaluated inside the kernel: closed loop, no action tensor,
        no per-step launch.  obs0 [E, Np, D] = the observation the first action is computed from
        (`reset()`'s, or `obs[-1]` of the previous rollout).  `norm`: "agent" divides each pursuer's action
        by its own norm (the reference's Visualizer calls the policy per agent); "env" divides all of an env's
        actions by one norm, as rltools' decrollout calls it with the env's Np observations as one batch
        (madrl_ww_set_heuristic_norm).  Returns (actions [T,E,Np,2] or None, obs, rew, done, info)."""
        if norm not in self._heuristic_norms:
            raise ValueError("norm must be 'agent' or 'env', got %r" % (norm,))
        code = self._heuristic_norms[norm]
        if code != self._heuristic_norm:
            _lib.check(self._L.madrl_ww_set_heuristic_norm(self._h, code))
            self._heuristic_norm = code
            self._launch_settings_changed()
        return self._rollout_heuristic(T, obs0, auto_reset, out, record_actions, actions_out)


class MAWaterWorld(DropInEnv):
    """Drop-in for the reference class (same constructor, waterworld.py:77-81)."""

    def __init__(self, n_pursuers, n_evaders, n_coop=2, n_poison=10, radius=0.015,
                 obstacle_radius=0.2, obstacle_loc=np.array([0.5, 0.5]), ev_speed=0.01,
                 poison_speed=0.01, n_sensors=30, sensor_range=0.2, action_scale=0.01,
                 poison_reward=-1., food_reward=1., encounter_reward=.05, control_penalty=-.5,
                 reward_mech='local', addid=True, speed_features=True, **kwargs):
        EzPickle.__init__(self, n_pursuers, n_evaders, n_coop, n_poison, radius, obstacle_radius,
                          obstacle_loc, ev_speed, poison_speed, n_sensors, sensor_range,
                          action_scale, poison_reward, food_reward, encounter_reward,
                          control_penalty, reward_mech, addid, speed_features, **kwargs)
        self.n_pursuers, self.n_evaders, self.n_coop, self.n_poison = n_pursuers, n_evaders, n_coop, n_poison
        self.radius, self.obstacle_radius, self.obstacle_loc = radius, obstacle_radius, obstacle_loc
        self.ev_speed, self.poison_speed = ev_speed, poison_speed
        self.n_sensors, self.sensor_range, self.action_scale = n_sensors, sensor_range, action_scale
        self.poison_reward, self.food_reward = poison_reward, food_reward
        self.encounter_reward, self.control_penalty = encounter_reward, control_penalty
        self._reward_mech, self._addid, self._speed_features = reward_mech, addid, speed_features
        self._engine_kwargs = dict(device=kwargs.pop('device', None), dtype=kwargs.pop('dtype', torch.float32))
        self._seed_value = kwargs.pop('seed', 0)
        self._env_id = kwargs.pop('env_id', 0)
        self._pursuers = [Archea(i + 1, radius, n_sensors, sensor_range, addid, speed_features)
                          for i in range(n_pursuers)]
        self._timesteps = 0
        self.setup()

    def _make_engine(self, n_envs, **kw):
        # looks up the module-level class at call time, so that a test double can stand in for it
        return BatchedMAWaterWorld(n_envs, n_pursuers=self.n_pursuers, n_evaders=self.n_evaders, n_coop=self.n_coop,
                                   n_poison=self.n_poison, radius=self.radius, obstacle_radius=self.obstacle_radius,
                                   obstacle_loc=self.obstacle_loc, ev_speed=self.ev_speed,
                                   poison_speed=self.poison_speed, n_sensors=self.n_sensors,
                                   sensor_range=self.sensor_range, action_scale=self.action_scale,
                                   poison_reward=self.poison_reward, food_reward=self.food_reward,
                                   encounter_reward=self.encounter_reward, control_penalty=self.control_penalty,
                                   reward_mech=self._reward_mech, addid=self._addid,
                                   speed_features=self._speed_features, seed=self._seed_value,
                                   **self._engine_kwargs, **kw)

    @property
    def timestep_limit(self):
        return 1000

    @property
    def agents(self):
        return self._pursuers

    def reset(self):
        obs = self._engine.reset().cpu().numpy().astype(np.float64)
        self._timesteps = 1  # reset consumes one internal step (waterworld.py:172)
        return [obs[0, i] for i in range(self.n_pursuers)]

    @property
    def is_terminal(self):
        return self._timesteps >= self.timestep_limit

    def render(self, screen_size=800, rate=10, mode='human'):
        """The frame the reference's render draws (waterworld.py:438-479), as a NumPy RGB uint8 array
        [screen_size, screen_size, 3] (BatchedMAWaterWorld.render_frames).  No window is opened: `rate` and `mode`
        are accepted for the reference's signature and unused."""
        return self._frame(screen_size=screen_size)

    def step(self, action_Np2):
        a = np.asarray(action_Np2, dtype=np.float64).reshape((self.n_pursuers, 2))  # waterworld.py:221-222
        obs, rew, done, info = self._engine.step(a[None], auto_reset=False)
        obs = obs.cpu().numpy().astype(np.float64)
        self._timesteps += 1
        return ([obs[0, i] for i in range(self.n_pursuers)], rew[0].cpu().numpy().astype(np.float64),
                bool(done[0].item()),
                dict(evcatches=int(info['evcatches'][0].item()), pocatches=int(info['pocatches'][0].item())))
