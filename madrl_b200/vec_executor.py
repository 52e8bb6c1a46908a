"""GPU-batched stand-in for rllab's ``VecEnvExecutor``
(rllab/sandbox/rocky/tf/envs/vec_env_executor.py:8-48): same methods and return types
(``reset() -> list``, ``step(action_n) -> (obs list, rewards ndarray, dones ndarray,
env_infos dict of arrays)``, ``num_envs``, ``action_space``, ``observation_space``,
``terminate()``), with the horizon cut-off and auto-reset-in-place done on the device.
"""
import numpy as np
import torch

from .spaces import Discrete


class BatchedVecExecutor(object):
    """`n_envs` copies of the drop-in env `proto_env` on one batched engine (the env's `_make_engine`)."""

    def __init__(self, proto_env, n_envs, max_path_length):
        self._proto = proto_env
        self._engine = proto_env._make_engine(n_envs, max_path_length=max_path_length)
        self._n = n_envs
        self.max_path_length = max_path_length
        self.ts = np.zeros(n_envs, dtype='int')
        # discrete moves (Pursuit) are int32, continuous ones float64 until the engine casts them to its dtype
        self._act_dtype = np.int32 if isinstance(self.action_space, Discrete) else np.float64

    @property
    def num_envs(self):
        return self._n

    @property
    def action_space(self):
        return self._proto.agents[0].action_space

    @property
    def observation_space(self):
        return self._proto.agents[0].observation_space

    def reset(self):
        obs = self._engine.reset().cpu().numpy().astype(np.float64)
        self.ts[:] = 0
        return [obs[i] for i in range(self._n)]

    def step(self, action_n):
        # engine.step reshapes the actions to [n_envs, agents, *action shape]
        a = torch.as_tensor(np.asarray(action_n, dtype=self._act_dtype))
        obs, rew, done, info = self._engine.step(a, auto_reset=True)
        obs = obs.cpu().numpy().astype(np.float64)
        dones = done.cpu().numpy().astype(bool)
        self.ts += 1
        self.ts[dones] = 0
        infos = {k: v.cpu().numpy() for k, v in info.items()}
        return [obs[i] for i in range(self._n)], rew.cpu().numpy().astype(np.float64), dones, infos

    def terminate(self):
        pass
