"""rllab's DDPG replay pool on the device: whole rollouts in, minibatches out, with CUDA kernels.

``ReplayPool`` is ``MAReplayPool`` (rllab/rllab/algos/ddpg.py:85-145) as ``DDPG.train`` fills it in decentralized
mode, the runners' default for ``--algo thddpg`` (Waterworld and Hostage; Pursuit's actions are not a Box).  It
sits between a rollout (``engine.rollout`` or ``PolicyRollout``) and the caller's Q-function and actor updates, as
``postproc.process_samples*`` does for TRPO.  See madrl_b200/csrc/replay.cu for the kernels.
"""
import ctypes as C

import torch

from . import _lib
from ._lib import _ptr


class ReplayPool(object):
    """A ring of `max_pool_size` transitions (observation, action, reward, next observation, terminal) in device
    memory, filled from rollouts and sampled with replacement.  The defaults are DDPG's.

    ``add(obs, actions, rew, done, obs_before, term, path_len0, timestep0, max_path_length, timestep_limit)`` adds the
    transitions DDPG.train would have added had each env run its loop (ddpg.py:285-353), in (t, env, agent) order:

    * observation ``obs[t-1]`` (``obs_before`` at t = 0), action ``actions[t]``, reward
      ``float32(float64(rew[t]) * scale_reward)`` (the reference keeps float64), terminal ``done[t]``;
    * next observation ``term[t]`` where ``done[t]`` is set, else ``obs[t]`` (with auto-reset ``obs[t]`` holds the
      reset observation there).  ``term`` is the engine's ``set_terminal_obs`` tensor of this rollout, and required;
    * ``path_len0`` / ``timestep0``: clones of ``engine.state["path_len"]`` and ``["timestep"]`` taken before the
      launch.  A done step whose path reached ``max_path_length`` in an env that did not terminate by itself
      (``timestep < timestep_limit``) is a horizon cut (ddpg.py:310): dropped, or stored with terminal = 1 when
      ``include_horizon_terminal_transitions``.  This is exact for Waterworld.  Hostage also ends on the bomb or
      when every hostage is saved; when that happens exactly at the horizon step the rollout cannot tell it from a
      cut, and the pool treats it as one, where the reference stores it with terminal = True.

    When one add keeps more transitions than the pool holds, only the last `max_pool_size` land.  ``top``,
    ``bottom`` and ``size`` move as ``add_sample`` moves them.

    ``random_batch(B)`` / ``random_batches(n, B)`` return dicts of ``observations``, ``actions``, ``rewards``,
    ``terminals``, ``next_observations`` and ``indices`` with B rows ([n, B, ...] for random_batches), drawn
    uniformly over the slots [0, size - 1): exactly the set ``MAReplayPool.random_batch``'s rejection loop accepts.
    Indices come from a Philox stream keyed by (`seed`, draw counter).  One deliberate deviation: the reference
    returns the observations as ``next_observations`` (ddpg.py:140), which leaves the stored next observations unused
    and the Q target meaningless; this pool returns the stored next observations.

    All bookkeeping, the draw counter included, lives in device memory: ``add`` and ``random_batches`` make no host
    synchronisation and no allocation after their first call at a shape, so they can be captured in a CUDA graph
    with a ``PolicyRollout``, and each replay draws fresh indices.  ``random_batch`` checks ``size > B`` (the
    reference's assertion) with a host read, except while the current stream is capturing: the caller then makes
    sure of it, as DDPG's ``min_pool_size`` does.  The returned batches are views of buffers the next call with the
    same (n, B) overwrites.

    Only decentralized mode: the reference's DDPG raises for concurrent mode, and its centralized branch cannot
    store the per-agent reward vector these envs return; both raise NotImplementedError.  Each rank of a sharded run
    keeps the pool of its own envs; give the ranks different seeds.
    """

    def __init__(self, max_pool_size, n_agents, obs_dim, action_dim, device, obs_dtype=torch.float32,
                 scale_reward=0.1, include_horizon_terminal_transitions=False, seed=0, mode="decentralized"):
        if mode != "decentralized":
            raise NotImplementedError("ReplayPool supports decentralized mode only, got %r" % (mode,))
        if obs_dtype not in (torch.float32, torch.bfloat16):
            raise TypeError("obs_dtype must be torch.float32 or torch.bfloat16, got %s" % obs_dtype)
        if int(max_pool_size) < 1 or int(n_agents) < 1 or int(obs_dim) < 1 or int(action_dim) < 1:
            raise ValueError("max_pool_size, n_agents, obs_dim and action_dim must be >= 1")
        self._L = _lib.lib()
        self.max_pool_size, self.n_agents = int(max_pool_size), int(n_agents)
        self.obs_dim, self.action_dim, self.obs_dtype = int(obs_dim), int(action_dim), obs_dtype
        self.scale_reward = float(scale_reward)
        self.include_horizon_terminal_transitions = bool(include_horizon_terminal_transitions)
        self.seed = int(seed) & 0xFFFFFFFFFFFFFFFF
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("ReplayPool lives on a CUDA device, got %s" % self.device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        M, D, Ad, dev = self.max_pool_size, self.obs_dim, self.action_dim, self.device
        self.observations = torch.zeros((M, D), dtype=obs_dtype, device=dev)
        self.next_observations = torch.zeros((M, D), dtype=obs_dtype, device=dev)
        self.actions = torch.zeros((M, Ad), dtype=torch.float32, device=dev)
        self.rewards = torch.zeros(M, dtype=torch.float32, device=dev)
        self.terminals = torch.zeros(M, dtype=torch.uint8, device=dev)
        self._ctl = torch.zeros(4, dtype=torch.int64, device=dev)   # top, bottom, size, draw counter
        self._ws = {}
        self._out = {}
        self._sfx = "bf16" if obs_dtype == torch.bfloat16 else "f32"

    def _workspace(self, T, E):
        ws = self._ws.get((T, E))
        if ws is None:
            n = C.c_size_t()
            _lib.check(self._L.madrl_replay_workspace_size(T, E, C.byref(n)))
            ws = self._ws[(T, E)] = torch.empty(int(n.value), dtype=torch.uint8, device=self.device)
        return ws

    def add(self, obs, actions, rew, done, obs_before, term, path_len0, timestep0, max_path_length, timestep_limit):
        """Insert one rollout: obs [T, E, A, D], actions float32 [T, E, A, action_dim], rew float32 [T, E, A], done
        uint8 [T, E], obs_before [E, A, D], term [T, E, A, D], path_len0 / timestep0 int32 [E]."""
        A, D, Ad, dev, od = self.n_agents, self.obs_dim, self.action_dim, self.device, self.obs_dtype
        T, E = _lib.require_tensor(done, "done", torch.uint8, (None, None), dev).shape
        _lib.require_tensor(obs, "obs", od, (T, E, A, D), dev)
        _lib.require_tensor(actions, "actions", torch.float32, (T, E, A, Ad), dev)
        _lib.require_tensor(rew, "rew", torch.float32, (T, E, A), dev)
        _lib.require_tensor(obs_before, "obs_before", od, (E, A, D), dev)
        _lib.require_tensor(term, "term", od, (T, E, A, D), dev)
        _lib.require_tensor(path_len0, "path_len0", torch.int32, (E,), dev)
        _lib.require_tensor(timestep0, "timestep0", torch.int32, (E,), dev)
        ws = self._workspace(T, E)
        fn = getattr(self._L, "madrl_replay_add_" + self._sfx)
        with torch.cuda.device(dev):
            _lib.check(fn(T, E, A, D, Ad, self.max_pool_size, _ptr(obs), _ptr(actions), _ptr(rew), _ptr(done),
                          _ptr(obs_before), _ptr(term), _ptr(path_len0), _ptr(timestep0), int(max_path_length),
                          int(timestep_limit), int(self.include_horizon_terminal_transitions), self.scale_reward,
                          _ptr(self.observations), _ptr(self.next_observations), _ptr(self.actions),
                          _ptr(self.rewards), _ptr(self.terminals), _ptr(self._ctl), _ptr(ws), _lib.stream(dev)))

    def random_batches(self, n, batch_size):
        """n minibatches of `batch_size` rows in one launch: a dict of [n, batch_size, ...] tensors."""
        n, B = int(n), int(batch_size)
        if n < 1 or B < 1:
            raise ValueError("n and batch_size must be >= 1, got %d, %d" % (n, B))
        out = self._out.get((n, B))
        if out is None:
            dev, D, Ad = self.device, self.obs_dim, self.action_dim
            out = self._out[(n, B)] = dict(
                observations=torch.empty((n, B, D), dtype=self.obs_dtype, device=dev),
                actions=torch.empty((n, B, Ad), dtype=torch.float32, device=dev),
                rewards=torch.empty((n, B), dtype=torch.float32, device=dev),
                terminals=torch.empty((n, B), dtype=torch.uint8, device=dev),
                next_observations=torch.empty((n, B, D), dtype=self.obs_dtype, device=dev),
                indices=torch.empty((n, B), dtype=torch.int64, device=dev))
        fn = getattr(self._L, "madrl_replay_sample_" + self._sfx)
        with torch.cuda.device(self.device):
            _lib.check(fn(n, B, self.obs_dim, self.action_dim, self.max_pool_size, self.seed, _ptr(self.observations),
                          _ptr(self.next_observations), _ptr(self.actions), _ptr(self.rewards), _ptr(self.terminals),
                          _ptr(self._ctl), _ptr(out["indices"]), _ptr(out["observations"]),
                          _ptr(out["next_observations"]), _ptr(out["actions"]), _ptr(out["rewards"]),
                          _ptr(out["terminals"]), _lib.stream(self.device)))
        return dict(out)

    def random_batch(self, batch_size):
        """One minibatch (ddpg.py:118-141): a dict of [batch_size, ...] tensors.  Raises ValueError unless
        size > batch_size, except during stream capture (see the class docstring)."""
        if not torch.cuda.is_current_stream_capturing() and not self.size > batch_size:
            raise ValueError("random_batch(%d) needs more than %d transitions in the pool, it holds %d"
                             % (batch_size, batch_size, self.size))
        return {k: v[0] for k, v in self.random_batches(1, batch_size).items()}

    @property
    def size(self):
        """Transitions in the pool (a host read: synchronises with the device)."""
        return int(self._ctl[2].item())

    def get_state(self):
        """The ring counters and the draw counter: {top, bottom, size, draws} (a host read)."""
        top, bottom, size, draws = (int(x) for x in self._ctl.tolist())
        return dict(top=top, bottom=bottom, size=size, draws=draws)

    def set_state(self, state):
        """Restore what get_state returned (the pool's arrays are the caller's to save and restore)."""
        M = self.max_pool_size
        top, bottom, size, draws = (int(state[k]) for k in ("top", "bottom", "size", "draws"))
        if not (0 <= size <= M and 0 <= top < M and 0 <= bottom < M and draws >= 0):
            raise ValueError("bad replay pool state %r for max_pool_size %d" % (state, M))
        self._ctl.copy_(torch.tensor([top, bottom, size, draws], dtype=torch.int64))
