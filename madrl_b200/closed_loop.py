"""Closed-loop rollouts with the caller's PyTorch policy, captured as one CUDA graph.

``PolicyRollout(engine, policy, T)`` runs T lockstep steps of a ``Batched*`` engine in which every action
comes from ``policy`` evaluated on the observation of the step before, as rllab's and rltools' samplers do.
On the first call the T steps -- policy kernels, the engine's one-step rollout launches, the recording of
the policy's extras and the reset of recurrent state -- are captured unrolled into one
``torch.cuda.CUDAGraph``; later calls copy the inputs in and replay it.  The policy stays in PyTorch (any
architecture: MLP, GRU, LSTM, conv), and the env kernels stay policy-free.

The outputs are the tensors ``postproc.process_samples_recurrent`` / ``process_samples_concurrent`` and
``rltools_sampler.process_samples`` take, with ``obs_before = obs0``.

With ``frame_stack=B`` and / or ``standardizer=`` the policy reads observations wrapped as the reference's
``StandardizedEnv`` inside ``ObservationBuffer`` wrap them, one fused kernel per step (madrl_obs_wrap_step_*).
"""
import collections
import contextlib

import torch

from . import _lib
from ._lib import _ptr

Rollout = collections.namedtuple("Rollout", "actions obs rew done info extras state policy_obs")


def _map_state(fn, state):
    """`fn` over a recurrent state: None, a tensor, or a (nested) tuple / list of tensors."""
    if state is None:
        return None
    if isinstance(state, torch.Tensor):
        return fn(state)
    return type(state)(_map_state(fn, s) for s in state)


def reset_state(state, done):
    """`state` with every env whose `done` (uint8 [E]) is set zeroed: the leading axis of each state tensor is
    the env axis.  rllab's recurrent sampler starts every episode from the policy's initial (zero) state."""
    def zero(s):
        if s.shape[0] != done.shape[0]:
            raise ValueError("recurrent state tensors must have the env axis (%d) first, got %s"
                             % (done.shape[0], tuple(s.shape)))
        return s.masked_fill(done.view((-1,) + (1,) * (s.dim() - 1)).bool(), 0)
    return _map_state(zero, state)


class PolicyRollout(object):
    """T closed-loop steps of `engine` driven by `policy`, as one CUDA graph replay (or eagerly, `graph=False`).

    ``policy(obs [E, A, D], state) -> (actions, extras, state)`` is any PyTorch callable that is safe to capture
    in a CUDA graph (no host synchronisation, no data-dependent Python control flow, no host copies):

    * ``obs`` has the engine's obs_dtype (bfloat16 engines hand the policy bfloat16 rows);
    * ``actions`` is anything ``copy_`` can write into the engine's action slot [E, A, *act_tail]: it is cast to
      the engine's action dtype inside the graph.  Pursuit's categorical policies sample int64 categories; they are
      cast to the kernel's int32 there, unchecked, so they must already lie in {0, .., 4};
    * ``extras`` is a dict of per-step tensors (rllab's ``mean`` / ``log_std`` agent_infos, ``logits``, ...); the
      entries named in `record` (all when None) are recorded as [T, E, A, ...];
    * ``state`` is the recurrent state (None, a tensor or a tuple of tensors, each with the env axis first).
      After step t it is zeroed for every env whose ``done[t]`` is set, so that a GRU or LSTM restarts with each
      episode as rllab's recurrent sampler does.

    At step t the policy reads observation slot t-1 of the trajectory (``obs0`` for t = 0) and its actions go to
    slot t of ``actions``; the engine then writes slot t of ``obs``, ``rew``, ``done`` and ``info``, and, with
    ``engine.set_terminal_obs(term)`` (term [T, E, A, D]) and `auto_reset`, slot t of ``term``.  Every pointer is
    fixed at capture, so there is no device step counter and no extra copy of the observations.

    The engine runs with `obs_cache` during the loop; its own setting is restored afterwards.  The default (None) is
    _lib.OBS_CACHE_KEEP on float32 engines -- the policy reads each step's observation rows right after the launch
    that wrote them, so they are stored at normal L2 priority instead of evict-first -- and _lib.OBS_CACHE_STREAM on
    the float64 verification engines, which have no KEEP kernels (asking for KEEP there raises EngineError).

    The capture is redone when T, the engine, its obs dtype, its terminal-observation tensor, the state's shapes or
    any host-side setting a launch copies into its kernel parameters changes: ``engine.seed``, ``set_launch`` and
    Pursuit's ``set_params`` (the curriculum hook) (``engine.launch_settings`` counts them).  So a curriculum update
    or a re-seed between calls takes effect as it would in an eager loop.  A call raises ValueError while
    Waterworld's ``set_peers`` is in effect: each launch of the fused peer exchange writes its rows from step 0 of
    the gather buffers, so one-step launches would overwrite each other.  The first call with graph=True first runs the policy twice on a side stream
    (torch.cuda.graphs' warm-up: lazy library initialisation must not happen during capture); this touches no env
    state.

    The graph also holds the policy's tensors by address: its weights must be updated IN PLACE (``optimizer.step()``,
    ``param.data.copy_(new)``).  Rebinding a parameter to a new tensor (``param.data = new``, which is what
    ``torch.nn.utils.vector_to_parameters`` and many TRPO ``set_flat_params`` do, or a new module) leaves the replays
    on the old weights without an error; copy into the existing tensors, or build a new PolicyRollout after such an
    update.

    Randomness: torch's CUDA generator is graph-safe, so ``torch.randn`` / ``Categorical.sample`` inside the policy
    draw fresh noise at every replay.  The draws are not those of an eager loop from the same seed: at capture the
    generator assigns the graph's random kernels one block of Philox offsets and moves its offset past that block
    at each replay, whereas the eager loop advances it kernel by kernel.

    Observation wrappers (the reference's runners wrap the env as ``ObservationBuffer(StandardizedEnv(env),
    buffer_size)``):
    * ``standardizer``: a ``postproc.Standardizer`` of the engine's (E, A, D) on its device.  With
      ``enable_obsnorm`` the policy reads observations standardised by the per-env running estimates, updated at
      every step in the reference's order (at a done step the terminal observation first, then the reset one); the
      Standardizer's float64 state is updated in place, so it carries over between calls and to open-loop use.
      Its reward side (``enable_rewnorm``, ``scale_reward``) feeds no policy input and is applied to ``rew`` once
      after the T steps (``Standardizer.rew``, inside the graph), which equals per-step application.
    * ``frame_stack=B`` (1..8): the policy reads the last B observations as ``[E, A, D, B]`` (the newest in slot
      B-1; after a reset every slot holds the reset observation).  ``obs.reshape(E, A, D * B)`` is the reference's
      ``buffer.flatten()``.  ``obs0`` is then ``[E, A, D, B]``.
    Either option runs one fused kernel after each step's launch (policy -> env launch -> wrapper kernel ->
    recurrent-state reset).  ``obs`` then holds the standardised observations (with obsnorm) and
    ``policy_obs[t]`` the wrapped observation step t returned: a new [T, E, A, D, B] buffer with B > 1 (at C2,
    T = 256, B = 4: 17.9 GB in float32, 8.9 GB in bfloat16), ``obs`` itself with B = 1.  The sample-processing
    passes take ``policy_obs.view(T, E, A, D * B)`` with ``obs_before = obs0.view(E, A, D * B)``.  Obsnorm needs
    the terminal observations: the ``set_terminal_obs`` tensor when the caller has one, otherwise a private
    one-step buffer, set for the loop and unset afterwards.  The start of a run::

        o = engine.reset()
        std.obs(o)                                           # the reset observation updates the estimate
        obs0 = postproc.FrameStack(E, A, D, B, dev, engine.obs_dtype).reset(o)   # or o itself with B = 1

    and each later call takes the previous call's ``policy_obs[-1]``.  The wrappers need float32 or bfloat16
    observations, ``auto_reset`` and, for Pursuit, ``flatten=True`` (ObservationBuffer takes 1-D observations).

    ``__call__(obs0, state0=None)`` returns a ``Rollout`` (actions, obs, rew, done, info, extras, state, policy_obs)
    of VIEWS of the rollout's buffers: the next call overwrites them, so clone what must outlive it.
    """

    def __init__(self, engine, policy, T, auto_reset=True, record=None, graph=True, obs_cache=None, frame_stack=1,
                 standardizer=None):
        self.engine, self.policy, self.T = engine, policy, T
        self.auto_reset, self.record, self.graph, self.obs_cache = auto_reset, record, graph, obs_cache
        self.frame_stack, self.standardizer = frame_stack, standardizer
        self._key = None
        self._graph = None
        self._check_wrappers()

    def _check_wrappers(self):
        """Raise for wrapper options the kernels or the reference do not support."""
        B, std, eng = self.frame_stack, self.standardizer, self.engine
        if not isinstance(B, int) or not 1 <= B <= 8:
            raise ValueError("frame_stack must be an int in [1, 8], got %r" % (B,))
        if B == 1 and std is None:
            return
        opt = "frame_stack" if std is None else "standardizer"
        if not self.auto_reset:
            raise ValueError("%s needs auto_reset=True (the wrappers restart at each env's reset)" % opt)
        if eng.obs_dtype not in (torch.float32, torch.bfloat16):
            raise TypeError("%s needs float32 or bfloat16 observations, the engine's are %s" % (opt, eng.obs_dtype))
        if getattr(eng, "flatten", True) is False:
            raise ValueError("%s needs a Pursuit engine with flatten=True (ObservationBuffer takes 1-D observations)"
                             % opt)
        if std is not None:
            from .postproc import Standardizer
            if not isinstance(std, Standardizer):
                raise TypeError("standardizer must be a postproc.Standardizer, got %r" % type(std))
            shape = (eng.n_envs, eng._n_acting, eng.obs_dim)
            for t, n in ((std.obs_mean, "obs_mean"), (std.obs_var, "obs_var")):
                _lib.require_tensor(t, "standardizer." + n, torch.float64, shape, eng.device)
            for t, n in ((std.rew_mean, "rew_mean"), (std.rew_var, "rew_var")):
                _lib.require_tensor(t, "standardizer." + n, torch.float64, shape[:2], eng.device)

    def _wrapped(self):
        """The fused wrapper kernel runs after every step."""
        std = self.standardizer
        return self.frame_stack > 1 or (std is not None and bool(std.enable_obsnorm))

    def _obs0_shape(self):
        eng = self.engine
        return (eng.n_envs, eng._n_acting, eng.obs_dim) + ((self.frame_stack,) if self.frame_stack > 1 else ())

    def _settings(self, state0):
        eng, std = self.engine, self.standardizer
        term = eng._term_obs if self.auto_reset else None
        wrap = None if std is None else (
            id(std), tuple(t.data_ptr() for t in (std.obs_mean, std.obs_var, std.rew_mean, std.rew_var)),
            float(std.obs_alpha), float(std.rew_alpha), float(std.eps), bool(std.enable_obsnorm),
            bool(std.enable_rewnorm), float(std.scale_reward))
        return (self.T, id(eng), eng.obs_dtype, None if term is None else (term.data_ptr(), tuple(term.shape)),
                eng.launch_settings, self.auto_reset, self.graph, self._obs_cache(), self.record,
                tuple((tuple(s.shape), s.dtype) for s in _flat(state0)), state0 is None, self.frame_stack, wrap)

    def _obs_cache(self):
        if self.obs_cache is not None:
            return self.obs_cache
        return _lib.OBS_CACHE_STREAM if self.engine.dtype == torch.float64 else _lib.OBS_CACHE_KEEP

    def _allocate(self, state0):
        eng, T = self.engine, self.T
        if int(T) < 1:
            raise ValueError("T must be >= 1, got %r" % (T,))
        E, A, dev = eng.n_envs, eng._n_acting, eng.device
        self._act = torch.zeros((T, E, A) + eng._act_tail, dtype=eng._act_dtype, device=dev)
        self._traj = tuple(torch.zeros(s, dtype=dt, device=dev) for dt, s in eng._trajectory_shapes(T))
        self._obs0 = torch.zeros(self._obs0_shape(), dtype=eng.obs_dtype, device=dev)
        self._state0 = _map_state(torch.clone, state0)
        self._term = eng._term_obs if self.auto_reset else None
        if self._term is not None:
            _lib.require_tensor(self._term, "the set_terminal_obs tensor", eng.obs_dtype, (T, E, A, eng.obs_dim), dev)
        self._check_wrappers()
        std = self.standardizer
        obsnorm = std is not None and bool(std.enable_obsnorm)
        # the terminal observations obsnorm reads: a private one-step buffer when the caller keeps none
        self._term1 = None
        if obsnorm and self._term is None:
            self._term1 = torch.zeros((1, E, A, eng.obs_dim), dtype=eng.obs_dtype, device=dev)
        self._stats = (std.obs_mean, std.obs_var) if obsnorm else None
        self._policy_obs = self._traj[0]
        if self.frame_stack > 1:
            self._policy_obs = torch.zeros((T,) + self._obs0_shape(), dtype=eng.obs_dtype, device=dev)
        self._extras = None   # allocated at the first policy call: shapes and dtypes are the policy's
        self._graph = None

    def _wrap_step(self, t):
        """madrl_obs_wrap_step_* of step t: standardise obs[t] (and term[t]) in place, stack into policy_obs[t]."""
        eng, B = self.engine, self.frame_stack
        obs, _, done, _ = self._traj
        E, A, D = eng.n_envs, eng._n_acting, eng.obs_dim
        term = None
        if self._stats is not None:
            term = self._term1[0] if self._term1 is not None else self._term[t]
        prev = out = None
        if B > 1:
            prev = self._obs0 if t == 0 else self._policy_obs[t - 1]
            out = self._policy_obs[t]
        mean, var = self._stats if self._stats is not None else (None, None)
        std = self.standardizer
        fn = getattr(_lib.lib(), "madrl_obs_wrap_step_%s" % ("bf16" if eng.obs_dtype == torch.bfloat16 else "f32"))
        _lib.check(fn(E, A, D, B, _ptr(obs[t]), _ptr(term), _ptr(done[t]), _ptr(prev), _ptr(out), _ptr(mean),
                      _ptr(var), float(std.obs_alpha) if std is not None else 0.0,
                      float(std.eps) if std is not None else 0.0, _lib.stream(eng.device)))

    def _record_buffers(self, extras):
        keys = extras.keys() if self.record is None else self.record
        return {k: torch.zeros((self.T,) + tuple(extras[k].shape), dtype=extras[k].dtype, device=self.engine.device)
                for k in keys}

    def _loop(self):
        """The T steps on the current stream, from and into the fixed buffers -> the final state."""
        eng = self.engine
        obs, rew, done, info = self._traj
        state = self._state0
        prev = self._obs0
        wrapped = self._wrapped()
        for t in range(self.T):
            a, extras, state = self.policy(prev, state)
            if self._extras is None:
                self._extras = self._record_buffers(extras)
            self._act[t].copy_(a)
            for k, buf in self._extras.items():
                buf[t].copy_(extras[k])
            if self._term is not None:
                eng.set_terminal_obs(self._term[t:t + 1])
            eng.rollout(self._act[t:t + 1], auto_reset=self.auto_reset,
                        out=(obs[t:t + 1], rew[t:t + 1], done[t:t + 1], info[t:t + 1]))
            if wrapped:
                self._wrap_step(t)
            state = reset_state(state, done[t])
            prev = self._policy_obs[t]
        if self.standardizer is not None:
            self.standardizer.rew(rew)
        return state

    @contextlib.contextmanager
    def _engine_settings(self):
        """The engine with our obs cache mode (set before any capture begins, so a refused mode raises there) and
        our private terminal-observation buffer, if any; its own mode and terminal-observation tensor are restored
        after."""
        eng = self.engine
        keep_mode, keep_term = eng.obs_cache, eng._term_obs
        eng.set_obs_cache(self._obs_cache())
        try:
            if self._term1 is not None:
                eng.set_terminal_obs(self._term1)
            yield
        finally:
            eng.set_obs_cache(keep_mode)
            if self._term is not None or self._term1 is not None:
                eng.set_terminal_obs(keep_term)

    def _capture(self):
        dev = self.engine.device
        side = torch.cuda.Stream(dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(2):
                self.policy(self._obs0, self._state0)
        torch.cuda.current_stream(dev).wait_stream(side)
        g = torch.cuda.CUDAGraph()
        with self._engine_settings(), torch.cuda.graph(g):
            self._state_out = self._loop()
        self._graph = g

    def __call__(self, obs0, state0=None):
        eng = self.engine
        if getattr(eng, "_peer_keepalive", None) is not None:
            raise ValueError("PolicyRollout runs one launch per step, and every launch would write its peer rows "
                             "from step 0 of the gather buffers: clear_peers() first")
        _lib.require_tensor(obs0, "obs0", eng.obs_dtype, self._obs0_shape(), eng.device, contiguous=False)
        with torch.cuda.device(eng.device):
            key = self._settings(state0)
            if key != self._key:
                self._allocate(state0)
                self._key = key
            self._obs0.copy_(obs0)
            for d, s in zip(_flat(self._state0), _flat(state0)):
                d.copy_(s)
            if self.graph:
                if self._graph is None:
                    self._capture()
                self._graph.replay()
                state = self._state_out
            else:
                with self._engine_settings():
                    state = self._loop()
        obs, rew, done, info = self._traj
        return Rollout(self._act, obs, rew, done, info, dict(self._extras), state, self._policy_obs)


def _flat(state):
    if state is None:
        return []
    if isinstance(state, torch.Tensor):
        return [state]
    return [x for s in state for x in _flat(s)]
