"""What the three env families share on the Python side.

``BatchedEngine`` is the base of ``BatchedMAWaterWorld``, ``BatchedPursuitEvade`` and
``BatchedHostageWorld``: one handle of the ``madrl_<abi>_*`` C ABI, its state blob in HBM, and the entry
points every family has.  A family declares its ABI prefix, its layout struct, the action shape of one
agent, the info shape of one env and the info keys of ``step()``; its constructor builds the config
struct and hands it to ``BatchedEngine.__init__``.

``DropInEnv`` is the base of the drop-in env classes (``MAWaterWorld``, ``PursuitEvade``,
``ContinuousHostageWorld``): a one-env engine built by the family's ``_make_engine``, and rllab's
batched plug-in hook (``vectorized`` / ``vec_env_executor``; rllab/sandbox/rocky/tf/envs/base.py:97-103).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import _ptr
from .core import AbstractMAEnv, EzPickle


class BatchedEngine(object):
    _abi = None       # C ABI prefix: madrl_<_abi>_*
    _Layout = None    # ctypes struct filled by madrl_<_abi>_state_layout
    _act_tail = ()    # action shape of one acting agent
    _info_tail = ()   # info shape of one env
    _info_keys = ()   # step() info keys: one per info column, or a single key for the whole row

    def __init__(self, cfg, n_acting, device, dtype, act_dtype, create_args=(), obs_dtype=None):
        """`n_acting`: agents that act and observe per env; `dtype`: rewards (and state);
        `act_dtype`: actions; `create_args`: family arguments of madrl_<abi>_create before the blob;
        `obs_dtype`: observations, `dtype` (None) or torch.bfloat16 (fp32 engines only)."""
        obs_dtype = dtype if obs_dtype is None else obs_dtype
        if obs_dtype not in (dtype, torch.bfloat16) or (obs_dtype == torch.bfloat16 and dtype != torch.float32):
            raise ValueError("obs_dtype must be %s or torch.bfloat16 (with float32 rewards), got %s" % (dtype, obs_dtype))
        if not torch.cuda.is_available():
            raise _lib.EngineError("madrl_b200 needs a CUDA device (there is no CPU fallback)")
        self._L = _lib.lib()
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None \
            else torch.device(device)
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.cfg, self._n_acting, self.dtype, self._act_dtype = cfg, n_acting, dtype, act_dtype
        self.layout = self._Layout()
        _lib.check(self._fn("state_layout")(C.byref(cfg), C.byref(self.layout)))
        self.obs_dim = int(self.layout.obs_dim)
        with torch.cuda.device(self.device):
            self._blob = torch.zeros(int(self.layout.total_bytes), dtype=torch.uint8, device=self.device)
            h = C.c_void_p()
            _lib.check(self._fn("create")(C.byref(cfg), *create_args, _ptr(self._blob), C.byref(h)))
        self._h = h
        self.obs_dtype = obs_dtype
        self._term_obs = None   # set_terminal_obs
        if obs_dtype == torch.bfloat16:
            _lib.check(self._fn("set_obs_format")(self._h, _lib.OBS_BF16))

    def _fn(self, name):
        return getattr(self._L, "madrl_%s_%s" % (self._abi, name))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._fn("destroy")(h)

    def _view(self, off, dtype, shape):
        n = int(np.prod(shape)) * torch.empty((), dtype=dtype).element_size()
        return self._blob[off:off + n].view(dtype).view(*shape)

    def set_terminal_obs(self, term_obs):
        """Keep the terminal observations of done steps: `term_obs` (same shape / obs_dtype as the obs tensor
        of the following auto-reset rollouts, which check it) receives, at the [t, e] slots where `done` is set,
        the observation the env returned BEFORE it was reset in place (StandardizedEnv needs it,
        madrl_environments/__init__.py:283-291).  None switches it off."""
        _lib.require_tensor(term_obs, "term_obs", self.obs_dtype, (None, self.n_envs, self._n_acting, self.obs_dim),
                            self.device, optional=True)
        self._term_obs = term_obs
        _lib.check(self._fn("set_terminal_obs")(self._h, _ptr(term_obs)))

    # Counts the calls that change host-side handle settings a rollout launch copies into its kernel parameters
    # (seed, set_launch, the families' set_params / set_peers): a CUDA graph holding earlier launches is stale
    # once it changes (closed_loop.PolicyRollout re-captures).
    launch_settings = 0

    def _launch_settings_changed(self):
        self.launch_settings += 1

    def set_launch(self, warps_per_block=0, blocks_per_sm=0):
        _lib.check(self._fn("set_launch")(self._h, warps_per_block, blocks_per_sm))
        self._launch_settings_changed()

    def seed(self, seed=None):
        with torch.cuda.device(self.device):
            _lib.check(self._fn("seed")(self._h, 0 if seed is None else int(seed), _lib.stream(self.device)))
        self._launch_settings_changed()
        return [seed]

    def reset(self, mask=None, out=None):
        """reset() of the masked envs (all if None) -> obs [E, A, D]."""
        shape = (self.n_envs, self._n_acting, self.obs_dim)
        obs = out if out is not None else torch.zeros(shape, dtype=self.obs_dtype, device=self.device)
        if out is not None:
            _lib.require_tensor(out, "out", self.obs_dtype, shape, self.device)
        if mask is not None:
            mask = _lib.require_tensor(mask.to(device=self.device, dtype=torch.uint8).contiguous(), "mask", torch.uint8,
                                       (self.n_envs,), self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._fn("reset")(self._h, _ptr(mask), _ptr(obs), _lib.stream(self.device)))
        return obs

    def _trajectory_shapes(self, T):
        """(dtype, shape) of obs, rew, done and info of a T-step rollout."""
        E, A = self.n_envs, self._n_acting
        return ((self.obs_dtype, (T, E, A, self.obs_dim)), (self.dtype, (T, E, A)), (torch.uint8, (T, E)),
                (torch.int32, (T, E) + self._info_tail))

    def _outputs(self, T, out, auto_reset):
        """The trajectory buffers of a T-step device rollout: `out` after checking dtype / shape /
        contiguity / placement, or new ones.  An auto-reset rollout also writes the set_terminal_obs
        tensor, which must then have the shape of its obs tensor."""
        if auto_reset and self._term_obs is not None:
            _lib.require_tensor(self._term_obs, "the set_terminal_obs tensor", self.obs_dtype,
                                (T, self.n_envs, self._n_acting, self.obs_dim), self.device)
        if out is None:   # spelled out: this is on the per-step path of the single-env drop-ins
            E, A, dev = self.n_envs, self._n_acting, self.device
            return (torch.empty((T, E, A, self.obs_dim), dtype=self.obs_dtype, device=dev),
                    torch.empty((T, E, A), dtype=self.dtype, device=dev),
                    torch.empty((T, E), dtype=torch.uint8, device=dev),
                    torch.empty((T, E) + self._info_tail, dtype=torch.int32, device=dev))
        obs, rew, done, info = out
        for t, n, (dt, s) in zip(out, ("obs", "rew", "done", "info"), self._trajectory_shapes(T)):
            _lib.require_tensor(t, n, dt, s, self.device)
        return obs, rew, done, info

    def rollout(self, actions, auto_reset=True, out=None):
        """T lockstep steps in one kernel launch.  actions [T, E, A, *act_tail] ->
        (obs [T,E,A,D], rew [T,E,A], done [T,E] uint8, info [T,E,*info_tail] int32)."""
        actions = actions.to(device=self.device, dtype=self._act_dtype).contiguous()
        T = _lib.require_tensor(actions, "actions", self._act_dtype,
                                (None, self.n_envs, self._n_acting) + self._act_tail, self.device).shape[0]
        obs, rew, done, info = self._outputs(T, out, auto_reset)
        with torch.cuda.device(self.device):
            _lib.check(self._fn("rollout")(self._h, T, _ptr(actions), _ptr(obs), _ptr(rew),
                                           _ptr(done), _ptr(info), int(auto_reset), _lib.stream(self.device)))
        return obs, rew, done, info

    def _rollout_heuristic(self, T, obs0, auto_reset, out, record_actions, actions_out, *extra, fn="rollout_heuristic",
                           mid=()):
        """madrl_<abi>_<fn>; `mid`: the family's arguments after the actions buffer, `extra`: those before the
        stream."""
        E, A = self.n_envs, self._n_acting
        _lib.require_tensor(obs0, "obs0", self.obs_dtype, (E, A, self.obs_dim), self.device)
        obs, rew, done, info = self._outputs(T, out, auto_reset)
        act_shape = (T, E, A) + self._act_tail
        if actions_out is not None:   # caller-owned buffer for the actions taken (no allocation in a rollout loop)
            act = _lib.require_tensor(actions_out, "actions_out", self._act_dtype, act_shape, self.device)
        else:
            act = torch.empty(act_shape, dtype=self._act_dtype, device=self.device) if record_actions else None
        with torch.cuda.device(self.device):
            _lib.check(self._fn(fn)(self._h, T, _ptr(obs0), _ptr(act), *mid, _ptr(obs), _ptr(rew), _ptr(done),
                                    _ptr(info), int(auto_reset), *extra, _lib.stream(self.device)))
        return act, obs, rew, done, info

    def set_obs_cache(self, mode):
        """L2 policy of the observation stores of rollout() and step(): _lib.OBS_CACHE_STREAM (the default,
        evict-first) or _lib.OBS_CACHE_KEEP (normal priority, for a policy that reads each step's observations
        right after it; float32 engines only).  The values written are the same either way."""
        _lib.check(self._fn("set_obs_cache")(self._h, int(mode)))
        self.obs_cache = int(mode)

    obs_cache = _lib.OBS_CACHE_STREAM

    def step(self, actions, auto_reset=False, out=None, **rollout_kw):
        """One lockstep step.  actions [E, A, *act_tail] (or anything reshapeable to it).  `out`: caller buffers
        (obs [E, A, D], rew [E, A], done [E], info [E, *info_tail]) written instead of new tensors; the
        returned values are then views of them.  `rollout_kw`: the family's further rollout() arguments."""
        a = torch.as_tensor(actions, device=self.device, dtype=self._act_dtype).reshape(
            (1, self.n_envs, self._n_acting) + self._act_tail)
        if out is not None:
            out = tuple(t.unsqueeze(0) if isinstance(t, torch.Tensor) else t for t in out)
        obs, rew, done, info = self.rollout(a, auto_reset=auto_reset, out=out, **rollout_kw)
        if len(self._info_keys) == 1:
            return obs[0], rew[0], done[0], {self._info_keys[0]: info[0]}
        return obs[0], rew[0], done[0], {k: info[0, :, i] for i, k in enumerate(self._info_keys)}

    RENDER_MAX_SIZE = 32768   # largest frame edge of madrl_*_render
    RENDER_MAX_REACH = float(1 << 29)   # radii and |sensor_range| * screen_size must stay below it (pixels)

    def _frame_ids(self, env_ids):
        """`env_ids` as the int32 device tensor the frame kernels read.  A sequence or a host tensor is checked here
        (ValueError for an id outside [0, n_envs)); a CUDA tensor is not read back, which would synchronise with
        the device, and the frame of an id outside the range comes back all zero (DESIGN §4.10).  An int64 id
        outside the range is made -1 on the device first, so that the int32 cast cannot wrap it onto an env."""
        if isinstance(env_ids, torch.Tensor) and env_ids.device.type == "cuda":
            if env_ids.dtype not in (torch.int32, torch.int64) or env_ids.dim() != 1:
                raise TypeError("env_ids must be a 1-D int32 or int64 tensor, got %s of shape %s"
                                % (env_ids.dtype, tuple(env_ids.shape)))
            ids = env_ids.to(device=self.device)
            if ids.dtype == torch.int64:
                ids = ids.masked_fill((ids < 0) | (ids >= self.n_envs), -1)
            ids = ids.to(dtype=torch.int32).contiguous()
        else:
            a = np.asarray(env_ids.numpy() if isinstance(env_ids, torch.Tensor) else env_ids)
            if a.ndim != 1 or not (a.size == 0 or np.issubdtype(a.dtype, np.integer)):
                raise TypeError("env_ids must be a 1-D sequence of ints, got %r" % (env_ids,))
            if a.size and (a.min() < 0 or a.max() >= self.n_envs):
                raise ValueError("env_ids must lie in [0, %d), got %d .. %d" % (self.n_envs, a.min(), a.max()))
            ids = torch.as_tensor(a.astype(np.int32), device=self.device)
        if ids.numel() < 1:
            raise ValueError("env_ids must name at least one env")
        return ids

    def _render(self, env_ids, shape, out, *args):
        """madrl_<abi>_render of `env_ids` into `out` (or a new tensor) of shape [n, *shape]; `args`: the family's
        arguments between the ids and the output."""
        if any(s < 1 or s > self.RENDER_MAX_SIZE for s in shape[:2]):
            raise ValueError("a frame must be 1 to %d pixels a side, got %d x %d" % (self.RENDER_MAX_SIZE, shape[1],
                                                                                   shape[0]))
        ids = self._frame_ids(env_ids)
        shape = (ids.numel(),) + tuple(shape)
        if out is None:
            out = torch.empty(shape, dtype=torch.uint8, device=self.device)
        _lib.require_tensor(out, "out", torch.uint8, shape, self.device)
        with torch.cuda.device(self.device):
            _lib.check(self._fn("render")(self._h, ids.numel(), _ptr(ids), *args, _ptr(out), _lib.stream(self.device)))
        return out

    def _render_sensor_frames(self, env_ids, screen_size, out):
        """Waterworld's and Hostage's render_frames: S x S frames drawn with the float64 sensor direction table."""
        S = int(screen_size)
        if S != screen_size:
            raise TypeError("screen_size must be an int, got %r" % (screen_size,))
        r = float(self.cfg.sensor_range)
        if not abs(r) * S < self.RENDER_MAX_REACH:   # NaN fails it too
            raise ValueError("a sensor_range of %r at screen_size %d reaches 2^29 pixels or more" % (r, S))
        dirs = getattr(self, "_sensor_dirs", None)
        if dirs is None:   # built once on the host, as the reference builds its sensors (waterworld.py:29-30)
            ang = np.linspace(0., 2. * np.pi, self.cfg.n_sensors + 1)[:-1]
            dirs = self._sensor_dirs = torch.as_tensor(np.stack([np.cos(ang), np.sin(ang)]), device=self.device)
        return self._render(env_ids, (S, S, 3), out, S, _ptr(dirs))

    def rollout_host(self, actions, obs, rew, done, info, auto_reset=True, obs_last=False):
        """rollout() with HOST tensors (pinned for full PCIe speed); the copies are inside the call,
        chunked and overlapped with the compute (csrc/host_pipeline.cuh).  `obs_last=True`: only the last
        step's observations come back (obs is [E, A, D]) -- the policy-on-device mode."""
        T = actions.shape[0]
        E, A = self.n_envs, self._n_acting
        _lib.require_tensor(actions, "actions", self._act_dtype, (T, E, A) + self._act_tail, 'cpu')
        shapes = self._trajectory_shapes(T)
        if obs_last:
            shapes = ((self.obs_dtype, (E, A, self.obs_dim)),) + shapes[1:]
        for t, n, (dt, s) in zip((obs, rew, done, info), ("obs", "rew", "done", "info"), shapes):
            _lib.require_tensor(t, n, dt, s, 'cpu')
        with torch.cuda.device(self.device):
            _lib.check(self._fn("rollout_host2")(self._h, T, _ptr(actions), _ptr(obs), _ptr(rew), _ptr(done),
                                                 _ptr(info), int(auto_reset), 1 if obs_last else 0))
        return obs, rew, done, info


class DropInEnv(AbstractMAEnv, EzPickle):
    """Base of the drop-in env classes.  A family sets `_reward_mech`, `_seed_value` and `_env_id` and
    defines `_make_engine(n_envs, **kw)`, which builds its batched engine from the env's attributes."""

    vectorized = True  # rllab batched plug-in hook (tf/envs/base.py:97-103)

    def setup(self):
        """(Re)build the engine from the current attributes (set_param_values contract)."""
        self._engine = self._make_engine(1, env_id_base=self._env_id)

    @property
    def reward_mech(self):
        return self._reward_mech

    def get_param_values(self):
        return self.__dict__

    def seed(self, seed=None):
        self._seed_value = 0 if seed is None else int(seed)
        self._engine.seed(self._seed_value)
        return [seed]

    def _frame(self, **kw):
        """Env 0's frame (render_frames of the engine) as a NumPy RGB uint8 array; no window is opened."""
        return self._engine.render_frames([0], **kw)[0].cpu().numpy()

    def vec_env_executor(self, n_envs, max_path_length):
        from .vec_executor import BatchedVecExecutor
        return BatchedVecExecutor(self, n_envs, max_path_length)
