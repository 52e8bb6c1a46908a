"""Device-side consumers of the rollout tensors (SURVEY.md 8f rows 1-3): what the reference does
right after ``env.step`` in its sampler loop, as streaming passes over ``[T, E, A, ...]`` tensors.

* ``gae``            rllab ``BaseSampler.process_samples`` (rllab/rllab/sampler/base.py:48-68)
* ``FrameStack``     ``ObservationBuffer`` (madrl_environments/__init__.py:143-196)
* ``Standardizer``   ``StandardizedEnv``   (madrl_environments/__init__.py:204-291)
* ``center_advantages`` / ``explained_variance``  the whole-batch statistics of
                     ``process_samples`` (base.py:69-86; rllab/rllab/algos/util.py:7-12,
                     rllab/rllab/misc/special.py:51-59)
* ``LinearFeatureBaseline``  rllab's default baseline (rllab/rllab/baselines/linear_feature_baseline.py):
                     ``predict`` before ``gae``, ``fit`` after it (base.py:52-55, :163-168)
* ``to_paths``       the per-agent ``paths`` dicts of ``dec_rollout``
                     (rllab/rllab/sampler/ma_sampler.py:52-100), built on the host from gathered
                     tensors for callers that still want rllab's list-of-paths format.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import _ptr


def _stream(dev):
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def _require_dtype(t, name, dtypes=(torch.float32,)):
    """The passes read and write raw buffers: a tensor of another dtype must not reach them."""
    if t is not None and t.dtype not in dtypes:
        raise TypeError("%s must be %s, got %s" % (name, " or ".join(str(d) for d in dtypes), t.dtype))


def _obs_fn(name, dtype):
    """The f32 or bf16 entry point of an observation pass."""
    return getattr(_lib.lib(), "madrl_%s_%s" % (name, "bf16" if dtype == torch.bfloat16 else "f32"))


_OBS_DTYPES = (torch.float32, torch.bfloat16)


def gae(rew, values, done, discount, gae_lambda, last_value=None):
    """rew, values [T,E,A] float32 cuda; done [T,E] uint8 -> (advantages, returns) [T,E,A].

    Paths end where ``done`` is set (bootstrap 0, base.py:57) and at the end of the rollout
    (bootstrap ``last_value`` [E,A] if given, else 0)."""
    for t, n in ((rew, "rew"), (values, "values"), (last_value, "last_value")):
        _require_dtype(t, n)
    _require_dtype(done, "done", (torch.uint8,))
    rew, values, done = rew.contiguous(), values.contiguous(), done.contiguous()
    T, E, A = rew.shape
    adv, ret = torch.empty_like(rew), torch.empty_like(rew)
    lv = last_value.contiguous() if last_value is not None else None
    with torch.cuda.device(rew.device):
        _lib.check(_lib.lib().madrl_gae_f32(T, E, A, _ptr(rew), _ptr(values), _ptr(done), _ptr(lv),
                                            float(discount), float(gae_lambda), _ptr(adv), _ptr(ret),
                                            _stream(rew.device)))
    return adv, ret


MOMENTS_STATS, MOMENTS_WS = 9, 4096            # include/madrl_b200.h


def _moments_buffers(dev):
    return (torch.empty(MOMENTS_STATS, dtype=torch.float64, device=dev),
            torch.empty(MOMENTS_WS, dtype=torch.float64, device=dev))


def center_advantages(adv, center=True, positive=False, inplace=False):
    """``util.center_advantages`` / ``util.shift_advantages_to_positive`` over every sample of the
    batch (base.py:82-86 applies them to the concatenation of all paths): float64 mean / population
    std / min computed on the device, deterministic.  Returns the processed tensor (same shape)."""
    _require_dtype(adv, "adv")
    out = adv.contiguous() if inplace else adv.contiguous().clone()
    stats, ws = _moments_buffers(out.device)
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().madrl_center_advantages_f32(out.numel(), _ptr(out), int(bool(center)),
                                                          int(bool(positive)), _ptr(stats), _ptr(ws),
                                                          _stream(out.device)))
    return out


def moments(a, b=None):
    """float64 [9] cuda tensor: means, population variances and minima of the series a, b, b - a
    taken over every element (NumPy's two-pass ``var``)."""
    _require_dtype(a, "a")
    _require_dtype(b, "b")
    a = a.contiguous()
    b = b.contiguous() if b is not None else None
    assert b is None or b.numel() == a.numel()
    stats, ws = _moments_buffers(a.device)
    with torch.cuda.device(a.device):
        _lib.check(_lib.lib().madrl_moments_f32(a.numel(), _ptr(a), _ptr(b), _ptr(stats), _ptr(ws),
                                                _stream(a.device)))
    return stats


def explained_variance(ypred, y):
    """``special.explained_variance_1d`` (special.py:51-59) of baseline predictions against returns,
    over every sample of the batch; one 72-byte device->host read."""
    st = moments(ypred, y).cpu().numpy()
    var_pred, vary, var_res = float(st[3]), float(st[4]), float(st[5])
    if np.isclose(vary, 0):
        return 0 if var_pred > 0 else 1
    return 1 - var_res / (vary + 1e-8)


class FrameStack(object):
    """ObservationBuffer for a whole env batch: the last ``buffer_size`` observations of every
    agent stacked on a new minor axis; a reset fills every slot with the reset observation.
    ``dtype``: the observations' (torch.float32, or torch.bfloat16 for an engine built with
    ``obs_dtype=torch.bfloat16``); the stack keeps it (values are only moved)."""

    def __init__(self, n_envs, n_agents, obs_dim, buffer_size, device, dtype=torch.float32):
        _require_dtype(torch.empty(0, dtype=dtype), "dtype", _OBS_DTYPES)
        self.shape, self.dtype = (n_envs, n_agents, obs_dim, buffer_size), dtype
        self.carry = torch.zeros(self.shape, dtype=dtype, device=device)   # __init__.py:150

    def reset(self, obs0):
        """obs0 [E,A,D] from engine.reset() -> stacked [E,A,D,B] (__init__.py:186-196)."""
        _require_dtype(obs0, "obs0", (self.dtype,))
        self.carry.copy_(obs0.unsqueeze(-1).expand(self.shape))
        return self.carry.clone()

    def rollout(self, obs, done):
        """obs [T,E,A,D], done [T,E] from engine.rollout(auto_reset=True) -> [T,E,A,D,B]."""
        _require_dtype(obs, "obs", (self.dtype,))
        _require_dtype(done, "done", (torch.uint8,))
        obs, done = obs.contiguous(), done.contiguous()
        T = obs.shape[0]
        E, A, D, B = self.shape
        assert tuple(obs.shape) == (T, E, A, D) and tuple(done.shape) == (T, E), (obs.shape, done.shape)
        out = torch.empty((T, E, A, D, B), dtype=self.dtype, device=obs.device)
        with torch.cuda.device(obs.device):
            _lib.check(_obs_fn("frame_stack", self.dtype)(T, E, A, D, B, _ptr(obs), _ptr(done),
                                                          _ptr(self.carry), _ptr(out), _stream(obs.device)))
        return out


class Standardizer(object):
    """StandardizedEnv's running observation / reward normalisation for a whole env batch
    (one running estimate per env, agent and observation coordinate, as each reference env keeps
    its own).  Under auto-reset the rollout's obs slot of a done step holds the reset observation; the
    reference's estimate also sees the terminal one (step() standardises it, then reset() the new
    one, madrl_environments/__init__.py:283-291).  Pass `done` and the `terminal_obs` side tensor
    (`engine.set_terminal_obs`) to `obs()` to reproduce that order exactly; without them the estimate
    sees the reset observation only."""

    def __init__(self, n_envs, n_agents, obs_dim, device, scale_reward=1., enable_obsnorm=False,
                 enable_rewnorm=False, obs_alpha=0.001, rew_alpha=0.001, eps=1e-8):
        self.scale_reward, self.enable_obsnorm, self.enable_rewnorm = scale_reward, enable_obsnorm, enable_rewnorm
        self.obs_alpha, self.rew_alpha, self.eps = obs_alpha, rew_alpha, eps
        self.obs_mean = torch.zeros((n_envs, n_agents, obs_dim), dtype=torch.float64, device=device)
        self.obs_var = torch.ones((n_envs, n_agents, obs_dim), dtype=torch.float64, device=device)
        self.rew_mean = torch.zeros((n_envs, n_agents), dtype=torch.float64, device=device)
        self.rew_var = torch.ones((n_envs, n_agents), dtype=torch.float64, device=device)

    def obs(self, obs, done=None, terminal_obs=None):
        """In place on obs [T,E,A,D] (or [E,A,D]); with `done` [T,E] and `terminal_obs` [T,E,A,D] the
        terminal observations update the estimate first (and are standardised in place as well).
        float32 or bfloat16 observations; bfloat16 ones take the same float64 arithmetic on the widened
        values and are rounded once, at the store."""
        if not self.enable_obsnorm:
            return obs
        _require_dtype(obs, "obs", _OBS_DTYPES)
        x = obs if obs.dim() == 4 else obs.unsqueeze(0)
        assert x.is_contiguous() and x[0].numel() == self.obs_mean.numel(), (x.shape, self.obs_mean.shape)
        if terminal_obs is not None:
            _require_dtype(terminal_obs, "terminal_obs", (x.dtype,))
            _require_dtype(done, "done", (torch.uint8,))
            assert done is not None and terminal_obs.shape == x.shape and terminal_obs.is_contiguous()
            E = x.shape[1]
            with torch.cuda.device(x.device):
                _lib.check(_obs_fn("standardize_obs_terminal", x.dtype)(
                    x.shape[0], E, self.obs_mean.numel() // E, _ptr(x), _ptr(terminal_obs), _ptr(done.contiguous()),
                    _ptr(self.obs_mean), _ptr(self.obs_var), self.obs_alpha, self.eps, _stream(x.device)))
            return obs
        with torch.cuda.device(x.device):
            _lib.check(_obs_fn("standardize", x.dtype)(x.shape[0], self.obs_mean.numel(), _ptr(x),
                                                       _ptr(self.obs_mean), _ptr(self.obs_var), self.obs_alpha,
                                                       self.eps, 1, 1.0, 1, _stream(x.device)))
        return obs

    def rew(self, rew):
        """In place on rew [T,E,A]: optional running-std division, then scale_reward."""
        _require_dtype(rew, "rew")
        assert rew.is_contiguous() and rew[0].numel() == self.rew_mean.numel(), rew.shape
        with torch.cuda.device(rew.device):
            _lib.check(_lib.lib().madrl_standardize_f32(rew.shape[0], self.rew_mean.numel(), _ptr(rew),
                                                        _ptr(self.rew_mean), _ptr(self.rew_var), self.rew_alpha,
                                                        self.eps, 0, float(self.scale_reward),
                                                        int(self.enable_rewnorm), _stream(rew.device)))
        return rew


class EpisodeStats(object):
    """DiagnosticsWrapper's per-episode statistics for a whole env batch
    (madrl_environments/__init__.py:314-369): episode reward per agent, its agent-mean, the
    discounted return of the agent-mean reward and the episode length, emitted at the steps where
    an episode closes (``done`` or ``max_traj_len`` reached)."""

    def __init__(self, n_envs, n_agents, device, discount=0.99, max_traj_len=500):
        self.n_envs, self.n_agents, self.discount, self.max_traj_len = n_envs, n_agents, discount, max_traj_len
        self.carry = torch.zeros((n_envs, n_agents + 3), dtype=torch.float64, device=device)

    def rollout(self, rew, done):
        """rew [T,E,A] float32, done [T,E] uint8 -> dict(end [T,E] bool, episode_reward [T,E,A],
        episode_avg_reward [T,E], episode_disc_return [T,E], episode_length [T,E])."""
        _require_dtype(rew, "rew")
        _require_dtype(done, "done", (torch.uint8,))
        rew, done = rew.contiguous(), done.contiguous()
        T, E, A = rew.shape
        dev = rew.device
        ep_r = torch.empty((T, E, A), dtype=torch.float32, device=dev)
        ep_d = torch.empty((T, E), dtype=torch.float32, device=dev)
        ep_l = torch.empty((T, E), dtype=torch.int32, device=dev)
        ep_e = torch.empty((T, E), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().madrl_episode_stats_f32(T, E, A, _ptr(rew), _ptr(done), float(self.discount),
                                                          int(self.max_traj_len), _ptr(self.carry), _ptr(ep_r),
                                                          _ptr(ep_d), _ptr(ep_l), _ptr(ep_e), _stream(dev)))
        return dict(end=ep_e.bool(), episode_reward=ep_r, episode_avg_reward=ep_r.mean(dim=-1),
                    episode_disc_return=ep_d, episode_length=ep_l)


def _require_shape(t, name, shape):
    if tuple(t.shape) != tuple(shape):
        raise ValueError("%s must have shape %s, got %s" % (name, tuple(shape), tuple(t.shape)))


class LinearFeatureBaseline(object):
    """rllab's ``LinearFeatureBaseline`` (rllab/rllab/baselines/linear_feature_baseline.py) over the rows of a
    rollout, pooled over envs and agents (the decentralized mode: one baseline for every agent's paths).

    Row (t, e, a) is the observation action t was taken in -- with ``obs_before`` [E,A,D] (what
    ``engine.rollout(auto_reset=True)`` returns plus the observations before the launch) row t uses
    ``obs[t-1]`` (``obs_before`` for t = 0), as ``pack_paths`` does; without it ``obs[t]`` as given.  Its time
    index is its 0-based position in its path (paths cut at ``done``), plus ``t0[e]`` (int32 [E]) on env e's
    first path: pass the engine's ``state['path_len']`` read before the launch so that a path begun in an
    earlier launch continues its index.  Features ``[clip(o,±10), clip(o,±10)², i/100, (i/100)², (i/100)³, 1]``
    (Df = 2D + 4) are built on the device from the observation rows, never stored: ``fit`` forms the float64
    normal equations ``[F y]ᵀ[F y]`` on the FP64 tensor cores (``madrl_lfb_normal_eq_*``), optionally
    all-reduces them over a ``torch.distributed`` group, and solves ``(FᵀF + reg·I) c = Fᵀy`` by Cholesky on
    the device; only if that fails does it fall back to rllab's host ``lstsq`` with its retry loop.
    Observations: float32 or bfloat16 (widened exactly: a bfloat16 call equals the call on ``obs.float()``).
    Centralized control is the view ``obs.view(T, E, 1, A * D)``."""

    def __init__(self, obs_dim, device, reg_coeff=1e-5):
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.obs_dim, self.device, self.reg_coeff = int(obs_dim), device, reg_coeff
        self.n_features = 2 * self.obs_dim + 4
        self._coeffs = None

    def get_param_values(self):
        """float64 coefficients [Df] (NumPy), or None before the first fit."""
        return None if self._coeffs is None else self._coeffs.cpu().numpy()

    def set_param_values(self, val):
        if val is None:
            self._coeffs = None
            return
        c = torch.as_tensor(np.asarray(val, dtype=np.float64) if not torch.is_tensor(val) else val)
        _require_dtype(c, "coefficients", (torch.float64,))
        _require_shape(c, "coefficients", (self.n_features,))
        self._coeffs = c.to(self.device).contiguous().clone()

    def _rows(self, obs, done, obs_before, t0, returns=None):
        """Validates the rollout tensors (before any pointer reaches a kernel) and runs the path plan."""
        for t, n in ((obs, "obs"), (done, "done"), (obs_before, "obs_before"), (t0, "t0"), (returns, "returns")):
            if t is not None and not torch.is_tensor(t):
                raise TypeError("%s must be a torch.Tensor, got %r" % (n, type(t)))
        _require_dtype(obs, "obs", _OBS_DTYPES)
        _require_dtype(obs_before, "obs_before", (obs.dtype,))
        _require_dtype(done, "done", (torch.uint8,))
        _require_dtype(t0, "t0", (torch.int32,))
        _require_dtype(returns, "returns")
        if obs.dim() != 4:
            raise ValueError("obs must be [T, E, A, D], got shape %s" % (tuple(obs.shape),))
        T, E, A, D = obs.shape
        if D != self.obs_dim:
            raise ValueError("obs has %d features per row, the baseline was built for %d" % (D, self.obs_dim))
        _require_shape(done, "done", (T, E))
        if obs_before is not None:
            _require_shape(obs_before, "obs_before", (E, A, D))
        if t0 is not None:
            _require_shape(t0, "t0", (E,))
        if returns is not None:
            _require_shape(returns, "returns", (T, E, A))
        for t, n in ((obs, "obs"), (done, "done"), (obs_before, "obs_before"), (t0, "t0"), (returns, "returns")):
            if t is not None and t.device != self.device:
                raise ValueError("%s must live on %s, got %s" % (n, self.device, t.device))
        if T * E * A >= 2 ** 31:
            raise ValueError("T*E*A must be < 2^31, got %d" % (T * E * A))
        L = _lib.lib()
        done = done.contiguous()
        seg_s = torch.empty((T, E), dtype=torch.int32, device=self.device)
        seg_l = torch.empty((T, E), dtype=torch.int32, device=self.device)
        n_ep = torch.empty((E,), dtype=torch.int32, device=self.device)
        ep_rec = torch.empty((E, T, 3), dtype=torch.int32, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(L.madrl_paths_plan(T, E, A, _ptr(done), _ptr(seg_s), _ptr(seg_l), _ptr(n_ep), _ptr(ep_rec),
                                          _stream(self.device)))
        cont = lambda x: None if x is None else x.contiguous()          # noqa: E731
        return (T, E, A, D), cont(obs), cont(obs_before), cont(t0), seg_s

    def normal_equations(self, obs, done, returns, obs_before=None, t0=None):
        """G = [F y]ᵀ[F y], float64 [Df+1, Df+1] on the device: FᵀF, with Fᵀy as row and column Df."""
        (T, E, A, D), obs, obs_before, t0, seg_s = self._rows(obs, done, obs_before, t0, returns)
        returns = returns.contiguous()
        L = _lib.lib()
        nbytes = C.c_size_t()
        _lib.check(L.madrl_lfb_workspace_size(D, C.byref(nbytes)))
        ws = torch.empty(nbytes.value // 8, dtype=torch.float64, device=self.device)
        G = torch.empty((self.n_features + 1, self.n_features + 1), dtype=torch.float64, device=self.device)
        with torch.cuda.device(self.device):
            _lib.check(_obs_fn("lfb_normal_eq", obs.dtype)(T, E, A, D, _ptr(obs), _ptr(obs_before), _ptr(seg_s),
                                                           _ptr(t0), _ptr(returns), _ptr(G), _ptr(ws),
                                                           _stream(self.device)))
        return G

    def solve(self, G):
        """Coefficients from normal equations G (as `normal_equations` returns them), rllab's regularisation."""
        Df = self.n_features
        M, b = G[:Df, :Df], G[:Df, Df]
        Lc, info = torch.linalg.cholesky_ex(M + self.reg_coeff * torch.eye(Df, dtype=G.dtype, device=G.device))
        if int(info) == 0:
            c = torch.cholesky_solve(b.unsqueeze(1), Lc).squeeze(1)
            if bool(torch.isfinite(c).all()):
                return c
        # the factorisation failed: rllab's loop (linear_feature_baseline.py:29-37) on the host
        Mn, bn, reg = M.cpu().numpy(), b.cpu().numpy(), self.reg_coeff
        for _ in range(5):
            c = np.linalg.lstsq(Mn + reg * np.identity(Df), bn, rcond=None)[0]
            if np.all(np.isfinite(c)):
                break
            reg *= 10
        return torch.from_numpy(c).to(G.device)

    def fit(self, obs, done, returns, obs_before=None, t0=None, group=None):
        """Fit to ``returns`` [T,E,A] float32 (``gae``'s second output).  With a ``torch.distributed`` group the
        normal equations are summed over its ranks before the solve (every rank gets the pooled coefficients;
        no observation moves)."""
        G = self.normal_equations(obs, done, returns, obs_before, t0)
        if group is not None:
            import torch.distributed as dist
            dist.all_reduce(G, op=dist.ReduceOp.SUM, group=group)
        self._coeffs = self.solve(G)

    def predict(self, obs, done, obs_before=None, t0=None):
        """values [T,E,A] float32 = features(row) . coefficients, evaluated in float64; zeros before the first fit."""
        (T, E, A, D), obs, obs_before, t0, seg_s = self._rows(obs, done, obs_before, t0)
        values = torch.empty((T, E, A), dtype=torch.float32, device=self.device)
        if self._coeffs is None:
            return values.zero_()
        with torch.cuda.device(self.device):
            _lib.check(_obs_fn("lfb_predict", obs.dtype)(T, E, A, D, _ptr(obs), _ptr(obs_before), _ptr(seg_s),
                                                         _ptr(t0), _ptr(self._coeffs), _ptr(values),
                                                         _stream(self.device)))
        return values


def to_paths(obs, actions, rew, done, infos=None):
    """Split time-major rollout arrays [T,E,A,...] (numpy or cpu tensors) into rllab-style paths:
    one dict per (env, agent, episode) with ``observations/actions/rewards/env_infos`` arrays, the
    format ``dec_rollout`` returns (ma_sampler.py:88-100).  ``obs[t]`` is the observation the action
    ``actions[t]`` was taken in, i.e. callers pass obs shifted by one step (reset obs first)."""
    obs, actions, rew, done = [np.asarray(x) for x in (obs, actions, rew, done)]
    T, E, A = rew.shape
    infos = {k: np.asarray(v) for k, v in (infos or {}).items()}
    paths = []
    for e in range(E):
        ends = list(np.nonzero(done[:, e])[0] + 1)
        if not ends or ends[-1] != T:
            ends.append(T)
        start = 0
        for end in ends:
            for a in range(A):
                paths.append(dict(observations=obs[start:end, e, a], actions=actions[start:end, e, a],
                                  rewards=rew[start:end, e, a],
                                  env_infos={k: v[start:end, e] for k, v in infos.items()},
                                  env=e, agent=a, terminated=bool(done[end - 1, e])))
            start = end
    return paths


class PackedPaths(object):
    """rllab-style paths of one rollout, resident on the device (see `pack_paths`).

    ``observations [N, D]``, ``actions [N, ...]``, ``rewards [N]`` with N = T*E*A rows in path order;
    ``env_infos[k] [E*T]`` in (env, time) order; per path p (ordered env, episode, agent -- the order of
    the host ``to_paths``): ``offset[p]``, ``length[p]``, ``env[p]``, ``agent[p]``, ``terminated[p]`` and
    ``info_offset[p]`` (first row of the path's steps in the env_infos arrays).
    """

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def __len__(self):
        return int(self.offset.shape[0])

    def path(self, p):
        """Path p as the dict ``dec_rollout`` returns (ma_sampler.py:88-100); zero-copy views."""
        o, n, io = int(self.offset[p]), int(self.length[p]), int(self.info_offset[p])
        return dict(observations=self.observations[o:o + n], actions=self.actions[o:o + n],
                    rewards=self.rewards[o:o + n],
                    env_infos={k: v[io:io + n] for k, v in self.env_infos.items()},
                    env=int(self.env[p]), agent=int(self.agent[p]), terminated=bool(self.terminated[p]))

    def to_list(self):
        """All paths as NumPy dicts (ONE device->host copy per packed array, then views)."""
        host = PackedPaths(**{k: (v.cpu().numpy() if torch.is_tensor(v) else
                                  ({kk: vv.cpu().numpy() for kk, vv in v.items()} if isinstance(v, dict) else v))
                              for k, v in self.__dict__.items()})
        return [host.path(p) for p in range(len(host))]


def pack_paths(obs, actions, rew, done, infos=None, obs_before=None):
    """Device-side ``to_paths``: rollout tensors [T,E,A,...] (CUDA) -> `PackedPaths`.

    Episodes are cut at ``done`` (and at the end of the rollout).  ``obs_before`` [E,A,D] = the
    observations the first actions were taken in (the reset / previous rollout's last observations):
    when given, ``obs`` is what ``engine.rollout(auto_reset=True)`` returned (the observation AFTER each
    step, the reset observation on a done step) and the packed ``observations`` are shifted so that row t
    is the observation action t was taken in -- what rllab stores (ma_sampler.py:71-77).  Without it,
    ``obs`` is used as is (the host ``to_paths`` contract).  Two kernels of csrc/postproc.cu: a plan pass
    over ``done`` and one HBM-bound row permutation per tensor; no host loop.  Tensors of 4-byte elements,
    and bfloat16 observations (2-byte rows, ``madrl_paths_pack_u16``)."""
    for name, x in [("obs", obs), ("actions", actions), ("rew", rew)] + sorted((infos or {}).items()):
        if x.element_size() not in (2, 4) or (x.element_size() == 2 and x.dtype != torch.bfloat16):
            raise TypeError("pack_paths packs 4-byte elements and bfloat16; %s is %s" % (name, x.dtype))
    _require_dtype(done, "done", (torch.uint8,))
    L = _lib.lib()
    T, E, A = rew.shape
    dev = rew.device
    done = done.contiguous()
    seg_s = torch.empty((T, E), dtype=torch.int32, device=dev)
    seg_l = torch.empty((T, E), dtype=torch.int32, device=dev)
    n_ep = torch.empty((E,), dtype=torch.int32, device=dev)
    ep_rec = torch.zeros((E, T, 3), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        st = _stream(dev)
        _lib.check(L.madrl_paths_plan(T, E, A, _ptr(done), _ptr(seg_s), _ptr(seg_l), _ptr(n_ep), _ptr(ep_rec), st))

        def pack(x, per_agent, first=None):
            x = x.contiguous()
            assert x.shape[0] == T and x.shape[1] == E, (x.dtype, x.shape)
            assert not per_agent or x.shape[2] == A, x.shape
            n_agents = A if per_agent else 1
            tail = tuple(x.shape[3:] if per_agent else x.shape[2:])
            D = max(1, int(np.prod(tail)))
            out = torch.empty((T * E * n_agents,) + tail, dtype=x.dtype, device=dev)
            if first is not None:
                first = first.to(x.dtype).contiguous()
                assert first.shape == x.shape[1:], (first.shape, x.shape)
            # per-env tensors (n_agents = 1): the row offset e*T + s + (t - s) = e*T + t for any (s, L)
            fn = L.madrl_paths_pack_u16 if x.element_size() == 2 else L.madrl_paths_pack_u32
            _lib.check(fn(T, E, n_agents, D, _ptr(x), _ptr(first), _ptr(seg_s), _ptr(seg_l), _ptr(out), st))
            return out

        packed_obs = pack(obs, True, obs_before)
        packed_act = pack(actions, True)
        packed_rew = pack(rew, True)
        packed_info = {k: pack(v, False) for k, v in (infos or {}).items()}
    # per-path records from the (tiny) per-episode records: plain tensor ops, no host loop
    slot = torch.arange(T, device=dev).unsqueeze(0)
    live = slot < n_ep.unsqueeze(1)                                   # [E, T] valid episode slots
    e_idx, _ = torch.nonzero(live, as_tuple=True)
    rec = ep_rec[live]                                                # [n_episodes_total, 3] in (env, episode) order
    s, Ln, term = rec[:, 0].long(), rec[:, 1].long(), rec[:, 2]
    a_idx = torch.arange(A, device=dev)
    offset = ((e_idx * T * A + s * A).unsqueeze(1) + a_idx.unsqueeze(0) * Ln.unsqueeze(1)).reshape(-1)
    rep = lambda v: v.unsqueeze(1).expand(-1, A).reshape(-1)          # noqa: E731
    return PackedPaths(observations=packed_obs, actions=packed_act, rewards=packed_rew, env_infos=packed_info,
                       offset=offset, length=rep(Ln), env=rep(e_idx), agent=a_idx.repeat(rec.shape[0]),
                       terminated=rep(term).bool(), info_offset=rep(e_idx * T + s))
