"""Device-side consumers of the rollout tensors (SURVEY.md 8f rows 1-3): what the reference does
right after ``env.step`` in its sampler loop, as streaming passes over ``[T, E, A, ...]`` tensors.

* ``gae``            rllab ``BaseSampler.process_samples`` (rllab/rllab/sampler/base.py:48-68)
* ``FrameStack``     ``ObservationBuffer`` (madrl_environments/__init__.py:143-196)
* ``Standardizer``   ``StandardizedEnv``   (madrl_environments/__init__.py:204-291)
* ``center_advantages`` / ``explained_variance``  the whole-batch statistics of
                     ``process_samples`` (base.py:69-86; rllab/rllab/algos/util.py:7-12,
                     rllab/rllab/misc/special.py:51-59)
* ``LinearFeatureBaseline``  rllab's default baseline (rllab/rllab/baselines/linear_feature_baseline.py):
                     ``predict`` before ``gae``, ``fit`` after it (base.py:52-55, :163-168); one per agent
                     with ``n_agents`` (concurrent control)
* ``process_samples_concurrent``  the concurrent branch of ``BatchMASampler.process_samples``
                     (rllab/sandbox/rocky/tf/samplers/batch_ma_sampler.py:64-123, :184-188)
* ``to_paths``       the per-agent ``paths`` dicts of ``dec_rollout``
                     (rllab/rllab/sampler/ma_sampler.py:52-100), built on the host from gathered
                     tensors for callers that still want rllab's list-of-paths format.
* ``pad_paths`` / ``path_statistics`` / ``process_samples_recurrent``  the recurrent branch of
                     ``process_samples`` (base.py:105-161; per agent, batch_ma_sampler.py:124-181): paths
                     zero-padded to the longest one with a ``valids`` mask, and the sampler's return statistics
                     (base.py:170-180).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import _ptr

# Argument checks (_lib.require_tensor): every tensor of a call is checked against the shape derived from its
# first tensor and must sit on that tensor's device.  That device is checked last (it must be CUDA, and where an
# object owns state, the state's device), so that a call on host tensors reports a wrong dtype or shape first.


def _obs_fn(name, dtype):
    """The f32 or bf16 entry point of an observation pass."""
    return getattr(_lib.lib(), "madrl_%s_%s" % (name, "bf16" if dtype == torch.bfloat16 else "f32"))


def _paths_plan(done, A):
    """How a rollout is cut into paths (at ``done`` and at the end of the rollout): madrl_paths_plan over done [T,E]
    uint8 on its CUDA device, enqueued without a host synchronisation.  Returns int32 seg_s, seg_l [T,E] (start and
    length of the path holding each step), n_ep [E] (paths per env) and ep_rec [E,T,3] (per path of each env: start,
    length, terminated; zero past the env's last path)."""
    from .whole_paths import whole_paths_of
    wp = whole_paths_of(done)
    if wp is not None:     # a WholePathBatch's [N, 1] view: the plan built from its path table, one thread per row
        return wp.plan()
    T, E = done.shape
    dev = done.device
    seg_s = torch.empty((T, E), dtype=torch.int32, device=dev)
    seg_l = torch.empty((T, E), dtype=torch.int32, device=dev)
    n_ep = torch.empty((E,), dtype=torch.int32, device=dev)
    ep_rec = torch.zeros((E, T, 3), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().madrl_paths_plan(T, E, A, _ptr(done.contiguous()), _ptr(seg_s), _ptr(seg_l), _ptr(n_ep),
                                               _ptr(ep_rec), _lib.stream(dev)))
    return seg_s, seg_l, n_ep, ep_rec


_OBS_DTYPES = (torch.float32, torch.bfloat16)
_PACKED_DTYPES = (torch.float32, torch.int32, torch.uint32, torch.bfloat16)   # pack_paths moves 4- and 2-byte words


def gae(rew, values, done, discount, gae_lambda, last_value=None):
    """rew, values [T,E,A] float32 cuda; done [T,E] uint8 -> (advantages, returns) [T,E,A].

    Paths end where ``done`` is set (bootstrap 0, base.py:57) and at the end of the rollout
    (bootstrap ``last_value`` [E,A] if given, else 0).  On the ``done`` of ``WholePathBatch.as_rollout()`` one thread
    per (path, agent) walks the batch's paths (every one ends at ``done``, so ``last_value`` is unused, as in the
    serial walk), with the serial walk's arithmetic."""
    T, E, A = _lib.require_tensor(rew, "rew", torch.float32, (None, None, None), None, contiguous=False).shape
    dev = rew.device
    _lib.require_tensor(values, "values", torch.float32, (T, E, A), dev, contiguous=False)
    _lib.require_tensor(done, "done", torch.uint8, (T, E), dev, contiguous=False)
    _lib.require_tensor(last_value, "last_value", torch.float32, (E, A), dev, contiguous=False, optional=True)
    _lib.require_tensor(rew, "rew", torch.float32, (T, E, A), "cuda", contiguous=False)
    rew, values, done = rew.contiguous(), values.contiguous(), done.contiguous()
    adv, ret = torch.empty_like(rew), torch.empty_like(rew)
    lv = last_value.contiguous() if last_value is not None else None
    from .whole_paths import whole_paths_of
    wp = whole_paths_of(done)
    if wp is not None:
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().madrl_gae_paths_f32(wp.n_paths, A, _ptr(wp.path_start), _ptr(rew), _ptr(values),
                                                      float(discount), float(gae_lambda), _ptr(adv), _ptr(ret),
                                                      _lib.stream(dev)))
        return adv, ret
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().madrl_gae_f32(T, E, A, _ptr(rew), _ptr(values), _ptr(done), _ptr(lv),
                                            float(discount), float(gae_lambda), _ptr(adv), _ptr(ret),
                                            _lib.stream(dev)))
    return adv, ret


MOMENTS_STATS, MOMENTS_WS = 9, 4096            # include/madrl_b200.h
AGENTS_MAX = 1024                               # include/madrl_b200.h MADRL_AGENTS_MAX


def _agent_columns(t, name):
    """(rows, A) of a float32 tensor whose last axis is the agent; raises before any library call.  Its
    device is left to the caller."""
    _lib.require_tensor(t, name, torch.float32, (...,), None, contiguous=False)
    if t.dim() < 1 or t.shape[-1] < 1 or t.numel() == 0:
        raise ValueError("%s must have a non-empty last (agent) axis, got shape %s" % (name, tuple(t.shape)))
    A = int(t.shape[-1])
    if A > AGENTS_MAX:
        raise ValueError("%s has %d agents, at most %d are supported" % (name, A, AGENTS_MAX))
    return t.numel() // A, A


def _moments(a, b, A, group):
    """float64 [A, 9] moments of the columns of a, b [rows, A] (the whole batch is A = 1), over every rank of a
    ``torch.distributed`` group (None: this rank's rows): the sums and row counts pooled give the means, the sums of
    squared deviations about those means pooled give the population variances (NumPy's two passes over the union
    of the shards), the minima pool by their minimum.  `dist.pool_sum` combines in rank order, so every rank gets
    the same bits.  The row counts stay a float64 device tensor: a division by a host scalar may be computed as a
    multiplication by its reciprocal, which can differ in the last bit from the division."""
    from .dist import _pooled, pool_min, pool_sum
    rows, dev = a.numel() // A, a.device
    stats = torch.empty((A, MOMENTS_STATS), dtype=torch.float64, device=dev)
    ws = torch.empty((A, MOMENTS_WS), dtype=torch.float64, device=dev)
    fn, stream = _lib.lib().madrl_moments_pass_f32, _lib.stream(dev)
    with torch.cuda.device(dev):
        _lib.check(fn(rows, A, _ptr(a), _ptr(b), 0, _ptr(stats), _ptr(ws), stream))
        count = torch.full((A, 1), float(rows), dtype=torch.float64, device=dev)
        # a group pools the sums and the row counts in one exchange
        sums, n = _pooled(lambda p, g: pool_sum(torch.cat(p, dim=1), g).split(3, dim=1), (stats[:, 0:3], count),
                          group)
        _pooled(lambda m, g: m.copy_(pool_min(m, g)), stats[:, 6:9], group)
        torch.div(sums, n, out=stats[:, 0:3])
        _lib.check(fn(rows, A, _ptr(a), _ptr(b), 1, _ptr(stats), _ptr(ws), stream))
        torch.div(_pooled(pool_sum, stats[:, 3:6], group), n, out=stats[:, 3:6])
    return stats


def center_advantages(adv, center=True, positive=False, inplace=False, per_agent=False, group=None):
    """``util.center_advantages`` / ``util.shift_advantages_to_positive`` over every sample of the
    batch (base.py:82-86 applies them to the concatenation of all paths): float64 mean / population
    std / min computed on the device, deterministic.  Returns the processed tensor (same shape).
    ``per_agent=True``: the last axis of ``adv`` (e.g. [T,E,A]) is the agent, and each agent's samples are
    centred with their own statistics, as the concurrent sampler does per agent
    (batch_ma_sampler.py:102-106).  ``group``: a ``torch.distributed`` group whose ranks hold the shards of one
    batch: the statistics are the whole batch's (`moments` with ``group``), the same on every rank."""
    if per_agent:
        rows, A = _agent_columns(adv, "adv")
    _lib.require_tensor(adv, "adv", torch.float32, (...,), "cuda", contiguous=False)
    out = adv.contiguous() if inplace else adv.contiguous().clone()
    if not per_agent:
        rows, A = out.numel(), 1
    stats = _moments(out, None, A, group)
    with torch.cuda.device(out.device):
        _lib.check(_lib.lib().madrl_center_apply_f32(rows, A, _ptr(out), _ptr(stats), int(bool(center)),
                                                     int(bool(positive)), _lib.stream(out.device)))
    return out


def moments(a, b=None, group=None):
    """float64 [9] cuda tensor: means, population variances and minima of the series a, b, b - a
    (b of a's shape) taken over every element (NumPy's two-pass ``var``).  ``group``: a ``torch.distributed``
    group whose ranks hold the shards of one batch: the moments of the whole batch, the same bits on every rank
    (a one-rank group gives ``group=None``'s bits)."""
    _lib.require_tensor(a, "a", torch.float32, (...,), None, contiguous=False)
    _lib.require_tensor(b, "b", torch.float32, tuple(a.shape), a.device, contiguous=False, optional=True)
    _lib.require_tensor(a, "a", torch.float32, (...,), "cuda", contiguous=False)
    return _moments(a.contiguous(), None if b is None else b.contiguous(), 1, group)[0]


def moments_agents(a, b=None, group=None):
    """float64 [A, 9] cuda tensor: ``moments`` of each agent's samples, the agent being the last axis of
    a (and b), e.g. [T,E,A].  ``group`` as for `moments`."""
    _, A = _agent_columns(a, "a")
    _lib.require_tensor(b, "b", torch.float32, tuple(a.shape), a.device, contiguous=False, optional=True)
    _lib.require_tensor(a, "a", torch.float32, (...,), "cuda", contiguous=False)
    return _moments(a.contiguous(), None if b is None else b.contiguous(), A, group)


def _explained_variance_1d(st):
    var_pred, vary, var_res = float(st[3]), float(st[4]), float(st[5])
    if np.isclose(vary, 0):
        return 0 if var_pred > 0 else 1
    return 1 - var_res / (vary + 1e-8)


def explained_variance(ypred, y, per_agent=False, group=None):
    """``special.explained_variance_1d`` (special.py:51-59) of baseline predictions against returns,
    over every sample of the batch; one 72-byte device->host read.  ``per_agent=True``: one value per
    agent (the last axis), over that agent's samples -- a list of A floats.  ``group`` as for `moments`."""
    if per_agent:
        return [_explained_variance_1d(st) for st in moments_agents(ypred, y, group).cpu().numpy()]
    return _explained_variance_1d(moments(ypred, y, group).cpu().numpy())


class FrameStack(object):
    """ObservationBuffer for a whole env batch: the last ``buffer_size`` observations of every
    agent stacked on a new minor axis; a reset fills every slot with the reset observation.
    ``dtype``: the observations' (torch.float32, or torch.bfloat16 for an engine built with
    ``obs_dtype=torch.bfloat16``); the stack keeps it (values are only moved)."""

    def __init__(self, n_envs, n_agents, obs_dim, buffer_size, device, dtype=torch.float32):
        if dtype not in _OBS_DTYPES:
            raise TypeError("dtype must be torch.float32 or torch.bfloat16, got %s" % dtype)
        self.shape, self.dtype = (n_envs, n_agents, obs_dim, buffer_size), dtype
        self.carry = torch.zeros(self.shape, dtype=dtype, device=device)   # __init__.py:150

    def reset(self, obs0):
        """obs0 [E,A,D] from engine.reset() -> stacked [E,A,D,B] (__init__.py:186-196)."""
        _lib.require_tensor(obs0, "obs0", self.dtype, (...,), None, contiguous=False)   # copied by torch, not the ABI
        self.carry.copy_(obs0.unsqueeze(-1).expand(self.shape))
        return self.carry.clone()

    def rollout(self, obs, done):
        """obs [T,E,A,D], done [T,E] from engine.rollout(auto_reset=True) -> [T,E,A,D,B]."""
        E, A, D, B = self.shape
        T = _lib.require_tensor(obs, "obs", self.dtype, (None, E, A, D), None, contiguous=False).shape[0]
        _lib.require_tensor(done, "done", torch.uint8, (T, E), obs.device, contiguous=False)
        _lib.require_tensor(self.carry, "FrameStack.carry", self.dtype, self.shape, "cuda")
        _lib.require_tensor(obs, "obs", self.dtype, (T, E, A, D), self.carry.device, contiguous=False)
        obs, done = obs.contiguous(), done.contiguous()
        out = torch.empty((T, E, A, D, B), dtype=self.dtype, device=obs.device)
        with torch.cuda.device(obs.device):
            _lib.check(_obs_fn("frame_stack", self.dtype)(T, E, A, D, B, _ptr(obs), _ptr(done),
                                                          _ptr(self.carry), _ptr(out), _lib.stream(obs.device)))
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
        E, A, D = self.obs_mean.shape
        x = obs.unsqueeze(0) if torch.is_tensor(obs) and obs.dim() == 3 else obs
        T = _lib.require_tensor(x, "obs", _OBS_DTYPES, (None, E, A, D), None).shape[0]
        if terminal_obs is not None:
            _lib.require_tensor(terminal_obs, "terminal_obs", x.dtype, (T, E, A, D), x.device)
            _lib.require_tensor(done, "done", torch.uint8, (T, E), x.device, contiguous=False)
        _lib.require_tensor(self.obs_mean, "Standardizer.obs_mean", torch.float64, (E, A, D), "cuda")
        _lib.require_tensor(x, "obs", x.dtype, (T, E, A, D), self.obs_mean.device)
        if terminal_obs is not None:
            with torch.cuda.device(x.device):
                _lib.check(_obs_fn("standardize_obs_terminal", x.dtype)(
                    T, E, A * D, _ptr(x), _ptr(terminal_obs), _ptr(done.contiguous()),
                    _ptr(self.obs_mean), _ptr(self.obs_var), self.obs_alpha, self.eps, _lib.stream(x.device)))
            return obs
        with torch.cuda.device(x.device):
            _lib.check(_obs_fn("standardize", x.dtype)(T, self.obs_mean.numel(), _ptr(x),
                                                       _ptr(self.obs_mean), _ptr(self.obs_var), self.obs_alpha,
                                                       self.eps, 1, 1.0, 1, _lib.stream(x.device)))
        return obs

    def rew(self, rew):
        """In place on rew [T,E,A]: optional running-std division, then scale_reward."""
        E, A = self.rew_mean.shape
        T = _lib.require_tensor(rew, "rew", torch.float32, (None, E, A), None).shape[0]
        _lib.require_tensor(self.rew_mean, "Standardizer.rew_mean", torch.float64, (E, A), "cuda")
        _lib.require_tensor(rew, "rew", torch.float32, (T, E, A), self.rew_mean.device)
        with torch.cuda.device(rew.device):
            _lib.check(_lib.lib().madrl_standardize_f32(T, self.rew_mean.numel(), _ptr(rew),
                                                        _ptr(self.rew_mean), _ptr(self.rew_var), self.rew_alpha,
                                                        self.eps, 0, float(self.scale_reward),
                                                        int(self.enable_rewnorm), _lib.stream(rew.device)))
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
        E, A = self.n_envs, self.n_agents
        T = _lib.require_tensor(rew, "rew", torch.float32, (None, E, A), None, contiguous=False).shape[0]
        _lib.require_tensor(done, "done", torch.uint8, (T, E), rew.device, contiguous=False)
        _lib.require_tensor(self.carry, "EpisodeStats.carry", torch.float64, (E, A + 3), "cuda")
        _lib.require_tensor(rew, "rew", torch.float32, (T, E, A), self.carry.device, contiguous=False)
        rew, done, dev = rew.contiguous(), done.contiguous(), rew.device
        ep_r = torch.empty((T, E, A), dtype=torch.float32, device=dev)
        ep_d = torch.empty((T, E), dtype=torch.float32, device=dev)
        ep_l = torch.empty((T, E), dtype=torch.int32, device=dev)
        ep_e = torch.empty((T, E), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            _lib.check(_lib.lib().madrl_episode_stats_f32(T, E, A, _ptr(rew), _ptr(done), float(self.discount),
                                                          int(self.max_traj_len), _ptr(self.carry), _ptr(ep_r),
                                                          _ptr(ep_d), _ptr(ep_l), _ptr(ep_e), _lib.stream(dev)))
        return dict(end=ep_e.bool(), episode_reward=ep_r, episode_avg_reward=ep_r.mean(dim=-1),
                    episode_disc_return=ep_d, episode_length=ep_l)


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
    Centralized control is the view ``obs.view(T, E, 1, A * D)``.

    Concurrent control (``n_agents=A``): one baseline per agent, as rllab's concurrent sampler keeps
    (batch_ma_sampler.py:64-188).  Agent a is fitted on its own rows (t, e, a) only; ``fit`` forms all A
    systems in one launch (``madrl_lfb_normal_eq_agents_*``) and solves them with one batched Cholesky, and
    ``predict`` evaluates agent a with coefficient row a.  The coefficients are [A, Df].

    ``shared=True`` reproduces the reference runner instead, which lists ONE baseline object A times
    (runners/rurllab.py:275-276): within one ``process_samples`` call agent a >= 1 is predicted with the
    coefficients just fitted on agent a-1's paths, agent 0 with the previous call's fit on agent A-1's paths
    (zeros before the first fit), and the object ends holding agent A-1's fit.  After ``fit`` the rows held
    are therefore ``[previous fit's row A-1 (zeros before any fit), this fit's rows 0..A-2]``; ``carry``
    is this fit's row A-1, the object's own coefficients, which the next fit gives agent 0.  Because a
    rollout's returns do not depend on the values, ``process_samples_concurrent`` fits a shared baseline
    before it predicts and still gives the reference's numbers."""

    def __init__(self, obs_dim, device, reg_coeff=1e-5, n_agents=None, shared=False):
        if shared and n_agents is None:
            raise ValueError("shared=True models one baseline object listed once per agent: it needs n_agents")
        if n_agents is not None and not (1 <= int(n_agents) <= AGENTS_MAX):
            raise ValueError("n_agents must be in [1, %d], got %r" % (AGENTS_MAX, n_agents))
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
        self.obs_dim, self.device, self.reg_coeff = int(obs_dim), device, reg_coeff
        self.n_agents = None if n_agents is None else int(n_agents)
        self.shared = bool(shared)
        self.n_features = 2 * self.obs_dim + 4
        self._coeffs = None
        self._carry = None

    # The kernels' feature map: madrl_lfb_* (rllab's); a subclass with another map names its entry points and the
    # extra arguments they take after the returns (normal equations) or t0 (predict).
    _kernels = "lfb"

    def _map_args(self):
        return ()

    def _coef_shape(self):
        return (self.n_features,) if self.n_agents is None else (self.n_agents, self.n_features)

    def _as_coeffs(self, val, name, shape):
        c = torch.as_tensor(np.asarray(val, dtype=np.float64) if not torch.is_tensor(val) else val)
        return _lib.require_tensor(c, name, torch.float64, shape, None, contiguous=False)

    def get_param_values(self):
        """float64 coefficients [Df] ([A, Df] per agent) (NumPy), or None before the first fit."""
        return None if self._coeffs is None else self._coeffs.cpu().numpy()

    def set_param_values(self, val, carry=None):
        """``carry`` [Df] (shared flavour only): the coefficients the next fit gives agent 0; None = zeros, as
        before any fit."""
        if carry is not None and not self.shared:
            raise ValueError("carry only exists for shared=True")
        if carry is not None:
            cc = self._as_coeffs(carry, "carry", (self.n_features,))
        if val is None:
            self._coeffs = None
        else:
            c = self._as_coeffs(val, "coefficients", self._coef_shape())
            self._coeffs = c.to(self.device).contiguous().clone()
        if self.shared:
            self._carry = None if carry is None else cc.to(self.device).contiguous().clone()

    @property
    def carry(self):
        """Shared flavour: the last fit's agent A-1 coefficients [Df] (NumPy), None before any fit."""
        return None if self._carry is None else self._carry.cpu().numpy()

    def _rows(self, obs, done, obs_before, t0, returns=None):
        """Validates the rollout tensors (before any pointer reaches a kernel) and runs the path plan."""
        T, E, A, D = _lib.require_tensor(obs, "obs", _OBS_DTYPES, (None, None, self.n_agents, self.obs_dim), None,
                                         contiguous=False).shape
        dev = obs.device
        _lib.require_tensor(done, "done", torch.uint8, (T, E), dev, contiguous=False)
        _lib.require_tensor(obs_before, "obs_before", obs.dtype, (E, A, D), dev, contiguous=False, optional=True)
        _lib.require_tensor(t0, "t0", torch.int32, (E,), dev, contiguous=False, optional=True)
        _lib.require_tensor(returns, "returns", torch.float32, (T, E, A), dev, contiguous=False, optional=True)
        if self.device.type != "cuda":
            raise ValueError("this baseline lives on %s: its normal equations and predictions need a CUDA device"
                             % self.device)
        _lib.require_tensor(obs, "obs", obs.dtype, (T, E, A, D), self.device, contiguous=False)
        if T * E * A >= 2 ** 31:
            raise ValueError("T*E*A must be < 2^31, got %d" % (T * E * A))
        seg_s = _paths_plan(done, A)[0]
        cont = lambda x: None if x is None else x.contiguous()          # noqa: E731
        return (T, E, A, D), cont(obs), cont(obs_before), cont(t0), seg_s

    def normal_equations(self, obs, done, returns, obs_before=None, t0=None):
        """G = [F y]ᵀ[F y], float64 [Df+1, Df+1] on the device: FᵀF, with Fᵀy as row and column Df.
        Per agent: [A, Df+1, Df+1], agent a's system from its rows only."""
        (T, E, A, D), obs, obs_before, t0, seg_s = self._rows(obs, done, obs_before, t0, returns)
        returns = returns.contiguous()
        L = _lib.lib()
        nbytes = C.c_size_t()
        per_agent = self.n_agents is not None
        if per_agent:
            _lib.check(getattr(L, "madrl_%s_agents_workspace_size" % self._kernels)(D, A, C.byref(nbytes)))
        else:
            _lib.check(getattr(L, "madrl_%s_workspace_size" % self._kernels)(D, C.byref(nbytes)))
        ws = torch.empty(nbytes.value // 8, dtype=torch.float64, device=self.device)
        Dc = self.n_features + 1
        G = torch.empty(((A,) if per_agent else ()) + (Dc, Dc), dtype=torch.float64, device=self.device)
        fn = _obs_fn(self._kernels + ("_normal_eq_agents" if per_agent else "_normal_eq"), obs.dtype)
        with torch.cuda.device(self.device):
            _lib.check(fn(T, E, A, D, _ptr(obs), _ptr(obs_before), _ptr(seg_s), _ptr(t0), _ptr(returns),
                          *self._map_args(), _ptr(G), _ptr(ws), _lib.stream(self.device)))
        return G

    def _host_lstsq(self, M, b):
        """rllab's loop (linear_feature_baseline.py:29-37) on the host."""
        Df = self.n_features
        Mn, bn, reg = M.cpu().numpy(), b.cpu().numpy(), self.reg_coeff
        for _ in range(5):
            c = np.linalg.lstsq(Mn + reg * np.identity(Df), bn, rcond=None)[0]
            if np.all(np.isfinite(c)):
                break
            reg *= 10
        return torch.from_numpy(c).to(M.device)

    def solve(self, G):
        """Coefficients from normal equations G (as `normal_equations` returns them), rllab's regularisation.
        A stack [A, Df+1, Df+1] is solved by one batched Cholesky; only the agents whose factorisation fails
        take the host loop, the others keep their Cholesky solution."""
        Df = self.n_features
        if G.dim() == 3:
            M, b = G[:, :Df, :Df], G[:, :Df, Df]
            eye = torch.eye(Df, dtype=G.dtype, device=G.device)
            Lc, info = torch.linalg.cholesky_ex(M + self.reg_coeff * eye)
            c = torch.cholesky_solve(b.unsqueeze(-1), Lc).squeeze(-1)
            ok = ((info == 0) & torch.isfinite(c).all(dim=1)).cpu()
            for a in torch.nonzero(~ok).flatten().tolist():
                c[a] = self._host_lstsq(M[a], b[a])
            return c
        M, b = G[:Df, :Df], G[:Df, Df]
        Lc, info = torch.linalg.cholesky_ex(M + self.reg_coeff * torch.eye(Df, dtype=G.dtype, device=G.device))
        if int(info) == 0:
            c = torch.cholesky_solve(b.unsqueeze(1), Lc).squeeze(1)
            if bool(torch.isfinite(c).all()):
                return c
        # the factorisation failed: rllab's loop (linear_feature_baseline.py:29-37) on the host
        return self._host_lstsq(M, b)

    def fit(self, obs, done, returns, obs_before=None, t0=None, group=None):
        """Fit to ``returns`` [T,E,A] float32 (``gae``'s second output).  With a ``torch.distributed`` group the
        normal equations (the per-agent stack) are summed over its ranks before the solve (every rank gets the
        pooled coefficients; no observation moves)."""
        G = self.normal_equations(obs, done, returns, obs_before, t0)
        if group is not None:
            import torch.distributed as dist
            dist.all_reduce(G, op=dist.ReduceOp.SUM, group=group)
        c = self.solve(G)
        if self.shared:
            prev = self._carry if self._carry is not None else torch.zeros_like(c[0])
            self._coeffs = torch.cat([prev.unsqueeze(0), c[:-1]]).contiguous()
            self._carry = c[-1].clone()
        else:
            self._coeffs = c.contiguous()

    def predict(self, obs, done, obs_before=None, t0=None):
        """values [T,E,A] float32 = features(row) . coefficients, evaluated in float64; zeros before the first fit.
        Per agent: row (t, e, a) with coefficient row a."""
        (T, E, A, D), obs, obs_before, t0, seg_s = self._rows(obs, done, obs_before, t0)
        values = torch.empty((T, E, A), dtype=torch.float32, device=self.device)
        if self._coeffs is None:
            return values.zero_()
        fn = _obs_fn(self._kernels + ("_predict" if self.n_agents is None else "_predict_agents"), obs.dtype)
        with torch.cuda.device(self.device):
            _lib.check(fn(T, E, A, D, _ptr(obs), _ptr(obs_before), _ptr(seg_s), _ptr(t0), *self._map_args(),
                          _ptr(self._coeffs), _ptr(values), _lib.stream(self.device)))
        return values


def process_samples_concurrent(baseline, obs, done, rew, discount, gae_lambda, obs_before=None, t0=None,
                               center_adv=True, positive_adv=False, group=None):
    """The non-recurrent concurrent branch of rllab's ``BatchMASampler.process_samples``
    (batch_ma_sampler.py:64-123) and its baseline fit (:184-188) over one rollout, for every agent at once.

    Per agent, in the reference's order: predict with the agent's baseline, GAE advantages and discounted
    returns per path (``gae``: paths end at ``done`` and at the end of the rollout, bootstrap 0), the explained
    variance of the predictions over the agent's samples, ``center_advantages`` / ``shift_advantages_to_positive``
    over the agent's samples, then the fit to the agent's returns.  ``baseline``: a ``LinearFeatureBaseline``
    with ``n_agents``; with ``shared=True`` the runner's single object (see the class), which is fitted first
    -- the returns do not depend on the values -- and then predicts.

    obs [T,E,A,D], done [T,E] uint8, rew [T,E,A] float32 (cuda) -> (values, advantages, returns) [T,E,A] and the
    A explained variances (a list of floats).  ``group``: a ``torch.distributed`` group whose ranks hold the env
    shards of one batch: the fit's normal equations are summed over its ranks, and the explained variances and
    the centring statistics are the whole batch's (`moments_agents` with ``group``)."""
    if not isinstance(baseline, LinearFeatureBaseline) or baseline.n_agents is None:
        raise ValueError("process_samples_concurrent needs a LinearFeatureBaseline built with n_agents")
    T, E, A, _ = _lib.require_tensor(obs, "obs", _OBS_DTYPES, (None, None, baseline.n_agents, baseline.obs_dim),
                                     None, contiguous=False).shape
    _lib.require_tensor(rew, "rew", torch.float32, (T, E, A), obs.device, contiguous=False)
    values, adv, ret, ev = _sampler_core(baseline, obs, done, rew, discount, gae_lambda, obs_before, t0, center_adv,
                                         positive_adv, True, group)
    if not baseline.shared:
        baseline.fit(obs, done, ret, obs_before, t0, group)
    return values, adv, ret, ev


def _sampler_core(baseline, obs, done, rew, discount, gae_lambda, obs_before, t0, center, positive, per_agent, group):
    """What both branches of ``process_samples`` do before the baseline fit, in the reference's order: predict, `gae`,
    the explained variance and `center_advantages` (per agent with ``per_agent``).  A shared baseline is fitted first
    (the returns do not depend on the values); the caller fits any other one last.  -> (values, adv, ret, ev)."""
    if baseline.shared:
        _, ret = gae(rew, torch.zeros_like(rew), done, discount, gae_lambda)
        baseline.fit(obs, done, ret, obs_before, t0, group)
        values = baseline.predict(obs, done, obs_before, t0)
        adv, _ = gae(rew, values, done, discount, gae_lambda)
    else:
        values = baseline.predict(obs, done, obs_before, t0)
        adv, ret = gae(rew, values, done, discount, gae_lambda)
    ev = explained_variance(values, ret, per_agent, group)
    if center or positive:
        adv = center_advantages(adv, center, positive, inplace=True, per_agent=per_agent, group=group)
    return values, adv, ret, ev


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
    over ``done`` and one HBM-bound row permutation per tensor; no host loop, and one 16-byte device->host read
    (the path count, `_PathTable`).  Tensors of 4-byte elements,
    and bfloat16 observations (2-byte rows, ``madrl_paths_pack_u16``)."""
    T, E, A = _lib.require_tensor(obs, "obs", _PACKED_DTYPES, (None, None, None, ...), None,
                                  contiguous=False).shape[:3]
    dev = obs.device
    _lib.require_tensor(actions, "actions", _PACKED_DTYPES, (T, E, A, ...), dev, contiguous=False)
    _lib.require_tensor(rew, "rew", _PACKED_DTYPES, (T, E, A), dev, contiguous=False)
    _lib.require_tensor(done, "done", torch.uint8, (T, E), dev, contiguous=False)
    for k, v in (infos or {}).items():
        _lib.require_tensor(v, "infos[%r]" % (k,), _PACKED_DTYPES, (T, E, ...), dev, contiguous=False)
    if obs_before is not None:   # taken in the observations' dtype
        obs_before = _lib.require_tensor(obs_before.to(obs.dtype).contiguous(), "obs_before", obs.dtype,
                                         tuple(obs.shape[1:]), dev)
    _lib.require_tensor(obs, "obs", obs.dtype, (T, E, A, ...), "cuda", contiguous=False)
    table = _PathTable(done, A, agent_major=False)
    env, agent, s, Ln = table.rec.long().t().contiguous()
    infos = {k: table.pack(v, per_agent=False) for k, v in (infos or {}).items()}
    return PackedPaths(observations=table.pack(obs, first=obs_before), actions=table.pack(actions),
                       rewards=table.pack(rew), env_infos=infos, offset=env * T * A + s * A + agent * Ln, length=Ln,
                       env=env, agent=agent, terminated=table.terminated, info_offset=env * T + s)


# ---------------------------------------------------------------- the recurrent branch of process_samples
# rllab pads every path of a batch to the longest one for a recurrent policy (base.py:105-161,
# tensor_utils.pad_tensor_n) and marks the real steps with ``valids``.  Here the padded tensors are written
# straight from the rollout by madrl_paths_pad_* (one pass, each output word written once, the padding included),
# from a per-path record table built on the device.

MODES = ("decentralized", "concurrent", "centralized")


def _check_mode(mode):
    if mode not in MODES:
        raise ValueError("mode must be one of %s, got %r" % (", ".join(MODES), mode))


class _PathTable(object):
    """The paths of one rollout (episodes cut at ``done`` and at the end of the rollout, `_paths_plan`) as the
    record table of madrl_paths_pad_*: int32 [P, 4] = (env, agent, start step, length).  Order (env, episode, agent),
    or agent-major (agent, env, episode) for concurrent control.  P and the longest length L come from one 16-byte
    device->host read.  ``seg_s`` / ``seg_l`` of the plan drive madrl_paths_pack_*."""

    def __init__(self, done, A, agent_major):
        T, E = done.shape
        dev = done.device
        self.seg_s, self.seg_l, n_ep, ep_rec = _paths_plan(done, A)
        n, L = (int(v) for v in torch.stack([n_ep.sum(), ep_rec[:, :, 1].max().long()]).cpu())
        live = torch.arange(T, device=dev).unsqueeze(0) < n_ep.unsqueeze(1)
        slot = torch.nonzero_static(live, size=n)                 # (env, episode) of every episode, in that order
        ep = ep_rec[slot[:, 0], slot[:, 1]]
        agents, eps = torch.arange(A, device=dev), torch.arange(n, device=dev)
        if agent_major:
            a, j = agents.repeat_interleave(n), eps.repeat(A)
        else:
            a, j = agents.repeat(n), eps.repeat_interleave(A)
        self.rec = torch.stack([slot[j, 0], a, ep[j, 0].long(), ep[j, 1].long()], dim=1).to(torch.int32).contiguous()
        self.terminated = ep[j, 2].bool()
        self.T, self.E, self.A, self.P, self.L = T, E, A, n * A, L
        self.lead = (A, n) if agent_major else (n * A,)

    def _copy(self, kind, x, per_agent, first, rows, sizes, plan):
        """madrl_paths_<kind>_u32 / _u16 (by the element size) from x [T,E,A,...] (per agent) or [T,E,...] (per env:
        each agent's path gets its env's rows) into a new [rows, ...]; ``first``: the one-step shift.  ``sizes`` and
        ``plan`` (tensors) are the entry point's own arguments after the row width and after ``first``."""
        x = x.contiguous()
        tail = tuple(x.shape[3:] if per_agent else x.shape[2:])
        out = torch.empty((rows,) + tail, dtype=x.dtype, device=x.device)
        fn = getattr(_lib.lib(), "madrl_paths_%s_%s" % (kind, "u16" if x.element_size() == 2 else "u32"))
        with torch.cuda.device(x.device):
            _lib.check(fn(self.T, self.E, self.A if per_agent else 1, max(1, int(np.prod(tail))), *sizes, _ptr(x),
                          _ptr(None if first is None else first.contiguous()), *map(_ptr, plan), _ptr(out),
                          _lib.stream(x.device)))
        return out

    def pack(self, x, per_agent=True, first=None):
        """x [T,E,A,...] (per agent) -> its rows in path order (`PackedPaths`); per env, [T,E,...] -> (env, time)
        order, since the row of (t, e) in a path starting at s is e*T + s + (t - s) = e*T + t."""
        rows = self.T * self.E * (self.A if per_agent else 1)
        return self._copy("pack", x, per_agent, first, rows, (), (self.seg_s, self.seg_l))

    def pad(self, x, per_agent=True, first=None):
        """x [T,E,A,...] (per agent) or [T,E,...] (per env) -> [*lead, L, ...], zero past each path's end."""
        out = self._copy("pad", x, per_agent, first, self.P * self.L, (self.P, self.L), (self.rec,))
        return out.view(self.lead + (self.L,) + out.shape[1:])

    def valids(self):
        """float32 [*lead, L]: 1 on a path's steps, 0 on its padding."""
        L = self.L
        v = torch.arange(L, device=self.rec.device).unsqueeze(0) < self.rec[:, 3:4]
        return v.to(torch.float32).view(self.lead + (L,))

    def sums(self, rew, ret):
        """float64 [*lead] per path: the sum of its rewards in time order and its first return."""
        rew, ret = rew.contiguous(), ret.contiguous()
        s = torch.empty(self.P, dtype=torch.float64, device=rew.device)
        f = torch.empty(self.P, dtype=torch.float64, device=rew.device)
        with torch.cuda.device(rew.device):
            _lib.check(_lib.lib().madrl_path_sums_f32(self.T, self.E, self.A, self.P, _ptr(rew), _ptr(ret),
                                                      _ptr(self.rec), _ptr(s), _ptr(f), _lib.stream(rew.device)))
        return s.view(self.lead), f.view(self.lead)

    def records(self):
        """The per-path fields of `PaddedPaths`."""
        r = self.rec.long()
        return {k: r[:, c].view(self.lead) for c, k in enumerate(("env", "agent", "start", "length"))} | \
            dict(terminated=self.terminated.view(self.lead))


class PaddedPaths(object):
    """rllab's recurrent sample batch of one rollout, resident on the device (see `pad_paths`).

    ``observations [P, L, D]``, ``actions [P, L, ...]``, ``rewards [P, L]``, ``valids [P, L]`` float32 (1 on a
    path's steps, 0 on its padding), ``env_infos[k] [P, L, ...]``, ``agent_infos[k] [P, L, ...]``, and per path
    ``env``, ``agent``, ``start``, ``length`` (int64) and ``terminated`` (bool) [P].  Concurrent control: every
    field has a leading agent axis, [A, P_a, L, ...] and [A, P_a]."""

    def __init__(self, **kw):
        self.__dict__.update(kw)


def _recurrent_inputs(mode, obs, actions, rew, done, infos, obs_before, agent_infos, obs_dtypes, rew_dtypes,
                      t0=None):
    """Checks the rollout tensors of the recurrent branch (every one before any pointer reaches the library) and
    returns them in the mode's layout: centralized control is the view of one agent whose observation, action and
    agent_infos rows are the agents' side by side, with agent 0's reward (all agents' are equal there,
    ma_sampler.py:27-29)."""
    _check_mode(mode)
    T, E, A = _lib.require_tensor(obs, "obs", obs_dtypes, (None, None, None, ...), None, contiguous=False).shape[:3]
    dev = obs.device
    _lib.require_tensor(actions, "actions", _PACKED_DTYPES, (T, E, A, ...), dev, contiguous=False)
    _lib.require_tensor(rew, "rew", rew_dtypes, (T, E, A), dev, contiguous=False)
    _lib.require_tensor(done, "done", torch.uint8, (T, E), dev, contiguous=False)
    _lib.require_tensor(obs_before, "obs_before", obs.dtype, tuple(obs.shape[1:]), dev, contiguous=False,
                        optional=True)
    _lib.require_tensor(t0, "t0", torch.int32, (E,), dev, contiguous=False, optional=True)
    infos, agent_infos = dict(infos or {}), dict(agent_infos or {})
    for k, v in infos.items():
        _lib.require_tensor(v, "infos[%r]" % (k,), _PACKED_DTYPES, (T, E, ...), dev, contiguous=False)
    for k, v in agent_infos.items():
        _lib.require_tensor(v, "agent_infos[%r]" % (k,), _PACKED_DTYPES, (T, E, A, ...), dev, contiguous=False)
    if mode == "centralized" and not torch.equal(rew, rew[..., :1].expand_as(rew)):
        raise ValueError("centralized control needs the agents' rewards equal at every step (one reward per env)")
    _lib.require_tensor(obs, "obs", obs.dtype, (T, E, A, ...), "cuda", contiguous=False)
    if T * E * A >= 2 ** 31:
        raise ValueError("T*E*A must be < 2^31, got %d" % (T * E * A))
    if mode == "centralized":
        side = lambda x: x.contiguous().view(T, E, 1, -1)             # noqa: E731
        obs, actions, rew = side(obs), side(actions), rew[..., :1]
        obs_before = None if obs_before is None else obs_before.contiguous().view(E, 1, -1)
        agent_infos = {k: side(v) for k, v in agent_infos.items()}
    return obs, actions, rew, done.contiguous(), infos, obs_before, agent_infos


def _pad_all(table, obs, actions, rew, infos, obs_before, agent_infos):
    return dict(observations=table.pad(obs, first=obs_before), actions=table.pad(actions),
                rewards=table.pad(rew), valids=table.valids(),
                env_infos={k: table.pad(v, per_agent=False) for k, v in infos.items()},
                agent_infos={k: table.pad(v) for k, v in agent_infos.items()})


def pad_paths(obs, actions, rew, done, infos=None, obs_before=None, agent_infos=None, mode="decentralized"):
    """Rollout tensors [T,E,A,...] (CUDA) -> `PaddedPaths`: rllab's recurrent batch layout (base.py:105-161), every
    path zero-padded to L = the longest path.

    Paths are cut at ``done`` and at the end of the rollout.  ``obs_before`` [E,A,...]: as in `pack_paths`, row i
    of a path is then the observation its action was taken in.  ``infos`` {k: [T,E,...]} are per env: each agent's
    path holds a copy of its env's rows, as ``dec_rollout`` gives it (ma_sampler.py:79-81).  ``agent_infos``
    {k: [T,E,A,...]}: the policy's per-agent outputs (means, log-stds), padded the same way.  Path order per
    ``mode``:

    * ``"decentralized"``  (env, episode, agent), the order of `to_paths` / `pack_paths`;
    * ``"concurrent"``     agent a's paths in (env, episode) order, under a leading agent axis [A, P_a, L, ...]
                           (all agents share the episode cuts, hence P_a and L);
    * ``"centralized"``    one path per episode of the view obs [T,E,1,A*D], actions [T,E,1,A*k] (agent_infos
                           likewise) and reward ``rew[..., 0]``; ValueError unless all agents' rewards are equal.

    Tensors of 4-byte elements, and bfloat16 (2-byte) ones.  One plan launch, one 16-byte device->host read
    (P and L), one padding launch per tensor."""
    obs, actions, rew, done, infos, obs_before, agent_infos = _recurrent_inputs(
        mode, obs, actions, rew, done, infos, obs_before, agent_infos, _PACKED_DTYPES, _PACKED_DTYPES)
    table = _PathTable(done, obs.shape[2], mode == "concurrent")
    return PaddedPaths(mode=mode, **_pad_all(table, obs, actions, rew, infos, obs_before, agent_infos),
                       **table.records())


_STAT_KEYS = ("AverageDiscountedReturn", "AverageReturn", "StdReturn", "MaxReturn", "MinReturn")


def _statistics(sums, first_ret):
    """base.py:144-147 and :170-180 over the paths of the last axis: one dict, or a list of one per row."""
    vals = torch.stack([first_ret.mean(-1), sums.mean(-1), sums.std(-1, correction=0), sums.max(-1).values,
                        sums.min(-1).values], dim=-1).cpu().numpy()
    out = [dict(zip(_STAT_KEYS, map(float, row)), NumTrajs=int(sums.shape[-1])) for row in vals.reshape(-1, 5)]
    return out if sums.dim() == 2 else out[0]


def _pooled_statistics(sums, first_ret, group):
    """`_statistics` over the paths of every rank of `group` (None: this rank's): each rank's per-path values,
    8 bytes each, gathered in rank order (`dist.pool_cat`) -- for env-contiguous shards the unsharded batch's
    path order, so the statistics are the unsharded ones bit for bit, and those of one rank its own."""
    from .dist import _pooled, pool_cat
    return _statistics(*_pooled(lambda p, g: pool_cat(torch.stack(p), g).unbind(0), (sums, first_ret), group))


def path_returns(rew, ret, done, per_agent=False):
    """Per path (episodes cut at ``done``): the undiscounted return ``sum(path["rewards"])`` (float64, in time
    order) and the first return ``path["returns"][0]`` -- float64 tensors [P] in (env, episode, agent) order, or
    [A, P_a] with ``per_agent=True`` (agent a's paths in (env, episode) order).  rew, ret [T,E,A] float32
    (``ret``: `gae`'s second output); centralized control passes ``rew[..., :1]`` and its returns."""
    T, E, A = _lib.require_tensor(rew, "rew", torch.float32, (None, None, None), None, contiguous=False).shape
    _lib.require_tensor(ret, "ret", torch.float32, (T, E, A), rew.device, contiguous=False)
    _lib.require_tensor(done, "done", torch.uint8, (T, E), rew.device, contiguous=False)
    _lib.require_tensor(rew, "rew", torch.float32, (T, E, A), "cuda", contiguous=False)
    if T * E * A >= 2 ** 31:
        raise ValueError("T*E*A must be < 2^31, got %d" % (T * E * A))
    return _PathTable(done, A, per_agent).sums(rew, ret)


def path_statistics(rew, ret, done, per_agent=False, group=None):
    """The return statistics both branches of ``process_samples`` log (base.py:144-147, :170-180):
    ``AverageDiscountedReturn`` (mean of the paths' first returns), ``AverageReturn``, ``StdReturn`` (population),
    ``MaxReturn``, ``MinReturn`` (over the paths' undiscounted returns) and ``NumTrajs``, as Python numbers in a
    dict; ``per_agent=True`` (concurrent control): a list of A dicts, agent a's over its own paths.  Arguments as
    `path_returns`.  Unlike `EpisodeStats` every path counts, including the unfinished one at the end of the
    rollout, and nothing is averaged over agents.  ``group``: a ``torch.distributed`` group whose ranks hold the env
    shards of one batch: the statistics are over the paths of every rank, the same on every rank and equal to the
    unsharded batch's (`_pooled_statistics`)."""
    return _pooled_statistics(*path_returns(rew, ret, done, per_agent), group)


def process_samples_recurrent(baseline, obs, actions, rew, done, discount, gae_lambda, mode, obs_before=None,
                              t0=None, infos=None, agent_infos=None, center_adv=True, group=None):
    """The recurrent branch of rllab's ``process_samples`` over one rollout (base.py:48-68, :105-180;
    concurrent control: once per agent, batch_ma_sampler.py:124-188), in the reference's order: baseline
    predictions, GAE advantages and discounted returns per path (`gae`), the explained variance, advantage
    centring, padding (`pad_paths`), the baseline fit.

    ``baseline``: a `LinearFeatureBaseline` -- pooled with ``obs_dim = D`` (decentralized), with ``n_agents = A``
    (concurrent; ``shared=True`` is fitted first, as in `process_samples_concurrent`), pooled with
    ``obs_dim = A*D`` (centralized).  obs [T,E,A,D] float32 or bfloat16, actions [T,E,A,...], rew [T,E,A] float32,
    done [T,E] uint8; ``obs_before``, ``t0`` as for the baseline, ``infos``, ``agent_infos`` as for `pad_paths`.
    ``group``: a ``torch.distributed`` group whose ranks hold the env shards of one batch: the baseline's normal
    equations are summed over its ranks, the explained variance and the centring use the whole batch's moments,
    and the return statistics are over every rank's paths (`path_statistics` with ``group``).  Padding stays per
    rank: each rank's batch holds its own paths.

    Two quirks of the reference are kept: the branch has no ``positive_adv`` (rllab ignores the flag there), and
    centring always divides by ``std + 1e-8``.  Centring is over every sample (per agent for concurrent control)
    and comes before the padding, so padded advantages are 0.

    Returns a dict: the ``samples_data`` keys of base.py:151-161 (``observations``, ``actions``, ``advantages``,
    ``rewards``, ``returns``, ``valids``, ``agent_infos``, ``env_infos``) padded as `pad_paths` pads them, ``paths``
    = the `PaddedPaths` of the batch (the same tensors and the per-path records), ``values`` [T,E,A] (the
    predictions), ``ExplainedVariance`` and the `path_statistics` keys.  Concurrent control: leading agent axes
    and one statistic per agent (lists of A).  The entropy term needs the policy's distribution: it stays the
    caller's, from the padded ``agent_infos`` and ``valids``."""
    _check_mode(mode)
    if not isinstance(baseline, LinearFeatureBaseline):
        raise ValueError("process_samples_recurrent needs a LinearFeatureBaseline")
    _lib.require_tensor(obs, "obs", _OBS_DTYPES, (None, None, None, None), None, contiguous=False)
    concurrent = mode == "concurrent"
    if concurrent != (baseline.n_agents is not None):
        raise ValueError("mode %r needs a LinearFeatureBaseline %s n_agents" % (mode, "with" if concurrent else
                                                                                 "without"))
    obs, actions, rew, done, infos, obs_before, agent_infos = _recurrent_inputs(
        mode, obs, actions, rew, done, infos, obs_before, agent_infos, _OBS_DTYPES, (torch.float32,), t0)
    values, adv, ret, ev = _sampler_core(baseline, obs, done, rew, discount, gae_lambda, obs_before, t0, center_adv,
                                         False, concurrent, group)
    table = _PathTable(done, obs.shape[2], concurrent)
    data = _pad_all(table, obs, actions, rew, infos, obs_before, agent_infos)
    data.update(advantages=table.pad(adv), returns=table.pad(ret))
    stats = _pooled_statistics(*table.sums(rew, ret), group)
    if not baseline.shared:
        baseline.fit(obs, done, ret, obs_before, t0, group)
    out = dict(data, paths=PaddedPaths(mode=mode, **data, **table.records()), values=values, ExplainedVariance=ev)
    if concurrent:
        out.update({k: [s[k] for s in stats] for k in _STAT_KEYS + ("NumTrajs",)})
    else:
        out.update(stats)
    return out
