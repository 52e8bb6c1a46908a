"""rltools' sample processing on the rollout tensors: what ``Sampler.process``
(rltools/rltools/samplers/__init__.py:35-88) and its baselines do between a rollout and the TRPO step, on the
device, for the three control modes of the rltools runner (runners/rurltools.py:127-191).

* ``RunningStandardizer``     ``nn.Standardizer`` (rltools/rltools/nn.py:533-592): count-weighted running mean and
                              mean square per column, in the reference's float32 / float64 arithmetic.
* ``LinearFeatureBaseline``   rltools/rltools/baselines/linear.py: features ``[obsnorm(o), i/100, (i/100)², 1]``,
                              the normal equations on the device, a Cholesky solve that raises like SciPy's.
* ``time_baseline``           the time-dependent baseline ``simplev`` (samplers/__init__.py:46-52).
* ``process_samples``         ``Sampler.process``: reward normalisation, q, ``simplev``, predictions, the two
                              explained variances, the ``v_r < 0`` fallback to ``simplev``, GAE, the fit.
* ``sample_fields``           the fields ``sample()`` logs (samplers/serial.py:36-47, :75-85, :114-130).

Paths are cut at ``done`` and at the end of the rollout, as `postproc.pack_paths` cuts them; with ``obs_before``
row t of a path is the observation its action was taken in.  Modes as in `postproc.pad_paths`: ``decentralized``
(one batch of every agent's paths, one baseline), ``concurrent`` (one batch and one independent baseline per agent:
``LinearFeatureBaseline(n_agents=A)``), ``centralized`` (the view obs [T,E,1,A*D] with agent 0's reward).
"""
import ctypes as C

import numpy as np
import torch

from . import _lib, postproc
from ._lib import _ptr
from .postproc import _OBS_DTYPES, AGENTS_MAX, _check_mode, _paths_plan


def _state_device(device):
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device() if torch.cuda.is_available() else 0)
    return device


class RunningStandardizer(object):
    """``nn.Standardizer(dim, eps)`` (rltools/rltools/nn.py:533-592): state ``count``, ``mean``, ``meansq`` in float32
    (the TensorFlow variables' dtype), initially 0, 0 and 1.  ``n_agents=A``: A independent standardisers in one
    object (concurrent control: each agent's baseline owns its obsnorm), state [A] / [A, dim].

    ``update`` takes the batch's column sums of x and x² in float64 on the device (``madrl_running_moments_*``,
    deterministic) and mixes them as the reference does: ``a = count / (count + N)`` in float32, then
    ``mean <- f32(f32(a * mean) + f32(1 - a) * sum / N)`` with the sum in float64, likewise ``meansq``.  ``stdev``
    is ``sqrt(meansq - mean² + eps)`` in float32 and ``standardize`` divides by ``f32(stdev + eps)`` in float64."""

    def __init__(self, dim, device, n_agents=None, eps=1e-6):
        if n_agents is not None and not (1 <= int(n_agents) <= AGENTS_MAX):
            raise ValueError("n_agents must be in [1, %d], got %r" % (AGENTS_MAX, n_agents))
        self.dim, self.eps, self.device = int(dim), eps, _state_device(device)
        self.n_agents = None if n_agents is None else int(n_agents)
        lead = () if self.n_agents is None else (self.n_agents,)
        self.count = torch.zeros(lead, dtype=torch.float32, device=self.device)
        self.mean = torch.zeros(lead + (self.dim,), dtype=torch.float32, device=self.device)
        self.meansq = torch.ones(lead + (self.dim,), dtype=torch.float32, device=self.device)
        self._refresh()

    def _refresh(self):
        """stdev and the kernels' obsnorm table [..., 2, D] float64 = (mean, f32(stdev + eps))."""
        eps = torch.tensor(self.eps, dtype=torch.float32, device=self.device)
        self.stdev = torch.sqrt(self.meansq - self.mean * self.mean + eps)
        self.denom = self.stdev + eps
        self.norm_table = torch.stack([self.mean.double(), self.denom.double()], dim=-2).contiguous()

    def get_param_values(self):
        """(count, mean, meansq) as float32 NumPy arrays."""
        return tuple(t.cpu().numpy() for t in (self.count, self.mean, self.meansq))

    def set_param_values(self, count, mean, meansq):
        for name, val in (("count", count), ("mean", mean), ("meansq", meansq)):
            cur = getattr(self, name)
            t = torch.as_tensor(np.asarray(val, np.float32) if not torch.is_tensor(val) else val)
            _lib.require_tensor(t, name, torch.float32, tuple(cur.shape), None, contiguous=False)
            cur.copy_(t)
        self._refresh()

    def _sums(self, x, obs_before, groups):
        """float64 [G, 2, D] column sums of x and x² over the rows of each group, and the rows per group.  x [..., D]
        with G = 1, or [..., G, D]; obs_before [E, A, D] (x [T, E, A, D]): the one-step observation shift."""
        D = self.dim
        lead = (None,) * (x.dim() - 1 if groups == 1 else x.dim() - 2)
        want = lead + ((D,) if groups == 1 else (groups, D))
        _lib.require_tensor(x, "x", _OBS_DTYPES, want, None, contiguous=False)
        if x.numel() == 0:
            raise ValueError("x must hold at least one row")
        shift = 0
        if obs_before is not None:
            if x.dim() != 4:
                raise ValueError("obs_before needs x as [T, E, A, D], got shape %s" % (tuple(x.shape),))
            _lib.require_tensor(obs_before, "obs_before", x.dtype, tuple(x.shape[1:]), x.device, contiguous=False)
            shift = x[0].numel() // D
            obs_before = obs_before.contiguous()
        if self.device.type != "cuda":
            raise ValueError("this standardiser lives on %s: its batch statistics need a CUDA device" % self.device)
        _lib.require_tensor(x, "x", x.dtype, tuple(x.shape), self.device, contiguous=False)
        x = x.contiguous()
        R = x.numel() // (D * groups)
        L = _lib.lib()
        nbytes = C.c_size_t()
        _lib.check(L.madrl_running_moments_workspace_size(groups, D, C.byref(nbytes)))
        ws = torch.empty(nbytes.value // 8, dtype=torch.float64, device=self.device)
        sums = torch.empty((groups, 2, D), dtype=torch.float64, device=self.device)
        fn = postproc._obs_fn("running_moments", x.dtype)
        with torch.cuda.device(self.device):
            _lib.check(fn(R, groups, D, shift, _ptr(x), _ptr(obs_before), _ptr(sums), _ptr(ws),
                          _lib.stream(self.device)))
        return sums, R

    def _mix(self, count, mean, meansq, sums, n):
        """nn.py:568-579 on float32 state: returns the new (count, mean, meansq)."""
        a = count / (count + n)
        b = (1.0 - a).double()
        new_mean = ((a.unsqueeze(-1) * mean).double() + b.unsqueeze(-1) * (sums[..., 0, :] / n)).float()
        new_meansq = ((a.unsqueeze(-1) * meansq).double() + b.unsqueeze(-1) * (sums[..., 1, :] / n)).float()
        return count + n, new_mean, new_meansq

    def update(self, x, obs_before=None):
        """x [..., D] (every row; [..., A, D] with n_agents: agent a's rows update standardiser a); rows of a
        rollout [T, E, A, D] with ``obs_before`` are the observations the actions were taken in."""
        groups = 1 if self.n_agents is None else self.n_agents
        sums, n = self._sums(x, obs_before, groups)
        if self.n_agents is None:
            sums = sums[0]
        self.count, self.mean, self.meansq = self._mix(self.count, self.mean, self.meansq, sums, n)
        self._refresh()

    def update_per_agent(self, x, obs_before=None):
        """One update per agent, in agent order, with agent a's rows of x [..., A, D]: rltools' concurrent optimizer
        updates its single reward normaliser this way (algos/policyopt.py:221-231).  Needs n_agents=None."""
        if self.n_agents is not None:
            raise ValueError("update_per_agent updates one standardiser A times: it needs n_agents=None")
        if x.dim() < 2 or not 1 <= x.shape[-2] <= AGENTS_MAX:
            raise ValueError("x must be [..., A, D] with A in [1, %d], got shape %s" % (AGENTS_MAX, tuple(x.shape)))
        sums, n = self._sums(x, obs_before, int(x.shape[-2]))
        count, mean, meansq = self.count, self.mean, self.meansq
        for a in range(sums.shape[0]):
            count, mean, meansq = self._mix(count, mean, meansq, sums[a], n)
        self.count, self.mean, self.meansq = count, mean, meansq
        self._refresh()

    def standardize(self, x, centered=True):
        """``(x - mean) / f32(stdev + eps)`` in float64 (``centered=False``: no mean), rounded to float32.  x float32
        or bfloat16 [..., D] ([..., A, D] with n_agents)."""
        _lib.require_tensor(x, "x", _OBS_DTYPES, (...,), self.device, contiguous=False)
        tail = (self.dim,) if self.n_agents is None else (self.n_agents, self.dim)
        if tuple(x.shape[-len(tail):]) != tail:
            raise ValueError("x must end in %s, got shape %s" % (tail, tuple(x.shape)))
        y = x.double()
        if centered:
            y = y - self.mean.double()
        return (y / self.denom.double()).float()


class LinearFeatureBaseline(postproc.LinearFeatureBaseline):
    """rltools' ``LinearFeatureBaseline`` (rltools/rltools/baselines/linear.py) over the rows of a rollout.

    Row (t, e, a), ``obs_before`` and ``t0`` as in `postproc.LinearFeatureBaseline` (t0 continues a path's time
    index across rollouts; rltools itself always starts at 0).  Features ``[obsnorm.standardize(o), i/100,
    (i/100)², 1]`` (Df = D + 3), built on the device (``madrl_lfbr_*``); ``obsnorm`` is a `RunningStandardizer`
    when ``enable_obsnorm`` (rltools updates it from the iteration-0 extra batch only, algos/policyopt.py:49-54),
    else None (``NoOpStandardizer``: the raw observations).  ``fit`` solves ``(FᵀF + reg·I) w = Fᵀq`` by a Cholesky
    factorisation on the device, batched per agent, and raises ``numpy.linalg.LinAlgError`` where one fails, as
    ``scipy.linalg.solve(..., sym_pos=True)`` does: there is no fallback.  Before the first fit the coefficients
    are zero (predictions are 0).  ``n_agents=A``: one independent baseline, and obsnorm, per agent (concurrent
    control); centralized control is the view ``obs.view(T, E, 1, A * D)`` with ``obs_dim = A * D``.

    ``get_param_values`` / ``set_param_values`` cover the coefficients and ``obsnorm``'s state (count, mean, meansq):
    ``(coefficients, obsnorm state or None)``, so a resumed run standardises as the saved one did."""

    _kernels = "lfbr"

    def __init__(self, obs_dim, device, enable_obsnorm, n_agents=None, reg_coeff=1e-5):
        super(LinearFeatureBaseline, self).__init__(obs_dim, device, reg_coeff=reg_coeff, n_agents=n_agents)
        self.n_features = self.obs_dim + 3
        self.obsnorm = RunningStandardizer(self.obs_dim, self.device, self.n_agents) if enable_obsnorm else None

    def _map_args(self):
        if self.obsnorm is None:
            return (_ptr(None),)
        shape = (2, self.obs_dim) if self.n_agents is None else (self.n_agents, 2, self.obs_dim)
        return (_ptr(_lib.require_tensor(self.obsnorm.norm_table, "obsnorm table", torch.float64, shape,
                                         self.device)),)

    def get_param_values(self):
        """(coefficients [Df] or [A, Df] float64, or None before the first fit; the obsnorm's (count, mean, meansq)
        float32 arrays, or None without an obsnorm)."""
        coef = super(LinearFeatureBaseline, self).get_param_values()
        return coef, (None if self.obsnorm is None else self.obsnorm.get_param_values())

    def set_param_values(self, val):
        """``val``: what `get_param_values` returned."""
        coef, norm = val
        if (norm is None) != (self.obsnorm is None):
            raise ValueError("the saved state %s an obsnorm, this baseline %s one" % (
                "has" if norm is not None else "has no", "has" if self.obsnorm is not None else "has no"))
        super(LinearFeatureBaseline, self).set_param_values(coef)
        if norm is not None:
            self.obsnorm.set_param_values(*norm)

    def update_obsnorm(self, obs, obs_before=None):
        """The baseline's obsnorm update from a batch's observation rows (a no-op without obsnorm)."""
        if self.obsnorm is not None:
            self.obsnorm.update(obs, obs_before)

    def solve(self, G):
        """Coefficients from normal equations G ([Df+1, Df+1] or [A, Df+1, Df+1]): one (batched) Cholesky; raises
        ``numpy.linalg.LinAlgError`` naming the agents whose matrix is not positive definite."""
        Df = self.n_features
        M, b = G[..., :Df, :Df], G[..., :Df, Df]
        Lc, info = torch.linalg.cholesky_ex(M + self.reg_coeff * torch.eye(Df, dtype=G.dtype, device=G.device))
        bad = torch.nonzero(info.reshape(-1)).flatten().tolist()
        if bad:
            raise np.linalg.LinAlgError("the regularised normal equations are not positive definite%s" % (
                "" if G.dim() == 2 else " (agents %s)" % bad))
        return torch.cholesky_solve(b.unsqueeze(-1), Lc).squeeze(-1)


def _check_rollout(q_like, name, done, t0):
    T, E, A = _lib.require_tensor(q_like, name, torch.float32, (None, None, None), None, contiguous=False).shape
    _lib.require_tensor(done, "done", torch.uint8, (T, E), q_like.device, contiguous=False)
    _lib.require_tensor(t0, "t0", torch.int32, (E,), q_like.device, contiguous=False, optional=True)
    _lib.require_tensor(q_like, name, torch.float32, (T, E, A), "cuda", contiguous=False)
    if T * E * A >= 2 ** 31:
        raise ValueError("T*E*A must be < 2^31, got %d" % (T * E * A))
    return T, E, A


def time_baseline(q, done, t0=None, per_agent=False):
    """The time-dependent baseline of ``Sampler.process`` (samplers/__init__.py:46-52): for each time index i (a
    row's position in its path, plus ``t0[e]`` on env e's first path -- the baseline's own index), the mean of q
    over the paths that reach i.  q [T,E,A] float32, done [T,E] uint8 (cuda).  Returns ``simplev`` [T,E,A] float32
    (each row's bin mean), the float64 bin sums and the int32 counts [G, L] (G = A with ``per_agent``, one set of
    bins per agent; else 1 over every agent's rows; L = the largest index + 1).  Deterministic; one 4-byte
    device->host read (L)."""
    T, E, A = _check_rollout(q, "q", done, t0)
    G = A if per_agent else 1
    if G > AGENTS_MAX:
        raise ValueError("q has %d agents, at most %d are supported" % (A, AGENTS_MAX))
    dev = q.device
    seg_s, _, n_ep, ep_rec = _paths_plan(done, A)
    last = ep_rec[:, :, 1].max()
    if t0 is not None:
        last = torch.maximum(last, (t0.to(torch.int32) + ep_rec[:, 0, 1]).max())
    L = int(last)
    if L < 1:
        raise ValueError("t0 must be >= 0")
    q, t0 = q.contiguous(), (None if t0 is None else t0.contiguous())
    nbytes = C.c_size_t()
    lib = _lib.lib()
    _lib.check(lib.madrl_time_baseline_workspace_size(G, L, C.byref(nbytes)))
    ws = torch.empty(max(1, nbytes.value), dtype=torch.uint8, device=dev)
    bin_sum = torch.empty((G, L), dtype=torch.float64, device=dev)
    bin_cnt = torch.empty((G, L), dtype=torch.int32, device=dev)
    simplev = torch.empty_like(q)
    with torch.cuda.device(dev):
        _lib.check(lib.madrl_time_baseline_f32(T, E, A, int(bool(per_agent)), L, _ptr(q), _ptr(seg_s), _ptr(n_ep),
                                               _ptr(ep_rec), _ptr(t0), _ptr(bin_sum), _ptr(bin_cnt), _ptr(simplev),
                                               _ptr(ws), _lib.stream(dev)))
    return simplev, bin_sum, bin_cnt


def _mode_view(mode, obs, done, rew, obs_before):
    """Checks the rollout tensors and returns them in the mode's layout (centralized: one agent whose observation
    row is the agents' side by side, with agent 0's reward)."""
    _check_mode(mode)
    T, E, A = _lib.require_tensor(obs, "obs", _OBS_DTYPES, (None, None, None, None), None, contiguous=False).shape[:3]
    dev = obs.device
    _lib.require_tensor(rew, "rew", torch.float32, (T, E, A), dev, contiguous=False)
    _lib.require_tensor(done, "done", torch.uint8, (T, E), dev, contiguous=False)
    _lib.require_tensor(obs_before, "obs_before", obs.dtype, tuple(obs.shape[1:]), dev, contiguous=False,
                        optional=True)
    _lib.require_tensor(obs, "obs", obs.dtype, tuple(obs.shape), "cuda", contiguous=False)
    if mode == "centralized":
        if not torch.equal(rew, rew[..., :1].expand_as(rew)):
            raise ValueError("centralized control needs the agents' rewards equal at every step (one reward per env)")
        obs = obs.contiguous().view(T, E, 1, -1)
        obs_before = None if obs_before is None else obs_before.contiguous().view(E, 1, -1)
        rew = rew[..., :1]
    return obs, done, rew.contiguous(), obs_before


def _explained(st):
    """1 - var(q - x) / (var(q) + 1e-8) from moments(q, x) (population variances; no isclose branch)."""
    return 1.0 - st[..., 5] / (st[..., 3] + 1e-8)


def process_samples(baseline, obs, done, rew, discount, gae_lambda, rewnorm=None, mode="decentralized",
                    obs_before=None, t0=None, group=None):
    """rltools' ``Sampler.process`` (samplers/__init__.py:35-88) over one rollout, in its order:

    1. ``r' = r / f32(stdev + eps)`` with ``rewnorm`` (a `RunningStandardizer(1)`; None = ``NoOpStandardizer``);
    2. q = the discounted return of r' per path (`postproc.gae`; paths end at ``done`` and the rollout's end);
    3. ``simplev`` = `time_baseline` of q (per agent in concurrent mode);
    4. v = ``baseline.predict`` (``baseline=None``: ``ZeroBaseline``, v = 0);
    5. ``tv_r`` and ``v_r`` = ``1 - var(q - x) / (var(q) + 1e-8)`` for x = simplev and x = v;
    6. if ``v_r < 0`` the values become ``simplev`` (the reference's "XXX HACK");
    7. GAE(γ, λ) with r' and the values chosen, bootstrap 0 at each path's end;
    8. ``baseline.fit`` to q (summed over a ``torch.distributed`` ``group``'s ranks if given).

    obs [T,E,A,D] float32 or bfloat16, done [T,E] uint8, rew [T,E,A] float32 (cuda); ``obs_before``, ``t0`` as for
    the baseline.  ``baseline``: `LinearFeatureBaseline` with ``obs_dim = D`` (decentralized), ``n_agents = A``
    (concurrent), ``obs_dim = A*D`` (centralized).  Returns a dict: ``advantages``, ``q`` and ``values`` (the values
    used) float32 [T,E,A] ([T,E,1] centralized), and ``v_r``, ``tv_r`` (floats), ``fallback`` (bool); in concurrent
    mode these three are lists of A, one per agent.  The statistics cost one 144-byte device->host read
    (``A * 144`` concurrent), besides `time_baseline`'s 4 bytes."""
    obs, done, rew, obs_before = _mode_view(mode, obs, done, rew, obs_before)
    per_agent = mode == "concurrent"
    if baseline is not None:
        if not isinstance(baseline, LinearFeatureBaseline):
            raise ValueError("baseline must be a rltools_sampler.LinearFeatureBaseline or None")
        if per_agent != (baseline.n_agents is not None):
            raise ValueError("mode %r needs a LinearFeatureBaseline %s n_agents" % (
                mode, "with" if per_agent else "without"))
    if rewnorm is not None and (rewnorm.dim != 1 or rewnorm.n_agents is not None):
        raise ValueError("rewnorm must be a RunningStandardizer(1) without n_agents")
    rew_n = rew if rewnorm is None else rewnorm.standardize(rew.unsqueeze(-1), centered=False).squeeze(-1)
    if baseline is None:
        values = torch.zeros_like(rew_n)
    else:
        values = baseline.predict(obs, done, obs_before, t0)
    adv, q = postproc.gae(rew_n, values, done, discount, gae_lambda)
    simplev = time_baseline(q, done, t0, per_agent)[0]
    mom = postproc.moments_agents if per_agent else postproc.moments
    st = torch.stack([mom(q, values), mom(q, simplev)]).cpu().numpy()
    v_r, tv_r = _explained(st[0]), _explained(st[1])
    fallback = v_r < 0
    if np.any(fallback):
        mask = torch.from_numpy(np.asarray(fallback).reshape(-1)).to(q.device)
        values = torch.where(mask, simplev, values) if per_agent else simplev
        adv, _ = postproc.gae(rew_n, values, done, discount, gae_lambda)
    if baseline is not None:
        baseline.fit(obs, done, q, obs_before, t0, group)
    if per_agent:
        v_r, tv_r, fallback = [float(x) for x in v_r], [float(x) for x in tv_r], [bool(x) for x in fallback]
    else:
        v_r, tv_r, fallback = float(v_r), float(tv_r), bool(fallback)
    return dict(advantages=adv, q=q, values=values, v_r=v_r, tv_r=tv_r, fallback=fallback)


def sample_fields(rew, done, mode="decentralized"):
    """The fields rltools' ``sample()`` logs (samplers/serial.py:36-47, :75-85, :114-130) from a rollout's raw
    rewards: ``ret`` (mean over paths of the undiscounted reward sums), ``batch`` (paths), ``avglen`` (int of the
    mean length), ``maxlen``, ``minlen`` and ``ravg`` (mean reward per step).  Concurrent control averages ``ret``,
    ``batch`` and ``ravg`` over the agents (their paths share the cuts, so the lengths are every agent's);
    centralized control counts one path per episode with agent 0's reward.  rew [T,E,A] float32, done [T,E] uint8."""
    _check_mode(mode)
    _check_rollout(rew, "rew", done, None)
    if mode == "centralized":
        rew = rew[..., :1].contiguous()
    per_agent = mode == "concurrent"
    table = postproc._PathTable(done, rew.shape[2], per_agent)
    sums, _ = table.sums(rew, rew)
    lens = table.rec[:, 3].view(table.lead).double()
    steps = lens.sum(-1)
    vals = torch.stack([sums.mean(-1), sums.sum(-1) / steps, lens.mean(-1), lens.max(-1).values,
                        lens.min(-1).values], dim=-1).reshape(-1, 5).cpu().numpy()
    ret, ravg, avglen, maxlen, minlen = vals.mean(0) if per_agent else vals[0]
    return dict(ret=float(ret), batch=float(sums.shape[-1]) if per_agent else int(sums.shape[-1]),
                avglen=int(avglen), maxlen=int(maxlen), minlen=int(minlen), ravg=float(ravg))
