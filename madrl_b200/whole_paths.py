"""rllab's sample batch of whole paths on the device: ``BatchMASampler.obtain_samples`` with ``whole_paths=True``
(rllab/sandbox/rocky/tf/samplers/batch_ma_sampler.py:40-57, ma_sampler.py:52-100, stateful_pool.py:102-190).

``WholePathSampler(engine, policy, batch_size, max_path_length)`` resets every env and runs ``PolicyRollout``
launches of ``chunk`` steps until the paths finished so far hold ``batch_size`` env-steps and every env has ended
the path it was running then (the selection rule of DESIGN §4.9).  After each launch ``madrl_whole_paths_fold``
folds its ``done`` columns into per-env records on the device, and the host reads one status word to decide whether
to launch again.  Then ``madrl_whole_paths_gather`` copies the kept rows of every launch into one flat, path-major
``WholePathBatch``: env 0's paths in order, then env 1's, and so on.

The batch is a rollout of one env with ``t0 = 0``: ``batch.as_rollout()`` gives ``(obs [N,1,A,D], done [N,1],
rew [N,1,A], obs_before [1,A,D])`` in the auto-reset convention the processing passes take, and its ``done`` carries
the batch's path table, so ``postproc.gae``, the linear baselines, ``process_samples_concurrent``,
``process_samples_recurrent`` / ``pad_paths``, ``path_statistics`` and ``rltools_sampler.process_samples`` cut its
paths from ``path_start`` with one thread per path or row (``madrl_paths_plan_flat``, ``madrl_gae_paths_f32``)
rather than walking the N rows of the view serially.  The results are the serial kernels' bit for bit.

With ``group=`` (a ``torch.distributed`` group whose ranks each hold one shard of the env batch, built by
``dist.make_sharded``) the selection is the whole batch's: each launch, ``madrl_whole_paths_steps`` writes the
rank's count increment of every step, ``dist.pool_sum`` adds them over the ranks, and
``madrl_whole_paths_fold_pooled`` advances the one count by the sums, so t* is the same on every rank and each rank
keeps exactly the rows of its envs that the unsharded selection keeps.  The ranks' batches, concatenated in
group-rank order (``path_start`` and ``env_rows`` shifted by the rows of the lower ranks), are the unsharded batch.
"""
import collections

import torch

from . import _lib
from ._lib import _ptr
from .closed_loop import PolicyRollout, _map_state
from .dist import _world, pool_min, pool_sum


class WholePathBatch(object):
    """The rows of the kept paths, env-major and path-major (N rows, P paths, A agents):

    * ``obs [N, A, W]``: the observation each action was taken in (the policy's input; with ``frame_stack`` B > 1
      the stacked one, W = D * B, the reference's ``buffer.flatten()``);
    * ``actions [N, A, ...]``, ``rew [N, A]``, ``infos [N, ...]`` (the engine's env infos), ``extras`` {k: [N, ...]}
      (the policy's agent_infos);
    * ``path_start`` int32 [P + 1]: path p is rows ``path_start[p] .. path_start[p + 1] - 1``;
    * ``done`` uint8 [N]: set on each path's last row (every path of the batch ends there);
    * ``obs_before [A, W]``: ``obs[0]``, the observation before the batch's first step;
    * ``env_rows`` int32 [E]: the first row of each env's paths; ``n_steps``: the lockstep steps the sampler ran;
      ``t_star``: the step at which the finished paths reached ``batch_size``."""

    def __init__(self, obs_store, actions, rew, infos, extras, path_start, done, env_rows, n_steps, t_star):
        self._obs_store = obs_store                  # [N + 1, A, W]: row N is zeros, so the shifted view has N rows
        self.obs, self.obs_before = obs_store[:-1], obs_store[0]
        self.actions, self.rew, self.infos, self.extras = actions, rew, infos, extras
        self.path_start, self.done, self.env_rows = path_start, done, env_rows
        self.n_steps, self.t_star = int(n_steps), int(t_star)
        self._plan = None

    def __len__(self):
        return int(self.done.shape[0])

    @property
    def n_paths(self):
        return int(self.path_start.shape[0]) - 1

    def as_rollout(self):
        """(obs [N,1,A,W], done [N,1], rew [N,1,A], obs_before [1,A,W]): the batch as an auto-reset rollout of one env
        (``obs[t]`` the observation after step t, so row t's own observation is ``obs[t-1]``, ``obs_before`` for
        t = 0).  Pass them, with ``t0=None``, to any sample-processing pass; other per-row tensors are
        ``x.unsqueeze(1)`` (actions, extras) or ``infos.unsqueeze(1)``."""
        N, A = len(self), self.rew.shape[1]
        done = self.done.view(N, 1)
        done._whole_paths = self
        return self._obs_store[1:].view(N, 1, A, -1), done, self.rew.view(N, 1, A), self._obs_store[:1]

    def owns(self, done):
        """True if `done` is this batch's [N, 1] done view."""
        return tuple(done.shape) == (len(self), 1) and done.data_ptr() == self.done.data_ptr()

    def plan(self):
        """madrl_paths_plan's outputs for the [N, 1] view, built from path_start (cached): seg_s, seg_l [N, 1],
        n_ep [1], ep_rec [1, N, 3]."""
        if self._plan is None:
            N, P, dev = len(self), self.n_paths, self.done.device
            seg_s = torch.empty((N, 1), dtype=torch.int32, device=dev)
            seg_l = torch.empty((N, 1), dtype=torch.int32, device=dev)
            n_ep = torch.empty((1,), dtype=torch.int32, device=dev)
            ep_rec = torch.zeros((1, N, 3), dtype=torch.int32, device=dev)
            with torch.cuda.device(dev):
                _lib.check(_lib.lib().madrl_paths_plan_flat(N, P, _ptr(self.path_start), _ptr(seg_s), _ptr(seg_l),
                                                            _ptr(n_ep), _ptr(ep_rec), _lib.stream(dev)))
            self._plan = (seg_s, seg_l, n_ep, ep_rec)
        return self._plan


def whole_paths_of(done):
    """The `WholePathBatch` whose ``as_rollout()`` done view `done` is, or None."""
    wp = getattr(done, "_whole_paths", None)
    return wp if wp is not None and wp.owns(done) else None


_Launch = collections.namedtuple("_Launch", "first policy_obs actions rew info extras")


class _Selection(object):
    """The device side of one batch: ``add`` folds each launch of T steps of E envs (madrl_whole_paths_fold) and
    keeps its outputs, ``batch`` gathers the kept rows (madrl_whole_paths_finish / _gather).  `max_steps`: the
    capacity of the done columns kept for the path table.  `group`: the ranks that shard the batch (None or one
    rank: this rank holds all of it); every rank must add its launches in step."""

    def __init__(self, E, T, batch_size, max_steps, device, group=None):
        self.E, self.T, self.batch_size, self.S, self.device = E, T, int(batch_size), int(max_steps), device
        self.carry = torch.tensor([-1, -1, 0], dtype=torch.int32, device=device).repeat_interleave(E)
        self.acc = torch.tensor([0, -1, 0, 0, 0], dtype=torch.int64, device=device)
        self.done_stage = torch.zeros((self.S, E), dtype=torch.uint8, device=device)
        self.launches = []
        self.status = None
        self.group = group if group is not None and _world(group) > 1 else None
        if self.group is not None:
            self.inc = torch.empty(T, dtype=torch.int64, device=device)
            self.pooled_inc = torch.zeros(T, dtype=torch.int64, device=device)

    @property
    def n_steps(self):
        return len(self.launches) * self.T

    def add(self, first, policy_obs, actions, rew, done, info, extras):
        """Fold one launch ([T, E, ...] tensors, owned by the selection from now on; `first` [E, ...]: the policy's
        input before its first step) -> True once the batch is complete.  One 40-byte device->host read; over
        several ranks, until t* is known, a sum of the T step increments over the ranks, and then the minimum of
        their finished flags, so that every rank completes at the same launch."""
        T, E, t = self.T, self.E, self.n_steps
        if t + T > self.S:
            raise RuntimeError("no whole-path batch after %d steps: the engine's paths must end within its "
                               "max_path_length" % t)
        _lib.require_tensor(done, "done", torch.uint8, (T, E), self.device)
        self.launches.append(_Launch(first, policy_obs, actions, rew, info, extras))
        self.done_stage[t:t + T].copy_(done)
        L, d = _lib.lib(), _ptr(self.done_stage[t:t + T])
        with torch.cuda.device(self.device):
            stream = _lib.stream(self.device)
            if self.group is None:
                _lib.check(L.madrl_whole_paths_fold(T, E, t, self.batch_size, d, _ptr(self.carry), _ptr(self.acc),
                                                    stream))
                self.status = self.acc.cpu()
                return bool(self.status[2])
            if self.status is None or self.status[1] < 0:      # t* not known yet: pool this launch's increments
                _lib.check(L.madrl_whole_paths_steps(T, E, t, d, _ptr(self.carry), _ptr(self.inc), stream))
                self.pooled_inc = pool_sum(self.inc, self.group)
            _lib.check(L.madrl_whole_paths_fold_pooled(T, E, t, self.batch_size, d, _ptr(self.pooled_inc),
                                                       _ptr(self.carry), _ptr(self.acc), stream))
            status = torch.cat([self.acc, pool_min(self.acc[2:3], self.group)]).cpu()
        self.status = status[:5]
        return bool(status[5])

    def batch(self):
        """The `WholePathBatch` of a complete selection."""
        E, T, dev, L = self.E, self.T, self.device, _lib.lib()
        t_star, N, P = (int(v) for v in self.status[[1, 3, 4]])
        first = self.launches[0]
        A = first.rew.shape[2]
        pobs = first.policy_obs.view(T, E, A, -1)
        if (N + 1) * A >= 2 ** 31:
            raise ValueError("the batch has %d rows of %d agents: N*A must be < 2^31" % (N, A))

        def flat(x, rows=N):
            return torch.empty((rows,) + tuple(x.shape[2:]), dtype=x.dtype, device=dev)

        env_off = torch.empty(2 * E, dtype=torch.int32, device=dev)
        path_start = torch.empty(P + 1, dtype=torch.int32, device=dev)
        done = torch.empty(N, dtype=torch.uint8, device=dev)
        obs_store = flat(pobs, N + 1)
        obs_store[N].zero_()
        out = (obs_store, flat(first.actions), flat(first.rew), flat(first.info),
               {k: flat(v) for k, v in first.extras.items()})
        with torch.cuda.device(dev):
            stream = _lib.stream(dev)
            _lib.check(L.madrl_whole_paths_finish(E, self.S, _ptr(self.done_stage), _ptr(self.carry), _ptr(env_off),
                                                  _ptr(path_start), _ptr(done), stream))
            for j, ln in enumerate(self.launches):
                srcs = [(ln.policy_obs.view(T, E, A, -1), ln.first, obs_store), (ln.actions, None, out[1]),
                        (ln.rew, None, out[2]), (ln.info, None, out[3])]
                srcs += [(v, None, out[4][k]) for k, v in ln.extras.items()]
                for src, fst, dst in srcs:
                    _lib.require_tensor(src, "launch tensor", dst.dtype, (T, E) + tuple(dst.shape[1:]), dev)
                    slab = src[0, 0].numel() * src.element_size()
                    _lib.check(L.madrl_whole_paths_gather(T, E, slab, j * T, _ptr(src), _ptr(fst), _ptr(self.carry),
                                                          _ptr(env_off), _ptr(dst), stream))
        return WholePathBatch(obs_store, out[1], out[2], out[3], out[4], path_start, done, env_off[:E],
                              self.n_steps, t_star)


class WholePathSampler(object):
    """rllab's whole-path batch (DESIGN §4.9) of `engine` driven by `policy` (the ``PolicyRollout`` interface).

    ``max_path_length`` must be the engine's (its horizon cut ends the paths).  The sampler runs ``PolicyRollout``
    launches of ``chunk`` steps with ``auto_reset=True``; ``frame_stack`` / ``standardizer`` are its observation
    wrappers, started as ``evaluate_policy`` starts them.  E, the engine's env count, should be on the order of
    ``batch_size / mean path length``: the batch overshoots ``batch_size`` by up to E unfinished paths, and fewer
    envs mean more lockstep steps.

    ``sampler(state0=None)`` resets the engine (and zeroes a copy of the recurrent state `state0`, whose shapes it
    takes) and returns a `WholePathBatch`.  Each launch's outputs are copied aside before the next launch overwrites
    them, so the memory held is about twice the rows the sampler ran.

    ``group``: a ``torch.distributed`` group whose ranks each hold one shard of the env batch (engines built by
    ``dist.make_sharded`` with the group's rank and size).  The selection is then the whole batch's: one count of
    finished env-steps over every rank's envs, one t* and one number of launches on every rank.  Each rank returns
    its own envs' rows; concatenated in group-rank order, with ``path_start`` and ``env_rows`` shifted by the rows
    of the lower ranks, they are the batch an unsharded sampler returns on the same envs.  Every rank must call the
    sampler together.  At construction the ranks check, in one collective, that their shards tile the batch in
    group-rank order and that they pass the same ``batch_size``, ``max_path_length`` and ``chunk``; otherwise every
    rank raises ValueError.  ``group=None`` or a one-rank group: this rank holds the whole batch."""

    def __init__(self, engine, policy, batch_size, max_path_length, chunk=64, frame_stack=1, standardizer=None,
                 graph=True, group=None):
        if int(batch_size) != batch_size or batch_size < 1:
            raise ValueError("batch_size must be a positive int, got %r" % (batch_size,))
        if int(chunk) != chunk or chunk < 1:
            raise ValueError("chunk must be a positive int, got %r" % (chunk,))
        mpl = int(engine.cfg.max_path_length)
        if int(max_path_length) != mpl or mpl < 1:
            raise ValueError("max_path_length (%r) must equal the engine's, which must be > 0 (got %d): the engine's "
                             "horizon cut ends the paths" % (max_path_length, mpl))
        self.engine, self.policy, self.group = engine, policy, group
        self.batch_size, self.max_path_length, self.chunk = int(batch_size), mpl, int(chunk)
        from .evaluate import _global_envs
        self.n_envs_global = _global_envs(engine, group, (("batch_size", self.batch_size),
                                                          ("max_path_length", mpl), ("chunk", self.chunk)))
        self.frame_stack, self.standardizer = frame_stack, standardizer
        self.loop = PolicyRollout(engine, policy, self.chunk, auto_reset=True, graph=graph, frame_stack=frame_stack,
                                  standardizer=standardizer)

    def max_steps(self):
        """The most lockstep steps a call can run: every path ends within max_path_length steps, so the finished
        paths reach batch_size by step ceil(batch_size / E) + max_path_length - 1, and the paths running then end
        within max_path_length more; rounded up to whole launches.  E is the whole batch's env count, so every
        rank of a group has the same capacity."""
        E = getattr(self, "n_envs_global", self.engine.n_envs)
        mpl, T = self.max_path_length, self.chunk
        steps = -(-self.batch_size // E) + 2 * mpl
        return -(-steps // T) * T

    def _first_obs(self):
        from .postproc import FrameStack
        eng = self.engine
        o = eng.reset()
        if self.standardizer is not None:
            self.standardizer.obs(o)
        if self.frame_stack == 1:
            return o
        return FrameStack(eng.n_envs, eng._n_acting, eng.obs_dim, self.frame_stack, eng.device,
                          eng.obs_dtype).reset(o)

    def __call__(self, state0=None):
        eng = self.engine
        with torch.cuda.device(eng.device):
            sel = _Selection(eng.n_envs, self.chunk, self.batch_size, self.max_steps(), eng.device, self.group)
            obs0 = self._first_obs()
            state = _map_state(torch.zeros_like, state0)
            while True:
                r = self.loop(obs0, state)
                pobs = r.policy_obs.clone()
                if sel.add(obs0, pobs, r.actions.clone(), r.rew.clone(), r.done, r.info.clone(),
                           {k: v.clone() for k, v in r.extras.items()}):
                    return sel.batch()
                obs0, state = pobs[-1], r.state
