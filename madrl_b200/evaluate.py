"""Policy evaluation over whole episodes on the device: rltools' ``evaluate_policy`` (rltools/rltools/util.py:141-231).

``evaluate_policy(engine, policy, n_trajs, discount, mode)`` evaluates a PyTorch policy through ``PolicyRollout``;
``evaluate_heuristic(engine, n_trajs, discount, mode)`` evaluates the reference's hand-written policy inside the
rollout kernels.  Both return the dict ``evaluate_policy`` returns:

* decentralized / concurrent: ``ret``, ``retstd`` and ``disc_ret`` as float64 arrays [A] (one entry per agent, as
  the reference's lists), and each info key as an [A] array of the mean per-episode info sum;
* centralized: ``ret``, ``disc_ret`` and each info key's mean as floats.

``disc_ret`` is what the reference computes: the mean of the discounted reward-to-go q_t over the episodes' rewards
zero-padded to the longest episode, ``discount(r_B_T, disc).mean()`` (util.py:228) = sum of every q_t / (B * Lmax).

Each env of the engine runs episodes back to back from ``engine.reset()``; an episode ends at ``done``, the engine's
``max_path_length`` being the reference's ``max_traj_len``.  With K = ceil(n_trajs / E) the evaluation runs
K * max_path_length steps, so every env completes at least K episodes, and the first K of env e are records
k * E + e; the statistics take records 0 .. n_trajs - 1.  The rollout runs in launches of ``chunk`` steps;
``madrl_eval_episodes_*`` folds each launch into the records on the device, and the records are read to the host
once, at the end.

With ``group`` (a ``torch.distributed`` group whose ranks each hold one shard of the env batch, built by
``dist.make_sharded``) E is the global batch: K = ceil(n_trajs / E_global), each rank records its own envs' episodes,
and the reading gathers every rank's records into the unsharded order k * E_global + global env id.  The env
kernels key their random streams by the global env id and do the same work per env whatever the shard, so the
result equals the unsharded evaluation's, on every rank.  Before any record moves, the ranks exchange their
shards and check that they tile [0, E_global) in group-rank order; otherwise every rank raises ValueError (an engine
that `make_sharded` placed with torchrun's WORLD rank and size does not tile a smaller data-parallel group: build it
with ``rank=`` and ``world=`` of the group).

Differences from the reference (DESIGN §8): exactly ``n_trajs`` episodes (its workers also
return the episodes still running when the n_trajs-th arrives); each env's first K episodes (not the first
n_trajs to finish anywhere, which over-represents short episodes); Philox streams instead of one
``np.random.seed`` per trajectory; q stays finite where discount^t underflows.
"""
import numpy as np
import torch

from . import _lib
from ._lib import _ptr

MODES = ("centralized", "decentralized", "concurrent")


def _global_envs(engine, group, same=()):
    """The envs of the whole batch: the engine's own, or with a group of several ranks the global size of the
    shards, once every rank has checked that they tile it.  The ranks exchange their (lo, hi, E_global) in one
    collective and apply the same rule to what they gathered, so they all raise or all go on.  `same`: (name, int)
    pairs that every rank must pass alike, exchanged and checked in the same collective."""
    from .dist import _world, pool_cat
    if group is None or _world(group) == 1:
        return engine.n_envs
    shard = getattr(engine, "shard", None)
    mine = (-1, -1, -1) if shard is None or int(shard[1]) - int(shard[0]) != engine.n_envs else shard
    mine = tuple(mine) + tuple(int(v) for _, v in same)
    got = pool_cat(torch.tensor(mine, dtype=torch.int64, device=engine.device).view(len(mine), 1),
                   group).cpu().numpy()
    lo, hi, size = got[:3]
    E = int(size[0])
    if not (lo[0] == 0 and (lo[1:] == hi[:-1]).all() and (hi > lo).all() and hi[-1] == E and (size == E).all()):
        raise ValueError("an evaluation over several ranks needs engines built by dist.make_sharded whose shards "
                         "tile the batch in group-rank order; got (lo, hi, n_envs_global) = %s"
                         % [tuple(int(v) for v in c) for c in zip(lo, hi, size)])
    for (name, _), v in zip(same, got[3:]):
        if (v != v[0]).any():
            raise ValueError("%s differs across the ranks: %s" % (name, [int(x) for x in v]))
    return E


def _plan(engine, n_trajs, discount, mode, chunk, group=None):
    """(max_traj_len, K) of an evaluation; raises ValueError for arguments the evaluation cannot run."""
    if mode not in MODES:
        raise ValueError("mode must be one of %s, got %r" % (", ".join(MODES), mode))
    if int(n_trajs) != n_trajs or n_trajs < 1:
        raise ValueError("n_trajs must be a positive int, got %r" % (n_trajs,))
    if not 0.0 <= float(discount) <= 1.0:
        raise ValueError("discount must be in [0, 1], got %r" % (discount,))
    if int(chunk) != chunk or chunk < 1:
        raise ValueError("chunk must be a positive int, got %r" % (chunk,))
    mpl = int(engine.cfg.max_path_length)
    if mpl < 1:
        raise ValueError("evaluation needs an engine built with max_path_length > 0 (the reference's max_traj_len)")
    return mpl, -(-int(n_trajs) // _global_envs(engine, group))


class EpisodeRecords(object):
    """The device side of one evaluation: the carry and the records of ``madrl_eval_episodes_*`` for ``engine``'s
    E envs and A agents, K episodes per env.  ``add(rew, done, info)`` after each launch of the rollout;
    ``read(n)`` copies records 0 .. n-1 to the host in one transfer -> (ret [n, A], qsum [n, A], len [n],
    info_sum [n, C])."""

    def __init__(self, engine, K, discount):
        self.E, self.A, self.K, self.discount = engine.n_envs, engine._n_acting, int(K), float(discount)
        self.C = int(np.prod(engine._info_tail))   # Pursuit's [T, E] info is one column
        self.dtype, dev = engine.dtype, engine.device
        n, A, C = self.K * self.E, self.A, self.C
        self.carry = torch.zeros((self.E, A, _lib.EVAL_CARRY_WORDS), dtype=torch.int64, device=dev)
        self.ret = torch.zeros((n, A), dtype=torch.float64, device=dev)
        self.qsum = torch.zeros((n, A), dtype=torch.float64, device=dev)
        self.info_sum = torch.zeros((n, C), dtype=torch.int64, device=dev)
        self.len = torch.zeros((n,), dtype=torch.int32, device=dev)

    def add(self, rew, done, info):
        """Fold one launch's rew [T, E, A], done [T, E] and info [T, E, *info_tail] into the records."""
        E, A, C, dev = self.E, self.A, self.C, self.carry.device
        T = _lib.require_tensor(rew, "rew", self.dtype, (None, E, A), dev).shape[0]
        _lib.require_tensor(done, "done", torch.uint8, (T, E), dev)
        _lib.require_tensor(info.view(T, E, C), "info", torch.int32, (T, E, C), dev)
        fn = _lib.lib().madrl_eval_episodes_f64 if self.dtype == torch.float64 else _lib.lib().madrl_eval_episodes_f32
        with torch.cuda.device(dev):
            _lib.check(fn(T, E, A, C, _ptr(rew), _ptr(done), _ptr(info), self.discount, self.K, _ptr(self.carry),
                          _ptr(self.ret), _ptr(self.qsum), _ptr(self.len), _ptr(self.info_sum), _lib.stream(dev)))

    def read(self, n, group=None):
        """Records 0 .. n-1.  ``group``: those of the whole batch, from every rank's records gathered in one
        exchange (`dist.pool_cat` over env-contiguous shards), in the order k * E_global + global env id."""
        from .dist import _pooled, pool_cat
        K, E, A, C = self.K, self.E, self.A, self.C
        fields = (self.ret, self.qsum, self.info_sum, self.len.view(-1, 1))
        rec = torch.cat([f.view(K, E, -1).view(torch.uint8) for f in fields], dim=2)      # [K, E, bytes per record]
        rec = _pooled(pool_cat, rec.transpose(1, 2), group).transpose(1, 2).reshape(-1, rec.shape[2])[:n]
        rec = rec.cpu().numpy()
        o1, o2, o3 = 8 * A, 16 * A, 16 * A + 8 * C
        return (rec[:, :o1].copy().view(np.float64), rec[:, o1:o2].copy().view(np.float64),
                rec[:, o3:].copy().view(np.int32)[:, 0], rec[:, o2:o3].copy().view(np.int64))


def statistics(ret, qsum, length, info_sum, mode, info_keys):
    """evaluate_policy's dict (util.py:219-231) from n episode records: ret / qsum float64 [n, A], length [n],
    info_sum [n, C] with one column per name of `info_keys`."""
    B, A = ret.shape
    lmax = int(length.max())
    infos = {k: float(np.mean(info_sum[:, c])) for c, k in enumerate(info_keys)}
    if mode == "centralized":
        # centrollout keeps one reward per step and asserts that every agent's is the same (samplers/__init__.py:115)
        if not (np.array_equal(ret, np.repeat(ret[:, :1], A, 1)) and np.array_equal(qsum, np.repeat(qsum[:, :1], A, 1))):
            raise ValueError("centralized evaluation needs the same reward for every agent (reward_mech='global')")
        return dict(ret=float(ret[:, 0].mean()), disc_ret=float(qsum[:, 0].sum() / (B * lmax)), **infos)
    return dict(ret=ret.mean(axis=0), retstd=ret.std(axis=0), disc_ret=qsum.sum(axis=0) / (B * lmax),
                **{k: np.full(A, v) for k, v in infos.items()})


def evaluate_policy(engine, policy, n_trajs, discount, mode, chunk=64, state0=None, frame_stack=1, standardizer=None,
                    graph=True, group=None):
    """rltools' evaluate_policy for a PyTorch `policy` (the ``PolicyRollout`` interface: ``policy(obs, state) ->
    (actions, extras, state)``), run as ``PolicyRollout`` launches of `chunk` steps (one more of the remaining
    steps).  `state0`: the policy's initial recurrent state (zeroed again at every episode start by the loop).
    `frame_stack` / `standardizer`: the observation wrappers of ``PolicyRollout``, started as its docstring
    describes (the reset observation updates the standardiser, then fills the stack); the standardiser's state
    is updated in place.  The rewards recorded are the ones the rollout returns (after the standardiser's reward
    side, if enabled).  The engine is reset first; it is left where the evaluation ended.  ``group``: evaluate over
    the env shards of its ranks (see the module docstring); every rank gets the whole batch's dict."""
    from .closed_loop import PolicyRollout
    from .postproc import FrameStack
    mpl, K = _plan(engine, n_trajs, discount, mode, chunk, group)
    rec = EpisodeRecords(engine, K, discount)
    steps = K * mpl
    with torch.cuda.device(engine.device):
        o = engine.reset()
        if standardizer is not None:
            standardizer.obs(o)
        obs0 = o if frame_stack == 1 else FrameStack(engine.n_envs, engine._n_acting, engine.obs_dim, frame_stack,
                                                     engine.device, engine.obs_dtype).reset(o)
        state = state0
        for T, n in ((chunk, steps // chunk), (steps % chunk, 1)):
            if T == 0 or n == 0:
                continue
            loop = PolicyRollout(engine, policy, T, record=(), graph=graph, frame_stack=frame_stack,
                                 standardizer=standardizer)
            for _ in range(n):
                r = loop(obs0, state)
                rec.add(r.rew, r.done, r.info)
                obs0, state = r.policy_obs[-1], r.state
    return statistics(*rec.read(int(n_trajs), group), mode, engine._info_keys)


def evaluate_heuristic(engine, n_trajs, discount, mode, chunk=64, norm="env", py2_division=True, group=None):
    """rltools' evaluate_policy for the reference's hand-written policy of the engine's family, evaluated inside
    the rollout kernels (``rollout_heuristic``) in launches of `chunk` steps:

    * Waterworld: `norm` "env" (the default) divides an env's actions by one norm, as rltools' decrollout calls
      heuristics/waterworld.py with the env's observations as one batch; "agent" by each pursuer's own norm.
    * Pursuit: the per-agent policy of heuristics/pursuit.py; `py2_division` as in ``rollout_heuristic``.
    * Hostage: the reference has no heuristic; raises ValueError.

    The engine is reset first; it is left where the evaluation ended.  ``group`` as for `evaluate_policy`."""
    fam = engine._abi
    if fam == "hostage":
        raise ValueError("the reference has no Hostage heuristic policy")
    if fam == "ww" and norm not in ("agent", "env"):
        raise ValueError("norm must be 'agent' or 'env', got %r" % (norm,))
    mpl, K = _plan(engine, n_trajs, discount, mode, chunk, group)
    rec = EpisodeRecords(engine, K, discount)
    steps = K * mpl
    kw = dict(norm=norm) if fam == "ww" else dict(py2_division=py2_division)
    with torch.cuda.device(engine.device):
        obs0 = engine.reset()
        bufs = engine._outputs(min(chunk, steps), None, True)
        t = 0
        while t < steps:
            T = min(chunk, steps - t)
            _, obs, rew, done, info = engine.rollout_heuristic(T, obs0, auto_reset=True, out=[b[:T] for b in bufs],
                                                               record_actions=False, **kw)
            rec.add(rew, done, info)
            obs0.copy_(obs[T - 1])
            t += T
    return statistics(*rec.read(int(n_trajs), group), mode, engine._info_keys)
