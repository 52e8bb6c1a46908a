"""Cases, a rank harness and whole-batch references for the calls that pool over the ranks of a sharded batch
(``group=``): tests/test_sharded_edges_gpu.py and tests/test_sharded_samples_gpu.py run them on the device over
gloo (every rank on one GPU) or NCCL, tests/test_emulated_pooled.py runs the split tables through the warp emulator.

Shards are explicit env ranges, not only `dist.shard_range`'s balanced ones: one-env shards, very uneven shards and
shards whose own statistics (largest time index, minimum, longest path) are far from the batch's.  The whole-batch
references are float64 NumPy (tests/postproc_edges.py, oracle/rltools_oracle.py, oracle/eval_oracle.py) or the
goldens of tests/golden/ written by the reference's own code.

``run_ranks(world, backend, fn, payload)`` spawns one process per rank; ``run_cases`` as ``fn`` runs every case of
the payload in one go, reports each case's exception instead of raising it, and returns picklable NumPy results.
"""
import datetime
import os
import socket
import time
import traceback

import numpy as np

import postproc_edges as pe
from oracle import rltools_oracle as ro

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden")

# explicit env ranges per rank: SPLITS[E][W] = shard sizes in rank order; never W > E (make_sharded refuses an
# empty shard, and so does this suite)
SPLITS = {2: {2: ((1, 1),)},
          3: {2: ((1, 2), (2, 1)), 3: ((1, 1, 1),)},
          4: {2: ((2, 2), (1, 3), (3, 1)), 3: ((1, 1, 2), (2, 1, 1)), 4: ((1, 1, 1, 1),)}}
# a collective that one rank never reaches fails the test after this long instead of stalling it
TIMEOUT_S = 120
MOM_BLOCKS = pe.csrc_default("MADRL_MOM_BLOCKS", "postproc.cu")


def bounds(sizes):
    """[(lo, hi)] of consecutive shards of the given sizes."""
    c = np.concatenate([[0], np.cumsum(sizes)]).astype(int)
    return [(int(c[r]), int(c[r + 1])) for r in range(len(sizes))]


def splits(E, W):
    return SPLITS.get(E, {}).get(W, ())


def ulps(got, want):
    """The largest distance in float32 ulps between two float32 arrays."""
    g, w = np.asarray(got, np.float32).view(np.int32), np.asarray(want, np.float32).view(np.int32)
    return int(np.max(np.abs(g.astype(np.int64) - w.astype(np.int64)))) if g.size else 0


def to_np(x):
    import torch
    if torch.is_tensor(x):
        return x.detach().cpu().numpy()
    if isinstance(x, dict):
        return {k: to_np(v) for k, v in x.items()}
    if isinstance(x, (list, tuple)):
        return type(x)(to_np(v) for v in x)
    return x


def bits_equal(a, b, path="out"):
    """The same keys, types and bytes all the way down."""
    if isinstance(a, dict):
        assert sorted(a, key=str) == sorted(b, key=str), path
        for k in a:
            bits_equal(a[k], b[k], "%s[%r]" % (path, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            bits_equal(x, y, "%s[%d]" % (path, i))
    elif isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        a, b = np.asarray(a), np.asarray(b)
        assert a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes(), path
    else:
        assert type(a) is type(b) and (a == b or (a != a and b != b)), (path, a, b)


# ---------------------------------------------------------------- rank harness

class CaseError(object):
    """A case's exception on one rank, as text (exceptions do not always pickle)."""

    def __init__(self, text):
        self.text = text

    def __repr__(self):
        return "CaseError(%s)" % self.text


def free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


class Rank(object):
    """What a case knows about its process: rank, world, device and the WORLD group."""

    def __init__(self, rank, world, dev, group):
        self.rank, self.world, self.dev, self.group = rank, world, dev, group


def _rank_main(rank, world, port, backend, fn, payload, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch
    import torch.distributed as dist
    dev = "cuda:%d" % (rank if backend == "nccl" else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world, timeout=datetime.timedelta(seconds=TIMEOUT_S))
    try:
        try:
            torch.cuda.reset_peak_memory_stats(dev)
            res = fn(Rank(rank, world, dev, dist.group.WORLD), payload)
            torch.cuda.synchronize(dev)
            res["peak_bytes"] = int(torch.cuda.max_memory_allocated(dev))
        except Exception:
            res = CaseError(traceback.format_exc())
        q.put((rank, res))
    finally:
        dist.destroy_process_group()


def run_ranks(world, backend, fn, payload, timeout=1200):
    """Spawn `world` processes (all on cuda:0 for gloo, one GPU each for NCCL), each running
    ``fn(Rank, payload) -> dict``; returns {rank: dict}.  A rank that dies without reporting fails the call; every
    child still alive when this returns or raises is killed and joined."""
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = free_port()
    procs = [ctx.Process(target=_rank_main, args=(r, world, port, backend, fn, payload, q)) for r in range(world)]
    try:
        for p in procs:
            p.start()
        got, t_end = {}, time.monotonic() + timeout
        while len(got) < world:
            try:
                r, res = q.get(timeout=5)
                got[r] = res
                continue
            except Exception:                    # queue.Empty: check that every rank still to report is alive
                pass
            dead = [r for r, p in enumerate(procs) if r not in got and p.exitcode is not None]
            if dead:
                raise RuntimeError("ranks %s exited (codes %s) without a result" % (
                    dead, [procs[r].exitcode for r in dead]))
            if time.monotonic() > t_end:
                raise RuntimeError("ranks %s did not report within %d s" % (sorted(set(range(world)) - set(got)),
                                                                             timeout))
        for p in procs:
            p.join(120)
            assert p.exitcode == 0, p.exitcode
        for r, res in got.items():
            assert not isinstance(res, CaseError), "rank %d: %s" % (r, res.text)
        return got
    finally:
        for p in procs:
            if p.is_alive():
                p.kill()
            p.join()


def run_cases(ctx, cases):
    """`run_ranks`'s fn for a list of (key, fn, args): {key: fn(ctx, *args) or CaseError}, in list order."""
    out = {}
    for key, fn, args in cases:
        try:
            out[key] = fn(ctx, *args)
        except Exception:
            out[key] = CaseError(traceback.format_exc())
    return out


def result(got, key):
    """{rank: result of case `key`}, failing with every rank's traceback if a rank's case raised."""
    res = {r: got[r][key] for r in sorted(got)}
    bad = {r: v.text for r, v in res.items() if isinstance(v, CaseError)}
    assert not bad, "case %r failed:\n%s" % (key, "\n".join("rank %d: %s" % kv for kv in bad.items()))
    return res


def cut(arrays, lo, hi):
    """Env columns [lo, hi) of rollout arrays ([T, E, ...], and [E, ...] for obs_before)."""
    return {k: (v[lo:hi] if k == "obs_before" else v[:, lo:hi]).copy() for k, v in arrays.items()}


# ---------------------------------------------------------------- policies

def rowwise(obs, W):
    """obs [..., D] @ W [D, K] as a sum over D in a fixed order: each row's result does not depend on how many rows
    the batch holds (a GEMM's may, through the algorithm the library picks for the shape), so a policy built on it
    acts on a shard's envs exactly as on the whole batch's."""
    W = W.to(obs.dtype)
    acc = obs[..., :1] * W[0]
    for d in range(1, W.shape[0]):
        acc = acc + obs[..., d:d + 1] * W[d]
    return acc


class Linear(object):
    """A fixed deterministic policy: tanh of a linear map of the observation (the same weights on every rank)."""

    def __init__(self, D, seed, device):
        import torch
        self.W = torch.randn(D, 2, generator=torch.Generator().manual_seed(seed)).to(device) * 0.1

    def __call__(self, obs, state):
        import torch
        return torch.tanh(rowwise(obs, self.W)), {}, state


class Stacked(object):
    """`Linear` over a frame stack [E, A, D, B] flattened per agent."""

    def __init__(self, D, B, seed, device):
        self.pol = Linear(D * B, seed, device)

    def __call__(self, obs, state):
        return self.pol(obs.reshape(obs.shape[0], obs.shape[1], -1), state)


class Argmax(object):
    """Pursuit's argmax of a fixed linear map of the flattened observation."""

    def __init__(self, D, seed, device):
        import torch
        self.W = torch.randn(D, 5, generator=torch.Generator().manual_seed(seed)).to(device)

    def __call__(self, obs, state):
        return rowwise(obs.reshape(obs.shape[0], obs.shape[1], -1), self.W).argmax(-1), {}, state


def map_pool():
    return np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))


# ---------------------------------------------------------------- (a) golden training loops

def replay_device(settings, rollouts, mode, dtype, dev="cuda", group=None):
    """rltools' training loop on the device over the golden's rollouts (rollout 0 is the extra batch that updates
    the baselines' obsnorm and the reward normaliser, each later one is processed, then the reward normaliser is
    updated), every call pooled over `group`.  Yields (k, process_samples result or None, baseline, rewnorm)."""
    import torch
    from madrl_b200 import rltools_sampler as rs
    pm = "decentralized" if mode == "zero" else mode
    A, D = rollouts[0]["obs"].shape[2:]
    dev = torch.device(dev)
    od = A * D if pm == "centralized" else D
    bl = None if mode == "zero" else rs.LinearFeatureBaseline(od, dev, settings["obsnorm"],
                                                              n_agents=A if pm == "concurrent" else None)
    rewnorm = rs.RunningStandardizer(1, dev) if settings["rewnorm"] else None
    for k, it in enumerate(rollouts):
        obs = torch.from_numpy(it["obs"]).to(dev, dtype)
        done = torch.from_numpy(it["done"]).to(dev)
        rew = torch.from_numpy(it["rew_cent"] if pm == "centralized" else it["rew"]).to(dev)
        ob = None if "obs_before" not in it else torch.from_numpy(it["obs_before"]).to(dev, dtype)
        out = None
        if k > 0:
            out = rs.process_samples(bl, obs, done, rew, settings["discount"], settings["gae_lambda"], rewnorm, pm,
                                     obs_before=ob, group=group)
        elif bl is not None:
            if pm == "centralized":
                bl.update_obsnorm(obs.reshape(obs.shape[0], obs.shape[1], 1, -1),
                                  None if ob is None else ob.reshape(ob.shape[0], 1, -1), group=group)
            else:
                bl.update_obsnorm(obs, ob, group=group)
        if rewnorm is not None:
            r = rew[..., :1] if pm == "centralized" else rew
            (rewnorm.update_per_agent if pm == "concurrent" else rewnorm.update)(r.unsqueeze(-1), group=group)
        yield k, out, bl, rewnorm


def rltools_golden(name):
    return ro.golden_case(np.load(os.path.join(GOLDEN, "rltools_samples_ref.npz")), name)


def rltools_loop(dev, group, case, mode, lo=None, hi=None):
    """The device training loop over the golden case's rollouts (env columns [lo, hi) if given): per rollout the
    processed outputs, the coefficients, obsnorm and rewnorm states, and sample_fields of every mode."""
    import torch
    from madrl_b200 import rltools_sampler as rs
    settings, rollouts = rltools_golden(case)
    if lo is not None:
        rollouts = [cut(it, lo, hi) for it in rollouts]
    dtype = torch.bfloat16 if case == "plain" else torch.float32
    kw = {} if group is None else dict(group=group)
    out = []
    for k, res, bl, rn in replay_device(settings, rollouts, mode, dtype, dev, group):
        rec = {}
        if res is not None:
            rec.update(q=res["q"], advantages=res["advantages"], values=res["values"], v_r=res["v_r"],
                       tv_r=res["tv_r"], fallback=res["fallback"])
        if bl is not None:
            rec["w"] = bl.get_param_values()[0]
            if bl.obsnorm is not None:
                rec["obsnorm"] = bl.obsnorm.get_param_values()
        if rn is not None:
            rec["rewnorm"] = rn.get_param_values()
        if mode == "decentralized":
            it = rollouts[k]
            rec["fields"] = {m: rs.sample_fields(torch.from_numpy(it["rew_cent"] if m == "centralized" else it["rew"])
                                                 .to(dev), torch.from_numpy(it["done"]).to(dev), m, **kw)
                             for m in ("decentralized", "concurrent", "centralized")}
        out.append(rec)
    return to_np(out)


def rank_rltools(ctx, case, sizes, mode):
    lo, hi = bounds(sizes)[ctx.rank]
    return rltools_loop(ctx.dev, ctx.group, case, mode, lo, hi)


RECURRENT_CASES = ("ragged", "bf16_int")
RECURRENT_RUNS = ("decentralized", "concurrent_independent", "concurrent_shared", "centralized")
RECURRENT_BF16 = dict(ragged=(False,), bf16_int=(False, True))
RECURRENT_STATS = ("AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "StdReturn",
                   "MaxReturn", "MinReturn")
EXACT_STATS = ("AverageReturn", "StdReturn", "MaxReturn", "MinReturn", "NumTrajs")


def recurrent_golden(case):
    """(npz, [iteration dicts], env-info key, agent-info key) of a case of recurrent_samples_ref.npz."""
    z = np.load(os.path.join(GOLDEN, "recurrent_samples_ref.npz"))
    its = []
    for n in range(2):
        pre = "%s/it%d/" % (case, n)
        its.append({k[len(pre):]: z[k] for k in z.files if k.startswith(pre) and k.count("/") == 2})
    ik = next(k.split(".")[-1] for k in z.files if k.startswith(case + "/decentralized/it0/env_infos."))
    ak = next(k.split(".")[-1] for k in z.files if k.startswith(case + "/decentralized/it0/agent_infos."))
    return z, its, ik, ak


def recurrent_loop(dev, group, case, run, bf16, lo=None, hi=None):
    """Both iterations of process_samples_recurrent with one baseline: per iteration and path list (one, or one per
    agent) the padded observations, valids, returns, advantages and the statistics, and the coefficients."""
    import torch
    from madrl_b200.postproc import LinearFeatureBaseline, process_samples_recurrent
    z, its, ik, ak = recurrent_golden(case)
    settings = z[case + "/settings"]
    mode = run.split("_")[0]
    T, E, A, D = its[0]["obs"].shape
    if mode == "concurrent":
        bl = LinearFeatureBaseline(D, dev, n_agents=A, shared=run.endswith("shared"))
    else:
        bl = LinearFeatureBaseline(A * D if mode == "centralized" else D, dev)
    kw = {} if group is None else dict(group=group)
    out = []
    for it in its:
        if lo is not None:
            it = cut(it, lo, hi)
        cuda = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)          # noqa: E731
        obs, ob = cuda(it["obs"]), (cuda(it["obs_before"]) if "obs_before" in it else None)
        if bf16:
            obs, ob = obs.bfloat16(), (None if ob is None else ob.bfloat16())
        res = process_samples_recurrent(bl, obs, cuda(it["actions"]), cuda(it["rew_cent" if mode == "centralized"
                                                                            else "rew"]),
                                        cuda(it["done"]), settings[0], settings[1], mode, obs_before=ob,
                                        infos={ik: cuda(it["info"])}, agent_infos={ak: cuda(it["agent_info"])},
                                        center_adv=bool(settings[2]), **kw)
        lists = range(A) if mode == "concurrent" else (None,)
        pick = lambda x, a: x if a is None else x[a]                                  # noqa: E731
        rec = [dict({k: pick(res[k], a).double() if k != "valids" else pick(res[k], a)
                     for k in ("observations", "valids", "returns", "advantages")},
                    stats={k: pick(res[k], a) for k in RECURRENT_STATS}) for a in lists]
        out.append(dict(lists=rec, coeffs=bl.get_param_values()))
    return to_np(out)


def rank_recurrent(ctx, case, sizes, run, bf16):
    lo, hi = bounds(sizes)[ctx.rank]
    return recurrent_loop(ctx.dev, ctx.group, case, run, bf16, lo, hi)


def concurrent_golden(case):
    """(iterations, discount, gae_lambda, center, positive) of a case of linear_baseline_concurrent_ref.npz."""
    z = np.load(os.path.join(GOLDEN, "linear_baseline_concurrent_ref.npz"))
    its = [{k: z["%s/it%d/%s" % (case, n, k)] for k in ("obs", "obs_before", "done", "rew")} for n in range(2)]
    d, gl, center, positive = z[case + "/settings"]
    return z, its, float(d), float(gl), bool(center), bool(positive)


def concurrent_loop(dev, group, case, shared, lo=None, hi=None):
    """process_samples_concurrent over both iterations: values, advantages, returns, explained variances and the
    fits of each call ([A, Df]: the held rows, or the held rows 1..A-1 plus the carried row A-1 when shared)."""
    import torch
    from madrl_b200.postproc import LinearFeatureBaseline, process_samples_concurrent
    _, its, d, gl, center, positive = concurrent_golden(case)
    A, D = its[0]["obs"].shape[2:]
    b = LinearFeatureBaseline(D, dev, n_agents=A, shared=shared)
    kw = {} if group is None else dict(group=group)
    out = []
    for it in its:
        if lo is not None:
            it = cut(it, lo, hi)
        t = {k: torch.from_numpy(v).to(dev) for k, v in it.items()}
        values, adv, ret, ev = process_samples_concurrent(b, t["obs"], t["done"], t["rew"], d, gl,
                                                          obs_before=t["obs_before"], center_adv=center,
                                                          positive_adv=positive, **kw)
        held = b.get_param_values()
        fit = np.concatenate([held[1:], b.carry[None]]) if shared else held
        out.append(dict(values=values, adv=adv, ret=ret, ev=np.array(ev), fit=fit))
    return to_np(out)


def rank_concurrent(ctx, case, sizes, shared):
    lo, hi = bounds(sizes)[ctx.rank]
    return concurrent_loop(ctx.dev, ctx.group, case, shared, lo, hi)


# ---------------------------------------------------------------- (b) synthetic whole-batch checks

S_MOM = MOM_BLOCKS * 256
# shard row counts at the moments launch's block and grid-stride edges
MOMENT_ROWS = {2: ((S_MOM, 1), (255, 3 * S_MOM + 5)),
               3: ((S_MOM - 1, 1, S_MOM + 1), (255, 3 * S_MOM + 5, 256)),
               4: ((1, S_MOM - 1, 256, S_MOM + 1), (255, 3 * S_MOM + 5, 256, 1))}
# shard means far apart: a second pass about the local means, or a local minimum, is visibly wrong; the global
# minimum lives on rank 1
SHARD_OFFSETS = (1e4, -1e4, 0.0, 3e3)


def moment_shard(rows, A, r, seed):
    """x, y [rows, A] float32 of shard r."""
    x, y = pe.agent_columns(rows, A, seed + 17 * r)
    return x + np.float32(SHARD_OFFSETS[r]), y + np.float32(SHARD_OFFSETS[r])


def moments_of(x, y):
    """moments_want per agent column: [A, 9] float64."""
    return np.stack([pe.moments_want(x[:, a], y[:, a]) for a in range(x.shape[1])])


def centred_want(x, center, positive):
    """util.center_advantages then util.shift_advantages_to_positive over x's values, in float64."""
    from oracle import postproc_oracle as po
    v = np.asarray(x, np.float64)
    if center:
        v = po.center_advantages(v)
    if positive:
        v = po.shift_advantages_to_positive(v)
    return v


def rank_moments(ctx, sizes, A, seed, centre):
    import torch
    from madrl_b200 import postproc as pp
    x, y = moment_shard(sizes[ctx.rank], A, ctx.rank, seed)
    xd, yd = torch.from_numpy(x).to(ctx.dev), torch.from_numpy(y).to(ctx.dev)
    g = ctx.group
    out = dict(ma=pp.moments_agents(xd, yd, group=g), ma_nob=pp.moments_agents(xd, group=g))
    if A == 1:
        out.update(m=pp.moments(xd, yd, group=g), m_nob=pp.moments(xd, group=g))
    if centre:
        out["ev"] = (pp.explained_variance(xd, yd, group=g), pp.explained_variance(xd, yd, per_agent=True, group=g))
        out["ca"] = {(c, p, pa): pp.center_advantages(xd, bool(c), bool(p), per_agent=pa, group=g)
                     for c, p in pe.CENTRE_MODES for pa in (False, True)}
    return to_np(out)


# the global L lands on 127, 128, 129 and 257 (off and across the 128-thread bin block) while rank 1's own L is
# small; t0 = None takes L = T from rank 0's one env, which never finishes a path
TB_LS = (127, 128, 129, 257)
TB_SIZES = {2: (1, 3), 3: (1, 1, 2), 4: (1, 1, 1, 1)}


def tb_case(sizes, A, L, with_t0, seed):
    """q [T,E,A], done [T,E], t0 [E] or None: rank 0 (one env) never done, holding the largest index; rank 1 done on
    every step; the other ranks at random."""
    rs = np.random.RandomState(seed)
    E = int(sum(sizes))
    T = 40 if with_t0 else L
    (_, h0), (lo1, hi1) = bounds(sizes)[:2]
    done = (rs.rand(T, E) < 0.2).astype(np.uint8)
    done[:, :h0] = 0
    done[:, lo1:hi1] = 1
    t0 = None
    if with_t0:
        t0 = rs.randint(0, 20, size=E).astype(np.int32)
        t0[0] = L - T
    return pe.mixed_scale(rs, T, E, A), done, t0


def rank_time_baseline(ctx, sizes, A, L, with_t0, seed):
    import torch
    from madrl_b200 import rltools_sampler as rs
    q, done, t0 = tb_case(sizes, A, L, with_t0, seed)
    lo, hi = bounds(sizes)[ctx.rank]
    c = lambda x: None if x is None else torch.from_numpy(np.ascontiguousarray(x)).to(ctx.dev)    # noqa: E731
    out = {}
    for pa in (False, True):
        out[pa] = rs.time_baseline(c(q[:, lo:hi]), c(done[:, lo:hi]), None if t0 is None else c(t0[lo:hi]), pa,
                                   group=ctx.group)
    return to_np(out)


def ps_case(E, seed):
    """A rollout for process_samples with t0: obs [T,E,A,D], obs_before, done, rew (and equal-agent rewards for
    centralized control), t0 with its largest value on env 0."""
    rs = np.random.RandomState(seed)
    T, A, D = 23, 3, 4
    obs = (rs.randn(T, E, A, D) * 2 + 0.5).astype(np.float32)
    ob = rs.randn(E, A, D).astype(np.float32)
    done = (rs.rand(T, E) < 0.15).astype(np.uint8)
    rew = (obs[..., 0] - 0.5 * obs[..., 1] + rs.randn(T, E, A)).astype(np.float32)
    t0 = rs.randint(0, 30, size=E).astype(np.int32)
    t0[0] = 77
    return dict(obs=obs, obs_before=ob, done=done, rew=rew, rew_cent=np.repeat(rew[..., :1], A, 2), t0=t0)


def process_t0_loop(dev, group, mode, E, seed, lo=None, hi=None):
    """Two process_samples calls with t0 and a fixed reward normaliser and obsnorm (the second predicts with the
    first one's pooled fit)."""
    import torch
    from madrl_b200 import rltools_sampler as rs
    it = ps_case(E, seed)
    if lo is not None:
        it = dict(cut({k: v for k, v in it.items() if k != "t0"}, lo, hi), t0=it["t0"][lo:hi])
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in it.items()}
    pm = "decentralized" if mode == "zero" else mode
    A, D = it["obs"].shape[2:]
    od = A * D if pm == "centralized" else D
    bl = None if mode == "zero" else rs.LinearFeatureBaseline(od, dev, True, n_agents=A if pm == "concurrent" else None)
    if bl is not None:
        G = A if pm == "concurrent" else None
        lead = () if G is None else (G,)
        bl.obsnorm.set_param_values(np.full(lead, 50.0), np.full(lead + (od,), 0.25), np.full(lead + (od,), 2.5))
    rn = rs.RunningStandardizer(1, dev)
    rn.set_param_values(np.float32(40), np.float32([0.1]), np.float32([3.0]))
    kw = {} if group is None else dict(group=group)
    out = []
    for _ in range(2):
        r = rs.process_samples(bl, t["obs"], t["done"], t["rew_cent" if pm == "centralized" else "rew"], 0.99, 0.97,
                               rn, pm, obs_before=t["obs_before"], t0=t["t0"], **kw)
        out.append(dict(q=r["q"], advantages=r["advantages"], values=r["values"], v_r=r["v_r"], tv_r=r["tv_r"],
                        fallback=r["fallback"], w=None if bl is None else bl.get_param_values()[0]))
    return to_np(out)


def rank_process_t0(ctx, mode, sizes, seed):
    lo, hi = bounds(sizes)[ctx.rank]
    return process_t0_loop(ctx.dev, ctx.group, mode, int(sum(sizes)), seed, lo, hi)


def std_case(E, bf16, seed):
    """Two batches of (obs [T,E,A,D], obs_before [E,A,D]) float32, bfloat16-representable with bf16."""
    rs = np.random.RandomState(seed)
    cvt = (lambda x: pe.bf16_bits(x)[1]) if bf16 else (lambda x: x)
    T, A, D = 6, 3, 5
    return [(cvt((rs.randn(T, E, A, D) * 3 + np.arange(D)).astype(np.float32)),
             cvt((rs.randn(E, A, D) * 3 - 1).astype(np.float32))) for _ in range(2)]


def std_rows(obs, ob):
    """The rows an update with obs_before sees: [T*E, A, D] float64, obs_before first, in (t, e) order."""
    seen = np.concatenate([ob[None], obs[:-1]]).astype(np.float64)
    return seen.reshape(-1, seen.shape[2], seen.shape[3])


def standardizer_states(dev, group, E, bf16, seed, lo=None, hi=None):
    """After each batch: (count, mean, meansq) of update, update with n_agents, update_per_agent and the
    baseline's update_obsnorm."""
    import torch
    from madrl_b200 import rltools_sampler as rs
    batches = std_case(E, bf16, seed)
    T, _, A, D = batches[0][0].shape
    st, sa, su = rs.RunningStandardizer(D, dev), rs.RunningStandardizer(D, dev, n_agents=A), rs.RunningStandardizer(
        D, dev)
    bl = rs.LinearFeatureBaseline(D, dev, True)
    kw = {} if group is None else dict(group=group)
    out = []
    for obs, ob in batches:
        if lo is not None:
            obs, ob = obs[:, lo:hi], ob[lo:hi]
        o = torch.from_numpy(np.ascontiguousarray(obs)).to(dev)
        b = torch.from_numpy(np.ascontiguousarray(ob)).to(dev)
        if bf16:
            o, b = o.bfloat16(), b.bfloat16()
        st.update(o, b, **kw)
        sa.update(o, b, **kw)
        su.update_per_agent(o, b, **kw)
        bl.update_obsnorm(o, b, **kw)
        out.append(dict(update=st.get_param_values(), agents=sa.get_param_values(),
                        per_agent=su.get_param_values(), obsnorm=bl.obsnorm.get_param_values()))
    return out


def rank_standardizers(ctx, sizes, bf16, seed):
    lo, hi = bounds(sizes)[ctx.rank]
    return standardizer_states(ctx.dev, ctx.group, int(sum(sizes)), bf16, seed, lo, hi)


def standardizer_want(E, bf16, seed):
    """The oracle's states after each batch, updated on the concatenated rows of the whole batch."""
    batches = std_case(E, bf16, seed)
    A, D = batches[0][0].shape[2:]
    st, su, sa = ro.Standardizer(D), ro.Standardizer(D), [ro.Standardizer(D) for _ in range(A)]
    out = []
    for obs, ob in batches:
        rows = std_rows(obs, ob)
        st.update(rows.reshape(-1, D))
        for a in range(A):
            sa[a].update(rows[:, a])
            su.update(rows[:, a])
        state = lambda s: (s.count.reshape(()), s.mean[0], s.meansq[0])                  # noqa: E731
        agents = (np.array([s.count[0] for s in sa], np.float32), np.stack([s.mean[0] for s in sa]),
                  np.stack([s.meansq[0] for s in sa]))
        out.append(dict(update=state(st), agents=agents, per_agent=state(su), obsnorm=state(st)))
    return out


def paths_case(sizes, seed):
    """rew [T,E,A], done [T,E]: rank 0's envs never done (the longest paths), the last rank's last env done on
    every step (the shortest), the others at random."""
    rs = np.random.RandomState(seed)
    T, E, A = 30, int(sum(sizes)), 3
    done = (rs.rand(T, E) < 0.15).astype(np.uint8)
    done[:, :sizes[0]] = 0
    done[:, E - 1] = 1
    return pe.mixed_scale(rs, T, E, A), done


def path_outputs(dev, group, sizes, seed, lo=None, hi=None):
    import torch
    from madrl_b200 import postproc as pp
    from madrl_b200 import rltools_sampler as rs
    rew, done = paths_case(sizes, seed)
    if lo is not None:
        rew, done = rew[:, lo:hi], done[:, lo:hi]
    r, d = (torch.from_numpy(np.ascontiguousarray(x)).to(dev) for x in (rew, done))
    kw = {} if group is None else dict(group=group)
    ret = pp.gae(r, torch.zeros_like(r), d, 0.99, 1.0)[1]
    return dict(stats=[pp.path_statistics(r, ret, d, pa, **kw) for pa in (False, True)],
                fields={m: rs.sample_fields(r, d, m, **kw) for m in ("decentralized", "concurrent", "centralized")})


def rank_paths(ctx, sizes, seed):
    lo, hi = bounds(sizes)[ctx.rank]
    return path_outputs(ctx.dev, ctx.group, sizes, seed, lo, hi)


# ---------------------------------------------------------------- (c) evaluation

def eval_golden():
    import json
    g = np.load(os.path.join(GOLDEN, "eval_ww_heuristic.npz"))
    return g, json.loads(str(g["case"]))


def rank_eval_golden(ctx, world):
    """The fp64 Waterworld heuristic golden (E = 3) from make_sharded shards over the first `world` ranks."""
    import torch
    from madrl_b200 import BatchedMAWaterWorld, evaluate_heuristic
    from madrl_b200.dist import make_sharded
    g, c = eval_golden()
    out = {}
    for chunk in (64, 17):
        eng = make_sharded(BatchedMAWaterWorld, c["E"], rank=ctx.rank, world=world, device=ctx.dev, seed=c["seed"],
                           env_id_base=c["env_id_base"], max_path_length=c["max_traj_len"], dtype=torch.float64,
                           **c["config"])
        out[chunk] = evaluate_heuristic(eng, c["n_trajs"], c["discount"], "decentralized", chunk=chunk,
                                        group=ctx.group)
    return out


EVAL_E = 7
EVAL_NTRAJS = (5, 7, 13, 14)           # fewer than E, E, one short of 2E, 2E
WW_EVAL = dict(n_pursuers=3, n_evaders=4, max_path_length=12)
EVAL_CHUNK = 5                         # does not divide max_path_length


def ww_eval_obs_dim():
    from madrl_b200 import BatchedMAWaterWorld
    return BatchedMAWaterWorld(1, device="cuda", **WW_EVAL).obs_dim


def evaluations(dev, group, rank=0, world=1):
    """evaluate_policy dicts: Waterworld over every n_trajs with and without graphs, with a frame stack and a
    standardiser, Hostage fp64 centralized and Pursuit with an argmax policy."""
    import torch
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade, evaluate_policy
    from madrl_b200.dist import make_sharded
    from madrl_b200.postproc import Standardizer
    kw = {} if group is None else dict(group=group)
    ww = lambda: make_sharded(BatchedMAWaterWorld, EVAL_E, rank=rank, world=world, device=dev, seed=8,  # noqa: E731
                              **WW_EVAL)
    D = ww().obs_dim
    pol = Linear(D, 0, dev)
    out = {}
    for n in EVAL_NTRAJS:
        for graph in (True, False):
            out["ww", n, graph] = evaluate_policy(ww(), pol, n, 0.97, "decentralized", chunk=EVAL_CHUNK, graph=graph,
                                                  **kw)
    eng = ww()
    std = Standardizer(eng.n_envs, eng._n_acting, D, dev, enable_obsnorm=True)
    out["ww_stack"] = evaluate_policy(eng, Stacked(D, 3, 2, dev), 13, 0.99, "decentralized", chunk=EVAL_CHUNK,
                                      frame_stack=3, standardizer=std, **kw)
    hw = make_sharded(BatchedHostageWorld, EVAL_E, 10, 16, 16, 4, 2, rank=rank, world=world, device=dev, seed=1,
                      max_path_length=15, dtype=torch.float64)
    out["hostage"] = evaluate_policy(hw, Linear(hw.obs_dim, 4, dev), 12, 0.99, "centralized", chunk=8, **kw)
    pe_eng = make_sharded(BatchedPursuitEvade, EVAL_E, map_pool(), rank=rank, world=world, n_evaders=30,
                          n_pursuers=8, obs_range=7, surround=True, sample_maps=True, device=dev, seed=2,
                          max_path_length=25)
    out["pursuit"] = evaluate_policy(pe_eng, Argmax(pe_eng.obs_dim, 3, dev), 13, 0.95, "decentralized", chunk=16,
                                     **kw)
    return to_np(out)


def rank_evaluations(ctx):
    return evaluations(ctx.dev, ctx.group, ctx.rank, ctx.world)


# ---------------------------------------------------------------- (d, e) groups and refusals

def refused(fn):
    """'refused' if fn() raises the shard check's ValueError, else what it returned or raised."""
    try:
        fn()
    except ValueError as ex:
        return "refused" if "make_sharded" in str(ex) else "ValueError: %s" % ex
    except Exception as ex:                             # noqa: BLE001 -- reported to the parent
        return "%s: %s" % (type(ex).__name__, ex)
    return "ran"


def refusals(dev, group, grank, gworld, rank, world):
    """Evaluations whose shards do not tile the batch: swapped shards, one rank without a shard and (with a group
    smaller than WORLD) engines placed by WORLD's rank and size."""
    from madrl_b200 import BatchedMAWaterWorld, evaluate_heuristic
    from madrl_b200.dist import make_sharded
    ww = lambda **kw: make_sharded(BatchedMAWaterWorld, 4, 5, 5, device=dev, seed=1, max_path_length=5,  # noqa: E731
                                   n_poison=10, n_sensors=30, **kw)
    ev = lambda eng: evaluate_heuristic(eng, 4, 0.99, "decentralized", group=group)    # noqa: E731
    out = dict(swapped=refused(lambda: ev(ww(rank=gworld - 1 - grank, world=gworld))))
    # one rank without a shard: only where the swapped shards were refused (on every rank alike) -- without the
    # collective check the other ranks would be left waiting in the record exchange
    out["mixed"] = "skipped" if out["swapped"] != "refused" else refused(
        lambda: ev(ww(rank=grank, world=gworld) if grank == 0 else
                   BatchedMAWaterWorld(2, 5, 5, device=dev, seed=1, max_path_length=5, n_poison=10, n_sensors=30)))
    if world > gworld:
        out["world_shards"] = refused(lambda: ev(ww(rank=rank, world=world)))
    # the group still exchanges in step after the refusals: a tiling evaluation runs
    out["after"] = to_np(ev(ww(rank=grank, world=gworld)))
    return out


def rank_refusals(ctx):
    return refusals(ctx.dev, ctx.group, ctx.rank, ctx.world, ctx.rank, ctx.world)


# the pooled entry points on one rank's shard of a heuristic Waterworld rollout

def pooled_suite(dev, group, rank=0, world=1, E_G=63, T=60, seed=3, eval_seed=8, pe_seed=6):
    """Every pooled entry point on this rank's `make_sharded` shard of one rollout (group=None, world=1: the
    unsharded batch)."""
    import torch
    from madrl_b200 import BatchedMAWaterWorld, BatchedPursuitEvade, evaluate_heuristic
    from madrl_b200 import postproc as pp
    from madrl_b200 import rltools_sampler as rs
    from madrl_b200.dist import make_sharded
    mpl, cfg = 25, dict(n_poison=10, n_sensors=30)
    kw = {} if group is None else dict(group=group)
    out = {}
    eng = make_sharded(BatchedMAWaterWorld, E_G, 5, 5, rank=rank, world=world, seed=seed, device=dev,
                       max_path_length=mpl, **cfg)
    out["lo"] = eng.shard[0]
    obs0 = eng.reset().clone()
    act, obs, rew, done, _ = eng.rollout_heuristic(T, obs0.clone(), auto_reset=True, norm="env")
    E, A = eng.n_envs, eng._n_acting
    obs, obs0 = obs.reshape(T, E, A, -1).float().contiguous(), obs0.reshape(E, A, -1).float().contiguous()
    D = obs.shape[-1]
    out["rew"], out["done"] = rew, done
    st, sa = rs.RunningStandardizer(D, dev), rs.RunningStandardizer(D, dev, n_agents=A)
    sr = rs.RunningStandardizer(1, dev)
    st.update(obs, obs0, **kw)
    sa.update(obs, obs0, **kw)
    sr.update_per_agent(rew.unsqueeze(-1), **kw)
    out["std"] = [s.get_param_values() for s in (st, sa, sr)]
    q = pp.gae(rew, torch.zeros_like(rew), done, 0.99, 1.0)[1]
    for pa in (False, True):
        out["tb", pa] = rs.time_baseline(q, done, None, pa, **kw)
    simplev = out["tb", False][0]
    out["mom"] = pp.moments(q, simplev, **kw)
    out["moma"] = pp.moments_agents(q, simplev, **kw)
    out["ev"] = (pp.explained_variance(simplev, q, **kw), pp.explained_variance(simplev, q, per_agent=True, **kw))
    out["ca"] = (pp.center_advantages(q, **kw), pp.center_advantages(q, True, True, per_agent=True, **kw))
    out["fields"] = [rs.sample_fields(rew, done, m, **kw) for m in ("decentralized", "concurrent", "centralized")]
    out["pstats"] = [pp.path_statistics(rew, q, done, pa, **kw) for pa in (False, True)]
    bl, rn = rs.LinearFeatureBaseline(D, dev, True), rs.RunningStandardizer(1, dev)
    bl.update_obsnorm(obs, obs0, **kw)
    rn.update(rew.unsqueeze(-1), **kw)
    out["ps"] = []
    for _ in range(2):
        r = rs.process_samples(bl, obs, done, rew, 0.99, 0.97, rewnorm=rn, obs_before=obs0, **kw)
        out["ps"].append((r["v_r"], r["tv_r"], r["fallback"], r["advantages"], bl.get_param_values()[0]))
    cb = pp.LinearFeatureBaseline(D, dev, n_agents=A)
    out["conc"] = [pp.process_samples_concurrent(cb, obs, done, rew, 0.99, 0.97, obs_before=obs0, **kw)
                   for _ in range(2)]
    rb = pp.LinearFeatureBaseline(D, dev)
    rec = pp.process_samples_recurrent(rb, obs, act, rew, done, 0.99, 0.97, "decentralized", obs_before=obs0, **kw)
    out["rec"] = {k: rec[k] for k in ("ExplainedVariance", "AverageReturn", "StdReturn", "MaxReturn", "MinReturn",
                                      "AverageDiscountedReturn", "NumTrajs")}
    ww = make_sharded(BatchedMAWaterWorld, E_G, 5, 5, rank=rank, world=world, seed=eval_seed, device=dev,
                      max_path_length=mpl, **cfg)
    out["eval_ww"] = evaluate_heuristic(ww, 100, 0.99, "decentralized", chunk=24, **kw)
    pe_eng = make_sharded(BatchedPursuitEvade, 21, map_pool(), rank=rank, world=world, n_evaders=30, n_pursuers=8,
                          obs_range=7, surround=True, sample_maps=True, seed=pe_seed, device=dev, max_path_length=40)
    out["eval_pe"] = evaluate_heuristic(pe_eng, 50, 0.99, "decentralized", chunk=24, py2_division=True, **kw)
    torch.cuda.synchronize(dev)
    return to_np(out)


def check_pooled(got, full, E_G=63):
    """got: {rank: pooled_suite(...)} of the ranks of one group; full: the unsharded pooled_suite.  Every pooled
    output has the same bytes on every rank and matches the unsharded call: counts, lengths, path counts, bin
    counts and the fallback exactly; float32 standardiser state and simplev within one float32 ulp; float64
    moments, explained variances and mean returns at rtol 1e-12; the baseline within 1e-9 of the unsharded fit;
    the heuristic evaluations exactly."""
    from madrl_b200.dist import shard_range
    W = len(got)
    rs_ = [got[r] for r in range(W)]
    his = [(r["lo"], r["lo"] + r["done"].shape[1]) for r in rs_]
    assert his == [shard_range(E_G, r, W) for r in range(W)]
    for r, (lo, hi) in zip(rs_, his):                       # the shards hold the unsharded batch's envs
        assert np.array_equal(r["rew"], full["rew"][:, lo:hi]) and np.array_equal(r["done"], full["done"][:, lo:hi])
    r0 = rs_[0]
    for r1 in rs_[1:]:
        for k in ("std", "mom", "moma", "ev", "fields", "pstats", "rec", "eval_ww", "eval_pe"):
            bits_equal(r0[k], r1[k], k)
        for k in (("tb", False), ("tb", True)):
            bits_equal(r0[k][1:], r1[k][1:], str(k))
        for i in range(2):
            bits_equal([x for j, x in enumerate(r0["ps"][i]) if j != 3], [x for j, x in enumerate(r1["ps"][i])
                                                                          if j != 3])
            bits_equal(r0["conc"][i][3], r1["conc"][i][3])
    for (g, w) in zip(r0["std"], full["std"]):
        assert np.array_equal(g[0], w[0]) and ulps(g[1], w[1]) <= 1 and ulps(g[2], w[2]) <= 1
    for pa in (False, True):
        s, bs, bc = full["tb", pa]
        assert np.array_equal(r0["tb", pa][2], bc)
        np.testing.assert_allclose(r0["tb", pa][1], bs, rtol=1e-12)
        for r, (lo, hi) in zip(rs_, his):
            assert ulps(r["tb", pa][0], s[:, lo:hi]) <= 1
    for k in ("mom", "moma"):     # the mean of q - simplev cancels to ~1e-10: an absolute floor at 1e-14 of the scale
        np.testing.assert_allclose(r0[k], full[k], rtol=1e-12, atol=1e-14 * np.abs(full[k]).max())
    np.testing.assert_allclose(r0["ev"][0], full["ev"][0], rtol=1e-12)
    np.testing.assert_allclose(r0["ev"][1], full["ev"][1], rtol=1e-12)
    for r, (lo, hi) in zip(rs_, his):
        for c in range(2):                   # centred values near 0 carry the means' rounding: an absolute bound
            np.testing.assert_allclose(r["ca"][c], full["ca"][c][:, lo:hi], rtol=1e-6, atol=1e-6)
    for g, w in zip(r0["fields"], full["fields"]):
        assert sorted(g) == sorted(w)
        for k in ("batch", "avglen", "maxlen", "minlen"):
            assert g[k] == w[k], k
        for k in ("ret", "ravg"):
            assert np.isclose(g[k], w[k], rtol=1e-12, atol=0), k
    for g, w in zip(r0["pstats"], full["pstats"]):
        for gd, wd in zip(g if isinstance(g, list) else [g], w if isinstance(w, list) else [w]):
            assert gd["NumTrajs"] == wd["NumTrajs"] and gd["MaxReturn"] == wd["MaxReturn"]
            assert gd["MinReturn"] == wd["MinReturn"]
            for k in ("AverageReturn", "StdReturn", "AverageDiscountedReturn"):
                assert np.isclose(gd[k], wd[k], rtol=1e-12, atol=0), k
    for i in range(2):
        v_r, tv_r, fb, _, coef = r0["ps"][i]
        wv, wtv, wfb, _, wcoef = full["ps"][i]
        assert fb == wfb
        assert np.isclose(v_r, wv, rtol=1e-12, atol=1e-12) and np.isclose(tv_r, wtv, rtol=1e-12, atol=1e-12)
        assert np.abs(coef - wcoef).max() <= 1e-9 * np.abs(wcoef).max()
        np.testing.assert_allclose(r0["conc"][i][3], full["conc"][i][3], rtol=1e-12, atol=1e-12)
    for k in ("NumTrajs", "MaxReturn", "MinReturn"):
        assert r0["rec"][k] == full["rec"][k], k
    for k in ("ExplainedVariance", "AverageReturn", "StdReturn", "AverageDiscountedReturn"):
        assert np.isclose(r0["rec"][k], full["rec"][k], rtol=1e-12, atol=0), k
    bits_equal(r0["eval_ww"], full["eval_ww"], "eval_ww")
    bits_equal(r0["eval_pe"], full["eval_pe"], "eval_pe")


SUBGROUP_SEEDS = ((11, 21, 31), (12, 22, 32))      # (rollout, Waterworld evaluation, Pursuit evaluation) per group
SUBGROUP_E = 21


def rank_subgroups(ctx):
    """Two groups of two ranks inside a four-rank world, each holding its own seeded batch (engines placed by the
    group's rank and size): the pooled suite and the refusals, per group."""
    import torch.distributed as dist
    groups = (dist.new_group([0, 1]), dist.new_group([2, 3]))
    k, grank = ctx.rank // 2, ctx.rank % 2
    seed, eval_seed, pe_seed = SUBGROUP_SEEDS[k]
    return dict(group=k, suite=pooled_suite(ctx.dev, groups[k], grank, 2, E_G=SUBGROUP_E, T=30, seed=seed,
                                            eval_seed=eval_seed, pe_seed=pe_seed),
                refusals=refusals(ctx.dev, groups[k], grank, 2, ctx.rank, ctx.world))
