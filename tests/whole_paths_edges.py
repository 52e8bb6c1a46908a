"""Cases and checks shared by the edge tests of whole-path sampling (madrl_b200/whole_paths.py, the
madrl_whole_paths_* and flat-batch kernels of csrc/postproc.cu): tests/test_emulated_whole_paths.py runs the small
cases in the warp emulator of tests/emu, tests/test_whole_paths_edges_gpu.py runs all of them on the device.

* `STREAMS`: scripted done streams from reset, each with a batch_size, a launch length T and the reason it is in the
  table: env counts at the fold's and scan's 256-env strides and the rows kernel's 128-thread blocks, where t* lands
  in its launch, where batch_size stands against the running count, length-1 paths at t*, an env that ends a launch
  after every other, launches in which some envs keep no rows.
* `worst_case`: the stream that needs the most steps `WholePathSampler.max_steps()` allows for.
* `GATHER_TENSORS`: slab shapes that reach each of the gather's 8 (word size, thread or warp per slab) cells, and
  `first` tensors whose alignment is worse than the source's.
* `PLAN_CASES`: path tables for madrl_paths_plan_flat and madrl_gae_paths_f32, checked against the serial kernels
  and a float64 per-path GAE."""
import collections
from types import SimpleNamespace

import numpy as np

import postproc_edges as pe
from oracle import whole_paths_oracle as wo

FOLD_THREADS, ROWS_THREADS = 256, 128     # whole_paths_fold / _scan CTA, whole_paths_rows blocks (csrc/postproc.cu)
EMU_MAX_E = 513                           # the emulator runs the streams up to this many envs

Stream = collections.namedtuple("Stream", "name why done batch_size T")


def ragged(seed, S, E, mpl, p_end):
    """A done stream from reset [S, E]: each env's paths end at random (probability p_end per step) or at mpl."""
    r = np.random.RandomState(seed).rand(S, E) < p_end
    done, n = np.zeros((S, E), np.uint8), np.zeros(E, np.int64)
    for t in range(S):
        n += 1
        d = r[t] | (n == mpl)
        done[t], n[d] = d, 0
    return done


def counts(done):
    """The finished env-steps after each step (the fold's running count)."""
    done = np.asarray(done).astype(bool)
    last, c, out = np.full(done.shape[1], -1, np.int64), 0, []
    for t in range(done.shape[0]):
        c += int(np.sum(t - last[done[t]]))
        last[done[t]] = t
        out.append(c)
    return np.array(out, np.int64)


def _placed(done, pred, Ts=range(2, 13)):
    """(batch_size, T) with the selection of `done` satisfying pred(t_star, end, T): batch_size one of the running
    counts (the threshold crossed at a path end) or one more."""
    c = counts(done)
    for bs in sorted(set(c[c > 0]) | set(c[c > 0] + 1)):
        sel = wo.select(done, bs)
        if sel is None:
            continue
        for T in Ts:
            if pred(sel[0], sel[1], T):
                return int(bs), T
    raise AssertionError("no batch_size / T places t* as asked")


def _streams():
    out = []
    # env counts: either side of the fold's and scan's 256-env strides and the rows kernel's 128-thread blocks;
    # E = 300 gives each scan thread two envs and leaves the last threads none
    for E in (1, 31, 33, 127, 128, 129, 255, 256, 257, 300, 511, 513, 4096, 4097):
        done = ragged(E, 40, E, 9, 0.2)
        out.append(Stream("E%d" % E, "env count at a thread-stride or block edge", done, 3 * E + 1, 7))
    base = ragged(101, 60, 5, 9, 0.2)
    # where t* lands in its launch
    bs, T = _placed(base, lambda ts, end, T: ts > 0 and ts % T == 0)
    out.append(Stream("tstar_first", "t* on the first step of a launch", base, bs, T))
    bs, T = _placed(base, lambda ts, end, T: ts % T == T - 1)
    out.append(Stream("tstar_last", "t* on the last step of a launch", base, bs, T))
    bs, T = _placed(base, lambda ts, end, T: 0 < ts % T < T - 1 and (end // T == ts // T).all())
    out.append(Stream("tstar_mid_closing", "t* mid-launch, every open path ends in that launch", base, bs, T))
    bs, T = _placed(base, lambda ts, end, T: end.max() // T - ts // T >= 2 and ts % T not in (0, T - 1))
    out.append(Stream("open_two_launches", "open paths end two or more launches after t*", base, bs, T))
    # where batch_size stands against the count
    c = counts(base)
    k = int(np.nonzero(base.any(1))[0][3])                       # a step at which some path ends
    out.append(Stream("bs_1", "batch_size 1: the first path end completes it", base, 1, 4))
    out.append(Stream("bs_exact", "batch_size the count at a path end", base, int(c[k]), 5))
    out.append(Stream("bs_exact_plus_1", "batch_size one more than the count at a path end", base, int(c[k]) + 1, 5))
    whole = base.copy()
    whole[-1] = 1
    out.append(Stream("bs_whole_stream", "batch_size the whole stream's count at its last done", whole,
                      int(counts(whole)[-1]), 6))
    # length-1 paths ending at t*
    ones = base.copy()
    t0 = 20
    ones[t0 - 1, :3] = ones[t0, :3] = 1
    out.append(Stream("len1_at_tstar", "paths of length 1 ending at t*", ones, int(counts(ones)[t0]), 3))
    # one env ends its last path mpl - 1 steps after t*, a launch after every other env; launches in which the
    # other envs keep no rows
    mpl, E = 9, 6
    late = np.zeros((40, E), np.uint8)
    late[:, :E - 1] = ragged(7, 40, E - 1, 3, 0.0)
    ts = 17
    late[ts - 1, E - 1] = late[ts - 1 - mpl, E - 1] = late[ts - 1 + mpl, E - 1] = 1
    bs = int(counts(late)[ts - 1]) + 1
    out.append(Stream("late_env", "one env ends at t* + mpl - 1, launches after the others", late, bs, 2))
    return out


STREAMS = _streams()


def selection(s):
    """(t_star, end) of a stream."""
    sel = wo.select(s.done, s.batch_size)
    assert sel is not None, s.name
    return sel


def launches(s):
    """The launches a stream's selection folds before it completes."""
    t_star, end = selection(s)
    return int(end.max()) // s.T + 1


def check_table():
    """The table reaches what its reasons say."""
    by = {s.name: s for s in STREAMS}
    for s in STREAMS:
        t_star, end = selection(s)
        assert wo.select(s.done[:t_star], s.batch_size) is None
    for name, pred in (("tstar_first", lambda ts, end, T: ts % T == 0),
                       ("tstar_last", lambda ts, end, T: ts % T == T - 1),
                       ("open_two_launches", lambda ts, end, T: end.max() // T - ts // T >= 2)):
        assert pred(*selection(by[name]), by[name].T), name
    ts, end = selection(by["len1_at_tstar"])
    assert (by["len1_at_tstar"].done[ts - 1:ts + 1, :3] == 1).all() and (end[:3] == ts).all()
    ts, end = selection(by["late_env"])
    T = by["late_env"].T
    assert end[-1] == ts + 8 and end[-1] // T > end[:-1].max() // T + 1      # envs 0..4 keep no rows at the end
    ts, end = selection(by["bs_whole_stream"])
    assert ts == by["bs_whole_stream"].done.shape[0] - 1 and (end == ts).all()
    assert selection(by["bs_1"])[0] == int(np.nonzero(by["bs_1"].done.any(1))[0][0])
    s = by["bs_exact"]
    assert s.done[selection(s)[0]].any() and counts(s.done)[selection(s)[0]] == s.batch_size


def max_steps(E, mpl, T, batch_size):
    """`WholePathSampler.max_steps()` of a sampler of E envs (the method itself, not a copy of its formula)."""
    from madrl_b200.whole_paths import WholePathSampler
    return WholePathSampler.max_steps(SimpleNamespace(engine=SimpleNamespace(n_envs=E), max_path_length=mpl,
                                                      chunk=T, batch_size=batch_size))


def worst_case(E=5, mpl=7, t_star=30, T=1):
    """(done, batch_size, capacity, tight, over) of the stream that needs the most steps with no path longer than
    mpl: every env but the last has run full-length paths and ends one at t*, the last env started a path at t*
    that runs mpl steps, and the count before t* is as small as those paths allow.  capacity = max_steps() for its
    E, mpl, T and batch_size.  The count argument bounds t* by ceil(bs / E) + mpl - 2, so `done` needs at most
    ceil(bs / E) + 2 mpl - 2 steps: max_steps() keeps at least two steps of slack.  `tight` and `over` lengthen the
    last path (past mpl, as an engine that does not cut its paths would) to end on the capacity's last step and one
    step past it."""
    S = t_star + mpl
    done = np.zeros((S, E), np.uint8)
    done[t_star::-mpl, :E - 1] = 1
    done[t_star - 1::-mpl, E - 1] = 1
    done[S - 1, E - 1] = 1
    bs = int(counts(done)[t_star - 1]) + 1
    cap = max_steps(E, mpl, T, bs)
    assert selection(Stream("worst", "", done, bs, T))[0] == t_star
    assert S <= cap
    tight, over = np.zeros((cap, E), np.uint8), np.zeros((cap + 1, E), np.uint8)
    for x in (tight, over):
        x[:S - 1] = done[:S - 1]
        x[-1, E - 1] = 1
    return done, bs, cap, tight, over


# ---------------------------------------------------------------- gather cells

# name -> (dtype, slab shape [A, ...]); the dispatch picks 16-, 4-, 2- or 1-byte words from the slab size and the
# pointers, then one thread per slab of at most 4 words or one warp per wider slab
GATHER_TENSORS = collections.OrderedDict([
    ("w16_thread", (np.float32, (2, 8))),       # 64 B: 4 words of 16 B
    ("w16_warp", (np.float32, (3, 8))),         # 96 B: 6 words of 16 B
    ("w4_thread", (np.float32, (3,))),          # 12 B: 3 words of 4 B
    ("w4_warp", (np.int32, (5,))),              # 20 B: 5 words of 4 B
    ("w2_thread", (np.uint16, (3,))),           # 6 B: 3 words of 2 B
    ("w2_warp", (np.uint16, (5,))),             # 10 B: 5 words of 2 B
    ("w1_thread", (np.uint8, (3,))),            # 3 B
    ("w1_warp", (np.uint8, (7,))),              # 7 B
])
# shifted tensors whose src and dst are 16-byte aligned with 16-byte slabs, but whose `first` is only 4- or
# 2-byte aligned: name -> (dtype, slab shape, byte offset of first in its buffer)
GATHER_FIRST = collections.OrderedDict([
    ("first_off4", (np.float32, (2, 8), 4)),   # 64 B slabs -> 16 words of 4 B (warp)
    ("first_off2", (np.uint16, (2, 8), 2)),    # 32 B slabs -> 16 words of 2 B (warp)
    ("first_off4_narrow", (np.float32, (4,), 4)),   # 16 B slabs -> 4 words of 4 B (thread)
])
SENTINEL = 0x5A


def gather_cell(slab_bytes, ptrs):
    """(word bytes, 'thread' | 'warp') madrl_whole_paths_gather launches for a slab size and its pointers."""
    bits = slab_bytes
    for p in ptrs:
        bits |= int(p or 0)
    word = next(w for w in (16, 4, 2, 1) if bits % w == 0)
    return word, "thread" if slab_bytes // word <= 4 else "warp"


ALL_CELLS = {(w, k) for w in (16, 4, 2, 1) for k in ("thread", "warp")}


def gather_inputs(S, E, seed):
    """name -> (x [S, E, ...], first [E, ...] or None, first's byte offset): random words for every gather cell,
    shifted (with `first`) or not."""
    rs = np.random.RandomState(seed)

    def words(dtype, shape):
        return rs.randint(0, 256, size=(int(np.prod(shape)) * np.dtype(dtype).itemsize,)).astype(np.uint8).view(
            dtype).reshape(shape)
    out = collections.OrderedDict()
    for k, (dt, sh) in GATHER_TENSORS.items():
        shifted = k.startswith("w16") or k == "w2_thread"
        out[k] = (words(dt, (S, E) + sh), words(dt, (E,) + sh) if shifted else None, 0)
    for k, (dt, sh, off) in GATHER_FIRST.items():
        out[k] = (words(dt, (S, E) + sh), words(dt, (E,) + sh), off)
    return out


def at_offset(x, off):
    """x copied into a larger NumPy buffer at `off` bytes past a 16-byte boundary (a view; keeps the buffer alive)."""
    buf = np.zeros(x.nbytes + 64, np.uint8)
    a = (-buf.ctypes.data) % 16 + off
    v = buf[a:a + x.nbytes].view(x.dtype).reshape(x.shape)
    v[...] = x
    return v


def check_gathered(got, x, end, first):
    """Every row written once, with the oracle's bytes (the sentinel would show a row never written; a duplicate
    write lands in a neighbour's row and breaks its bytes)."""
    want = wo.take(x, end, first)
    assert got.shape == want.shape and got.tobytes() == want.tobytes()


# ---------------------------------------------------------------- flat plan and GAE

PlanCase = collections.namedtuple("PlanCase", "name lengths A discount gae_lambda")


def _plan_cases():
    rs = np.random.RandomState(3)

    def split(N, P):
        """P path lengths summing to N, ragged."""
        cuts = np.sort(rs.choice(np.arange(1, N), P - 1, replace=False)) if P > 1 else np.array([], np.int64)
        return tuple(np.diff(np.concatenate([[0], cuts, [N]])).tolist())
    out = [PlanCase("N1", (1,), 3, 0.99, 0.95)]
    for N in (255, 256, 257, 3001):
        out.append(PlanCase("N%d_ragged" % N, split(N, max(1, N // 9)), 3, 0.99, 0.95))
    out += [PlanCase("P1_N257", (257,), 2, 0.99, 0.97),
            PlanCase("PN_N257", (1,) * 257, 2, 0.99, 0.97),
            PlanCase("PA127", split(400, 127), 1, 0.99, 0.95),
            PlanCase("PA128", split(400, 64), 2, 0.99, 0.95),
            PlanCase("PA129", split(400, 43), 3, 0.99, 0.95),
            PlanCase("one_path_1199", (5, 1199, 3), 2, 0.995, 0.97),
            PlanCase("discount0", split(300, 31), 3, 0.0, 0.95),
            PlanCase("discount1", split(300, 31), 3, 1.0, 1.0)]
    return out


PLAN_CASES = _plan_cases()


def plan_inputs(c, seed):
    """(path_start int32 [P + 1], done uint8 [N], rew, val float32 [N, 1, A]) of a plan case."""
    ps = np.concatenate([[0], np.cumsum(c.lengths)]).astype(np.int32)
    N = int(ps[-1])
    done = np.zeros(N, np.uint8)
    done[ps[1:] - 1] = 1
    rs = np.random.RandomState(seed)
    return ps, done, rs.randn(N, 1, c.A).astype(np.float32), rs.randn(N, 1, c.A).astype(np.float32)


def check_gae_float64(adv, ret, rew, val, done, discount, gae_lambda):
    """adv, ret [N, 1, A] within float32 ulps of rllab's GAE per path in float64 (base.py:57-63)."""
    pe.check_gae(np.asarray(adv), np.asarray(ret), rew, val, done.reshape(-1, 1), discount, gae_lambda, None)


# ---------------------------------------------------------------- whole-path batches pooled over ranks

def pooled_streams(W):
    """Per rank (E, done, batch_size, T), uneven on purpose: a rank with a single path, a rank whose longest path is
    longer than any other rank's (the time baseline's bin count comes from it), a rank of 257 envs."""
    single = np.zeros((12, 1), np.uint8)
    single[-1] = 1
    longest = ragged(31, 60, 4, 9, 0.2)
    longest[:, 1] = 0
    longest[39, 1] = 1                           # a 40-step path
    wide = ragged(32, 40, 257, 9, 0.2)
    if W == 2:
        single40 = np.zeros((40, 1), np.uint8)
        single40[-1] = 1
        ranks = [(single40, 40), (wide, 3 * 257)]
    else:
        ranks = [(wide, 3 * 257), (single, 12), (longest, 30)]
    return [(d.shape[1], d, bs, 5) for d, bs in ranks]


def pooled_tensors(W, rank, S, E, A=3, D=4):
    rs = np.random.RandomState(1000 * W + rank)
    return dict(obs=(rs.randn(S, E, A, D) * 2 + 0.5).astype(np.float32), first=rs.randn(E, A, D).astype(np.float32),
                rew=rs.randn(S, E, A).astype(np.float32), act=rs.randn(S, E, A, 2).astype(np.float32))


def pooled_batch(W, rank, dev):
    """Rank `rank`'s WholePathBatch, built by _Selection from its scripted stream."""
    import torch
    from madrl_b200.whole_paths import _Selection
    dev = torch.device(dev)
    E, done, bs, T = pooled_streams(W)[rank]
    S = -(-done.shape[0] // T) * T
    x = pooled_tensors(W, rank, S, E)
    d = np.zeros((S, E), np.uint8)
    d[:done.shape[0]] = done
    g = {k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in x.items()}
    dd = torch.from_numpy(d).to(dev)
    info = torch.zeros((S, E), dtype=torch.int32, device=dev)
    sel = _Selection(E, T, bs, S, dev)
    first = g["first"]
    for j in range(S // T):
        sl = slice(j * T, (j + 1) * T)
        if sel.add(first, g["obs"][sl].clone(), g["act"][sl].clone(), g["rew"][sl].clone(), dd[sl].contiguous(),
                   info[sl].clone(), {"mean": g["act"][sl].clone()}):
            break
        first = g["obs"][(j + 1) * T - 1].clone()
    return sel.batch()


def pooled_passes(obs, done, rew, ob, act, dev, group):
    """process_samples_concurrent (twice: the second predicts with the first's pooled fit),
    process_samples_recurrent in both modes and rltools' process_samples, with `group` (None: unsharded)."""
    import torch
    from madrl_b200 import postproc, rltools_sampler
    from sharded_edges import to_np
    kw = {} if group is None else dict(group=group)
    D, A = obs.shape[3], obs.shape[2]
    out = {}
    bl = postproc.LinearFeatureBaseline(D, dev, n_agents=A)
    out["conc"] = [postproc.process_samples_concurrent(bl, obs, done, rew, 0.99, 0.97, obs_before=ob, **kw)
                   for _ in range(2)]
    out["conc_coeffs"] = bl.get_param_values()
    for mode in ("decentralized", "concurrent"):
        bl = postproc.LinearFeatureBaseline(D, dev, n_agents=A if mode == "concurrent" else None)
        stats = []
        for _ in range(2):
            r = postproc.process_samples_recurrent(bl, obs, act, rew, done, 0.99, 0.97, mode, obs_before=ob,
                                                   agent_infos={"mean": act}, **kw)
            lists = r if isinstance(r, list) else [r]
            stats.append([{k: v for k, v in x.items() if not torch.is_tensor(v) and k != "paths"
                           and not isinstance(v, dict)} for x in lists])
        out[mode] = dict(stats=stats, coeffs=bl.get_param_values())
    rb = rltools_sampler.LinearFeatureBaseline(D, dev, True)
    rl = []
    for _ in range(2):
        r = rltools_sampler.process_samples(rb, obs, done, rew, 0.99, 0.97, mode="decentralized", obs_before=ob, **kw)
        rl.append({k: r[k] for k in ("q", "advantages", "values", "v_r", "tv_r", "fallback")})
    out["rltools"] = rl
    return to_np(out)


def pooled_rank(ctx, W):
    """One rank of the pooled whole-path processing: its batch's outputs with the WORLD group."""
    b = pooled_batch(W, ctx.rank, ctx.dev)
    obs, done, rew, ob = b.as_rollout()
    res = pooled_passes(obs, done, rew, ob, b.actions.unsqueeze(1), ctx.dev, ctx.group)
    res["N"] = len(b)
    return res
