"""Inputs and checks shared by the edge-case tests of the post-processing and linear-baseline kernels
(csrc/postproc.cu, csrc/baseline.cu): tests/test_postproc_edges_gpu.py runs them on the device through
madrl_b200.postproc, tests/test_emulated_postproc.py and the emulated baseline tests run them in the warp emulator
of tests/emu through the C ABI.  The cases sit at the block, tile, slice and stride edges of the kernels; every
check takes NumPy arrays and compares with the float64 oracles of oracle/, exactly where the arithmetic allows it
and otherwise within float32 ulps of the expected value."""
import os
import re
from fractions import Fraction

import numpy as np

from oracle import postproc_oracle as po

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "madrl_b200", "csrc")


def csrc_default(name, source):
    """The default value of a `#define name <int>` of a kernel source (what the product build uses)."""
    with open(os.path.join(CSRC, source)) as f:
        return int(re.search(r"#define %s (\d+)" % name, f.read()).group(1))


def f32_ulp(x):
    """float64 size of one float32 ulp at |x| (the smallest subnormal at 0)."""
    return np.spacing(np.abs(np.asarray(x, np.float64)).astype(np.float32)).astype(np.float64)


def bf16_bits(x):
    """Round-to-nearest-even bfloat16 bits of float32 x (uint16) and their exact float32 widening."""
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    b = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    return b, (b.astype(np.uint32) << 16).view(np.float32)


# ---------------------------------------------------------------- linear feature baseline (csrc/baseline.cu)

# obs_dims around the 64-column tiles of the Gram kernel ([obs | obs^2 | a, a^2, a^3, 1 | y], 2 D + 5 columns):
# the five time / constant / return columns cross a tile edge at D = 30, 31, 62, 63 and the obs^2 block ends on
# one at D = 32, 64
LFB_DIMS = (1, 2, 29, 30, 31, 32, 33, 61, 62, 63, 64)
# time indices where NumPy's al ** 3 (1 .. 50004, 199990) or glibc's pow (767, 1534, 3411, 196352) is 1 ulp
# off the correctly rounded cube on an x86-64 host
LFB_T0 = (0, 1, 2, 4, 8, 64, 99, 101, 128, 767, 1534, 3411, 50004, 99999, 196352, 199990)


def exact_time_features(idx):
    """(a, a^2, a^3) of time index idx: a = idx / 100 and a * a rounded once, a^3 the correctly rounded cube
    (exact rational arithmetic, not a pow())."""
    a = idx / 100.0
    return [a, a * a, float(Fraction(a) ** 3)]


def single_row_obs(D, k, bf16, rs):
    """D float32 observation values of a single-row case: exactly +-10, the next representable value beyond
    (float32 or bfloat16), +-inf and values just inside, rotated by k so that every position sees each of them,
    the rest random (some beyond the clip)."""
    beyond = 10.0625 if bf16 else float(np.nextafter(np.float32(10), np.float32(np.inf)))
    inside = 9.9375 if bf16 else float(np.nextafter(np.float32(10), np.float32(0)))
    special = [10.0, -10.0, beyond, -beyond, np.inf, -np.inf, inside, -inside]
    o = (rs.randn(D) * 8).astype(np.float32)
    for i in range(0, D, 2):
        o[i] = special[(k + i // 2) % len(special)]
    return bf16_bits(o)[1] if bf16 else o


def single_row_features(o, y, idx):
    """[clip(o), clip(o)^2, a, a^2, a^3, 1, y] of one row in float64; o holds the (widened) float32 values."""
    c = np.clip(np.asarray(o, np.float64), -10, 10)
    return np.concatenate([c, c * c, exact_time_features(idx), [1.0, float(y)]])


def lfb_case(T, E, A, D, p_done, seed, with_before=True, with_t0=True):
    """A random rollout for the baseline kernels: observations beyond the clip on some entries, several paths in
    env 0, returns, t0 and coefficients [2 D + 4]."""
    rs = np.random.RandomState(seed)
    obs = (rs.randn(T, E, A, D) * 6).astype(np.float32)
    obs_before = (rs.randn(E, A, D) * 6).astype(np.float32) if with_before else None
    done = (rs.rand(T, E) < p_done).astype(np.uint8)
    if T > 4:
        done[T // 2, 0] = done[T // 2 + 2, 0] = 1
    ret = rs.randn(T, E, A).astype(np.float32)
    t0 = rs.randint(0, 300, size=E).astype(np.int32) if with_t0 else None
    return dict(obs=obs, obs_before=obs_before, done=done, ret=ret, t0=t0)


def check_gram(G, G_ref):
    """|G - G_ref| <= 1e-12 sqrt(G_ii G_jj) (the bound of the existing baseline tests) and exact symmetry."""
    d = np.sqrt(np.outer(np.diag(G_ref), np.diag(G_ref)))
    err = np.abs(G - G_ref)
    assert np.all(err <= 1e-12 * d), (err / np.maximum(d, 1e-300)).max()
    assert np.array_equal(G, G.T)


def check_predict(vals, F, c):
    want = F.dot(c)
    tol = f32_ulp(want) + 1e-12 * np.abs(F * c).sum(axis=1)
    assert np.all(np.abs(np.asarray(vals, np.float64).reshape(-1) - want) <= tol)


# ---------------------------------------------------------------- whole-batch moments and advantage centring

def stride_sizes(blocks, threads=256):
    """Element counts at the block and grid-stride edges of a moments launch of `blocks` CTAs."""
    s = blocks * threads
    return (threads - 1, threads, threads + 1, s - 1, s, s + 1, 3 * s + 5)


def offset_series(n, seed):
    """(a, b) float32 with mean ~1e4 and unit-scale spread: a one-pass variance loses ~1e-9 relative."""
    rs = np.random.RandomState(seed)
    return (rs.randn(n) * 3 + 1e4).astype(np.float32), (rs.randn(n) + 1e4).astype(np.float32)


def moments_want(a, b):
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    s = (a64, b64, b64 - a64)
    return np.array([x.mean() for x in s] + [x.var() for x in s] + [x.min() for x in s])


def agent_columns(rows, A, seed):
    """x, y [rows, A] float32: per-agent scale and offset (every third agent around 1e4)."""
    rs = np.random.RandomState(seed)
    off = np.where(np.arange(A) % 3 == 0, 1e4, np.arange(A) * 0.5)
    x = (rs.randn(rows, A) * (1 + np.arange(A) % 5) + off).astype(np.float32)
    y = (x + rs.randn(rows, A)).astype(np.float32)
    return x, y


CENTRE_MODES = ((1, 0), (0, 1), (1, 1))


# ---------------------------------------------------------------- frame stack

def frame_stack_calls(E, A, D, seed, bf16=False):
    """Reset observations and three chained calls: done on each env's first step (every other env), done on
    every step, no done at all."""
    rs = np.random.RandomState(seed)
    cvt = (lambda x: bf16_bits(x)[1]) if bf16 else (lambda x: x)
    obs0 = cvt(rs.randn(E, A, D).astype(np.float32))
    calls = []
    for T, kind in ((5, "first"), (3, "every"), (6, "never")):
        obs = cvt(rs.randn(T, E, A, D).astype(np.float32))
        done = np.zeros((T, E), np.uint8)
        if kind == "first":
            done[0, ::2] = 1
            done[3, 1::3] = 1
        elif kind == "every":
            done[:] = 1
        calls.append((obs, done))
    return obs0, calls


def check_frame_stack(obs0, calls, outs, B):
    """outs: the calls' [T,E,A,D,B] results; bit for bit ObservationBuffer's."""
    obs = np.concatenate([o for o, _ in calls])
    done = np.concatenate([d for _, d in calls]).astype(bool)
    got = np.concatenate(outs)
    for e in range(obs.shape[1]):
        _, want = po.frame_stack_env(obs0[e].astype(np.float64), obs[:, e].astype(np.float64), done[:, e], B)
        assert np.array_equal(got[:, e].astype(np.float64), want), (B, e)


# ---------------------------------------------------------------- standardiser

STD_ALPHA, STD_EPS = 0.5, 1e-8
STD_X = (1.5, -3.0, 0.375, 1024.0, -2.0 ** -20, 96.0)      # dyadic float32 inputs


def _neighbours(b):
    """The float32 value of b, its float32 neighbours, and the float64 values next to it (which still round to it)."""
    f = np.float32(b)
    return [float(np.nextafter(f, np.float32(0))), float(f), float(np.nextafter(f, np.float32(np.inf))),
            float(np.nextafter(float(f), 0.0)), float(np.nextafter(float(f), np.inf))]


# updated variances v' on both paths of inv_std (csrc/postproc.cu): the exact one for (float)v' <= 1e-30f or
# >= 1e30f (0, subnormals, 1e-300, 1e300), the MUFU seed + Newton steps in between; both float32 boundaries
STD_TARGETS = tuple([0.0, 5e-324, 2.5e-310, 1e-300] + _neighbours(1e-30) + [1.0] + _neighbours(1e30) + [1e300])


def std_reward_case(reps=3):
    """Reward path (center = 0): rew_mean = x, so with alpha = 0.5 the update gives m' = x exactly, d = 0 and
    v' = v / 2; rew_var = 2 v' for each target v'.  Returns x float32, mean, var (float64) and the expected v'."""
    x, vt = np.meshgrid(np.array(STD_X, np.float32), np.array(STD_TARGETS))
    x, vt = np.tile(x.ravel(), reps), np.tile(vt.ravel(), reps)
    return x.copy(), x.astype(np.float64), 2 * vt, vt


def std_obs_case(reps=3):
    """Centred path (center = 1, alpha = 0.5): x - m' = d a power of two near sqrt(v')/3 (d^2 and alpha d^2 exact,
    so a contracted update gives the same v'), v = 2 v' - d^2.  x is set to 0 where x - d would round.  Returns
    x float32, mean, var and the updated m', v' as the kernel computes them."""
    xs, ms, vs = [], [], []
    for t in STD_TARGETS:
        for x in STD_X:
            d = 0.0 if t < 1e-290 else 2.0 ** (np.floor(np.log2(np.sqrt(t))) - 2)
            if any(Fraction(x) - Fraction(k * d) != Fraction(x - k * d) for k in (1, 2)):
                x = 0.0
            xs.append(x)
            ms.append(x - 2 * d)
            vs.append(2 * t - d * d)
    x = np.tile(np.array(xs, np.float32), reps)
    m, v = np.tile(np.array(ms), reps), np.tile(np.array(vs), reps)
    m1 = (1 - STD_ALPHA) * m + STD_ALPHA * x.astype(np.float64)
    d = x.astype(np.float64) - m1
    v1 = (1 - STD_ALPHA) * v + STD_ALPHA * d * d
    return x, m, v, m1, v1


def std_target_classes(v1):
    """float32 images of the updated variances: they must cover both sides of both inv_std boundaries."""
    with np.errstate(over="ignore"):
        f = v1.astype(np.float32)
    lo, hi = np.float32(1e-30), np.float32(1e30)
    return dict(exact_low=int((f <= lo).sum()), fast=int(((f > lo) & (f < hi)).sum()), exact_high=int((f >= hi).sum()))


def check_standardized(got, want):
    """got (float32) within one float32 ulp of the float64 `want`; returns how many differ from want rounded to
    float32 (near-ties of the Newton-refined reciprocal)."""
    got = np.asarray(got, np.float64).ravel()
    want = np.asarray(want, np.float64).ravel()
    err = np.abs(got - want)
    bad = ~(err <= f32_ulp(want))
    assert not bad.any(), (np.nonzero(bad)[0][:5], got[bad][:5], want[bad][:5])
    return int((got != want.astype(np.float32)).sum())


def terminal_case(T, E, P, seed):
    """Auto-reset observations with terminal observations on the side: env e % 3 == 0 is done at t = 0 only,
    e % 3 == 1 on every step, e % 3 == 2 never."""
    rs = np.random.RandomState(seed)
    obs = (rs.randn(T, E, P) * 2 + 0.5).astype(np.float32)
    term = (rs.randn(T, E, P) * 2 - 0.5).astype(np.float32)
    done = np.zeros((T, E), np.uint8)
    done[0, 0::3] = 1
    done[:, 1::3] = 1
    return obs, term, done


def check_terminal(x, tm, obs, term, done, alpha, mean):
    """x, tm: the standardised observations and terminal observations; StandardizedEnv's order (terminal, then
    reset observation) within a float32 ulp plus the float64 rounding of the running mean."""
    T, E, P = obs.shape
    for e in range(E):
        mine = po.StandardizeEnv(1, P, 1.0, True, False, alpha, 0.001)
        for t in range(T):
            for src, out in ((term, tm), (obs, x)):
                if src is term and not done[t, e]:
                    assert np.array_equal(tm[t, e], term[t, e])                   # untouched
                    continue
                v = src[t, e].astype(np.float64)
                want = mine.obs(v[None])[0]
                slack = 1e-12 * (np.abs(v) + np.abs(mine.obs_mean[0])) / (np.sqrt(mine.obs_var[0]) + 1e-8)
                assert np.all(np.abs(out[t, e].astype(np.float64) - want) <= f32_ulp(want) + slack), (t, e)
        assert np.allclose(mean[e], mine.obs_mean[0], rtol=1e-14, atol=1e-14)


# ---------------------------------------------------------------- GAE and episode statistics

GAE_PARAMS = ((0.99, 0.95), (1.0, 1.0), (0.0, 0.5))


def gae_case(T, E, A, seed):
    """rew, val [T,E,A], last [E,A], done [T,E]: env e % 4 == 0 done at t = 0, 1 at t = T - 1, 2 on every step,
    3 never."""
    rs = np.random.RandomState(seed)
    rew, val = rs.randn(T, E, A).astype(np.float32), rs.randn(T, E, A).astype(np.float32)
    last = rs.randn(E, A).astype(np.float32)
    done = np.zeros((T, E), np.uint8)
    done[0, 0::4] = 1
    done[T - 1, 1::4] = 1
    done[:, 2::4] = 1
    return rew, val, last, done


def check_gae(adv, ret, rew, val, done, discount, gae_lambda, last):
    T = rew.shape[0]
    scale = 1e-13 * T * (np.abs(rew).max() + 2 * np.abs(val).max() + (0 if last is None else np.abs(last).max()))
    for e in range(rew.shape[1]):
        a_o, r_o = po.gae_env(rew[:, e], val[:, e], done[:, e].astype(bool), discount, gae_lambda,
                              None if last is None else last[e])
        assert np.all(np.abs(adv[:, e] - a_o) <= f32_ulp(a_o) + scale), e
        assert np.all(np.abs(ret[:, e] - r_o) <= f32_ulp(r_o) + scale), e


def episode_stats_calls(E, A, kind, seed):
    """(max_traj_len, [(rew, done)] per call) of one scenario:
    len1      max_traj_len = 1: every step closes an episode;
    boundary  max_traj_len = 5 and calls of 5 steps: episodes end exactly at the call boundaries, done and
              max_traj_len on the same step (e % 3 == 0), a done mid-call shifting the boundary (e % 3 == 1);
    span3     one episode across three calls (the discount-power carry), closed by a done on the last step
              (every env but e % 5 == 0, which stays open)."""
    rs = np.random.RandomState(seed)
    if kind == "len1":
        mtl, lens = 1, (3, 4)
    elif kind == "boundary":
        mtl, lens = 5, (5, 5, 5)
    else:
        mtl, lens = 100, (4, 6, 5)
    calls = []
    for n, T in enumerate(lens):
        rew = rs.randn(T, E, A).astype(np.float32)
        done = np.zeros((T, E), np.uint8)
        if kind == "len1":
            done[:] = rs.rand(T, E) < 0.3
        elif kind == "boundary":
            if n == 0:
                done[4, 0::3] = 1
            if n == 1:
                done[2, 1::3] = 1
        elif n == len(lens) - 1:
            done[T - 1] = 1
            done[T - 1, 0::5] = 0
        calls.append((rew, done))
    return mtl, calls


def check_episode_stats(outs, calls, discount, mtl):
    """outs: per call (ep_reward [T,E,A] float32, ep_disc [T,E] float32, ep_len [T,E], ep_end [T,E])."""
    rew = np.concatenate([r for r, _ in calls]).astype(np.float64)
    done = np.concatenate([d for _, d in calls]).astype(bool)
    ep_r, ep_d, ep_l, ep_e = [np.concatenate([o[i] for o in outs]) for i in range(4)]
    for e in range(rew.shape[1]):
        recs = po.episode_stats_env(rew[:, e], done[:, e], discount, mtl)
        ends = [r[0] for r in recs]
        assert ends == list(np.nonzero(ep_e[:, e])[0]), e
        assert not ep_l[:, e][~ep_e[:, e].astype(bool)].any() and not ep_r[:, e][~ep_e[:, e].astype(bool)].any()
        for t, r, avg, disc, length in recs:
            assert np.array_equal(ep_r[t, e], r.astype(np.float32)), (t, e)      # the same float64 sum
            assert ep_l[t, e] == length
            s = rew[t - length + 1:t + 1, e]
            tol = f32_ulp(disc) + 1e-13 * length * np.abs(s).max()
            assert abs(float(ep_d[t, e]) - disc) <= tol, (t, e)
    return len(ends)


# ---------------------------------------------------------------- path packing

PACK_WORDS = (1, 2, 3, 4, 5, 31, 32, 33)       # one thread per row for D <= 4 words, one warp per row beyond
PACK_SHAPES = ((1, 131, 3, 0.5), (6, 150, 2, 1.0), (9, 140, 3, 0.3))   # T = 1; every episode one step; E > 128


def pack_case(T, E, A, D, p_done, itemsize, seed):
    """Random words (uint32 or uint16) as observations [T,E,A,D] and obs_before [E,A,D], int32 actions [T,E,A],
    float32 rewards, one int32 info per env and step."""
    rs = np.random.RandomState(seed)
    w = np.uint32 if itemsize == 4 else np.uint16
    words = lambda *s: rs.randint(0, 2 ** (8 * itemsize), size=s, dtype=np.uint64).astype(w)   # noqa: E731
    done = (rs.rand(T, E) < p_done).astype(np.uint8)
    return dict(obs=words(T, E, A, D), obs_before=words(E, A, D), act=rs.randint(0, 5, (T, E, A)).astype(np.int32),
                rew=rs.randn(T, E, A).astype(np.float32), info=rs.randint(0, 9, (T, E)).astype(np.int32),
                done=done)


def check_packed(c, shifted, paths, p_obs, p_act, p_rew, p_info):
    """paths: (env, agent, terminated, offset, length, info_offset) per path in pack order; the packed arrays
    against the host to_paths, bit for bit."""
    from madrl_b200.postproc import to_paths
    src = np.concatenate([c["obs_before"][None], c["obs"][:-1]]) if shifted else c["obs"]
    want = to_paths(src, c["act"], c["rew"], c["done"], dict(k=c["info"]))
    assert len(paths) == len(want)
    for (e, a, term, o, n, io), w in zip(paths, want):
        assert (e, a, term) == (w["env"], w["agent"], w["terminated"])
        assert np.array_equal(p_obs[o:o + n], w["observations"]), (e, a, o)
        assert np.array_equal(p_act[o:o + n], w["actions"]) and np.array_equal(p_rew[o:o + n], w["rewards"])
        assert np.array_equal(p_info[io:io + n], w["env_infos"]["k"])
    return len(paths)


def plan_paths(n_ep, ep_rec, T, A):
    """The path records of madrl_paths_plan's per-episode records, in pack order."""
    out = []
    for e in range(len(n_ep)):
        for j in range(n_ep[e]):
            s, L, term = ep_rec[e, j]
            out += [(e, a, bool(term), e * T * A + s * A + a * L, L, e * T + s) for a in range(A)]
    return out


def path_records(done, A, agent_major=False):
    """int32 [P, 4] (env, agent, start, length) of the paths of done [T, E] (cut at done and at the end of the
    rollout), in (env, episode, agent) order, or (agent, env, episode) with agent_major: the padded-path table."""
    T, E = done.shape
    eps = []
    for e in range(E):
        s = 0
        for t in range(T):
            if done[t, e] or t == T - 1:
                eps.append((e, s, t + 1 - s))
                s = t + 1
    recs = [(e, a, s, n) for a in range(A) for e, s, n in eps] if agent_major else \
        [(e, a, s, n) for e, s, n in eps for a in range(A)]
    return np.array(recs, np.int32).reshape(-1, 4)


def sequential_sum(x):
    """float64 sum of x from left to right, one rounding per term (Python >= 3.12's sum() of floats compensates)."""
    acc = 0.0
    for v in np.asarray(x, np.float64).ravel():
        acc += float(v)
    return acc


# ---------------------------------------------------------------- rltools' sample processing

def slice_rows(S):
    """Rows per group around a kernel's S row slices: one row, every slice empty but one or holding one row, and
    the 8-warp stride of a slice."""
    return tuple(sorted({r for r in (1, S - 1, S, S + 1, 8 * S - 1, 8 * S + 1) if r >= 1}))


def mixed_scale(rs, *shape):
    """float32 values whose magnitudes span 1e-3 .. 1e3 (so that an absolute error bound is not trivially loose)."""
    return (rs.randn(*shape) * 10.0 ** rs.randint(-3, 4, size=shape) + 0.25).astype(np.float32)


def check_column_sums(got, rows):
    """got [G, 2, D]: per group g the float64 column sums of x and x^2 over rows[:, g] (rows [n, G, D], widened
    float32, so every square is exact in float64), each within n 2^-52 sum|.| of NumPy's float64 sum."""
    n = rows.shape[0]
    for j, v in enumerate((rows, rows * rows)):
        err = np.abs(got[:, j] - v.sum(0))
        assert np.all(err <= n * 2.0 ** -52 * np.abs(v).sum(0)), (j, err.max())


def time_index(done, t0=None):
    """(idx, path) [T, E]: the time index of every (t, e) -- its position in its path plus t0[e] on env e's first
    path, the baseline's lfb_index -- and its path's number, paths numbered env by env in time order."""
    T, E = done.shape
    idx, path = np.zeros((T, E), np.int64), np.zeros((T, E), np.int64)
    p = 0
    for e in range(E):
        s = 0
        for t in range(T):
            idx[t, e] = t - s + (t0[e] if (t0 is not None and s == 0) else 0)
            path[t, e] = p
            if done[t, e] or t == T - 1:
                s, p = t + 1, p + 1
    return idx, path


def time_baseline_case(T, E, A, L, seed):
    """q [T,E,A], done [T,E] and t0 whose largest time index is L - 1: env 0 runs the whole horizon, env 1 ends a
    path on every step, the others at random.  L == T: no t0; L > T: env 0's t0 = L - T carries the index past T
    (the other envs' t0 stay below it)."""
    assert 1 <= T <= L
    rs = np.random.RandomState(seed)
    done = (rs.rand(T, E) < 0.2).astype(np.uint8)
    done[:, 0] = 0
    if E > 1:
        done[:, 1] = 1
    t0 = None
    if L > T:
        t0 = rs.randint(0, L - T + 1, size=E).astype(np.int32)
        t0[0] = L - T
    return mixed_scale(rs, T, E, A), done, t0


def check_time_baseline(simplev, bin_sum, bin_cnt, q, done, t0, per_agent):
    """Counts exact; sums within n 2^-52 sum|q| of NumPy's; simplev the returned bins' float64 quotient rounded to
    float32, bit for bit; and that quotient within float32 rounding of NumPy's nanmean over the NaN-padded paths
    (Sampler.process's simplev)."""
    T, E, A = q.shape
    idx, path = time_index(done, t0)
    G, L = (A if per_agent else 1), int(idx.max()) + 1
    assert bin_sum.shape == (G, L) and bin_cnt.shape == (G, L)
    q64 = q.astype(np.float64)
    s, c, mag = np.zeros((G, L)), np.zeros((G, L), np.int64), np.zeros((G, L))
    for a in range(A):
        g = a if per_agent else 0
        np.add.at(s[g], idx, q64[..., a])
        np.add.at(c[g], idx, 1)
        np.add.at(mag[g], idx, np.abs(q64[..., a]))
    assert np.array_equal(bin_cnt, c)
    tol = c * 2.0 ** -52 * mag
    assert np.all(np.abs(bin_sum - s) <= tol), np.abs(bin_sum - s).max()
    grp = np.arange(A) if per_agent else np.zeros(A, np.int64)
    got_bin = bin_sum[grp[None, None, :], idx[..., None]] / bin_cnt[grp[None, None, :], idx[..., None]]
    assert np.array_equal(simplev, got_bin.astype(np.float32))
    P = int(path.max()) + 1
    for g in range(G):
        agents = [g] if per_agent else list(range(A))
        pad = np.full((P * len(agents), L), np.nan)
        for k, a in enumerate(agents):
            pad[path * len(agents) + k, idx] = q64[..., a]
        m = c[g] > 0                     # a bin no row reaches (below a t0) is never read
        want = np.nanmean(pad[:, m], axis=0)
        got = bin_sum[g, m] / bin_cnt[g, m]
        assert np.all(np.abs(got - want) <= 4 * np.spacing(np.abs(want)) + tol[g, m] / c[g, m]), g


def lfbr_single_row_obs(D, k, bf16, rs):
    """D finite observation values for rltools' unclipped feature map: 0, +-1, +-1e30, +-2^-130 (subnormal in
    float32 and bfloat16), +-3e4, rotated by k so that every position sees each of them, the rest random."""
    special = [0.0, 1.0, -1.0, 1e30, -1e30, 2.0 ** -130, -2.0 ** -130, 3e4, -3e4]
    o = (rs.randn(D) * 8).astype(np.float32)
    for i in range(0, D, 2):
        o[i] = special[(k + i // 2) % len(special)]
    return bf16_bits(o)[1] if bf16 else o


def lfbr_features(seen, idx, norm):
    """rltools' features [(o - mu) / s, a, a * a, 1] (Df = D + 3) in float64 of rows seen [..., D] (widened
    float32), time indices idx [...] (a = idx / 100, one rounding) and norm [..., 2, D] = (mu, s) or None."""
    o = np.asarray(seen, np.float64)
    if norm is not None:
        o = (o - norm[..., 0, :]) / norm[..., 1, :]
    a = np.asarray(idx, np.float64)[..., None] / 100.0
    return np.concatenate([o, a, a * a, np.ones_like(a)], axis=-1)
