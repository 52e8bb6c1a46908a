"""Whole-path sampling over the ranks of a sharded batch (WholePathSampler with ``group=``, DESIGN §4.9) on the GPU:
W = 2, 3 and 4 gloo ranks on cuda:0, each holding an explicit env range (``env_id_base`` and ``.shard``, one-env and
very uneven shards), against an unsharded WholePathSampler on the global envs with the same seed, policy and chunk.
The ranks' batches, concatenated in rank order, must be the unsharded batch bit for bit: obs, actions, rew, infos,
extras and done, path_start and env_rows shifted by the rows of the lower ranks; t* and the steps run equal on every
rank and to the unsharded call's.

The policies are tests/sharded_edges.py's row-wise ones (Linear, Stacked, Argmax: each row's action does not depend
on the shard size) with a row-wise extras entry.  Cases: C2, C3 and C5 in float32 and C5 in bfloat16; chunk 1, 7 and
max_path_length; t* on a launch's first and last step; a rank on which no path ends before t*; a rank whose envs all
end launches before another rank's; a batch_size that no rank's own envs reach by t*; frame_stack 2 with a
standardiser (its state byte for byte); the refusals (shards that do not tile, batch_size, max_path_length or chunk
differing across ranks: every rank raises, none hangs); and process_samples_concurrent and rltools' process_samples
with ``group=`` on the ranks' batches against the same passes on the unsharded batch.
"""
import numpy as np
import pytest
import torch

import sharded_edges as se
import whole_paths_edges as wpe
from oracle import whole_paths_oracle as wo

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)

WW_C2 = dict(n_pursuers=5, n_evaders=5, n_poison=10, n_sensors=30)
PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
# few evaders, caught by one pursuer: paths end at many different steps before the horizon
PE_ENDS = dict(n_evaders=2, n_pursuers=8, obs_range=5, surround=False, n_catch=1, flatten=True, reward_mech='local',
               sample_maps=True)
HW_C5 = (10, 16, 16, 4, 2)
E, MPL = 24, 9
SIZES = {2: (1, 23), 3: (5, 1, 18), 4: (7, 1, 12, 4)}
ENDS_E, ENDS_MPL, ENDS_T = 32, 40, 3


def build(fam, n, mpl, lo=0, n_global=None, obs_dtype=None, seed=11):
    """`n` envs from global env `lo` of family `fam`; with n_global, the shard (lo, lo + n, n_global)."""
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    kw = dict(seed=seed, max_path_length=mpl, obs_dtype=obs_dtype, env_id_base=lo, device=DEV)
    if fam == "ww_c2":
        eng = BatchedMAWaterWorld(n, **dict(kw, **WW_C2))
    elif fam in ("pe_c3", "pe_ends"):
        eng = BatchedPursuitEvade(n, se.map_pool(), **dict(kw, **(PE_C3 if fam == "pe_c3" else PE_ENDS)))
    else:
        eng = BatchedHostageWorld(n, *HW_C5, **kw)
    if n_global is not None:
        eng.shard = (lo, lo + n, n_global)
    return eng


class WithExtras(object):
    """A row-wise policy of tests/sharded_edges.py on float32 observations, with a row-wise extras entry."""

    def __init__(self, pol):
        self.pol = pol

    def __call__(self, obs, state):
        act, _, state = self.pol(obs.float(), state)
        return act, {"row": act.float() * 0.5 - 1.0}, state


def policy(fam, eng, B=1):
    D = eng.obs_dim
    if fam.startswith("pe"):
        return WithExtras(se.Argmax(D * B, 3, DEV))
    return WithExtras(se.Linear(D, 0, DEV) if B == 1 else se.Stacked(D, B, 0, DEV))


def spec(key, fam, sizes, bs, chunk, mpl=MPL, dtype="f32", B=1, std=False):
    return dict(key=key, fam=fam, sizes=tuple(int(s) for s in sizes), bs=int(bs), chunk=int(chunk), mpl=mpl,
                dtype=dtype, B=B, std=std)


def sample(sp, lo, n, group=None, n_global=None):
    """(batch, standardiser or None) of a spec's sampler on envs [lo, lo + n)."""
    from madrl_b200 import WholePathSampler
    from madrl_b200.postproc import Standardizer
    eng = build(sp["fam"], n, sp["mpl"], lo, n_global, torch.bfloat16 if sp["dtype"] == "bf16" else None)
    std = Standardizer(n, eng._n_acting, eng.obs_dim, DEV, enable_obsnorm=True, obs_alpha=0.05) if sp["std"] else None
    s = WholePathSampler(eng, policy(sp["fam"], eng, sp["B"]), sp["bs"], sp["mpl"], chunk=sp["chunk"],
                         frame_stack=sp["B"], standardizer=std, group=group)
    return s(), std


def fields(b, std):
    out = dict(obs=b.obs, actions=b.actions, rew=b.rew, infos=b.infos, extras=b.extras, done=b.done,
               path_start=b.path_start, env_rows=b.env_rows, t_star=b.t_star, n_steps=b.n_steps)
    out = {k: (v.view(torch.int16) if torch.is_tensor(v) and v.dtype == torch.bfloat16 else v) for k, v in out.items()}
    if std is not None:
        out["std"] = (std.obs_mean, std.obs_var)
    return se.to_np(out)


def rank_sample(ctx, sp):
    lo, hi = se.bounds(sp["sizes"])[ctx.rank]
    return fields(*sample(sp, lo, hi - lo, ctx.group, sum(sp["sizes"])))


def check_concat(got, want, sizes):
    """got {rank: fields}, want: the unsharded fields."""
    W = len(sizes)
    for r in range(W):
        assert got[r]["t_star"] == want["t_star"] and got[r]["n_steps"] == want["n_steps"], r
    for k in ("obs", "actions", "rew", "infos", "done"):
        se.bits_equal(np.concatenate([got[r][k] for r in range(W)]), want[k], k)
    for k in want["extras"]:
        se.bits_equal(np.concatenate([got[r]["extras"][k] for r in range(W)]), want["extras"][k], k)
    rows = np.concatenate([[0], np.cumsum([len(got[r]["done"]) for r in range(W)])])
    ps = np.concatenate([got[r]["path_start"][:-1] + rows[r] for r in range(W)] + [[rows[-1]]]).astype(np.int32)
    se.bits_equal(ps, want["path_start"], "path_start")
    se.bits_equal(np.concatenate([got[r]["env_rows"] + rows[r] for r in range(W)]).astype(np.int32),
                  want["env_rows"], "env_rows")
    for r, (lo, hi) in enumerate(se.bounds(sizes)):
        assert len(got[r]["env_rows"]) == hi - lo
    if "std" in want:
        for i in range(2):
            se.bits_equal(np.concatenate([got[r]["std"][i] for r in range(W)]), want["std"][i], "std")


# ---------------------------------------------------------------- the cases

def ends_stream():
    """The done stream of PE_ENDS's global envs under its policy, from reset: [S, ENDS_E]."""
    from madrl_b200.closed_loop import PolicyRollout
    eng = build("pe_ends", ENDS_E, ENDS_MPL)
    r = PolicyRollout(eng, policy("pe_ends", eng), 6 * ENDS_MPL)(eng.reset())
    return r.done.cpu().numpy()


def sizes_with(cuts, W, n):
    """Shard sizes of n envs over W ranks with shard boundaries at every env of `cuts` (plus others as needed)."""
    b = sorted(set(c for c in cuts if 0 < c < n))
    extra = [c for c in range(1, n) if c not in b]
    b = sorted(b + extra[:W - 1 - len(b)])
    assert len(b) == W - 1
    return tuple(np.diff([0] + b + [n]).tolist())


def ends_cases(done, W):
    """Specs placed on the PE_ENDS stream: a rank with no path end before t*, a rank whose envs all end launches
    before another rank's last, and a batch_size no rank's own envs reach by t*."""
    first = np.argmax(done, 0)
    assert done.any(0).all() and first.min() < first.max(), "PE_ENDS paths all end at the same steps"
    out = []
    # the env whose first path ends last holds a rank (of its own where W allows); batch_size is the count one step
    # before any path on that rank ends, so t* comes from the other ranks' paths alone
    late = int(np.argmax(first))
    best = None
    for cuts in ([[late, late + 1]] if W >= 3 else [[late], [late + 1]]):
        sizes = sizes_with(cuts, W, ENDS_E)
        lo, hi = next(b for b in se.bounds(sizes) if b[0] <= late < b[1])
        if best is None or first[lo:hi].min() > best[0]:
            best = (int(first[lo:hi].min()), sizes, lo)
    m, sizes, lo = best
    bs = int(wpe.counts(done)[m - 1])
    assert bs >= 1 and wo.select(done, bs)[0] < m
    out.append((spec("no_end_before_tstar", "pe_ends", sizes, bs, ENDS_T, mpl=ENDS_MPL), dict(idle=lo)))
    # batch_size of two full horizons' steps: the env that ends first after t* holds a rank (of its own where W
    # allows) whose envs all end launches before the env that ends last
    bs = 2 * ENDS_MPL
    t_star, end = wo.select(done, bs)
    early = int(np.argmin(end))
    best = None
    for cuts in ([[early, early + 1]] if W >= 3 else [[early], [early + 1]]):
        sizes = sizes_with(cuts, W, ENDS_E)
        lo, hi = next(b for b in se.bounds(sizes) if b[0] <= early < b[1])
        if best is None or end[lo:hi].max() < best[0]:
            best = (int(end[lo:hi].max()), sizes, lo)
    last, sizes, lo = best
    assert last // ENDS_T < end.max() // ENDS_T, "the rank's envs end in the last launch"
    out.append((spec("rank_ends_early", "pe_ends", sizes, bs, ENDS_T, mpl=ENDS_MPL), dict(early=lo)))
    # balanced shards and a batch_size only the pooled count reaches by t*
    c = wpe.counts(done)
    bs = int(c[c > 0][len(c[c > 0]) // 2])
    sizes = tuple(np.diff([(ENDS_E * r) // W for r in range(W + 1)]).tolist())
    t_star = wo.select(done, bs)[0]
    for lo, hi in se.bounds(sizes):
        assert wpe.counts(done[:, lo:hi])[t_star] < bs
    out.append((spec("pooled_bs", "pe_ends", sizes, bs, ENDS_T, mpl=ENDS_MPL), {}))
    return out


def placed_cases(W):
    """t* on the first and on the last step of a launch of 7 (C5, from a long rollout of the unsharded envs)."""
    from madrl_b200.closed_loop import PolicyRollout
    eng = build("hw_c5", E, MPL)
    done = PolicyRollout(eng, policy("hw_c5", eng), 12 * MPL)(eng.reset()).done.cpu().numpy()
    out = []
    for key, pred in (("tstar_first", lambda ts, end, T: ts > 0 and ts % T == 0),
                      ("tstar_last", lambda ts, end, T: ts % T == T - 1)):
        bs, T = wpe._placed(done, pred, Ts=(7,))
        out.append((spec(key, "hw_c5", SIZES[W], bs, T), {}))
    return out


def cases(W):
    bs = 3 * E + 7
    out = [(spec("ww_c2", "ww_c2", SIZES[W], bs, 7), {}), (spec("pe_c3", "pe_c3", SIZES[W], bs, 7), {}),
           (spec("hw_c5", "hw_c5", SIZES[W], bs, 7), {}), (spec("hw_c5_bf16", "hw_c5", SIZES[W], bs, 7, dtype="bf16"), {}),
           (spec("chunk1", "ww_c2", SIZES[W], bs, 1), {}), (spec("chunk_mpl", "ww_c2", SIZES[W], bs, MPL), {}),
           (spec("stack_std", "ww_c2", SIZES[W][::-1], 2 * E * MPL + 3, 4, B=2, std=True), {})]
    return out + placed_cases(W) + ends_cases(ends_stream(), W)


# ---------------------------------------------------------------- refusals and the processing passes

def refusals(ctx):
    """Samplers whose ranks disagree: every rank must raise ValueError, and a sampler that agrees runs after."""
    from madrl_b200 import WholePathSampler
    W, r = ctx.world, ctx.rank
    sizes = SIZES[W]
    lo, hi = se.bounds(sizes)[r]
    out = {}

    def attempt(key, fn):
        try:
            fn()
            out[key] = "ran"
        except ValueError as ex:
            out[key] = "refused: " + str(ex).split(";")[0].split(":")[0]

    def sampler(mpl=MPL, bs=50, chunk=7, lo=lo, hi=hi):
        eng = build("ww_c2", hi - lo, mpl, lo, E)
        return WholePathSampler(eng, policy("ww_c2", eng), bs, mpl, chunk=chunk, group=ctx.group)
    slo, shi = se.bounds(sizes[::-1])[W - 1 - r]               # rank r holds rank W-1-r's envs of the mirror split
    attempt("swapped", lambda: sampler(lo=slo, hi=shi))
    attempt("batch_size", lambda: sampler(bs=50 + (r == W - 1)))
    attempt("max_path_length", lambda: sampler(mpl=MPL + (r == 0)))
    attempt("chunk", lambda: sampler(chunk=7 + r))
    out["after"] = fields(sampler()(), None)["t_star"]
    return out


def rank_passes(ctx, sp):
    lo, hi = se.bounds(sp["sizes"])[ctx.rank]
    b, _ = sample(sp, lo, hi - lo, ctx.group, sum(sp["sizes"]))
    obs, done, rew, ob = b.as_rollout()
    res = wpe.pooled_passes(obs, done, rew, ob, b.actions.unsqueeze(1), DEV, ctx.group)
    res["N"] = len(b)
    return res


PASSES = spec("passes", "ww_c2", (3, 1, 20), 4 * E, 5)


def jobs(W, specs):
    """The cases every rank runs, in one spawn per W (placed on streams the parent sampled)."""
    out = [(sp["key"], rank_sample, (sp,)) for sp in specs] + [("refusals", refusals, ())]
    return out + ([("passes", rank_passes, (PASSES,))] if W == 3 else [])


@pytest.fixture(scope="module", params=(2, 3, 4), ids=lambda w: "W%d" % w)
def ranks(request):
    W = request.param
    cs = cases(W)
    return W, cs, se.run_ranks(W, "gloo", se.run_cases, jobs(W, [sp for sp, _ in cs]))


def test_batches_concatenate_to_the_unsharded_batch(ranks):
    W, cs, got = ranks
    for sp, why in cs:
        res = se.result(got, sp["key"])
        want = fields(*sample(sp, 0, sum(sp["sizes"])))
        check_concat(res, want, sp["sizes"])
        bounds = se.bounds(sp["sizes"])
        t_star = want["t_star"]
        if "idle" in why:                    # the idle rank's env ends no path before t*
            r = next(i for i, (lo, hi) in enumerate(bounds) if lo == why["idle"])
            d, starts = res[r]["done"], list(res[r]["env_rows"]) + [len(res[r]["done"])]
            assert min(int(np.argmax(d[a:b])) for a, b in zip(starts[:-1], starts[1:])) > t_star
        if "early" in why:                   # that rank keeps no rows of the last launches
            r = next(i for i, (lo, hi) in enumerate(bounds) if lo == why["early"])
            d, starts = res[r]["done"], list(res[r]["env_rows"]) + [len(res[r]["done"])]
            assert max(b - a - 1 for a, b in zip(starts[:-1], starts[1:])) // sp["chunk"] < \
                want["n_steps"] // sp["chunk"] - 1
    assert [sp["key"] for sp, _ in cs][-5:] == ["tstar_first", "tstar_last", "no_end_before_tstar",
                                                "rank_ends_early", "pooled_bs"]


def test_disagreeing_ranks_all_refuse(ranks):
    W, _, got = ranks
    res = se.result(got, "refusals")
    for r in range(W):
        assert res[r]["swapped"].startswith("refused: an evaluation over several ranks needs engines"), res[r]
        for k in ("batch_size", "max_path_length", "chunk"):
            assert res[r][k] == "refused: %s differs across the ranks" % k, (k, res[r][k])
        assert res[r]["after"] == res[0]["after"]


def test_processing_on_the_ranks_batches(ranks):
    W, _, got = ranks
    if W != 3:
        pytest.skip("run over three ranks")
    res = se.result(got, "passes")
    b, _ = sample(PASSES, 0, sum(PASSES["sizes"]))
    obs, done, rew, ob = b.as_rollout()
    full = wpe.pooled_passes(obs, done, rew, ob, b.actions.unsqueeze(1), DEV, None)
    lens = [res[r]["N"] for r in range(W)]
    assert sum(lens) == len(b)
    for k in range(2):
        for r, (lo, hi) in enumerate(se.bounds(lens)):
            v, a, rt, _ = res[r]["conc"][k]
            fv, fa, frt, _ = full["conc"][k]
            assert np.array_equal(rt, frt[lo:hi])
            np.testing.assert_allclose(v, fv[lo:hi], rtol=1e-5, atol=1e-5 * np.abs(fv).max() + 1e-30)
            np.testing.assert_allclose(a, fa[lo:hi], rtol=1e-5, atol=1e-5 * np.abs(fa).max())
            q, fq = res[r]["rltools"][k], full["rltools"][k]
            assert np.array_equal(q["q"], fq["q"][lo:hi])
            for n in ("advantages", "values"):
                np.testing.assert_allclose(q[n], fq[n][lo:hi], rtol=1e-5, atol=1e-5 * np.abs(fq[n]).max() + 1e-30)
        np.testing.assert_allclose(res[0]["conc"][k][3], full["conc"][k][3], rtol=1e-9, atol=1e-9)
        assert np.array_equal(res[0]["rltools"][k]["fallback"], full["rltools"][k]["fallback"])
        np.testing.assert_allclose(res[0]["rltools"][k]["tv_r"], full["rltools"][k]["tv_r"], rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(res[0]["rltools"][k]["v_r"], full["rltools"][k]["v_r"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(res[0]["conc_coeffs"], full["conc_coeffs"], rtol=0,
                               atol=1e-9 * np.abs(full["conc_coeffs"]).max())
