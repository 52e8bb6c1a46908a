"""Pooled sample processing and evaluation (``group=``) over two to four uneven shards, on the GPU, against
whole-batch references.

One spawn per world size W in {2, 3, 4} (gloo, every rank on cuda:0) runs every case of that W; the checks run in
the parent after the ranks have exited.  Each case checks (i) that every pooled output has the same bytes on every
rank and (ii) that the outputs agree with a whole-batch reference: the goldens written by the reference's own code
(rltools' training loop, rllab's recurrent and concurrent branches, the fp64 Waterworld heuristic evaluation), the
float64 NumPy oracles, and the unsharded device call.  Shards come from the split tables of tests/sharded_edges.py:
one-env shards, very uneven ones, a shard without a finished path, a shard whose own largest time index is far
below the batch's, the global minimum and the largest t0 away from rank 0.  A group that is not WORLD (two groups
of two ranks inside four) and the evaluation's refusal of shards that do not tile the batch are covered too.  An
NCCL variant of the golden loops and the evaluations runs where the box has two GPUs or more.

Tolerances where an output is float32 arithmetic on pooled float64 state: the reduction order of the pooled sums
differs from the unsharded kernel's, so float32 state rounded from them may move by one ulp, and the baseline's
coefficients (normal equations summed by the collective) by ~1e-16 times the condition number.  Outputs that do not
depend on such state are compared bit for bit or at rtol 1e-12.
"""
import functools

import numpy as np
import pytest
import torch

import sharded_edges as se
from oracle import concurrent_baseline_oracle as cbo
from oracle import postproc_oracle as po
from oracle import rltools_oracle as ro

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
MODES = ("decentralized", "concurrent", "centralized", "zero")
RLTOOLS_CASES = (("ragged", 4), ("plain", 3))
RECURRENT_E = dict(ragged=4, bf16_int=3)
CONCURRENT_CASES = (("ragged", 3), ("beyond_clip", 2))
SEED = 5


def cases_for(W, golden_and_eval_only=False):
    """The payload of one spawn: every case of world size W."""
    cases = []
    for case, E in RLTOOLS_CASES:
        for sizes in se.splits(E, W):
            for mode in MODES:
                cases.append((("rltools", case, sizes, mode), se.rank_rltools, (case, sizes, mode)))
    for case, E in RECURRENT_E.items():
        for sizes in se.splits(E, W):
            for run in se.RECURRENT_RUNS:
                for bf16 in se.RECURRENT_BF16[case]:
                    cases.append((("recurrent", case, sizes, run, bf16), se.rank_recurrent, (case, sizes, run, bf16)))
    for case, E in CONCURRENT_CASES:
        for sizes in se.splits(E, W):
            for shared in (False, True):
                cases.append((("concurrent", case, sizes, shared), se.rank_concurrent, (case, sizes, shared)))
    if W <= 3:
        cases.append((("eval_golden",), se.rank_eval_golden, (W,)))
        cases.append((("evaluations",), se.rank_evaluations, ()))
    if golden_and_eval_only:
        return cases
    for i, rows in enumerate(se.MOMENT_ROWS[W]):
        for A in (1, 3, 32):
            cases.append((("moments", rows, A), se.rank_moments, (rows, A, SEED + A, i == 0 and A != 32)))
    for A in (1, 3):
        for L in se.TB_LS:
            for with_t0 in (False, True):
                cases.append((("time_baseline", A, L, with_t0), se.rank_time_baseline,
                              (se.TB_SIZES[W], A, L, with_t0, SEED + L)))
    for mode in MODES:
        cases.append((("process_t0", mode), se.rank_process_t0, (mode, se.splits(4, W)[0], SEED)))
    for E in (3, 4):
        for sizes in se.splits(E, W)[:1]:
            for bf16 in (False, True):
                cases.append((("standardizers", sizes, bf16), se.rank_standardizers, (sizes, bf16, SEED + E)))
    cases.append((("paths", se.splits(4, W)[-1]), se.rank_paths, (se.splits(4, W)[-1], SEED)))
    if W == 2:
        cases.append((("refusals",), se.rank_refusals, ()))
    if W == 4:
        cases.append((("subgroups",), se.rank_subgroups, ()))
    return cases


@pytest.fixture(scope="module", params=(2, 3, 4), ids=lambda w: "W%d" % w)
def gloo(request):
    W = request.param
    return W, se.run_ranks(W, "gloo", se.run_cases, cases_for(W))


def keys(got, kind):
    return [k for k in got[0] if isinstance(k, tuple) and k[0] == kind]


def each(got, kind, check, required=True):
    """check(key, {rank: result}) for every case of `kind`; a failure names its case.  A world size without such
    a case skips the test (`required`) or checks nothing."""
    ks = keys(got, kind)
    if not ks and required:
        pytest.skip("no %s case at %d ranks" % (kind, len(got)))
    for key in ks:
        res = se.result(got, key)
        try:
            check(key, res)
        except AssertionError as ex:
            raise AssertionError("case %r: %s" % (key, ex)) from ex


def same_on_every_rank(res, pick=lambda x: x, what="pooled"):
    for r in range(1, len(res)):
        se.bits_equal(pick(res[0]), pick(res[r]), what)


def bits_same(a, b):
    try:
        se.bits_equal(a, b)
    except AssertionError:
        return False
    return True


def close(got, want, scale_of, rtol, what):
    """allclose with an absolute floor at rtol of the whole batch's largest |value| (want may be a slice)."""
    scale = max(rtol * float(np.max(np.abs(scale_of))), 1e-30)
    np.testing.assert_allclose(got, want, rtol=rtol, atol=scale, err_msg=what)


def state_ulps(got, want, what):
    """A float32 standardiser state (count, mean, meansq): count exact, the others within one ulp."""
    assert np.array_equal(np.asarray(got[0]), np.asarray(want[0]).reshape(np.shape(got[0]))), what
    assert se.ulps(got[1], np.reshape(want[1], np.shape(got[1]))) <= 1, what
    assert se.ulps(got[2], np.reshape(want[2], np.shape(got[2]))) <= 1, what


# ---------------------------------------------------------------- (a) golden training loops

@functools.lru_cache(maxsize=None)
def rltools_full(case, mode):
    return se.rltools_loop(DEV, None, case, mode)


def check_rltools(got, required=True):
    golden = np.load(se.GOLDEN + "/rltools_samples_ref.npz")

    def check(key, res):
        _, case, sizes, mode = key
        settings, rollouts = se.rltools_golden(case)
        full = rltools_full(case, mode)
        oracle = list(ro.replay(settings, rollouts, mode))
        pm = "decentralized" if mode == "zero" else mode
        A = rollouts[0]["obs"].shape[2]
        nb = A if pm == "concurrent" else 1
        sub = lambda b: "a%d/" % b if pm == "concurrent" else ""                        # noqa: E731
        pick = lambda x, b: x[b] if pm == "concurrent" else x                           # noqa: E731
        for k, (_, ores, _, _) in enumerate(oracle):
            gk = "%s/%s/r%d/" % (case, mode, k)
            recs = [res[r][k] for r in range(len(res))]
            same_on_every_rank(recs, lambda x: {n: v for n, v in x.items()
                                                if n not in ("q", "advantages", "values")}, gk)
            r0, fk = recs[0], full[k]
            if ores is not None:
                done = rollouts[k]["done"]
                split = lambda flat, b: np.split(flat, np.cumsum([len(x) for x in ores[b]["q"]])[:-1])  # noqa: E731
                want = dict(q=ro.to_rollout([split(golden[gk + sub(b) + "q"], b) for b in range(nb)], done, A, pm),
                            advantages=ro.to_rollout([split(golden[gk + sub(b) + "adv"], b) for b in range(nb)],
                                                     done, A, pm),
                            values=ro.to_rollout([o["v"] for o in ores], done, A, pm))
                # the rows of each rank: the golden's rows of its envs (the unsharded test's tolerances), and the
                # unsharded device call's bits where the inputs they depend on are the same bits
                same_rewnorm = "rewnorm" not in fk or bits_same(res[0][k - 1]["rewnorm"], full[k - 1]["rewnorm"])
                for r, (lo, hi) in enumerate(se.bounds(sizes)):
                    for n in ("q", "advantages", "values"):
                        close(recs[r][n], want[n][:, lo:hi], want[n], 1e-5, gk + n)
                    if k == 1 and same_rewnorm:        # values are 0 before the first fit: q, adv, values bitwise
                        for n in ("q", "advantages", "values"):
                            assert np.array_equal(recs[r][n], fk[n][:, lo:hi]), gk + n
                    elif same_rewnorm:
                        assert np.array_equal(recs[r]["q"], fk["q"][:, lo:hi]), gk + "q"
                for b in range(nb):
                    st = golden[gk + sub(b) + "stats"]
                    assert abs(pick(r0["v_r"], b) - st[0]) < 1e-6 and abs(pick(r0["tv_r"], b) - st[1]) < 1e-6
                    assert pick(r0["fallback"], b) == bool(st[2])
                assert np.array_equal(r0["fallback"], fk["fallback"])
                if same_rewnorm:                       # tv_r depends on q and simplev only
                    np.testing.assert_allclose(r0["tv_r"], fk["tv_r"], rtol=1e-12, atol=1e-12)
                    if k == 1:
                        np.testing.assert_allclose(r0["v_r"], fk["v_r"], rtol=1e-12, atol=1e-12)
                if "w" in r0:
                    for b in range(nb):
                        gw = golden[gk + sub(b) + "w"]
                        np.testing.assert_allclose(pick(r0["w"], b), gw, rtol=1e-4, atol=1e-6 * np.max(np.abs(gw)))
                    assert np.abs(r0["w"] - fk["w"]).max() <= 1e-9 * np.abs(fk["w"]).max(), gk + "w"
            if "obsnorm" in r0:
                for b in range(nb):
                    g = golden[gk + sub(b) + "obsnorm"].astype(np.float32)
                    D = (len(g) - 1) // 2
                    state_ulps([pick(x, b) for x in r0["obsnorm"]], (g[0], g[1:1 + D], g[1 + D:]), gk + "obsnorm")
                state_ulps(r0["obsnorm"], fk["obsnorm"], gk + "obsnorm vs unsharded")
            if "rewnorm" in r0:
                g = golden[gk + "rewnorm"].astype(np.float32)
                state_ulps(r0["rewnorm"], (g[0], g[1:2], g[2:3]), gk + "rewnorm")
                state_ulps(r0["rewnorm"], fk["rewnorm"], gk + "rewnorm vs unsharded")
            if "fields" in r0:
                it = rollouts[k]
                for m, f in r0["fields"].items():
                    rew = it["rew_cent"] if m == "centralized" else it["rew"]
                    w = ro.sample_fields(ro.batches(it["obs"], rew.astype(np.float64), it["done"], None, m))
                    assert sorted(f) == sorted(w)
                    for n in ("batch", "avglen", "maxlen", "minlen"):
                        assert f[n] == w[n] == fk["fields"][m][n], (m, n)
                    for n in ("ret", "ravg"):
                        assert abs(f[n] - w[n]) <= 1e-12 * max(1.0, abs(w[n])), (m, n)
                        assert np.isclose(f[n], fk["fields"][m][n], rtol=1e-12, atol=0), (m, n)

    each(got, "rltools", check, required)


def golden_rows(done, lo, hi, per_episode):
    """Rows [p0, p1) of the golden's padded arrays that hold envs [lo, hi): paths in (env, episode[, agent]) order,
    `per_episode` rows per episode; and the longest path of those envs."""
    recs = se.pe.path_records(done, 1)
    before = int((recs[:, 0] < lo).sum())
    mine = recs[(recs[:, 0] >= lo) & (recs[:, 0] < hi)]
    return per_episode * before, per_episode * (before + len(mine)), int(mine[:, 3].max())


@functools.lru_cache(maxsize=None)
def recurrent_full(case, run, bf16):
    return se.recurrent_loop(DEV, None, case, run, bf16)


def check_recurrent(got, required=True):
    def check(key, res):
        _, case, sizes, run, bf16 = key
        z, its, _, _ = se.recurrent_golden(case)
        full = recurrent_full(case, run, bf16)
        mode = run.split("_")[0]
        A = its[0]["obs"].shape[2]
        for n, it in enumerate(its):
            pre = "%s/%s/it%d/" % (case, run, n)
            lists = [pre + "a%d/" % a for a in range(A)] if mode == "concurrent" else [pre]
            same_on_every_rank([res[r][n] for r in range(len(res))],
                               lambda x: (x["coeffs"], [lst["stats"] for lst in x["lists"]]), pre)
            fc = full[n]["coeffs"]
            assert np.abs(res[0][n]["coeffs"] - fc).max() <= 1e-9 * np.abs(fc).max(), pre + "coeffs"
            for j, gk in enumerate(lists):
                gret, gadv = z[gk + "returns"], z[gk + "advantages"]
                for r, (lo, hi) in enumerate(se.bounds(sizes)):
                    p0, p1, longest = golden_rows(it["done"], lo, hi, A if mode == "decentralized" else 1)
                    mine = res[r][n]["lists"][j]
                    L = mine["valids"].shape[-1]
                    assert L == longest, (r, L, longest)                 # padded to the rank's own longest path
                    for k in ("observations", "valids"):
                        assert np.array_equal(mine[k], z[gk + k][p0:p1, :L]), (r, k)
                    assert np.allclose(mine["returns"], gret[p0:p1, :L], rtol=1e-5, atol=1e-5 * np.abs(gret).max())
                    assert np.allclose(mine["advantages"], gadv[p0:p1, :L], rtol=1e-4,
                                       atol=1e-4 * np.abs(gadv).max())
                    for k in ("valids", "returns", "advantages", "observations"):      # the rest is padding
                        assert not z[gk + k][p0:p1, L:].any(), (r, k)
                stats = res[0][n]["lists"][j]["stats"]
                fstats = full[n]["lists"][j]["stats"]
                want = dict(zip(se.RECURRENT_STATS, z[gk + "stats"]))
                for k in se.EXACT_STATS:
                    assert np.isclose(stats[k], want[k], rtol=1e-12, atol=0), k
                    assert np.isclose(stats[k], fstats[k], rtol=1e-12, atol=0), k
                assert np.isclose(stats["AverageDiscountedReturn"], want["AverageDiscountedReturn"], rtol=1e-5,
                                  atol=1e-5 * np.abs(gret).max())
                assert np.isclose(stats["AverageDiscountedReturn"], fstats["AverageDiscountedReturn"], rtol=1e-12,
                                  atol=0)
                assert np.isclose(stats["ExplainedVariance"], want["ExplainedVariance"], rtol=1e-4, atol=1e-4)
                if n == 0 and not run.endswith("shared"):        # predictions are 0 before the first fit
                    assert np.isclose(stats["ExplainedVariance"], fstats["ExplainedVariance"], rtol=1e-12, atol=0)

    each(got, "recurrent", check, required)


@functools.lru_cache(maxsize=None)
def concurrent_full(case, shared):
    return se.concurrent_loop(DEV, None, case, shared)


def check_concurrent(got, required=True):
    def check(key, res):
        _, case, sizes, shared = key
        z, its, d, gl, center, positive = se.concurrent_golden(case)
        full = concurrent_full(case, shared)
        W = len(res)
        chain = cbo.concurrent_chain(its, shared, d, gl, center, positive, fits=[res[0][n]["fit"] for n in range(2)])
        for n, (it, ch) in enumerate(zip(its, chain)):
            same_on_every_rank([res[r][n] for r in range(W)], lambda x: (x["ev"], x["fit"]), "it%d" % n)
            whole = {k: np.concatenate([res[r][n][k] for r in range(W)], axis=1) for k in ("values", "adv", "ret")}
            assert np.allclose(whole["values"], ch["values"], rtol=1e-5, atol=1e-5 * np.abs(ch["values"]).max() +
                               1e-30)
            assert np.allclose(whole["ret"], ch["returns"], rtol=1e-5, atol=1e-5 * np.abs(ch["returns"]).max())
            assert np.allclose(whole["adv"], ch["advantages"], rtol=1e-4, atol=1e-4 * np.abs(ch["advantages"]).max())
            assert np.allclose(res[0][n]["ev"], ch["ev"], rtol=1e-4, atol=1e-4)
            rows, _ = cbo.agent_path_rows(it["done"])
            flavour = "shared" if shared else "independent"
            for a in range(it["obs"].shape[2]):
                g = z["%s/%s/it%d/ret%d" % (case, flavour, n, a)]
                assert np.allclose(whole["ret"][:, :, a].reshape(-1)[rows], g, rtol=1e-5, atol=1e-5 * np.abs(g).max())
                if n == 0 and not shared:
                    assert not whole["values"][:, :, a].any() and not z["%s/independent/it0/pred%d" % (case, a)].any()
            f = full[n]
            assert np.array_equal(whole["ret"], f["ret"])              # returns do not depend on the fit
            assert np.abs(res[0][n]["fit"] - f["fit"]).max() <= 1e-9 * np.abs(f["fit"]).max()
            if n == 0 and not shared:
                assert np.array_equal(whole["values"], f["values"])
                np.testing.assert_allclose(res[0][n]["ev"], f["ev"], rtol=1e-12, atol=1e-12)

    each(got, "concurrent", check, required)


# ---------------------------------------------------------------- (c) evaluation

def check_eval_golden(got, required=True):
    g, c = se.eval_golden()

    def check(key, res):
        same_on_every_rank(res)
        for chunk, d in res[0].items():
            for k in ("ret", "retstd", "disc_ret"):
                assert np.abs(d[k] - g[k]).max() < 1e-9, (chunk, k)
            for j, k in enumerate(g["info_keys"]):
                assert np.array_equal(d[str(k)], g["info"][:, j]), (chunk, k)

    each(got, "eval_golden", check, required)


@functools.lru_cache(maxsize=None)
def evaluations_full():
    return se.evaluations(DEV, None)


def check_evaluations(got, required=True):
    def check(key, res):
        full = evaluations_full()
        assert sorted(res[0], key=str) == sorted(full, key=str)
        for r in res:
            se.bits_equal(res[r], full, "rank %d" % r)

    each(got, "evaluations", check, required)


# ---------------------------------------------------------------- the tests


def test_rltools_training_loop_over_env_shards(gloo):
    check_rltools(gloo[1])


def test_recurrent_batches_over_env_shards(gloo):
    check_recurrent(gloo[1])


def test_concurrent_linear_baseline_over_env_shards(gloo):
    check_concurrent(gloo[1])


def test_moments_centring_and_explained_variance_against_float64(gloo):
    def check(key, res):
        _, rows, A = key
        same_on_every_rank(res, lambda x: {k: v for k, v in x.items() if k != "ca"})
        parts = [se.moment_shard(n, A, r, SEED + A) for r, n in enumerate(rows)]
        x, y = np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])
        want = se.moments_of(x, y)
        tol = dict(rtol=1e-10, atol=1e-12 * np.abs(want).max())
        np.testing.assert_allclose(res[0]["ma"], want, **tol)
        assert np.array_equal(res[0]["ma"][:, 6:9], want[:, 6:9])                # minima exactly
        np.testing.assert_allclose(res[0]["ma_nob"][:, [0, 3, 6]], want[:, [0, 3, 6]], **tol)
        from madrl_b200 import postproc as pp
        unsharded = pp.moments_agents(torch.from_numpy(x).to(DEV), torch.from_numpy(y).to(DEV)).cpu().numpy()
        np.testing.assert_allclose(res[0]["ma"], unsharded, rtol=1e-12, atol=1e-14 * np.abs(want).max())
        if A == 1:
            np.testing.assert_allclose(res[0]["m"], want[0], **tol)
            np.testing.assert_allclose(res[0]["m_nob"][[0, 3, 6]], want[0, [0, 3, 6]], **tol)
        if "ev" not in res[0]:
            return
        assert int(np.argmin(x.min(1))) >= rows[0]                               # the minimum is not rank 0's
        ev, ev_a = res[0]["ev"]
        assert abs(ev - po.explained_variance_1d(x.ravel(), y.ravel())) <= 1e-10
        assert np.allclose(ev_a, [po.explained_variance_1d(x[:, a], y[:, a]) for a in range(A)], rtol=0, atol=1e-10)
        for (c, p, pa) in res[0]["ca"]:
            got_ = np.concatenate([res[r]["ca"][c, p, pa] for r in range(len(res))])
            want_ = (np.stack([se.centred_want(x[:, a], c, p) for a in range(A)], 1) if pa else
                     se.centred_want(x.ravel(), c, p).reshape(x.shape))
            assert se.ulps(got_, want_.astype(np.float32)) <= 1, (c, p, pa)

    each(gloo[1], "moments", check)


def test_time_baseline_bins_over_uneven_shards(gloo):
    W = gloo[0]
    sizes = se.TB_SIZES[W]

    def check(key, res):
        _, A, L, with_t0 = key
        q, done, t0 = se.tb_case(sizes, A, L, with_t0, SEED + L)
        lo1, hi1 = se.bounds(sizes)[1]
        own = se.pe.time_index(done[:, lo1:hi1], None if t0 is None else t0[lo1:hi1])[0].max() + 1
        assert own < 128 and int(se.pe.time_index(done, t0)[0].max()) + 1 == L
        for pa in (False, True):
            same_on_every_rank(res, lambda x: x[pa][1:], "bins")
            simplev = np.concatenate([res[r][pa][0] for r in range(W)], axis=1)
            se.pe.check_time_baseline(simplev, res[0][pa][1], res[0][pa][2], q, done, t0, pa)

    each(gloo[1], "time_baseline", check)


@functools.lru_cache(maxsize=None)
def process_t0_full(mode, E):
    return se.process_t0_loop(DEV, None, mode, E, SEED)


def test_process_samples_with_t0_in_every_mode(gloo):
    W = gloo[0]
    sizes = se.splits(4, W)[0]

    def check(key, res):
        mode = key[1]
        full = process_t0_full(mode, sum(sizes))
        for i in range(2):
            recs = [res[r][i] for r in range(W)]
            same_on_every_rank(recs, lambda x: (x["v_r"], x["tv_r"], x["fallback"], x["w"]), "call %d" % i)
            f = full[i]
            tight = i == 0 or mode == "zero"         # predictions are 0: nothing depends on the pooled fit
            for r, (lo, hi) in enumerate(se.bounds(sizes)):
                assert np.array_equal(recs[r]["q"], f["q"][:, lo:hi])
                for n in ("advantages", "values"):
                    if tight:
                        assert np.array_equal(recs[r][n], f[n][:, lo:hi]), n
                    else:
                        close(recs[r][n], f[n][:, lo:hi], f[n], 1e-5, n)
            assert np.array_equal(recs[0]["fallback"], f["fallback"])
            np.testing.assert_allclose(recs[0]["tv_r"], f["tv_r"], rtol=1e-12, atol=1e-12)
            np.testing.assert_allclose(recs[0]["v_r"], f["v_r"], rtol=1e-12 if tight else 1e-6,
                                       atol=1e-12 if tight else 1e-6)
            if f["w"] is not None:
                assert np.abs(recs[0]["w"] - f["w"]).max() <= 1e-9 * np.abs(f["w"]).max()

    each(gloo[1], "process_t0", check)


@functools.lru_cache(maxsize=None)
def standardizers_full(E, bf16):
    return se.standardizer_states(DEV, None, E, bf16, SEED + E)


def test_standardisers_against_the_oracle_on_the_whole_batch(gloo):
    def check(key, res):
        _, sizes, bf16 = key
        E = sum(sizes)
        same_on_every_rank(res)
        want, full = se.standardizer_want(E, bf16, SEED + E), standardizers_full(E, bf16)
        for b in range(2):
            for k in ("update", "agents", "per_agent", "obsnorm"):
                state_ulps(res[0][b][k], want[b][k], (b, k))
                state_ulps(res[0][b][k], full[b][k], (b, k, "unsharded"))

    each(gloo[1], "standardizers", check)


def test_path_statistics_and_sample_fields(gloo):
    def check(key, res):
        sizes = key[1]
        same_on_every_rank(res)
        rew, done = se.paths_case(sizes, SEED)
        T, E, A = rew.shape
        full = se.path_outputs(DEV, None, sizes, SEED)
        recs = se.pe.path_records(done, A)
        sums = np.array([rew[s:s + n, e, a].astype(np.float64).sum() for e, a, s, n in recs])
        longest, shortest = recs[np.argmax(recs[:, 3])], recs[np.argmin(recs[:, 3])]
        ranks = [next(r for r, (lo, hi) in enumerate(se.bounds(sizes)) if lo <= p[0] < hi) for p in (longest,
                                                                                                     shortest)]
        assert ranks[0] != ranks[1]
        for pa, (g, w) in enumerate(zip(res[0]["stats"], full["stats"])):
            gl, wl = (g, w) if pa else ([g], [w])
            for a, (gd, wd) in enumerate(zip(gl, wl)):
                s = sums[recs[:, 1] == a] if pa else sums
                for k in ("NumTrajs", "MaxReturn", "MinReturn"):
                    assert gd[k] == wd[k], k
                assert gd["NumTrajs"] == len(s) and gd["MaxReturn"] == s.max() and gd["MinReturn"] == s.min()
                for k, v in (("AverageReturn", s.mean()), ("StdReturn", s.std())):
                    assert np.isclose(gd[k], v, rtol=1e-10, atol=1e-12 * np.abs(s).max()), k
                for k in ("AverageReturn", "StdReturn", "AverageDiscountedReturn"):
                    assert np.isclose(gd[k], wd[k], rtol=1e-12, atol=0), k
        for m, f in res[0]["fields"].items():
            r64 = (np.repeat(rew[..., :1], A, 2) if m == "centralized" else rew).astype(np.float64)
            w = ro.sample_fields(ro.batches(np.zeros((T, E, A, 1), np.float32), r64, done, None, m))
            for k in ("batch", "avglen", "maxlen", "minlen"):
                assert f[k] == w[k] == full["fields"][m][k], (m, k)
            for k in ("ret", "ravg"):
                assert abs(f[k] - w[k]) <= 1e-12 * max(1.0, abs(w[k])), (m, k)
                assert np.isclose(f[k], full["fields"][m][k], rtol=1e-12, atol=0), (m, k)

    each(gloo[1], "paths", check)


def test_fp64_heuristic_evaluation_over_shards_is_the_golden(gloo):
    if gloo[0] > 3:
        pytest.skip("the golden batch has 3 envs")
    check_eval_golden(gloo[1])


def test_evaluate_policy_over_shards_is_the_unsharded_dict(gloo):
    if gloo[0] > 3:
        pytest.skip("covered at W = 2 and 3")
    check_evaluations(gloo[1])


def test_refusals_of_shards_that_do_not_tile_the_batch(gloo):
    if gloo[0] != 2:
        pytest.skip("the two-rank world; the four-rank world checks them inside its subgroups")

    def check(key, res):
        for r in res:
            assert res[r]["swapped"] == "refused" and res[r]["mixed"] == "refused", res[r]
        same_on_every_rank(res, lambda x: x["after"], "after")

    each(gloo[1], "refusals", check)


@functools.lru_cache(maxsize=None)
def subgroup_full(k):
    seed, eval_seed, pe_seed = se.SUBGROUP_SEEDS[k]
    return se.pooled_suite(DEV, None, E_G=se.SUBGROUP_E, T=30, seed=seed, eval_seed=eval_seed, pe_seed=pe_seed)


def test_two_groups_inside_a_four_rank_world(gloo):
    if gloo[0] != 4:
        pytest.skip("needs four ranks")

    def check(key, res):
        for k in range(2):
            members = [r for r in res if res[r]["group"] == k]
            assert members == [2 * k, 2 * k + 1]
            se.check_pooled({i: res[r]["suite"] for i, r in enumerate(members)}, subgroup_full(k), se.SUBGROUP_E)
            for r in members:
                ref = res[r]["refusals"]
                assert ref["swapped"] == ref["mixed"] == ref["world_shards"] == "refused", (r, ref)
            same_on_every_rank({i: res[r]["refusals"]["after"] for i, r in enumerate(members)})
        assert not np.array_equal(res[0]["suite"]["mom"], res[2]["suite"]["mom"])      # nothing leaks across groups
        assert not np.array_equal(res[0]["suite"]["rew"], res[2]["suite"]["rew"])

    each(gloo[1], "subgroups", check)


def test_peak_device_memory_per_rank(gloo):
    W, got = gloo
    peaks = [got[r]["peak_bytes"] for r in range(W)]
    print("W=%d peak torch.cuda.max_memory_allocated per rank (MB): %s" % (W, [round(p / 2 ** 20, 1) for p in peaks]))
    assert max(peaks) < 2 * 2 ** 30


@pytest.fixture(scope="module")
def nccl():
    W = min(4, torch.cuda.device_count())
    if W < 2:
        pytest.skip("NCCL needs two GPUs")
    return se.run_ranks(W, "nccl", se.run_cases, cases_for(W, golden_and_eval_only=True))


def test_nccl_golden_loops_and_evaluations(nccl):
    for check in (check_rltools, check_recurrent, check_concurrent, check_eval_golden, check_evaluations):
        check(nccl, required=False)
