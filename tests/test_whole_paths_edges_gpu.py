"""Whole-path sampling (madrl_b200/whole_paths.py, DESIGN §4.9) on the GPU at the edges of its kernels, its launches,
its observation wrappers, its recurrent state and its ranks.

* Kernel level: every scripted stream of tests/whole_paths_edges.py (1 to 4097 envs: the fold's and scan's 256-env
  strides, the rows kernel's 128-thread blocks; t* on the first, last or a middle step of a launch; batch_size 1,
  equal to a count, one more, the whole stream; length-1 paths at t*; an env that ends launches after the others)
  through `_Selection`: acc, path_start, done, env_rows and the gathered tensors bit for bit against the vectorised
  oracle; every cell of the gather's word / thread-or-warp dispatch, with `first` only 4- or 2-byte aligned and a
  sentinel-filled destination; a fold after completion leaves acc and carry alone; the stream that needs the most
  steps completes at max_steps(), one step more raises before any fold.
* Sampler level, against one long PolicyRollout of the same seed (chained calls where it is too big): chunk 1, 7,
  mpl and one launch, graph and eager replay, C3 and C5, float32 and bfloat16; a GRU's state across launches and
  resets; frame_stack 2 and 4 with and without a standardiser (the stacked obs and obs_before, the standardiser's
  float64 state byte for byte); two calls in a row (the first batch unchanged, its done view still its own); the
  product shapes C2 (E = 4096, mpl 500, batch_size 12000, chunk 64) and C3 at E = 4096 with their peak device
  memory; the sampler's refusals.
* Processing on the flat view of a C3 batch (E = 256, paths up to mpl) against the float64 oracles of oracle/: gae,
  the linear feature baseline (plain and per agent), rltools' time baseline and path_statistics.
* Pooled processing of whole-path batches over W = 2 and 3 gloo ranks (uneven shards: a single-path rank, a rank
  with the longest path, a rank of 257 envs): process_samples_concurrent, process_samples_recurrent (both modes)
  and rltools' process_samples with ``group=``, the same bytes on every rank and the unsharded call's results on
  the ranks' batches concatenated into one [sum N, 1] rollout.
"""
import numpy as np
import pytest
import torch

import postproc_edges as pe
import sharded_edges as se
import whole_paths_edges as wpe
from madrl_b200 import WholePathSampler, _lib, postproc, rltools_sampler
from madrl_b200._lib import _ptr
from madrl_b200.closed_loop import PolicyRollout
from madrl_b200.whole_paths import _Selection, whole_paths_of
from oracle import baseline_oracle as bo
from oracle import postproc_oracle as po
from oracle import whole_paths_oracle as wo
from test_closed_loop_gpu import GRUPolicy
from test_whole_paths_gpu import Policy, engine

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda", 0)


def _np(x):
    return x.view(torch.int16).cpu().numpy() if x.dtype == torch.bfloat16 else x.cpu().numpy()


def _dev(x):
    return torch.from_numpy(np.ascontiguousarray(x)).to(DEV)


def _at_offset(x, off):
    """x on the device at `off` bytes past a 16-byte boundary, a view of a larger buffer."""
    buf = torch.empty(x.nbytes + 64, dtype=torch.uint8, device=DEV)
    v = buf[off:off + x.nbytes].view(_torch_dtype(x.dtype)).view(x.shape)
    v.copy_(_dev(x))
    assert v.data_ptr() % 16 == off
    return v


def _torch_dtype(dt):
    return {np.dtype(np.float32): torch.float32, np.dtype(np.int32): torch.int32, np.dtype(np.uint16): torch.int16,
            np.dtype(np.uint8): torch.uint8}[np.dtype(dt)]


def _t(x):
    return _dev(x.view(np.int16) if x.dtype == np.uint16 else x)


# ---------------------------------------------------------------- kernel level

def select_on_device(done, bs, T, S_run=None):
    """Fold `done` in launches of T through _Selection with random launch tensors -> (selection, batch, the
    sources name -> (x [S, E, ...], first or None) of the batch's fields)."""
    S, E = done.shape
    S_run = -(-S // T) * T if S_run is None else S_run
    d = np.zeros((S_run + T, E), np.uint8)
    d[:S] = done
    A = 3
    rs = np.random.RandomState(E)
    x = _dev(rs.randn(S_run + T, E, A, 4).astype(np.float32))
    x0 = _dev(rs.randn(E, A, 4).astype(np.float32))
    act = _dev(rs.randint(0, 5, (S_run + T, E, A)).astype(np.int32))
    rew = _dev(rs.randn(S_run + T, E, A).astype(np.float32))
    info = _dev(rs.randint(0, 9, (S_run + T, E, 2)).astype(np.int32))
    dd = _dev(d)
    sel = _Selection(E, T, bs, S_run, DEV)
    first = x0
    j = 0
    while True:
        sl = slice(j * T, (j + 1) * T)
        if sel.add(first, x[sl].clone(), act[sl].clone(), rew[sl].clone(), dd[sl].contiguous(), info[sl].clone(),
                   {"rew2": rew[sl].clone()}):
            break
        first = x[(j + 1) * T - 1].clone()
        j += 1
    return sel, sel.batch(), dict(obs=(x, x0), actions=(act, None), rew=(rew, None), infos=(info, None))


@pytest.mark.parametrize("s", wpe.STREAMS, ids=[s.name for s in wpe.STREAMS])
def test_selection_and_gather_match_oracle(s):
    t_star, end = wpe.selection(s)
    sel, batch, src = select_on_device(s.done, s.batch_size, s.T)
    acc = sel.acc.cpu().numpy()
    N = int(np.sum(end + 1))
    assert acc[1] == t_star and acc[2] == 1 and acc[3] == N and batch.t_star == t_star
    assert batch.n_steps == wpe.launches(s) * s.T
    np.testing.assert_array_equal(batch.path_start.cpu().numpy(), wo.path_start_np(s.done, end))
    np.testing.assert_array_equal(batch.done.cpu().numpy(), wo.take(s.done, end))
    np.testing.assert_array_equal(batch.env_rows.cpu().numpy(), wo.env_rows(end))
    for k, (x, first) in src.items():
        got = getattr(batch, k).cpu().numpy()
        want = wo.take(x.cpu().numpy(), end, None if first is None else first.cpu().numpy())
        assert got.tobytes() == want.tobytes(), k
    assert batch.extras["rew2"].cpu().numpy().tobytes() == wo.take(src["rew"][0].cpu().numpy(), end).tobytes()
    # a fold after completion returns on acc[2]: acc and carry unchanged
    acc0, carry0 = sel.acc.clone(), sel.carry.clone()
    ones = torch.ones((s.T, s.done.shape[1]), dtype=torch.uint8, device=DEV)
    _lib.check(_lib.lib().madrl_whole_paths_fold(s.T, s.done.shape[1], sel.n_steps, sel.batch_size, _ptr(ones),
                                                 _ptr(sel.carry), _ptr(sel.acc), _lib.stream(DEV)))
    assert torch.equal(sel.acc, acc0) and torch.equal(sel.carry, carry0)
    # every gather cell, into a sentinel-filled destination, `first` at 4- or 2-byte alignment
    if s.done.shape[1] > 600:
        return
    T, E = s.T, s.done.shape[1]
    S_run = len(sel.launches) * T
    cells = set()
    for k, (x, first, off) in wpe.gather_inputs(S_run, E, 7).items():
        slab = x[0, 0].nbytes
        src_d, dst = _t(x), torch.full((N * slab,), wpe.SENTINEL, dtype=torch.uint8, device=DEV)
        for j in range(len(sel.launches)):
            part = src_d[j * T:(j + 1) * T].contiguous()
            fst = None
            if first is not None:
                fst = _at_offset(first if j == 0 else x[j * T - 1], off)
            cells.add(wpe.gather_cell(slab, [part.data_ptr(), dst.data_ptr()] + ([] if fst is None else
                                                                                  [fst.data_ptr()])))
            _lib.check(_lib.lib().madrl_whole_paths_gather(T, E, slab, j * T, _ptr(part), _ptr(fst), _ptr(sel.carry),
                                                           _ptr(batch.env_rows), _ptr(dst), _lib.stream(DEV)))
        wpe.check_gathered(dst.cpu().numpy().view(x.dtype).reshape((N,) + x.shape[2:]), x, end, first)
    assert cells == wpe.ALL_CELLS


@pytest.mark.parametrize("T", [1, 4])
def test_worst_stream_at_the_capacity_of_max_steps(T):
    done, bs, cap, tight, over = wpe.worst_case(T=T)
    t_star, end = wo.select(done, bs)
    for stream in (done, tight):
        sel, batch, _ = select_on_device(stream, bs, T, S_run=cap)
        assert sel.done_stage.shape[0] == cap and batch.t_star == t_star
        e2 = wo.select(stream, bs)[1]
        np.testing.assert_array_equal(batch.path_start.cpu().numpy(), wo.path_start_np(stream, e2))
    # one step past the capacity: add raises before it copies or folds anything
    sel = _Selection(done.shape[1], T, bs, cap, DEV)
    d = _dev(over)
    x = torch.zeros((T, done.shape[1], 3, 4), device=DEV)
    for j in range(cap // T):
        assert not sel.add(x[0], x.clone(), x[..., 0].clone(), x[..., 0].clone(), d[j * T:(j + 1) * T].contiguous(),
                           x[..., 0, 0].int(), {})
    stage, acc = sel.done_stage.clone(), sel.acc.clone()
    with pytest.raises(RuntimeError):
        sel.add(x[0], x.clone(), x[..., 0].clone(), x[..., 0].clone(), torch.ones_like(d[:T]), x[..., 0, 0].int(), {})
    assert torch.equal(sel.done_stage, stage) and torch.equal(sel.acc, acc) and sel.done_stage.shape[0] == cap


# ---------------------------------------------------------------- sampler level

def long_rollout(eng, policy, steps, chunk=None, state0=None, frame_stack=1, standardizer=None, keep=None):
    """One long PolicyRollout from reset, as chained calls of `chunk` steps: (first [E, A, W], done, actions, rew,
    info, extras, policy_obs [S, E, A, W]) as NumPy (policy_obs only for the envs `keep`)."""
    chunk = steps if chunk is None else chunk
    o = eng.reset()
    if standardizer is not None:
        standardizer.obs(o)
    obs0 = o if frame_stack == 1 else postproc.FrameStack(eng.n_envs, eng._n_acting, eng.obs_dim, frame_stack,
                                                          eng.device, eng.obs_dtype).reset(o)
    E, A = eng.n_envs, eng._n_acting
    first = _np(obs0.reshape(E, A, -1))
    loop = PolicyRollout(eng, policy, chunk, frame_stack=frame_stack, standardizer=standardizer)
    state = None if state0 is None else torch.zeros_like(state0)
    parts = []
    for _ in range(-(-steps // chunk)):
        r = loop(obs0, state)
        pobs = r.policy_obs.reshape(chunk, E, A, -1)
        parts.append(dict(done=_np(r.done), actions=_np(r.actions), rew=_np(r.rew), info=_np(r.info),
                          extras={k: _np(v) for k, v in r.extras.items()},
                          pobs=_np(pobs if keep is None else pobs[:, keep])))
        obs0, state = r.policy_obs[-1].clone(), r.state
    cat = {k: np.concatenate([p[k] for p in parts]) for k in ("done", "actions", "rew", "info", "pobs")}
    cat["extras"] = {k: np.concatenate([p["extras"][k] for p in parts]) for k in parts[0]["extras"]}
    cat["first"] = first if keep is None else first[keep]
    return cat


def check_batch(batch, ref, bs, keep=None):
    """The batch against the oracle selection of the long rollout `ref`."""
    t_star, end = wo.select(ref["done"][:batch.n_steps], bs)
    assert batch.t_star == t_star
    np.testing.assert_array_equal(batch.path_start.cpu().numpy(), wo.path_start_np(ref["done"], end))
    np.testing.assert_array_equal(batch.done.cpu().numpy(), wo.take(ref["done"], end))
    np.testing.assert_array_equal(batch.env_rows.cpu().numpy(), wo.env_rows(end))
    for got, want in ((batch.actions, ref["actions"]), (batch.rew, ref["rew"]), (batch.infos, ref["info"])):
        np.testing.assert_array_equal(_np(got), wo.take(want, end))
    for k, v in ref["extras"].items():
        np.testing.assert_array_equal(_np(batch.extras[k]), wo.take(v, end), err_msg=k)
    if keep is None:
        np.testing.assert_array_equal(_np(batch.obs), wo.take(ref["pobs"], end, ref["first"]))
    else:
        rows = wo.env_rows(end)
        for i, e in enumerate(keep):
            got = _np(batch.obs[rows[e]:rows[e] + end[e] + 1])
            want = np.concatenate([ref["first"][i][None], ref["pobs"][:end[e], i]])
            np.testing.assert_array_equal(got, want, err_msg="env %d" % e)
    return t_star, end


def _fields(b):
    return dict(obs=b.obs, actions=b.actions, rew=b.rew, infos=b.infos, path_start=b.path_start, done=b.done,
                env_rows=b.env_rows, extras=b.extras, t_star=b.t_star, obs_before=b.obs_before)


def _same(a, b, what):
    if isinstance(a, dict):
        assert a.keys() == b.keys(), what
        for k in a:
            _same(a[k], b[k], "%s.%s" % (what, k))
    elif torch.is_tensor(a):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), what
    else:
        assert a == b, what


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("fam", ["pe_c3", "hw_c5"])
def test_batch_does_not_depend_on_the_launch_length(fam, dtype):
    E, mpl = 24, 9
    obs_dtype = torch.bfloat16 if dtype == "bf16" else None
    bs = 3 * E + 7
    eng = engine(fam, E, mpl, obs_dtype=obs_dtype)
    one = WholePathSampler(eng, Policy(eng), bs, mpl, chunk=1).max_steps()     # >= max_steps() at any chunk
    batches = {}
    for chunk in (1, 7, mpl, one):
        for graph in ((True, False) if chunk == 7 else (True,)):
            eng = engine(fam, E, mpl, obs_dtype=obs_dtype)
            batches[(chunk, graph)] = WholePathSampler(eng, Policy(eng), bs, mpl, chunk=chunk, graph=graph)()
    assert batches[(one, True)].n_steps == one                                  # one launch
    ref = batches[(7, True)]
    eng = engine(fam, E, mpl, obs_dtype=obs_dtype)
    check_batch(ref, long_rollout(eng, Policy(eng), ref.n_steps), bs)
    for key, b in batches.items():
        _same(_fields(b), _fields(ref), str(key))


def test_recurrent_state_carries_across_launches():
    E, mpl, chunk = 24, 9, 5
    eng = engine("ww_c2", E, mpl)
    pol = GRUPolicy(eng.obs_dim)
    h0 = torch.randn(E, eng._n_acting, 16, device=DEV)
    bs = 4 * E * mpl
    batch = WholePathSampler(eng, pol, bs, mpl, chunk=chunk)(h0)
    assert batch.n_steps // chunk >= 8
    ref_eng = engine("ww_c2", E, mpl)
    ref = long_rollout(ref_eng, pol, batch.n_steps, state0=h0)
    check_batch(batch, ref, bs)
    assert (ref["done"].sum(0) >= 3).all()         # every env restarted its state several times


@pytest.mark.parametrize("dtype", ["f32", "bf16"])
@pytest.mark.parametrize("norm", [False, True], ids=["plain", "obsnorm"])
@pytest.mark.parametrize("B", [2, 4])
def test_frame_stack_and_standardizer(B, norm, dtype):
    E, mpl, chunk = 16, 9, 4
    obs_dtype = torch.bfloat16 if dtype == "bf16" else None
    eng = engine("ww_c2", E, mpl, obs_dtype=obs_dtype)
    A, D = eng._n_acting, eng.obs_dim

    def std():
        return postproc.Standardizer(E, A, D, DEV, enable_obsnorm=True, obs_alpha=0.05) if norm else None
    s1 = std()
    bs = 2 * E * mpl + 3
    batch = WholePathSampler(eng, _StackedPolicy(Policy(eng), B), bs, mpl, chunk=chunk, frame_stack=B,
                             standardizer=s1)()
    ref_eng, s2 = engine("ww_c2", E, mpl, obs_dtype=obs_dtype), std()
    ref = long_rollout(ref_eng, _StackedPolicy(Policy(ref_eng), B), batch.n_steps, frame_stack=B, standardizer=s2)
    check_batch(batch, ref, bs)
    assert batch.obs.shape == (len(batch), A, D * B)
    np.testing.assert_array_equal(_np(batch.obs_before), ref["first"][0])
    obs, done, rew, before = batch.as_rollout()
    assert obs.shape == (len(batch), 1, A, D * B) and before.shape == (1, A, D * B)
    if norm:
        for n in ("obs_mean", "obs_var"):
            assert getattr(s1, n).cpu().numpy().tobytes() == getattr(s2, n).cpu().numpy().tobytes(), n


class _StackedPolicy(object):
    """Policy on the stacked observation [E, A, D, B] (its newest slot), so the stacked input drives the env."""

    def __init__(self, inner, B):
        self.inner, self.B = inner, B

    def __call__(self, obs, state):
        return self.inner(obs[..., -1] if obs.dim() == 4 else obs, state)


def test_two_calls_in_a_row():
    E, mpl, chunk = 24, 9, 5
    eng = engine("pe_c3", E, mpl)
    bs = 2 * E + 5
    s = WholePathSampler(eng, Policy(eng), bs, mpl, chunk=chunk)
    b1 = s()
    keep = {k: (v.clone() if torch.is_tensor(v) else dict((kk, vv.clone()) for kk, vv in v.items()) if
                isinstance(v, dict) else v) for k, v in _fields(b1).items()}
    n1 = b1.n_steps
    b2 = s()
    _same(_fields(b1), keep, "first batch after the second call")
    d1 = b1.as_rollout()[1]
    assert whole_paths_of(d1) is b1 and whole_paths_of(b2.as_rollout()[1]) is b2
    assert all(torch.equal(x, y) for x, y in zip(b1.plan(), postproc._paths_plan(d1.clone(), 1)))
    ref_eng = engine("pe_c3", E, mpl)
    PolicyRollout(ref_eng, Policy(ref_eng), n1)(ref_eng.reset())
    ref = long_rollout(ref_eng, Policy(ref_eng), b2.n_steps)
    check_batch(b2, ref, bs)


def _peak(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    out = fn()
    torch.cuda.synchronize()
    return out, torch.cuda.max_memory_allocated() - base


def _run_bytes(eng, batch, B=1):
    """The bytes one lockstep step of the sampler writes: policy_obs, actions, rew, info, extras."""
    E, A = eng.n_envs, eng._n_acting
    row = A * eng.obs_dim * B * eng.obs_dtype.itemsize + batch.actions[0].nbytes + batch.rew[0].nbytes + \
        batch.infos[0].nbytes + sum(v[0].nbytes for v in batch.extras.values()) + 1
    return E * row * batch.n_steps


@pytest.mark.parametrize("fam,E,mpl,bs,chunk", [("ww_c2", 4096, 500, 12000, 64),
                                                ("pe_c3", 4096, 100, 4096 * 50, 64)], ids=["C2", "C3"])
def test_product_shape(fam, E, mpl, bs, chunk):
    eng = engine(fam, E, mpl)
    s = WholePathSampler(eng, Policy(eng), bs, mpl, chunk=chunk)
    batch, peak = _peak(s)
    ran = _run_bytes(eng, batch)
    print("%s: %d steps, %d rows, %d paths; peak %.2f GB over %.2f GB of rows the sampler ran (%.2fx)" % (
        fam, batch.n_steps, len(batch), batch.n_paths, peak / 1e9, ran / 1e9, peak / ran))
    assert peak <= 2.5 * ran + (256 << 20)
    keep = [0, 255, 256, 257, 4095]
    ref_eng = engine(fam, E, mpl)
    ref = long_rollout(ref_eng, Policy(ref_eng), batch.n_steps, chunk=chunk, keep=keep)
    check_batch(batch, ref, bs, keep=keep)


def test_refusals():
    eng = engine("hw_c5", 4, 9)
    for bs in (0, -3, 2.5):
        with pytest.raises(ValueError):
            WholePathSampler(eng, Policy(eng), bs, 9)
    with pytest.raises(ValueError):
        WholePathSampler(eng, Policy(eng), 10, 9, chunk=0)
    sel = _Selection(2, 3, 10, 3, DEV)
    z = torch.zeros((3, 2), device=DEV)
    assert not sel.add(z[0], z.clone(), z.clone(), z.clone(), torch.zeros((3, 2), dtype=torch.uint8, device=DEV),
                       z.int(), {})
    with pytest.raises(RuntimeError):
        sel.add(z[0], z.clone(), z.clone(), z.clone(), torch.zeros((3, 2), dtype=torch.uint8, device=DEV), z.int(),
                {})


# ---------------------------------------------------------------- processing on the flat view

@pytest.fixture(scope="module")
def pe_batch():
    E, mpl = 256, 40
    eng = engine("pe_c3", E, mpl)
    batch = WholePathSampler(eng, Policy(eng), 4 * E * 10, mpl, chunk=16)()
    assert int(np.diff(batch.path_start.cpu().numpy()).max()) == mpl
    return batch


def test_processing_against_float64_oracles(pe_batch):
    b = pe_batch
    obs, done, rew, ob = b.as_rollout()
    N, _, A, D = obs.shape
    rs = np.random.RandomState(3)
    vals = rs.randn(N, 1, A).astype(np.float32)
    d, r = done.cpu().numpy(), rew.cpu().numpy()
    for disc, lam in ((0.99, 0.95), (1.0, 1.0)):
        adv, ret = postproc.gae(rew, _dev(vals), done, disc, lam)
        pe.check_gae(adv.cpu().numpy(), ret.cpu().numpy(), r, vals, d, disc, lam, None)
    ret = postproc.gae(rew, torch.zeros_like(rew), done, 0.99, 1.0)[1]
    o, obn, y = obs.cpu().numpy(), ob.cpu().numpy(), ret.cpu().numpy()
    F = bo.features(o, d, obn)
    for kw in (dict(), dict(n_agents=A)):
        bl = postproc.LinearFeatureBaseline(D, DEV, **kw)
        bl.fit(obs, done, ret, obs_before=ob)
        c = bl.get_param_values()
        v = bl.predict(obs, done, obs_before=ob).cpu().numpy()
        if not kw:
            yy = y.reshape(-1).astype(np.float64)
            assert bo.objective(F, yy, c) <= bo.objective(F, yy, bo.fit(F, yy)) * (1 + 1e-8)
            pe.check_predict(v, F, c)
        else:
            for a in range(A):
                Fa, ya = F[a::A], y[..., a].reshape(-1).astype(np.float64)
                assert bo.objective(Fa, ya, c[a]) <= bo.objective(Fa, ya, bo.fit(Fa, ya)) * (1 + 1e-8), a
                pe.check_predict(v[..., a].reshape(-1), Fa, c[a])
    for pa in (False, True):
        simplev, bin_sum, bin_cnt = (x.cpu().numpy() for x in rltools_sampler.time_baseline(ret, done, per_agent=pa))
        pe.check_time_baseline(simplev, bin_sum, bin_cnt, y, d, None, pa)
    ps = b.path_start.cpu().numpy()
    sums = np.array([[r[ps[p]:ps[p + 1], 0, a].astype(np.float64).sum() for a in range(A)]
                     for p in range(len(ps) - 1)]).reshape(-1)            # (path, agent) order
    disc = np.array([[po.gae_env(r[ps[p]:ps[p + 1], 0].astype(np.float64), np.zeros((ps[p + 1] - ps[p], A)),
                                 np.zeros(ps[p + 1] - ps[p], bool), 0.99, 1.0)[1][0, a] for a in range(A)]
                     for p in range(len(ps) - 1)]).reshape(-1)
    st = postproc.path_statistics(rew, ret, done, per_agent=False)
    assert st["NumTrajs"] == len(sums) and st["MaxReturn"] == sums.max() and st["MinReturn"] == sums.min()
    for k, v in (("AverageReturn", sums.mean()), ("StdReturn", sums.std())):
        assert np.isclose(st[k], v, rtol=1e-10, atol=1e-12 * np.abs(sums).max()), k
    assert np.isclose(st["AverageDiscountedReturn"], disc.mean(), rtol=1e-5, atol=1e-5 * np.abs(disc).max())


# ---------------------------------------------------------------- pooled over ranks

@pytest.fixture(scope="module", params=(2, 3), ids=lambda w: "W%d" % w)
def pooled(request):
    W = request.param
    got = se.run_ranks(W, "gloo", se.run_cases, [(("pooled",), wpe.pooled_rank, (W,))])
    return W, {r: se.result(got, ("pooled",))[r] for r in range(W)}


def test_pooled_whole_path_batches_over_ranks(pooled):
    W, res = pooled
    batches = [wpe.pooled_batch(W, r, DEV) for r in range(W)]
    lens = [len(b) for b in batches]
    assert [res[r]["N"] for r in range(W)] == lens
    plen = [int(np.diff(b.path_start.cpu().numpy()).max()) for b in batches]
    assert min(b.n_paths for b in batches) == 1 and plen.count(max(plen)) == 1
    assert any(b.env_rows.shape[0] == 257 for b in batches)
    # one unsharded [sum N, 1] auto-reset rollout: store = cat(obs_0, .., obs_{W-1}, zero row)
    A = batches[0].rew.shape[1]
    store = torch.cat([b.obs for b in batches] + [torch.zeros_like(batches[0].obs[:1])])
    Nt = sum(lens)
    obs, ob = store[1:].view(Nt, 1, A, -1), store[:1]
    done = torch.cat([b.done for b in batches]).view(Nt, 1)
    rew = torch.cat([b.rew for b in batches]).view(Nt, 1, A)
    act = torch.cat([b.actions for b in batches]).unsqueeze(1)
    full = wpe.pooled_passes(obs, done, rew, ob, act, DEV, None)
    for r in range(1, W):
        se.bits_equal(res[0]["conc_coeffs"], res[r]["conc_coeffs"], "conc coeffs")
        for m in ("decentralized", "concurrent"):
            se.bits_equal(res[0][m], res[r][m], m)
        for k in range(2):
            se.bits_equal({n: res[0]["rltools"][k][n] for n in ("v_r", "tv_r", "fallback")},
                          {n: res[r]["rltools"][k][n] for n in ("v_r", "tv_r", "fallback")}, "rltools")
            se.bits_equal(res[0]["conc"][k][3], res[r]["conc"][k][3], "conc ev")
    bounds = se.bounds(lens)
    for k in range(2):
        for r, (lo, hi) in enumerate(bounds):
            v, a, rt, _ = res[r]["conc"][k]
            fv, fa, frt, _ = full["conc"][k]
            assert np.array_equal(rt, frt[lo:hi])
            np.testing.assert_allclose(v, fv[lo:hi], rtol=1e-5, atol=1e-5 * np.abs(fv).max() + 1e-30)
            np.testing.assert_allclose(a, fa[lo:hi], rtol=1e-5, atol=1e-5 * np.abs(fa).max())
            q = res[r]["rltools"][k]
            fq = full["rltools"][k]
            assert np.array_equal(q["q"], fq["q"][lo:hi])
            for n in ("advantages", "values"):
                np.testing.assert_allclose(q[n], fq[n][lo:hi], rtol=1e-5, atol=1e-5 * np.abs(fq[n]).max() + 1e-30)
        np.testing.assert_allclose(res[0]["conc"][k][3], full["conc"][k][3], rtol=1e-9, atol=1e-9)
        assert np.array_equal(res[0]["rltools"][k]["fallback"], full["rltools"][k]["fallback"])
        np.testing.assert_allclose(res[0]["rltools"][k]["tv_r"], full["rltools"][k]["tv_r"], rtol=1e-9, atol=1e-9)
        np.testing.assert_allclose(res[0]["rltools"][k]["v_r"], full["rltools"][k]["v_r"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(res[0]["conc_coeffs"], full["conc_coeffs"], rtol=0,
                               atol=1e-9 * np.abs(full["conc_coeffs"]).max())
    for m in ("decentralized", "concurrent"):
        for k in range(2):
            for got, want in zip(res[0][m]["stats"][k], full[m]["stats"][k]):
                assert got.keys() == want.keys()
                for n in se.EXACT_STATS + ("AverageDiscountedReturn",):
                    assert np.allclose(got[n], want[n], rtol=1e-12, atol=0), (m, k, n)
                assert np.allclose(got["ExplainedVariance"], want["ExplainedVariance"], rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(res[0][m]["coeffs"], full[m]["coeffs"], rtol=0,
                                   atol=1e-9 * np.abs(full[m]["coeffs"]).max())
