"""Waterworld's writer-warp kernel at every layout it is built for, and at the geometry and timing edges of its ring
(needs a GPU).  The cases are tests/ww_writer_edges.py's table.

Every comparison of the writer with the one-warp kernel (set_obs_writer ON against OFF, bit for bit) also asserts,
from the library's launch log (madrl_ww_launch_log), which kernel each launch ran: were ww_use_writer to refuse the
writer, ON would compare the one-warp kernel with itself.  The writer's float32 observations are checked against the float64
oracle by teacher forcing, one writer launch per step, and the fp64 build checks each case's configuration against
the oracle over whole trajectories."""
import numpy as np
import pytest
import torch

import teacher_forced as TF
import ww_writer_edges as W
from madrl_b200 import BatchedMAWaterWorld, _lib
from oracle.philox import Stream
from oracle.waterworld_oracle import WaterworldOracle

pytestmark = pytest.mark.gpu

ON, OFF = _lib.WW_OBS_WRITER_ON, _lib.WW_OBS_WRITER_OFF
MPL, SEED = 5, 11
EDGE_CASES = [W.BY_NAME["c2"], W.BY_NAME["k64_plain"]]


# ------------------------------------------------------------------------------------------------ kernel identity
def launched(fn):
    """fn() with the library's launch log on -> (its result, [(name, grid)] of the ww_kernel launches, in launch order).
    madrl_ww_launch_log records the template arguments of the instantiation each launch ran and its gridDim.x, as the
    launch code passes them to the kernel; they are spelled as the demangled kernel name (ww_writer_edges.writer_kernel).
    The log is read on the host, so unlike a profiler session it cannot lose a launch."""
    L, fields, most = _lib.lib(), 10, 4096
    assert L.madrl_ww_launch_log(1, None, 0) >= 0
    try:
        out = fn()
    finally:
        recs = np.zeros((most, fields), np.int32)
        n = L.madrl_ww_launch_log(0, recs.ctypes.data, most)
    assert 0 <= n <= most, n
    real = {4: "float", 8: "double"}
    obs = {2: "unsigned short", 4: "float", 8: "double"}
    flag = ("false", "true")
    return out, [("void madrl::ww_kernel<%s, %s, %d, %d, %d, %s, %d, %s, %s>(madrl::WWParams<%s, %s>)" % (
        real[r], obs[o], opl, kch, kc, flag[peer], policy, flag[keep], flag[writer], real[r], obs[o]), int(grid))
        for r, o, opl, kch, kc, peer, policy, keep, writer, grid in recs[:n].tolist()]


def assert_writer(kernels, case, n=None):
    """Every ww_kernel launch ran the writer instantiation of `case` (and there were `n` of them)."""
    want = W.writer_kernel(case)
    assert kernels and all(name == want for name, _ in kernels), (want, kernels)
    if n is not None:
        assert len(kernels) == n, kernels


def assert_one_warp(kernels, n=None):
    assert kernels and not any(W.is_writer(name) for name, _ in kernels), kernels
    if n is not None:
        assert len(kernels) == n, kernels


def assert_ran(kernels, case, writer, n=None):
    if writer:
        assert_writer(kernels, case, n)
    else:
        assert_one_warp(kernels, n)


@pytest.fixture(scope="module")
def grid():
    """Blocks of the largest writer grid: WR_BLOCKS_PER_SM per SM (the tests check a launch reaches it)."""
    return torch.cuda.get_device_properties(0).multi_processor_count * W.WR_BLOCKS_PER_SM


# ------------------------------------------------------------------------------------------------ rollouts
def bits(x):
    return x.view(torch.int32) if x.dtype == torch.float32 else x


def make(case, E, mode, mpl=MPL, **kw):
    eng = BatchedMAWaterWorld(E, **case.cfg, device="cuda", seed=SEED, max_path_length=mpl, **kw)
    if mode is not None:
        eng.set_obs_writer(mode)
    return eng


def actions(case, T, E, seed):
    return torch.as_tensor(W.actions(np.random.RandomState(seed), T, E, case.Np)).cuda()


def buffers(eng, T, obs_offset=0):
    E, A, D = eng.n_envs, eng.n_pursuers, eng.obs_dim
    flat = torch.full((obs_offset + T * E * A * D,), float("nan"), device="cuda")
    return (flat[obs_offset:].view(T, E, A, D), torch.full((T, E, A), float("nan"), device="cuda"),
            torch.full((T, E), 255, dtype=torch.uint8, device="cuda"),
            torch.full((T, E, 2), -1, dtype=torch.int32, device="cuda"))


def run(eng, act, obs_offset=0, desync=False, auto_reset=True, prepare=None):
    """reset (then, with `desync`, a 3-step rollout and a masked reset of every other env, so that paths end at
    different steps within a group), `prepare(eng)`, and one rollout into NaN-filled buffers, with terminal
    observations when it auto-resets -> (outputs, state, ww_kernel launches of the rollout)."""
    E = eng.n_envs
    eng.reset()
    if desync:
        eng.rollout(act[:3], auto_reset=True)
        eng.reset(mask=(torch.arange(E, device="cuda") % 2).to(torch.uint8))
    if prepare is not None:
        prepare(eng)
    out = buffers(eng, act.shape[0], obs_offset)
    term = None
    if auto_reset:
        term = torch.full_like(out[0], -3.0)
        eng.set_terminal_obs(term)
    outs, kernels = launched(lambda: eng.rollout(act, auto_reset=auto_reset, out=out))
    eng.set_terminal_obs(None)
    return (tuple(outs) + ((term,) if auto_reset else ()), {k: v.clone() for k, v in eng.state.items()}), kernels


def assert_same(a, b):
    (got, got_state), (want, want_state) = a, b
    for k, (x, y) in enumerate(zip(got, want)):
        assert x.shape == y.shape and torch.equal(bits(x), bits(y)), ("obs", "rew", "done", "info", "term")[k]
    for k in want_state:
        assert torch.equal(bits(got_state[k]), bits(want_state[k])), k


def on_equals_off(case, E, T, seed=2, writer=None, mpl=MPL, **kw):
    """ON and OFF on the same rollout (run's keywords): the same bits, one launch each, ON on the writer (unless the
    case or `writer` says the launch falls back), OFF on the one-warp kernel -> (ON's outputs, ON's launches)."""
    act = actions(case, T, E, seed)
    got, k_on = run(make(case, E, ON, mpl), act, **kw)
    want, k_off = run(make(case, E, OFF, mpl), act, **kw)
    assert_ran(k_on, case, case.writer if writer is None else writer, 1)
    assert_one_warp(k_off, 1)
    assert_same(got, want)
    return got[0], k_on


# ------------------------------------------------------------------------------------------------ the case table
@pytest.mark.parametrize("case", W.CASES, ids=str)
def test_writer_equals_one_warp_kernel(case):
    """An auto-reset rollout of desynchronised envs over several groups, the last one partial where the stride rule
    allows it; collisions and catches happen."""
    E = case.E(60)
    outs, _ = on_equals_off(case, E, 24, desync=True)
    obs, done, info = outs[0], outs[2], outs[3]
    assert (done[:, 0::2] != done[:, 1::2]).any() and int(done.sum()) >= E * (24 // MPL)
    assert int(info.sum()) > 0, "no catch"
    assert min(W.tail_events(obs.cpu().numpy(), case)) > 0, "no evader or no poison collision"


@pytest.mark.parametrize("case", W.CASES, ids=str)
def test_auto_default_takes_writer_where_it_caps(case, grid):
    """AUTO runs the writer wherever the default cap applies and the writer is built for the layout (obj33 has a
    cap but more than 32 objects; stage_over no cap), and the one-warp kernel below 16 steps."""
    E, T = case.E(16 * grid), 16
    eng = make(case, E, None)
    cap = _lib.lib().madrl_ww_default_blocks_per_sm(eng._h, T)
    assert cap == (0 if case.name == "stage_over" else 16)
    eng.reset()
    act = actions(case, T, E, 3)
    _, k = launched(lambda: eng.rollout(act))
    assert_ran(k, case, case.writer and cap > 0, 1)
    _, k = launched(lambda: eng.rollout(act[:15]))
    assert_one_warp(k, 1)


def test_other_paths_never_take_writer():
    """bfloat16 observations, the fp64 build, KEEP stores, the fused peer exchange and the in-kernel heuristic
    policy run their own instantiations even with set_obs_writer(ON)."""
    case, E, T = W.BY_NAME["c2"], 64, 3
    act = actions(case, T, E, 4)
    for kw, setup in (({"obs_dtype": torch.bfloat16}, None), ({"dtype": torch.float64}, None),
                      ({}, lambda g: g.set_obs_cache(_lib.OBS_CACHE_KEEP)), ({}, "peers"), ({}, "heuristic")):
        eng = make(case, E, ON, **kw)
        obs0 = eng.reset()
        if callable(setup):
            setup(eng)
        if setup == "peers":
            keep = ([torch.zeros(1, E, T, 5, device="cuda")], [torch.zeros(1, E, T, dtype=torch.uint8, device="cuda")],
                    [torch.zeros(1, E, T, 2, dtype=torch.int32, device="cuda")])
            eng.set_peers(0, T, *keep)
        if setup == "heuristic":
            _, k = launched(lambda: eng.rollout_heuristic(T, obs0))
        else:
            _, k = launched(lambda: eng.rollout(act))
        assert_one_warp(k, 1)


@pytest.mark.parametrize("case", W.CASES, ids=str)
def test_writer_teacher_forced_against_oracle(case):
    """float32 writer launches of one step each, from the engine's own states, against the float64 oracle."""
    E, T = case.E(24), 6
    eng = make(case, E, ON, mpl=0)
    eng.reset()
    log, k = launched(lambda: TF.ww_self_teacher_forced(TF.TorchAdapter(eng), case.cfg, SEED, T, 0.7,
                                                        "ww_writer_" + case.name))
    assert_ran(k, case, case.writer, T)
    log.dump()
    assert log.checked_frac >= 0.98 and log.obs_frac >= 0.999, log.d


@pytest.mark.parametrize("case", W.CASES, ids=str)
def test_fp64_trajectories_match_oracle(case):
    """The fp64 build over whole trajectories: events exact, values within 1e-9 (checks the configuration)."""
    E, T, base = 4, 40, 300
    cfg = case.cfg
    eng = BatchedMAWaterWorld(E, **cfg, device="cuda", dtype=torch.float64, seed=SEED, env_id_base=base)
    obs0 = eng.reset().cpu().numpy()
    oracles = [WaterworldOracle(rng=Stream(SEED, base + e), **cfg) for e in range(E)]
    for e, o in enumerate(oracles):
        assert np.abs(np.array(o.reset()) - obs0[e]).max() < 1e-9, e
    act = np.random.RandomState(5).randn(T, E, case.Np, 2) * 0.7
    obs, rew, done, info = [x.cpu().numpy() for x in eng.rollout(torch.as_tensor(act), auto_reset=False)]
    for t in range(T):
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e])
            assert [ii['evcatches'], ii['pocatches']] == list(info[t, e]), (t, e)
            assert np.abs(np.array(oo) - obs[t, e]).max() < 1e-9, (t, e)
            assert np.abs(rr - rew[t, e]).max() < 1e-9, (t, e)
            assert bool(done[t, e]) == dd
    st = {k: v.cpu().numpy() for k, v in eng.state.items()}
    for e, o in enumerate(oracles):
        assert int(st['rng_counter'][e]) == o.np_random.counter and int(st['timestep'][e]) == o.t
    assert int(info.sum()) > 0, "no catch"
    assert min(W.tail_events(obs, case)) > 0, "no evader or no poison collision"


# ------------------------------------------------------------------------------------------------ geometry and timing
def group_counts(grid):
    """E around the writer grid: one partial group, one group, as many groups as blocks, one more, two rounds and a
    partial group."""
    return {"partial": 4, "one": 8, "grid": grid * 8, "grid+1": grid * 8 + 8, "2grid+half": 2 * grid * 8 + 4}


@pytest.mark.parametrize("which", ["partial", "one", "grid", "grid+1", "2grid+half"])
@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_group_counts(case, which, grid):
    E = group_counts(grid)[which]
    _, k = on_equals_off(case, E, 13, desync=True)
    assert k[0][1] == min((E + 7) // 8, grid), k   # the launch's grid: one block per group, up to the full grid


@pytest.mark.parametrize("T", [1, 2, 3, 7, 17])
@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_step_counts_with_multi_group_blocks(case, T, grid):
    """Blocks walk three or two groups through one ring: the slot index and phase carry across groups at odd
    offsets."""
    on_equals_off(case, 2 * grid * 8 + 4, T, seed=T, desync=True)


@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_done_every_step(case, grid):
    """max_path_length = 1: every step is done, so every step's terminal rows come from the staged slot."""
    outs, _ = on_equals_off(case, grid * 8 + 8, 9, mpl=1)
    assert bool(outs[2].bool().all())


@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_timestep_limit_done(case, grid):
    """Paths that end at the env's timestep limit (1000), at different steps in neighbouring envs."""
    E = grid * 8 + 8

    def near_limit(eng):
        eng.state["timestep"].copy_(990 + torch.arange(E, dtype=torch.int32, device="cuda") % 7)

    act = actions(case, 12, E, 6)
    got, k_on = run(make(case, E, ON, mpl=0), act, prepare=near_limit)
    want, k_off = run(make(case, E, OFF, mpl=0), act, prepare=near_limit)
    assert_writer(k_on, case, 1)
    assert_one_warp(k_off, 1)
    assert_same(got, want)
    done = got[0][2]
    assert int(done.sum()) == E and (done[:, 0] != done[:, 1]).any()


@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_no_auto_reset(case, grid):
    on_equals_off(case, grid * 8 + 8, 11, auto_reset=False)


@pytest.mark.parametrize("offset,writer", [(4, True), (1, False)], ids=["16B", "4B"])
@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_observation_base_offset(case, offset, writer):
    """An `out=` observation tensor 4 floats into its allocation (16-byte aligned, not 128) still takes the
    writer; 1 float falls back."""
    on_equals_off(case, case.E(100), 10, obs_offset=offset, writer=writer, desync=True)


@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_odd_stride_falls_back(case):
    on_equals_off(case, 101, 10, writer=False, desync=True)


@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_chained_auto_launches_equal_one_launch(case):
    """At AUTO, T = 20, 5 and 33 run the writer, the one-warp kernel and the writer again on the same envs; together
    they equal one 58-step launch of the one-warp kernel, terminal observations included."""
    E = case.E(4096)
    act = actions(case, 58, E, 7)
    eng = make(case, E, None)
    eng.reset()
    out, term = buffers(eng, 58), torch.full((58, E, case.Np, case.D), -3.0, device="cuda")
    t0 = 0
    for T, writer in ((20, True), (5, False), (33, True)):
        sl = slice(t0, t0 + T)
        eng.set_terminal_obs(term[sl])
        _, k = launched(lambda: eng.rollout(act[sl], out=tuple(x[sl] for x in out)))
        assert_ran(k, case, writer, 1)
        t0 += T
    eng.set_terminal_obs(None)
    got = (tuple(out) + (term,), {k: v.clone() for k, v in eng.state.items()})
    want, k = run(make(case, E, OFF), act)
    assert_one_warp(k, 1)
    assert_same(got, want)
    assert int(out[2].sum()) >= E * (58 // MPL)


@pytest.mark.parametrize("case", EDGE_CASES, ids=str)
def test_rollout_host_chunks(case):
    """rollout_host with chunks of 5 steps: every chunk is a writer launch shorter than 16 steps."""
    E, T = case.E(1024), 40
    act = actions(case, T, E, 8).cpu().pin_memory()
    res = []
    for mode in (ON, OFF):
        eng = make(case, E, mode)
        eng.reset()
        bufs = tuple(x.cpu().pin_memory() for x in buffers(eng, T))
        _lib.lib().madrl_set_host_chunk_bytes(bufs[0][0].numel() * 4 * 3)
        try:
            _, k = launched(lambda: eng.rollout_host(act, *bufs, auto_reset=True))
        finally:
            _lib.lib().madrl_set_host_chunk_bytes(0)
        assert_ran(k, case, mode == ON, 8)
        res.append((bufs, {n: v.clone() for n, v in eng.state.items()}))
    assert int(res[0][0][2].sum()) >= E * (T // MPL)
    assert_same(*res)
