"""Waterworld's fused peer exchange on one GPU (the PEER instantiation of ww_kernel, madrl_ww_set_peers), at every
staging edge of its rows, and the exchange primitives of csrc/exchange.cu.

The kernel stages the rows it sends in registers: a reward run covers rew_per = 32 // Np steps (lane s * Np + a holds
step s of agent a), a partial run is written at the end of the launch, and the done / info rows are flushed every 32
steps and at the last step.  RNG streams are keyed by the global env id, so W "ranks" run on one GPU: W engines with
env_id_base = r * E write slot r of the same destination buffers.  The reference is one unsharded engine of W * E envs
without peers.  Every destination starts as sentinels (NaN / 255 / -1) and has t_max > T steps; after the rollouts,
slot r, steps [0, T) hold the reference's rows of envs [r E, (r + 1) E), env-major, and everything else still holds
the sentinels.  Each rank's own outputs equal the reference's, bit for bit."""
import collections
import ctypes as C
import socket

import numpy as np
import pytest
import torch

from madrl_b200 import BatchedMAWaterWorld, _lib
from oracle.philox import Stream
from oracle.waterworld_oracle import WaterworldOracle

pytestmark = pytest.mark.gpu

SEED = 13
SENTINEL = dict(rew=float("nan"), done=255, info=-1)
DTYPES = dict(f32=torch.float32, f64=torch.float64)
# the sensor configuration of each instantiation ww_launch_t selects: compile-time K = 30 with speed features,
# any other K <= 32 (one sensor per lane), K > 32 (two sensors per lane)
KINDS = dict(kc30=dict(n_sensors=30, speed_features=True), plain=dict(n_sensors=12, speed_features=False),
             kch2=dict(n_sensors=40, speed_features=True))
# objects per env that select each OPL instantiation: ceil(objects / 32) objects per lane, rounded up to 1, 2, 4 or 8
N_OBJ = {1: 24, 2: 50, 4: 100, 8: 200}


class Case(collections.namedtuple("Case", "Np T kind opl dtype mpl auto_reset W slots n_dest E", defaults=(3,))):
    """One rollout of W ranks of E envs each, into n_dest destinations of `slots` slots and T + 2 steps."""

    @property
    def rew_per(self):
        return 32 // self.Np

    @property
    def t_max(self):
        return self.T + 2

    def cfg(self):
        n_obj = max(N_OBJ[self.opl], self.Np + 2)
        assert min(o for o in (1, 2, 4, 8) if 32 * o >= n_obj) == self.opl, self
        ne = (n_obj - self.Np) // 2
        return dict(n_pursuers=self.Np, n_evaders=ne, n_poison=n_obj - self.Np - ne, n_coop=1, radius=0.04,
                    **KINDS[self.kind])

    def __str__(self):
        return "np%d_t%d_%s_opl%d_%s_mpl%d%s_w%d_s%d_d%d" % (
            self.Np, self.T, self.kind, self.opl, self.dtype, self.mpl, "_ar" if self.auto_reset else "", self.W,
            self.slots, self.n_dest)


# For each Np (rew_per 32, 10, 6, 4, 2, 1, 1), T = 1, rew_per - 1, rew_per and rew_per + 1, and T = 31, 32, 33, 64, 97
# across the table: partial, exact and several 32-step flushes.  Each of the 24 (sensor instantiation, OPL, dtype)
# kernels runs at least once (32 pursuers leave no OPL = 1 layout).  max_path_length puts resets mid-run, on the last
# step and on 32-step flush boundaries (t = 31, 63, 95); some rollouts do not auto-reset.
CASES = [Case(*c) for c in [
    # Np, T, kind,  OPL, dtype, mpl, auto_reset, W, slots, n_dest
    (1, 1, "kc30", 1, "f32", 1, True, 2, 3, 1),
    (1, 31, "plain", 2, "f64", 8, True, 2, 2, 2),
    (1, 32, "kch2", 4, "f32", 8, True, 3, 3, 3),
    (1, 33, "kc30", 2, "f64", 11, True, 2, 3, 1),
    (1, 97, "plain", 4, "f32", 32, True, 2, 2, 2),
    (3, 1, "kch2", 8, "f64", 0, False, 2, 2, 1),
    (3, 9, "kc30", 4, "f32", 3, True, 2, 3, 2),
    (3, 10, "plain", 8, "f64", 4, False, 3, 4, 3),
    (3, 11, "kch2", 1, "f32", 5, True, 2, 2, 8),
    (5, 1, "kc30", 8, "f64", 0, True, 2, 2, 1),
    (5, 5, "plain", 1, "f32", 5, True, 2, 3, 2),
    (5, 6, "kch2", 2, "f64", 2, True, 2, 2, 1),
    (5, 7, "kc30", 1, "f64", 3, False, 2, 2, 3),
    (5, 64, "plain", 2, "f32", 16, True, 2, 3, 2),
    (8, 1, "kch2", 4, "f64", 1, False, 2, 2, 2),
    (8, 3, "kc30", 2, "f32", 0, True, 2, 3, 1),
    (8, 4, "plain", 4, "f64", 2, True, 3, 3, 2),
    (8, 5, "kch2", 8, "f32", 5, True, 2, 2, 1),
    (11, 1, "kc30", 4, "f64", 1, True, 2, 2, 1),
    (11, 2, "plain", 8, "f32", 0, False, 2, 3, 2),
    (11, 3, "kch2", 1, "f64", 3, True, 2, 2, 3),
    (17, 1, "kc30", 8, "f32", 1, True, 2, 2, 1),
    (17, 2, "plain", 1, "f64", 2, True, 2, 3, 2),
    (17, 33, "kch2", 2, "f32", 32, True, 2, 2, 1),
    (32, 1, "kc30", 2, "f32", 0, False, 2, 2, 1),
    (32, 2, "plain", 2, "f64", 1, True, 2, 3, 2),
    (32, 32, "kch2", 4, "f32", 8, True, 2, 2, 1),
]]


def test_table_covers_every_staging_edge():
    rew_per = {c.Np: c.rew_per for c in CASES}
    for Np, r in rew_per.items():
        steps = {c.T for c in CASES if c.Np == Np}
        assert {1, r, r + 1} | ({r - 1} if r > 1 else set()) <= steps, Np
    assert {31, 32, 33, 64, 97} <= {c.T for c in CASES}
    assert {1, 2, 4, 8} == {c.opl for c in CASES}
    assert len({(c.kind, c.opl, c.dtype) for c in CASES}) == 24
    resets = [c for c in CASES if c.auto_reset and c.mpl > 0]
    assert any(c.mpl < c.T and c.T % c.mpl == 0 for c in resets)                     # mid-run and on the last step
    assert any(c.T > 32 and 32 % c.mpl == 0 for c in resets)                        # on a flush boundary
    assert any(not c.auto_reset and 0 < c.mpl < c.T for c in CASES)                 # done stays set, no reset
    assert any(c.slots > c.W for c in CASES) and any(c.n_dest == 8 for c in CASES)


# ------------------------------------------------------------------------------------------------ helpers
def bits(x):
    return x.view({torch.float32: torch.int32, torch.float64: torch.int64}.get(x.dtype, x.dtype))


def make(c, E, base=0, dtype=None, **kw):
    return BatchedMAWaterWorld(E, **c.cfg(), device="cuda", seed=SEED, env_id_base=base, max_path_length=c.mpl,
                               dtype=dtype or DTYPES[c.dtype], **kw)


def actions(c, T, E, seed=0):
    g = torch.Generator("cuda").manual_seed(seed)
    return (torch.randn(T, E, c.Np, 2, device="cuda", generator=g, dtype=torch.float64) * 0.7).to(DTYPES[c.dtype])


def destinations(c, dtype=None):
    """n_dest sets of sentinel-filled (rew, done, info), each a distinct tensor."""
    S, E, t = c.slots, c.E, c.t_max
    return [(torch.full((S, E, t, c.Np), SENTINEL["rew"], dtype=dtype or DTYPES[c.dtype], device="cuda"),
             torch.full((S, E, t), SENTINEL["done"], dtype=torch.uint8, device="cuda"),
             torch.full((S, E, t, 2), SENTINEL["info"], dtype=torch.int32, device="cuda")) for _ in range(c.n_dest)]


def set_peers(eng, rank, t_max, dests):
    eng.set_peers(rank, t_max, [d[0] for d in dests], [d[1] for d in dests], [d[2] for d in dests])


def untouched(x):
    return bool(torch.isnan(x).all()) if x.is_floating_point() else bool((x == SENTINEL["done" if x.dtype == torch.uint8
                                                                                        else "info"]).all())


def assert_untouched(dests):
    for d in dests:
        assert all(untouched(x) for x in d)


def assert_rows(dests, W, E, T, rew, done, info):
    """Slot r, steps [0, T) of every destination hold the rows rew [T, W E, Np], done [T, W E], info [T, W E, 2] of
    envs [r E, (r + 1) E), env-major; steps >= T of slots [0, W) and every slot >= W still hold the sentinels."""
    for rew_d, done_d, info_d in dests:
        for r in range(W):
            s = slice(r * E, (r + 1) * E)
            assert torch.equal(bits(rew_d[r, :, :T]), bits(rew[:, s].transpose(0, 1))), ("rew", r)
            assert torch.equal(done_d[r, :, :T], done[:, s].t()), ("done", r)
            assert torch.equal(info_d[r, :, :T], info[:, s].transpose(0, 1)), ("info", r)
        for x in (rew_d, done_d, info_d):
            assert untouched(x[:W, :, T:]) and untouched(x[W:]), x.dtype


def assert_same(got, want):
    """The same tensors, bit for bit (got[k] against want[k])."""
    for k, (x, y) in enumerate(zip(got, want)):
        assert x.shape == y.shape and torch.equal(bits(x), bits(y)), k


def state_of(eng, envs=slice(None)):
    return {k: (v if k == "sensors" else v[envs]).clone() for k, v in eng.state.items()}


def sharded_rollout(c, dests, setup=None, term=False):
    """The reference of W E envs without peers, then W ranks of E envs each with peers into `dests`; asserts each
    rank's outputs (and terminal observations, with `term`) and final state equal the reference's -> the reference's
    (obs, rew, done, info)."""
    W, T, E = c.W, c.T, c.E
    act = actions(c, T, W * E)
    ref = make(c, W * E)
    ref.reset()
    if term:
        ref_term = torch.full((T, W * E, c.Np, ref.obs_dim), -3.0, dtype=ref.obs_dtype, device="cuda")
        ref.set_terminal_obs(ref_term)
    want = ref.rollout(act, auto_reset=c.auto_reset)
    for r in range(W):
        s = slice(r * E, (r + 1) * E)
        eng = make(c, E, base=r * E)
        eng.reset()
        if setup is not None:
            setup(eng)
        extra = ()
        if term:
            t_r = torch.full((T, E, c.Np, eng.obs_dim), -3.0, dtype=eng.obs_dtype, device="cuda")
            eng.set_terminal_obs(t_r)
            extra = ((t_r, ref_term[:, s]),)
        set_peers(eng, r, c.t_max, dests)
        got = eng.rollout(act[:, s], auto_reset=c.auto_reset)
        assert_same(tuple(got) + tuple(x for x, _ in extra), tuple(w[:, s] for w in want) + tuple(y for _, y in extra))
        got_state, want_state = state_of(eng), state_of(ref, s)
        for k in want_state:
            assert torch.equal(bits(got_state[k]), bits(want_state[k])), k
    torch.cuda.synchronize()
    return want


# ------------------------------------------------------------------------------------------------ the case table
@pytest.mark.parametrize("c", CASES, ids=str)
def test_peer_rows_equal_unsharded_rollout(c):
    dests = destinations(c)
    _, rew, done, info = sharded_rollout(c, dests)
    assert_rows(dests, c.W, c.E, c.T, rew, done, info)
    if c.mpl > 0:
        assert int(done.sum()) > 0


@pytest.mark.parametrize("dtype", ["f32", "f64"])
@pytest.mark.parametrize("blocks_per_sm", [0, 1])
def test_peer_rows_when_warps_step_several_envs(dtype, blocks_per_sm):
    """E = 2 SMs + 7 envs per rank: with one block per SM each warp steps two or three envs, so the env a lane's
    rows belong to changes inside a warp; with the default launch each warp steps one env.  T = 45: a partial
    32-step flush and a partial reward run; resets every 9 steps."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    c = Case(5, 45, "kc30", 1, dtype, 9, True, 2, 3, 2, E=2 * sms + 7)
    dests = destinations(c)
    _, rew, done, info = sharded_rollout(c, dests, setup=lambda g: g.set_launch(blocks_per_sm=blocks_per_sm))
    assert_rows(dests, c.W, c.E, c.T, rew, done, info)


def test_peer_rows_with_terminal_obs_keep_stores_and_writer():
    """set_terminal_obs, OBS_CACHE_KEEP and set_obs_writer(ON) together with peers: the peer instantiation runs,
    the values and the terminal observations equal the reference's, and the peer rows are right."""
    c = Case(5, 40, "kc30", 1, "f32", 7, True, 2, 2, 2)

    def setup(eng):
        eng.set_obs_cache(_lib.OBS_CACHE_KEEP)
        eng.set_obs_writer(_lib.WW_OBS_WRITER_ON)
    dests = destinations(c)
    _, rew, done, info = sharded_rollout(c, dests, setup=setup, term=True)
    assert_rows(dests, c.W, c.E, c.T, rew, done, info)


def test_fp64_peer_rows_match_oracle():
    """The fp64 build's peer rows against the float64 oracle of each global env id: events exact, rewards within
    1e-9."""
    c = Case(3, 12, "kc30", 1, "f64", 0, False, 2, 2, 1)
    E = c.E
    dests = destinations(c)
    sharded_rollout(c, dests)
    act = actions(c, c.T, c.W * E).cpu().numpy()
    rew_d, done_d, info_d = [x.cpu().numpy() for x in dests[0]]
    for g in range(c.W * E):
        r, e = divmod(g, E)
        o = WaterworldOracle(rng=Stream(SEED, g), **c.cfg())
        o.reset()
        for t in range(c.T):
            _, rr, dd, ii = o.step(act[t, g])
            assert np.abs(np.asarray(rr) - rew_d[r, e, t]).max() < 1e-9, (g, t)
            assert bool(done_d[r, e, t]) == dd and [ii['evcatches'], ii['pocatches']] == list(info_d[r, e, t]), (g, t)


# ------------------------------------------------------------------------------------------------ repeated launches
def test_alternating_buffer_sets_and_step():
    """PeerGather.arm's pattern: rollout 1 into set A, rollout 2 into set B (continuing the envs), then one step()
    into A.  Each launch writes its own steps from step 0 of the set it was given, and leaves the other set alone."""
    c = Case(5, 19, "kc30", 1, "f32", 7, True, 2, 3, 2)
    E, W, T = c.E, c.W, c.T
    A, B = destinations(c), destinations(c)
    act = [actions(c, T, W * E, k) for k in range(2)] + [actions(c, 1, W * E, 2)]
    ref = make(c, W * E)
    ref.reset()
    want = [ref.rollout(a, auto_reset=True) for a in act[:2]]
    o, r_, d, i = ref.step(act[2][0], auto_reset=True)
    want.append((o[None], r_[None], d[None], torch.stack((i["evcatches"], i["pocatches"]), -1)[None]))
    for r in range(W):
        s = slice(r * E, (r + 1) * E)
        eng = make(c, E, base=r * E)
        eng.reset()
        got = []
        for k, dests in enumerate((A, B)):
            set_peers(eng, r, c.t_max, dests)
            got.append(eng.rollout(act[k][:, s], auto_reset=True))
        set_peers(eng, r, c.t_max, A)
        o, r_, d, i = eng.step(act[2][0, s], auto_reset=True)
        got.append((o[None], r_[None], d[None], torch.stack((i["evcatches"], i["pocatches"]), -1)[None]))
        for g, w in zip(got, want):
            assert_same(g, tuple(x[:, s] for x in w))
    torch.cuda.synchronize()
    assert_rows(B, W, E, T, *want[1][1:])
    # A: the step's rows at step 0, rollout 1's at steps [1, T)
    assert_rows(A, W, E, T, *[torch.cat((s, r[1:])) for s, r in zip(want[2][1:], want[0][1:])])


def test_rollout_heuristic_writes_no_peer_rows():
    """The in-kernel heuristic policy runs its own instantiation, which has no peer stores: the buffers stay as they
    were and the outputs equal a heuristic rollout without peers."""
    c = Case(5, 35, "kc30", 1, "f32", 9, True, 1, 1, 2)
    a, b = make(c, c.E), make(c, c.E)
    dests = destinations(c)
    set_peers(b, 0, c.t_max, dests)
    got = b.rollout_heuristic(c.T, b.reset())
    want = a.rollout_heuristic(c.T, a.reset())
    torch.cuda.synchronize()
    assert_same(got, want)
    assert_untouched(dests)


# ------------------------------------------------------------------------------------------------ refusals
def test_launches_with_peers_that_are_refused_write_nothing():
    """A bfloat16 engine (the peer instantiation needs native observations), a rollout longer than t_max, the
    host-buffer rollout and a PolicyRollout (both run a rollout as several launches) all raise before any peer row is
    written."""
    from madrl_b200.closed_loop import PolicyRollout
    c = Case(5, 6, "kc30", 1, "f32", 4, True, 1, 1, 2)
    E, T = c.E, c.T
    act = actions(c, c.t_max + 1, E)

    bf = make(c, E, obs_dtype=torch.bfloat16)
    bf.reset()
    dests = destinations(c)
    set_peers(bf, 0, c.t_max, dests)
    with pytest.raises(_lib.EngineError, match="peer"):
        bf.rollout(act[:T])

    eng = make(c, E)
    eng.reset()
    set_peers(eng, 0, c.t_max, dests)
    with pytest.raises(_lib.EngineError, match="exceeds the peer buffers"):
        eng.rollout(act)
    host = [torch.zeros(s, dtype=dt).pin_memory() for dt, s in eng._trajectory_shapes(T)]
    with pytest.raises(_lib.EngineError, match="set_peers"):
        eng.rollout_host(act[:T].cpu().pin_memory(), *host)
    policy = lambda obs, state: (torch.zeros(E, c.Np, 2, device="cuda"), {}, state)   # noqa: E731
    with pytest.raises(ValueError, match="clear_peers"):
        PolicyRollout(eng, policy, T, graph=False)(eng.reset())
    torch.cuda.synchronize()
    assert_untouched(dests)
    # and all of them run once the peers are cleared
    eng.clear_peers()
    eng.rollout_host(act[:T].cpu().pin_memory(), *host)
    PolicyRollout(eng, policy, T, graph=False)(eng.reset())
    torch.cuda.synchronize()
    assert_untouched(dests)


def test_set_peers_checks_every_tensor():
    """Each malformed destination list is refused before a pointer reaches the library, and the engine then writes no
    peer rows."""
    c = Case(5, 6, "kc30", 1, "f32", 4, True, 2, 2, 1)
    E, T, Np, S = c.E, c.T, c.Np, c.slots
    eng = make(c, E)
    eng.reset()
    good = destinations(c)[0]
    rew, done, info = good
    full = lambda shape, dt, dev="cuda": torch.full(shape, -1, dtype=dt, device=dev)   # noqa: E731
    bad = [
        (TypeError, "rew_peers", 0, full((S, E, c.t_max, Np), torch.float64)),         # not the engine's dtype
        (TypeError, "done_peers", 1, full((S, E, c.t_max), torch.int8)),
        (TypeError, "info_peers", 2, full((S, E, c.t_max, 2), torch.int64)),
        (ValueError, "rew_peers", 0, full((S * E * c.t_max * Np,), torch.float32)),   # flat
        (ValueError, "rew_peers", 0, full((S, E, c.t_max, Np + 1), torch.float32)),
        (ValueError, "done_peers", 1, full((S, E - 1, c.t_max), torch.uint8)),
        (ValueError, "info_peers", 2, full((S, E, c.t_max + 1, 2), torch.int32)),      # not this t_max
        (ValueError, "info_peers", 2, full((S, E, c.t_max, 3), torch.int32)),
        (ValueError, "rew_peers", 0, full((S, E, c.t_max, Np), torch.float32, "cpu")),
        (ValueError, "done_peers", 1, full((S, E, 2 * c.t_max), torch.uint8)[:, :, ::2]),   # not contiguous
        (ValueError, "slots", 0, full((1, E, c.t_max, Np), torch.float32)),           # rank 1 writes slot 1
    ]
    for exc, what, k, t in bad:
        args = list(good)
        args[k] = t
        with pytest.raises(exc, match=what):
            set_peers(eng, 1, c.t_max, [tuple(args)])
    with pytest.raises(ValueError, match="1 to 8 destinations"):
        set_peers(eng, 0, c.t_max, [good] * 9)
    with pytest.raises(ValueError, match="1 to 8 destinations"):
        set_peers(eng, 0, c.t_max, [])
    with pytest.raises(ValueError, match="1 to 8 destinations"):
        eng.set_peers(0, c.t_max, [rew], [done, done], [info])
    with pytest.raises(ValueError, match="t_max"):
        set_peers(eng, -1, c.t_max, [good])
    # the library's own checks: nine destinations, and an info buffer that is not 8-byte aligned
    p = lambda ts: (C.c_void_p * len(ts))(*[t.data_ptr() for t in ts])   # noqa: E731
    assert _lib.lib().madrl_ww_set_peers(eng._h, 9, 0, c.t_max, p([rew] * 9), p([done] * 9), p([info] * 9)) == -1
    flat = full((S * E * c.t_max * 2 + 1,), torch.int32)
    shifted = flat[1:].view(S, E, c.t_max, 2)
    with pytest.raises(_lib.EngineError, match="8-byte aligned"):
        set_peers(eng, 0, c.t_max, [(rew, done, shifted)])
    eng.rollout(actions(c, T, E))
    torch.cuda.synchronize()
    assert_untouched([good])
    assert bool((flat == -1).all())


# ------------------------------------------------------------------------------------------------ exchange primitives
def test_stream_memory_operations_and_copies():
    """madrl_stream_write32 lands its value; madrl_stream_wait_geq32 on a value the stream has already written lets a
    later copy through; madrl_copy_async copies exactly 0, 1, 3 and 4097 bytes between unaligned addresses; NULL and
    misaligned flag addresses are refused before anything is enqueued.  No wait is ever for an unwritten value."""
    L = _lib.lib()
    assert L.madrl_stream_memops_available() == 1
    st = _lib.stream(torch.device("cuda", 0))
    flag = torch.zeros(4, dtype=torch.int32, device="cuda")
    addr = lambda t, off=0: C.c_void_p(t.data_ptr() + off)   # noqa: E731
    assert L.madrl_stream_write32(st, addr(flag, 4), 0xCAFE) == 0
    assert L.madrl_stream_write32(st, addr(flag, 12), 0xFFFFFFFF) == 0
    torch.cuda.synchronize()
    assert flag.tolist() == [0, 0xCAFE, 0, -1]

    src = torch.randint(0, 256, (8192,), dtype=torch.uint8, device="cuda")
    for n in (0, 1, 3, 4097):
        dst = torch.full((8192,), 0xEE, dtype=torch.uint8, device="cuda")
        assert L.madrl_stream_write32(st, addr(flag), n + 1) == 0
        assert L.madrl_stream_wait_geq32(st, addr(flag), n + 1) == 0     # written above, on the same stream
        assert L.madrl_stream_wait_geq32(st, addr(flag), n) == 0         # GEQ: an older value passes too
        assert L.madrl_copy_async(addr(dst, 3), addr(src, 1), n, st) == 0
        torch.cuda.synchronize()
        assert torch.equal(dst[3:3 + n], src[1:1 + n]), n
        assert bool((dst[:3] == 0xEE).all()) and bool((dst[3 + n:] == 0xEE).all()), n
    assert flag[0].item() == 4098

    for f, v in ((L.madrl_stream_write32, 1), (L.madrl_stream_wait_geq32, 0)):
        assert f(st, None, v) == -1
        assert f(st, addr(flag, 2), v) == -1
        assert b"4-byte aligned" in L.madrl_last_error()
    assert L.madrl_copy_async(None, addr(src), 4, st) == -1
    assert L.madrl_copy_async(addr(src), None, 4, st) == -1
    torch.cuda.synchronize()
    assert flag.tolist() == [4098, 0xCAFE, 0, -1]


def test_one_rank_exchange_end_to_end():
    """The 2-GPU test's worker as a one-rank NCCL group on cuda:0: PeerGather (root and all), AsyncRootGather with
    both completion protocols, madrl_ipc_alloc / _free and the exchange primitives.  With one rank, every wait is for
    a value the same stream has already written.  A worker still alive after the timeout is killed."""
    import torch.multiprocessing as mp
    from test_peer_gather_gpu import _worker
    ctx = mp.get_context("spawn")
    q = ctx.SimpleQueue()
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    p = ctx.Process(target=_worker, args=(0, 1, port, q))
    p.start()
    p.join(300)
    if p.is_alive():
        p.kill()
        p.join()
        pytest.fail("the one-rank exchange worker did not finish")
    assert p.exitcode == 0
    assert q.get() == (0, True)
