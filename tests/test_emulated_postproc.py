"""The trajectory post-processing kernels (madrl_b200/csrc/postproc.cu: GAE, frame stack,
standardiser, episode statistics, whole-batch moments / advantage centring) executed on the CPU by
the warp emulator of tests/emu and compared with oracle/postproc_oracle.py -- the GPU test
tests/test_postproc.py::test_cuda_* at small sizes, through the same C ABI."""
import numpy as np
import pytest

import postproc_edges as pe
from emu import build_emu, driver
from emu.driver import Guarded
from emu.driver import ptr as _p
from oracle import postproc_oracle as po

pytestmark = driver.needs_cxx


@pytest.fixture(scope="module")
def lib():
    return driver.load(())


def _data():
    rs = np.random.RandomState(2)
    T, E, A, D, B = 30, 5, 3, 7, 4
    return dict(T=T, E=E, A=A, D=D, B=B, obs0=rs.randn(E, A, D).astype(np.float32),
                obs=rs.randn(T, E, A, D).astype(np.float32), rew=rs.randn(T, E, A).astype(np.float32),
                val=rs.randn(T, E, A).astype(np.float32), last=rs.randn(E, A).astype(np.float32),
                done=(rs.rand(T, E) < 0.12).astype(np.uint8))


def test_gae(lib):
    d = _data()
    T, E, A = d['T'], d['E'], d['A']
    for lv in (None, d['last']):
        adv, ret = np.empty_like(d['rew']), np.empty_like(d['rew'])
        assert lib.madrl_gae_f32(T, E, A, _p(d['rew']), _p(d['val']), _p(d['done']), _p(lv), 0.99, 0.95, _p(adv),
                                 _p(ret), None) == 0
        for e in range(E):
            a_o, r_o = po.gae_env(d['rew'][:, e], d['val'][:, e], d['done'][:, e].astype(bool), 0.99, 0.95,
                                  None if lv is None else lv[e])
            assert np.abs(adv[:, e] - a_o).max() < 1e-4 and np.abs(ret[:, e] - r_o).max() < 1e-4


def test_frame_stack(lib):
    d = _data()
    T, E, A, D, B = d['T'], d['E'], d['A'], d['D'], d['B']
    carry = np.repeat(d['obs0'][..., None], B, axis=-1).copy()          # reset(): every slot = reset obs
    out = np.empty((T, E, A, D, B), np.float32)
    for t0, t1 in ((0, 11), (11, T)):                                       # two calls exercise the carry
        o = np.ascontiguousarray(d['obs'][t0:t1])
        dn = np.ascontiguousarray(d['done'][t0:t1])
        res = np.empty((t1 - t0, E, A, D, B), np.float32)
        assert lib.madrl_frame_stack_f32(t1 - t0, E, A, D, B, _p(o), _p(dn), _p(carry), _p(res), None) == 0
        out[t0:t1] = res
    for e in range(E):
        s0, so = po.frame_stack_env(d['obs0'][e].astype(np.float64), d['obs'][:, e].astype(np.float64),
                                    d['done'][:, e].astype(bool), B)
        assert np.array_equal(out[:, e], so.astype(np.float32))


def test_standardizer(lib):
    d = _data()
    T, E, A, D = d['T'], d['E'], d['A'], d['D']
    n = E * A * D
    mean, var = np.zeros(n), np.ones(n)
    x0, xo = d['obs0'].copy(), d['obs'].copy()
    assert lib.madrl_standardize_f32(1, n, _p(x0), _p(mean), _p(var), 0.05, 1e-8, 1, 1.0, 1, None) == 0
    assert lib.madrl_standardize_f32(T, n, _p(xo), _p(mean), _p(var), 0.05, 1e-8, 1, 1.0, 1, None) == 0
    rmean, rvar = np.zeros(E * A), np.ones(E * A)
    xr = d['rew'].copy()
    assert lib.madrl_standardize_f32(T, E * A, _p(xr), _p(rmean), _p(rvar), 0.02, 1e-8, 0, 0.5, 1, None) == 0
    for e in range(E):
        m = po.StandardizeEnv(A, D, 0.5, True, True, 0.05, 0.02)
        assert np.abs(m.obs(d['obs0'][e].astype(np.float64)) - x0[e]).max() < 1e-5
        for t in range(T):
            assert np.abs(m.obs(d['obs'][t, e].astype(np.float64)) - xo[t, e]).max() < 1e-5
            assert np.abs(m.rew(d['rew'][t, e].astype(np.float64)) - xr[t, e]).max() < 1e-5
        assert np.abs(m.obs_var - var.reshape(E, A, D)[e]).max() < 1e-12


def test_episode_stats(lib):
    d = _data()
    T, E, A = d['T'], d['E'], d['A']
    carry = np.zeros((E, A + 3))
    outs = dict(r=np.empty((T, E, A), np.float32), dsc=np.empty((T, E), np.float32),
                ln=np.empty((T, E), np.int32), end=np.empty((T, E), np.uint8))
    for t0, t1 in ((0, 13), (13, T)):
        r = np.ascontiguousarray(d['rew'][t0:t1]); dn = np.ascontiguousarray(d['done'][t0:t1])
        part = [np.empty((t1 - t0, E, A), np.float32), np.empty((t1 - t0, E), np.float32),
                np.empty((t1 - t0, E), np.int32), np.empty((t1 - t0, E), np.uint8)]
        assert lib.madrl_episode_stats_f32(t1 - t0, E, A, _p(r), _p(dn), 0.9, 12, _p(carry), *[_p(x) for x in part],
                                           None) == 0
        for k, x in zip(('r', 'dsc', 'ln', 'end'), part):
            outs[k][t0:t1] = x
    for e in range(E):
        recs = po.episode_stats_env(d['rew'][:, e].astype(np.float64), d['done'][:, e].astype(bool), 0.9, 12)
        assert [r[0] for r in recs] == list(np.nonzero(outs['end'][:, e])[0])
        for t, ep_r, avg, disc, length in recs:
            assert np.abs(outs['r'][t, e] - ep_r).max() < 1e-4 and abs(outs['dsc'][t, e] - disc) < 1e-4
            assert outs['ln'][t, e] == length


def test_moments_and_advantage_centring(lib):
    rs = np.random.RandomState(9)
    for n in (1, 3, 1050, 20000):        # 20000: every block of the (narrowed, see build_emu.py) grid loops
        adv = (rs.randn(n) * 3 + 1).astype(np.float32)
        ret = rs.randn(n).astype(np.float32)
        stats, ws = np.empty(9), np.empty(4096)
        assert lib.madrl_moments_f32(n, _p(adv), _p(ret), _p(stats), _p(ws), None) == 0
        a64, r64 = adv.astype(np.float64), ret.astype(np.float64)
        want = np.array([a64.mean(), r64.mean(), (r64 - a64).mean(), a64.var(), r64.var(), (r64 - a64).var(),
                         a64.min(), r64.min(), (r64 - a64).min()])
        assert np.allclose(stats, want, rtol=1e-10, atol=1e-12)
        for center, positive in ((1, 0), (0, 1), (1, 1)):
            x = adv.copy()
            assert lib.madrl_center_advantages_f32(n, _p(x), center, positive, _p(stats), _p(ws), None) == 0
            w = a64
            if center:
                w = po.center_advantages(w)
            if positive:
                w = po.shift_advantages_to_positive(w)
            assert np.abs(x - w).max() <= 1e-5 * max(1.0, np.abs(w).max())


def test_path_packing_kernels_equal_host_to_paths(lib):
    """madrl_paths_plan + madrl_paths_pack_u32 (the device-side `to_paths`) against the host triple
    loop of madrl_b200.postproc.to_paths: same paths in the same order, with and without the one-step
    observation shift."""
    from madrl_b200.postproc import to_paths
    rs = np.random.RandomState(4)
    for T, E, A, D, p_done in ((30, 5, 3, 7, 0.12), (9, 2, 1, 40, 0.4), (17, 3, 4, 1, 0.0)):
        obs = rs.randn(T, E, A, D).astype(np.float32)
        obs_before = rs.randn(E, A, D).astype(np.float32)
        act = rs.randint(0, 5, size=(T, E, A)).astype(np.int32)
        rew = rs.randn(T, E, A).astype(np.float32)
        info = rs.randint(0, 9, size=(T, E)).astype(np.int32)
        done = (rs.rand(T, E) < p_done).astype(np.uint8)
        seg_s, seg_l, n_ep, ep_rec = driver.paths_plan(lib, done, A)

        def pack(x, n_agents, first=None, per_agent=True):
            tail = x.shape[3:] if per_agent else x.shape[2:]
            out = np.zeros((T * E * n_agents,) + tail, x.dtype)
            Dw = max(1, int(np.prod(tail)))
            assert lib.madrl_paths_pack_u32(T, E, n_agents, Dw, _p(np.ascontiguousarray(x)), _p(first), _p(seg_s),
                                            _p(seg_l), _p(out), None) == 0
            return out
        for shifted in (False, True):
            p_obs = pack(obs, A, obs_before if shifted else None)
            p_act, p_rew, p_info = pack(act, A), pack(rew, A), pack(info, 1, per_agent=False)
            src_obs = np.concatenate([obs_before[None], obs[:-1]]) if shifted else obs
            want = to_paths(src_obs, act, rew, done, dict(k=info))
            got = []
            for e in range(E):
                for j in range(n_ep[e]):
                    s, L, term = ep_rec[e, j]
                    for a in range(A):
                        o = e * T * A + s * A + a * L
                        got.append(dict(observations=p_obs[o:o + L], actions=p_act[o:o + L], rewards=p_rew[o:o + L],
                                        env_infos=dict(k=p_info[e * T + s:e * T + s + L]), env=e, agent=a,
                                        terminated=bool(term)))
            assert len(got) == len(want)
            for g, w in zip(got, want):
                assert (g['env'], g['agent'], g['terminated']) == (w['env'], w['agent'], w['terminated'])
                for k in ('observations', 'actions', 'rewards'):
                    assert np.array_equal(g[k], w[k]), k
                assert np.array_equal(g['env_infos']['k'], w['env_infos']['k'])


def test_standardizer_with_terminal_observations_follows_the_reference_order(lib):
    """madrl_standardize_obs_terminal_f32 vs the StandardizedEnv oracle (pinned to the real wrapper in
    tests/test_postproc.py): at a done step the estimate sees the terminal observation first, then the
    reset observation (step() then reset(), madrl_environments/__init__.py:283-291)."""
    d = _data()
    T, E, A, D = d['T'], d['E'], d['A'], d['D']
    rs = np.random.RandomState(8)
    term = rs.randn(T, E, A, D).astype(np.float32)
    x, tm = d['obs'].copy(), term.copy()
    mean, var = np.zeros((E, A, D)), np.ones((E, A, D))
    assert lib.madrl_standardize_obs_terminal_f32(T, E, A * D, _p(x), _p(tm), _p(d['done']), _p(mean), _p(var),
                                                  0.05, 1e-8, None) == 0
    for e in range(E):
        mine = po.StandardizeEnv(A, D, 1.0, True, False, 0.05, 0.001)
        for t in range(T):
            if d['done'][t, e]:
                assert np.abs(np.array(mine.obs(term[t, e].astype(np.float64))) - tm[t, e]).max() < 1e-5, (t, e)
            else:
                assert np.array_equal(tm[t, e], term[t, e])          # untouched
            assert np.abs(np.array(mine.obs(d['obs'][t, e].astype(np.float64))) - x[t, e]).max() < 1e-5, (t, e)
        assert np.abs(np.array(mine.obs_mean) - mean[e]).max() < 1e-12


# ---------------------------------------------------------------- the edges of tests/test_postproc_edges_gpu.py
# The same cases and checks (tests/postproc_edges.py), with the size edges of this build: its moments grid is
# MADRL_MOM_BLOCKS CTAs of 256 threads (build_emu.GRID), so its stride edge is that times 256.

EMU_MOM_BLOCKS = build_emu.GRID["MADRL_MOM_BLOCKS"]


def test_moments_at_the_grid_stride_edges(lib):
    """n at the block edge and at one and three grid strides, data offset by 1e4 (a one-pass variance fails)."""
    for n in pe.stride_sizes(EMU_MOM_BLOCKS):
        a, b = pe.offset_series(n, n)
        stats, ws = np.full(9, np.nan), np.empty(4096)
        assert lib.madrl_moments_f32(n, _p(a), _p(b), _p(stats), _p(ws), None) == 0
        assert np.allclose(stats, pe.moments_want(a, b), rtol=1e-10, atol=1e-12), n


@pytest.mark.parametrize("A", [1, 2, 3, 257])
def test_agent_moments_and_centring_equal_pooled_bitwise(lib, A):
    """Agent a's statistics and centred column are the pooled call's on that column alone, bit for bit (same block
    loop, fold order and constant expressions).  A = 257: the per-agent constants of the centring kernel take a
    second pass of its strided loop; a launch then has 6 x 257 CTAs of fibers, so that case runs one centring
    mode and compares the agents on either side of 256 (the GPU test covers every agent and mode)."""
    rows = 2 * EMU_MOM_BLOCKS * 256 + 7 if A <= 3 else 45
    x, y = pe.agent_columns(rows, A, A)
    agents, modes = (range(A), pe.CENTRE_MODES) if A <= 3 else ((0, 255, 256), ((1, 1),))
    stats, ws = np.full((A, 9), np.nan), np.empty((A, 4096))
    st1, ws1 = np.empty(9), np.empty(4096)
    if A <= 3:
        assert lib.madrl_moments_agents_f32(rows, A, _p(x), _p(y), _p(stats), _p(ws), None) == 0
        for a in agents:
            xa, ya = np.ascontiguousarray(x[:, a]), np.ascontiguousarray(y[:, a])
            assert lib.madrl_moments_f32(rows, _p(xa), _p(ya), _p(st1), _p(ws1), None) == 0
            assert np.array_equal(stats[a], st1), a
    for center, positive in modes:
        xs = Guarded(x.shape, np.float32, x)
        assert lib.madrl_center_advantages_agents_f32(rows, A, _p(xs.arr), center, positive, _p(stats), _p(ws),
                                                      None) == 0
        got = xs.check("adv")
        for a in agents:
            xa = x[:, a].copy()
            assert lib.madrl_center_advantages_f32(rows, _p(xa), center, positive, _p(st1), _p(ws1), None) == 0
            assert np.array_equal(stats[a], st1) and np.array_equal(got[:, a], xa), (center, positive, a)


def test_frame_stack_every_buffer_size(lib):
    """B = 1..8, float32 and bfloat16, n = E*A*D over several blocks with a tail; three chained calls (done on a
    call's first step, on every step, never) bit for bit ObservationBuffer's; outputs and carry canary-guarded."""
    E, A, D = 37, 3, 29
    for bf16 in (False, True):
        obs0, calls = pe.frame_stack_calls(E, A, D, 5, bf16)
        dt = np.uint16 if bf16 else np.float32
        enc = (lambda v: pe.bf16_bits(v)[0]) if bf16 else (lambda v: v)                      # noqa: E731
        dec = (lambda v: (v.astype(np.uint32) << 16).view(np.float32)) if bf16 else np.copy   # noqa: E731
        fn = lib.madrl_frame_stack_bf16 if bf16 else lib.madrl_frame_stack_f32
        for B in range(1, 9):
            carry = Guarded((E, A, D, B), dt, enc(obs0)[..., None])
            outs = []
            for obs, done in calls:
                T = obs.shape[0]
                res = Guarded((T, E, A, D, B), dt, 0)
                src = np.ascontiguousarray(enc(obs))     # bound: _p keeps only the address of the array
                assert fn(T, E, A, D, B, _p(src), _p(done), _p(carry.arr), _p(res.arr), None) == 0
                carry.check("carry")
                outs.append(dec(res.check("out")))
            pe.check_frame_stack(obs0, calls, outs, B)


def test_standardizer_across_both_inv_std_paths(lib):
    """Running estimates set so that the updated variance v' lands on 0, subnormals, 1e-300, float32 1e-30 and its
    neighbours, 1, float32 1e30 and its neighbours and 1e300; one step, within a float32 ulp of the float64
    (x - m') / (sqrt(v') + eps); then pure scaling and the terminal-observation pass."""
    eps, alpha = pe.STD_EPS, pe.STD_ALPHA
    x, m, v, vt = pe.std_reward_case()
    n = x.size
    xr, mean, var = x.copy(), m.copy(), v.copy()
    assert lib.madrl_standardize_f32(1, n, _p(xr), _p(mean), _p(var), alpha, eps, 0, 0.5, 1, None) == 0
    assert np.array_equal(mean, m) and np.array_equal(var, vt)
    off = pe.check_standardized(xr, 0.5 * x.astype(np.float64) / (np.sqrt(vt) + eps))
    xs, mean, var = x.copy(), m.copy(), v.copy()
    assert lib.madrl_standardize_f32(1, n, _p(xs), _p(mean), _p(var), alpha, eps, 0, 0.5, 0, None) == 0
    assert np.array_equal(xs, (0.5 * x.astype(np.float64)).astype(np.float32))              # pure scaling
    assert np.array_equal(mean, m) and np.array_equal(var, v)
    x, m, v, m1, v1 = pe.std_obs_case()
    assert all(pe.std_target_classes(v1).values())
    xo, mean, var = x.copy(), m.copy(), v.copy()
    assert lib.madrl_standardize_f32(1, x.size, _p(xo), _p(mean), _p(var), alpha, eps, 1, 1.0, 1, None) == 0
    assert np.array_equal(mean, m1) and np.array_equal(var, v1)
    off += pe.check_standardized(xo, (x.astype(np.float64) - m1) / (np.sqrt(v1) + eps))
    assert off <= 2, off
    obs, term, done = pe.terminal_case(4, 7, 40, 3)
    T, E, P = obs.shape
    xt, tm, mean, var = obs.copy(), term.copy(), np.zeros((E, P)), np.ones((E, P))
    assert lib.madrl_standardize_obs_terminal_f32(T, E, P, _p(xt), _p(tm), _p(done), _p(mean), _p(var), 0.05, eps,
                                                  None) == 0
    pe.check_terminal(xt, tm, obs, term, done, 0.05, mean)


def test_gae_edges(lib):
    """E*A over several blocks with a tail; T = 1 and 17; done at t = 0, at T-1, on every step, never; with and
    without last_value; (gamma, lambda) in {(0.99, 0.95), (1, 1), (0, 0.5)}."""
    E, A = 301, 3
    for T in (1, 17):
        rew, val, last, done = pe.gae_case(T, E, A, T)
        for discount, lam in pe.GAE_PARAMS:
            for lv in (None, last):
                adv, ret = np.full_like(rew, np.nan), np.full_like(rew, np.nan)
                assert lib.madrl_gae_f32(T, E, A, _p(rew), _p(val), _p(done), _p(lv), discount, lam, _p(adv), _p(ret),
                                         None) == 0
                pe.check_gae(adv, ret, rew, val, done, discount, lam, lv)


@pytest.mark.parametrize("E,A,kind", [(131, 32, "len1"), (131, 3, "boundary"), (140, 5, "span3")])
def test_episode_stats_edges(lib, E, A, kind):
    mtl, calls = pe.episode_stats_calls(E, A, kind, 1)
    carry, outs = np.zeros((E, A + 3)), []
    for rew, done in calls:
        T = rew.shape[0]
        part = [np.empty((T, E, A), np.float32), np.empty((T, E), np.float32), np.empty((T, E), np.int32),
                np.empty((T, E), np.uint8)]
        assert lib.madrl_episode_stats_f32(T, E, A, _p(rew), _p(done), 0.9, mtl, _p(carry), *[_p(p) for p in part],
                                           None) == 0
        outs.append(part)
    assert pe.check_episode_stats(outs, calls, 0.9, mtl) > 0


@pytest.mark.parametrize("itemsize", [4, 2], ids=["u32", "u16"])
def test_path_packing_word_counts(lib, itemsize):
    """D in {1..5, 31, 32, 33} words (one thread per row up to 4, one warp beyond), with and without the
    obs_before shift; T = 1, episodes of one step, E > 128; bit for bit the host to_paths."""
    pack = lib.madrl_paths_pack_u32 if itemsize == 4 else lib.madrl_paths_pack_u16
    for k, D in enumerate(pe.PACK_WORDS):
        for shifted in (False, True):
            T, E, A, p_done = pe.PACK_SHAPES[(k + shifted) % len(pe.PACK_SHAPES)]
            c = pe.pack_case(T, E, A, D, p_done, itemsize, 10 * D + shifted)
            seg_s, seg_l, n_ep, ep_rec = driver.paths_plan(lib, c["done"], A)
            p_obs = Guarded((T * E * A, D), c["obs"].dtype, 0)
            assert pack(T, E, A, D, _p(c["obs"]), _p(c["obs_before"] if shifted else None), _p(seg_s), _p(seg_l),
                        _p(p_obs.arr), None) == 0
            words = []
            for x, n_agents in ((c["act"], A), (c["rew"], A), (c["info"], 1)):
                out = Guarded((T * E * n_agents,), x.dtype, 0)
                assert lib.madrl_paths_pack_u32(T, E, n_agents, 1, _p(x), None, _p(seg_s), _p(seg_l), _p(out.arr),
                                                None) == 0
                words.append(out.check("packed"))
            pe.check_packed(c, shifted, pe.plan_paths(n_ep, ep_rec, T, A), p_obs.check("packed obs"), *words)
