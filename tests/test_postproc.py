"""Post-processing passes: oracle vs what the REAL reference wrappers computed (CPU) and CUDA kernels
vs oracle (GPU)."""
import numpy as np
import pytest

from oracle import postproc_oracle as po
from oracle import ref_records as R
from oracle.postproc_oracle import StandardizeEnv, discount_cumsum, episode_stats_env, frame_stack_env, gae_env


def test_oracles_equal_reference_wrappers():
    """ObservationBuffer / StandardizedEnv (madrl_environments/__init__.py) on scripted inputs: their
    outputs are stored (oracle/ref_records.py)."""
    ref = np.load(R.RECORDS)
    obs0, obs, rew, B = R.wrapper_inputs()
    T, A, D = obs.shape
    o0, o = frame_stack_env(obs0, obs, np.zeros(T, bool), B)
    assert np.array_equal(ref["obsbuf_reset"], o0) and np.array_equal(ref["obsbuf_obs"], o)
    mine = StandardizeEnv(A, D, 0.5, True, True, 0.05, 0.02)
    assert np.array_equal(ref["std_reset"], mine.obs(obs0))
    for t in range(T):
        assert np.array_equal(ref["std_obs"][t], mine.obs(obs[t]))
        assert np.array_equal(ref["std_rew"][t], mine.rew(rew[t]))


def test_episode_stats_oracle_equals_reference_wrapper():
    """DiagnosticsWrapper's per-episode log entries (t, reward per agent, avg reward, discounted return,
    length), stored from the reference (oracle/ref_records.py)."""
    ref = np.load(R.RECORDS)["episode_stats"]
    obs0, obs, rew, done = R.episode_stats_inputs()
    A = obs0.shape[0]
    mine = episode_stats_env(rew, done, 0.9, 12)
    assert len(ref) == len(mine) >= 5
    for g, m in zip(ref, mine):
        assert g[0] == m[0] and np.array_equal(g[1:1 + A], m[1]) and g[A + 1] == m[2] and g[A + 2] == m[3]
        assert g[A + 3] == m[4]


def test_batch_statistics_oracle_equals_rllab_functions():
    """center_advantages / shift_advantages_to_positive / explained_variance_1d / discount_cumsum
    of the oracle against the reference's own functions (rllab/rllab/algos/util.py:7-12,
    rllab/rllab/misc/special.py:51-59,107-111), bit for bit; their outputs are stored
    (oracle/ref_records.py)."""
    ref = np.load(R.RECORDS)
    cases, r1, r2 = R.batch_stat_inputs()
    for n, (adv, y) in zip((1, 2, 17, 4096), cases):
        assert np.array_equal(po.center_advantages(adv), ref["center_%d" % n])
        assert np.array_equal(po.shift_advantages_to_positive(adv), ref["shift_%d" % n])
        assert po.explained_variance_1d(adv, y) == ref["ev_%d" % n]
        assert np.array_equal(discount_cumsum(adv, 0.97), ref["dcs_%d" % n])
    const = np.full(9, 2.5)
    assert po.explained_variance_1d(const, const) == ref["ev_const"][0] == 1
    assert po.explained_variance_1d(r1, const) == ref["ev_const"][1] == 0


def test_gae_oracle_matches_rllab_formulas():
    rs = np.random.RandomState(1)
    T, A = 30, 2
    rew, val = rs.randn(T, A), rs.randn(T, A)
    done = np.zeros(T, bool)
    done[[9, 19, 29]] = True
    adv, ret = gae_env(rew, val, done, 0.99, 0.95)
    for s, e in ((0, 10), (10, 20), (20, 30)):            # rllab: one call per complete path
        for a in range(A):
            b = np.append(val[s:e, a], 0)
            deltas = rew[s:e, a] + 0.99 * b[1:] - b[:-1]
            assert np.array_equal(adv[s:e, a], discount_cumsum(deltas, 0.99 * 0.95))
            assert np.array_equal(ret[s:e, a], discount_cumsum(rew[s:e, a], 0.99))
    assert ret[9, 0] == rew[9, 0]                          # a path's last step sees no future


def test_to_paths_splits_at_done():
    from madrl_b200.postproc import to_paths
    T, E, A = 6, 2, 2
    done = np.zeros((T, E), np.uint8)
    done[2, 0] = 1
    done[5, 1] = 1
    rew = np.arange(T * E * A, dtype=np.float32).reshape(T, E, A)
    paths = to_paths(np.zeros((T, E, A, 3)), np.zeros((T, E, A, 2)), rew, done, dict(x=np.ones((T, E))))
    lens = sorted((p['env'], p['agent'], len(p['rewards']), p['terminated']) for p in paths)
    assert lens == [(0, 0, 3, False), (0, 0, 3, True), (0, 1, 3, False), (0, 1, 3, True),
                    (1, 0, 6, True), (1, 1, 6, True)]
    assert all(p['env_infos']['x'].shape[0] == len(p['rewards']) for p in paths)


@pytest.mark.gpu
def test_cuda_postproc_matches_oracle():
    import torch
    from madrl_b200.postproc import EpisodeStats, FrameStack, Standardizer, gae
    rs = np.random.RandomState(2)
    T, E, A, D, B = 50, 7, 3, 11, 4
    obs0 = rs.randn(E, A, D).astype(np.float32)
    obs = rs.randn(T, E, A, D).astype(np.float32)
    rew = rs.randn(T, E, A).astype(np.float32)
    val = rs.randn(T, E, A).astype(np.float32)
    last = rs.randn(E, A).astype(np.float32)
    done = (rs.rand(T, E) < 0.1)
    dev = 'cuda'
    d_t = torch.as_tensor(done.astype(np.uint8), device=dev)
    # GAE
    for lv in (None, last):
        adv, ret = gae(torch.as_tensor(rew, device=dev), torch.as_tensor(val, device=dev), d_t, 0.99, 0.95,
                       None if lv is None else torch.as_tensor(lv, device=dev))
        for e in range(E):
            a_o, r_o = gae_env(rew[:, e], val[:, e], done[:, e], 0.99, 0.95, None if lv is None else lv[e])
            assert np.abs(adv[:, e].cpu().numpy() - a_o).max() < 1e-4
            assert np.abs(ret[:, e].cpu().numpy() - r_o).max() < 1e-4
    # frame stack (two consecutive rollouts exercise the carry)
    fs = FrameStack(E, A, D, B, dev)
    st0 = fs.reset(torch.as_tensor(obs0, device=dev)).cpu().numpy()
    o1 = fs.rollout(torch.as_tensor(obs[:20], device=dev), d_t[:20]).cpu().numpy()
    o2 = fs.rollout(torch.as_tensor(obs[20:], device=dev), d_t[20:]).cpu().numpy()
    for e in range(E):
        s0, so = frame_stack_env(obs0[e].astype(np.float64), obs[:, e].astype(np.float64), done[:, e], B)
        assert np.array_equal(st0[e], s0.astype(np.float32))
        assert np.array_equal(np.concatenate([o1, o2])[:, e], so.astype(np.float32))
    # standardizer
    sd = Standardizer(E, A, D, dev, scale_reward=0.5, enable_obsnorm=True, enable_rewnorm=True,
                      obs_alpha=0.05, rew_alpha=0.02)
    x0 = torch.as_tensor(obs0, device=dev).clone()
    sd.obs(x0)
    xo = torch.as_tensor(obs, device=dev).clone()
    xr = torch.as_tensor(rew, device=dev).clone()
    sd.obs(xo)
    sd.rew(xr)
    for e in range(E):
        m = StandardizeEnv(A, D, 0.5, True, True, 0.05, 0.02)
        assert np.abs(m.obs(obs0[e].astype(np.float64)) - x0[e].cpu().numpy()).max() < 1e-5
        for t in range(T):
            assert np.abs(m.obs(obs[t, e].astype(np.float64)) - xo[t, e].cpu().numpy()).max() < 1e-5
            assert np.abs(m.rew(rew[t, e].astype(np.float64)) - xr[t, e].cpu().numpy()).max() < 1e-5
        assert np.abs(m.obs_var - sd.obs_var[e].cpu().numpy()).max() < 1e-12
    # episode statistics (two calls exercise the carry)
    es = EpisodeStats(E, A, dev, discount=0.9, max_traj_len=12)
    r_t = torch.as_tensor(rew, device=dev)
    s1, s2 = es.rollout(r_t[:23], d_t[:23]), es.rollout(r_t[23:], d_t[23:])
    cat = {k: torch.cat([s1[k], s2[k]]).cpu().numpy() for k in s1}
    for e in range(E):
        recs = episode_stats_env(rew[:, e].astype(np.float64), done[:, e], 0.9, 12)
        assert [r[0] for r in recs] == list(np.nonzero(cat['end'][:, e])[0])
        for t, ep_r, avg, disc, length in recs:
            assert np.abs(cat['episode_reward'][t, e] - ep_r).max() < 1e-4
            assert abs(cat['episode_avg_reward'][t, e] - avg) < 1e-4 and abs(cat['episode_disc_return'][t, e] - disc) < 1e-4
            assert cat['episode_length'][t, e] == length


@pytest.mark.gpu
def test_cuda_batch_statistics_match_oracle():
    """center_advantages / moments (madrl_moments_pass_f32, madrl_center_apply_f32) against the oracle (float64
    NumPy on the same float32 inputs); tolerance 1e-5 relative to the value scale, results deterministic."""
    import torch
    from madrl_b200.postproc import center_advantages, explained_variance, moments
    import postproc_edges as pe
    rs = np.random.RandomState(9)
    cases = [(shape, 1.0) for shape in ((1,), (3,), (50, 7, 3), (256, 4096, 5))]
    # the block edge and the grid-stride edges of the moments launch, data offset by 1e4 so that a one-pass
    # variance would miss the rtol 1e-10 below
    cases += [((n,), 1e4) for n in pe.stride_sizes(pe.csrc_default("MADRL_MOM_BLOCKS", "postproc.cu"))]
    for shape, offset in cases:
        adv = (rs.randn(*shape) * 3 + offset).astype(np.float32)
        ret = rs.randn(*shape).astype(np.float32)
        a_t, r_t = torch.as_tensor(adv, device='cuda'), torch.as_tensor(ret, device='cuda')
        flat = adv.ravel().astype(np.float64)
        for center, positive in ((True, False), (False, True), (True, True), (False, False)):
            want = flat
            if center:
                want = po.center_advantages(want)
            if positive:
                want = po.shift_advantages_to_positive(want)
            got = center_advantages(a_t, center=center, positive=positive)
            assert got.shape == a_t.shape and got.data_ptr() != a_t.data_ptr()
            tol = 1e-5 * max(1.0, np.abs(want).max())
            assert np.abs(got.cpu().numpy().ravel() - want).max() <= tol
            again = center_advantages(a_t, center=center, positive=positive)
            assert torch.equal(got, again)                                 # deterministic reduction
        assert torch.equal(a_t, torch.as_tensor(adv, device='cuda'))       # input untouched
        st = moments(a_t, r_t).cpu().numpy()
        r64 = ret.ravel().astype(np.float64)
        want_st = np.array([flat.mean(), r64.mean(), (r64 - flat).mean(), flat.var(), r64.var(),
                            (r64 - flat).var(), flat.min(), r64.min(), (r64 - flat).min()])
        assert np.allclose(st, want_st, rtol=1e-10, atol=1e-12)
        ev = explained_variance(a_t, r_t)
        assert abs(ev - po.explained_variance_1d(flat, r64)) < 1e-9
    const = torch.full((64,), 2.5, device='cuda')
    assert explained_variance(const, const) == 1
    assert explained_variance(torch.as_tensor(rs.randn(64).astype(np.float32), device='cuda'), const) == 0
    out = center_advantages(const.clone(), inplace=True)                  # zero variance: 0 / 1e-8
    assert torch.equal(out, torch.zeros_like(out))


@pytest.mark.gpu
def test_cuda_moments_divide_the_pass_sums_by_the_rows():
    """`moments` and `moments_agents` equal, bit for bit, madrl_moments_pass_f32's two passes called directly with
    their sums divided by the rows in NumPy float64 (one IEEE division per value).  rows = 3 x 5^7, whose reciprocal
    is not exact: a multiplication by 1 / rows would differ in the last bit of some of the values."""
    import torch
    from madrl_b200 import _lib
    from madrl_b200._lib import _ptr
    from madrl_b200.postproc import moments, moments_agents
    rows, lib = 3 * 5 ** 7, _lib.lib()
    rs = np.random.RandomState(12)

    def passes(x, b, A):
        st = torch.full((A, 9), float("nan"), dtype=torch.float64, device="cuda")
        ws = torch.empty((A, 4096), dtype=torch.float64, device="cuda")
        want = np.empty((A, 9))
        for p in (0, 1):
            _lib.check(lib.madrl_moments_pass_f32(rows, A, _ptr(x), _ptr(b), p, _ptr(st), _ptr(ws),
                                                  _lib.stream(x.device)))
            want[:] = st.cpu().numpy()
            want[:, 3 * p:3 * p + 3] /= np.float64(rows)
            st.copy_(torch.from_numpy(want))
        return want

    for A in (1, 3):
        x = torch.as_tensor((rs.randn(rows, A) * 3 + 1e4).astype(np.float32), device="cuda")
        y = torch.as_tensor((rs.randn(rows, A) + 1).astype(np.float32), device="cuda")
        for b in (y, None):
            want = passes(x, b, A)
            assert np.array_equal(moments_agents(x, b).cpu().numpy(), want), (A, b is None)
            if A == 1:
                assert np.array_equal(moments(x.view(-1), None if b is None else b.view(-1)).cpu().numpy(), want[0])


@pytest.mark.gpu
def test_cuda_pack_paths_matches_host_to_paths():
    """Device-side path packing (csrc/postproc.cu paths_plan / paths_pack kernels, SURVEY 8f row 1:
    dec_rollout-shaped paths, rllab/rllab/sampler/ma_sampler.py:52-100) on a real Waterworld rollout
    with auto-reset, against the host `to_paths` triple loop."""
    import torch
    from madrl_b200 import BatchedMAWaterWorld
    from madrl_b200.postproc import pack_paths, to_paths
    E, T, mpl = 37, 50, 11
    eng = BatchedMAWaterWorld(E, 5, 5, n_coop=1, radius=0.04, seed=3, max_path_length=mpl)
    obs0 = eng.reset().clone()
    act = torch.randn(T, E, 5, 2, device="cuda") * 0.7
    obs, rew, done, info = eng.rollout(act, auto_reset=True)
    infos = dict(evcatches=info[..., 0].contiguous(), pocatches=info[..., 1].contiguous())
    pp = pack_paths(obs, act, rew, done, infos, obs_before=obs0)
    shifted = torch.cat([obs0.unsqueeze(0), obs[:-1]]).cpu()
    want = to_paths(shifted, act.cpu(), rew.cpu(), done.cpu(), {k: v.cpu() for k, v in infos.items()})
    got = pp.to_list()
    assert len(got) == len(want) == len(pp) and len(got) > E * 5 * (T // mpl)
    for g, w in zip(got, want):
        assert (g['env'], g['agent'], g['terminated']) == (w['env'], w['agent'], w['terminated'])
        for k in ('observations', 'actions', 'rewards'):
            assert np.array_equal(g[k], w[k]), k
        for k in infos:
            assert np.array_equal(g['env_infos'][k], w['env_infos'][k])
    one = pp.path(7)                       # zero-copy device views of one path
    assert one['observations'].is_cuda and one['observations'].shape == (int(pp.length[7]), eng.obs_dim)
    # a rollout without any done: one path per (env, agent) covering the whole rollout
    pp2 = pack_paths(obs, act, rew, torch.zeros_like(done), None)
    assert len(pp2) == E * 5 and int(pp2.length.min()) == T
    assert torch.equal(pp2.path(6)['observations'], obs[:, 1, 1])


@pytest.mark.gpu
def test_cuda_terminal_obs_side_tensor_and_standardizer_order():
    """engine.set_terminal_obs + Standardizer.obs(obs, done, terminal_obs) on the GPU: the side tensor
    holds the pre-reset observation of every done step, and the running estimate follows the reference
    order (terminal observation, then reset observation; madrl_environments/__init__.py:283-291)."""
    import torch
    from madrl_b200 import BatchedMAWaterWorld
    from madrl_b200.postproc import Standardizer
    E, T, mpl = 9, 23, 6
    mk = lambda: BatchedMAWaterWorld(E, 5, 5, seed=5, max_path_length=mpl)          # noqa: E731
    a, c = mk(), mk()
    a.reset(), c.reset()
    act = torch.randn(T, E, 5, 2, device="cuda") * 0.5
    term = torch.full((T, E, 5, a.obs_dim), -7.0, device="cuda")
    a.set_terminal_obs(term)
    obs, rew, done, _ = a.rollout(act, auto_reset=True)
    a.set_terminal_obs(None)
    assert int(done.sum()) == E * (T // mpl)
    for t in range(T):                                   # the same envs stepped without auto-reset
        o, _, d, _ = c.rollout(act[t:t + 1], auto_reset=False)
        hit = d[0].bool()
        assert torch.equal(term[t][hit], o[0][hit]) and bool((term[t][~hit] == -7.0).all())
        if hit.any():
            c.reset(mask=d[0])
    std = Standardizer(E, 5, a.obs_dim, "cuda", enable_obsnorm=True, obs_alpha=0.05)
    x, tm = obs.clone(), term.clone()
    std.obs(x, done, tm)
    obs_h, term_h, done_h = obs.cpu().numpy(), term.cpu().numpy(), done.cpu().numpy()
    for e in (0, 4, 8):
        mine = StandardizeEnv(5, a.obs_dim, 1.0, True, False, 0.05, 0.001)
        for t in range(T):
            if done_h[t, e]:
                assert np.abs(mine.obs(term_h[t, e].astype(np.float64)) - tm[t, e].cpu().numpy()).max() < 1e-4
            assert np.abs(mine.obs(obs_h[t, e].astype(np.float64)) - x[t, e].cpu().numpy()).max() < 1e-4, (t, e)
        assert np.abs(mine.obs_mean - std.obs_mean[e].cpu().numpy()).max() < 1e-9
