"""The post-processing and linear-baseline kernels (csrc/postproc.cu, csrc/baseline.cu) on the GPU at the shapes
and values where their indexing and arithmetic have edges: the Gram kernel's 64-column tiles, row slices and
accumulator flush, single rows whose normal equations are exactly the outer product of the features, the moments
grid stride and the per-agent constant loop, every frame-stack buffer size, both paths of the standardiser's
reciprocal square root, and the narrow / wide path-packing kernels.  Cases and checks are shared with the emulated
tests (tests/postproc_edges.py); the expected values come from the float64 oracles of oracle/."""
import numpy as np
import pytest
import torch

import postproc_edges as pe
from oracle import baseline_oracle as bo
from oracle import concurrent_baseline_oracle as cbo

pytestmark = pytest.mark.gpu
DEV = "cuda"


def cu(x):
    return None if x is None else torch.as_tensor(np.ascontiguousarray(x), device=DEV)


def obs_dev(x, bf16):
    """float32 values (bfloat16-representable when bf16) as a device tensor of the observation dtype."""
    t = cu(x)
    return None if t is None else (t.to(torch.bfloat16) if bf16 else t)


# ---------------------------------------------------------------- linear feature baseline

@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
def test_single_row_normal_equations_and_predictions_are_the_exact_features(bf16):
    """One row (T = E = A = 1): every MMA product has one non-zero term and the other slices add exact zeros, so
    G = outer(f, f) bit for bit, f = [clip(o), clip(o)^2, a, a^2, a^3, 1, y] with a^3 the correctly rounded cube.
    Observations at +-10, the next value beyond, +-inf; time indices where NumPy's or glibc's pow is an ulp off.
    With a unit coefficient vector, predict returns a feature rounded to float32: per time column for the pooled
    baseline, every column at once for a baseline with one agent per column."""
    from madrl_b200.postproc import LinearFeatureBaseline
    rs = np.random.RandomState(11 + bf16)
    done = torch.zeros((1, 1), dtype=torch.uint8, device=DEV)
    for D in pe.LFB_DIMS:
        Df = 2 * D + 4
        pooled, per = LinearFeatureBaseline(D, DEV), LinearFeatureBaseline(D, DEV, n_agents=Df)
        per.set_param_values(np.eye(Df))
        for before in (False, True):
            for k, t0 in enumerate(pe.LFB_T0):
                o = pe.single_row_obs(D, k, bf16, rs)
                y = np.float32(rs.randn() * 4)
                f = pe.single_row_features(o, y, t0)
                row = obs_dev(o.reshape(1, 1, 1, D), bf16)
                ob = None
                if before:                       # the row is obs_before's; obs[0] is never read
                    ob, row = row.reshape(1, 1, D), torch.full_like(row, float("nan"))
                t0_t = torch.tensor([t0], dtype=torch.int32, device=DEV)
                ret = torch.tensor([[[float(y)]]], device=DEV)
                G = pooled.normal_equations(row, done, ret, ob, t0_t).cpu().numpy()
                assert np.array_equal(G, np.outer(f, f)), (D, before, t0)
                for j in range(2 * D, Df):
                    pooled.set_param_values(np.eye(Df)[j])
                    v = pooled.predict(row, done, ob, t0_t).item()
                    assert v == np.float32(f[j]), (D, before, t0, j)
                rows = row.expand(1, 1, Df, D).contiguous()
                obs_b = None if ob is None else ob.expand(1, Df, D).contiguous()
                vals = per.predict(rows, done, obs_b, t0_t).cpu().numpy().reshape(-1)
                assert np.array_equal(vals, f[:Df].astype(np.float32)), (D, before, t0)
                if k % 4 == 0:                   # per-agent Gram: each agent's system is the same single row
                    GA = per.normal_equations(rows, done, ret.expand(1, 1, Df).contiguous(), obs_b, t0_t)
                    assert np.array_equal(GA.cpu().numpy(), np.broadcast_to(np.outer(f, f), GA.shape)), (D, t0)


def _gram_against_oracle(c, D, n_agents=None, bf16_too=False):
    from madrl_b200.postproc import LinearFeatureBaseline
    b = LinearFeatureBaseline(D, DEV, n_agents=n_agents)
    obs, ob, done, ret, t0 = cu(c["obs"]), cu(c["obs_before"]), cu(c["done"]), cu(c["ret"]), cu(c["t0"])
    G = b.normal_equations(obs, done, ret, ob, t0)
    assert torch.equal(G, b.normal_equations(obs, done, ret, ob, t0))        # same bits on a second call
    if bf16_too:                                                              # bf16 == the call on obs.float()
        o16, ob16 = obs.to(torch.bfloat16), None if ob is None else ob.to(torch.bfloat16)
        assert torch.equal(b.normal_equations(o16, done, ret, ob16, t0),
                           b.normal_equations(o16.float(), done, ret, None if ob16 is None else ob16.float(), t0))
    return b, G.cpu().numpy()


@pytest.mark.parametrize("D", pe.LFB_DIMS)
def test_gram_and_predict_at_tile_boundary_obs_dims(D):
    """273 rows (not a multiple of 32, 5-6 rows per slice) with the time / constant / return columns crossing a
    tile edge (D = 30, 31, 62, 63) or the obs^2 block ending on one (D = 32, 64)."""
    c = pe.lfb_case(13, 7, 3, D, 0.2, D)
    b, G = _gram_against_oracle(c, D, bf16_too=True)
    F = bo.features(c["obs"], c["done"], c["obs_before"], c["t0"])
    pe.check_gram(G, bo.normal_equations(F, c["ret"].reshape(-1)))
    coef = np.random.RandomState(D).randn(2 * D + 4)
    b.set_param_values(coef)
    vals = b.predict(cu(c["obs"]), cu(c["done"]), cu(c["obs_before"]), cu(c["t0"])).cpu().numpy()
    pe.check_predict(vals, F, coef)


SLICES = pe.csrc_default("MADRL_LFB_SLICES", "baseline.cu")          # 48 row slices
FLUSH = 2048                                                            # rows between accumulator flushes


@pytest.mark.parametrize("T,E,A,D", [
    (1, 1, 1, 31),                                  # one row
    (5, 3, 3, 30),                                  # fewer rows than slices
    (33, 31, 1, 33),                                # 1023 rows
    (32, SLICES * FLUSH // 96, 3, 31),              # every slice exactly one flush
    (SLICES * FLUSH - 1, 1, 1, 30),
    (SLICES * FLUSH + 1, 1, 1, 32),
], ids=["N1", "N45", "N1023", "N=S*2048", "N=S*2048-1", "N=S*2048+1"])
def test_gram_row_count_edges(T, E, A, D):
    c = pe.lfb_case(T, E, A, D, 0.02 if T > 100 else 0.2, T + D)
    _, G = _gram_against_oracle(c, D)
    F = bo.features(c["obs"], c["done"], c["obs_before"], c["t0"])
    pe.check_gram(G, bo.normal_equations(F, c["ret"].reshape(-1)))


@pytest.mark.parametrize("A,D", [(2, 30), (47, 31), (48, 32), (49, 33), (64, 62), (1024, 31)])
def test_per_agent_gram_at_slice_edges(A, D):
    """ceil(48 / A) slices per agent: 24 for A = 2 (most of them empty), 2 for A = 47, one from A = 48 on;
    each agent's system against the oracle on its own rows."""
    c = pe.lfb_case(4, 3, A, D, 0.3, A)
    _, G = _gram_against_oracle(c, D, n_agents=A, bf16_too=A <= 64)
    F = cbo.agent_features(c["obs"], c["done"], c["obs_before"], c["t0"])
    for a in range(A):
        pe.check_gram(G[a], bo.normal_equations(F[a], c["ret"][:, :, a].reshape(-1)))


@pytest.mark.parametrize("D", [1, 31, 32, 33, 65])
def test_per_agent_predict(D):
    from madrl_b200.postproc import LinearFeatureBaseline
    A = 5
    c = pe.lfb_case(9, 37, A, D, 0.2, 100 + D)
    coef = np.random.RandomState(D).randn(A, 2 * D + 4)
    b = LinearFeatureBaseline(D, DEV, n_agents=A)
    b.set_param_values(coef)
    vals = b.predict(cu(c["obs"]), cu(c["done"]), cu(c["obs_before"]), cu(c["t0"])).cpu().numpy()
    F = cbo.agent_features(c["obs"], c["done"], c["obs_before"], c["t0"])
    for a in range(A):
        pe.check_predict(vals[:, :, a], F[a], coef[a])


# ---------------------------------------------------------------- moments and advantage centring

@pytest.mark.parametrize("A", [1, 2, 255, 256, 257, 1024])
def test_agent_moments_and_centring_equal_pooled_bitwise(A):
    """moments_agents / center_advantages(per_agent=True) give agent a exactly what the pooled calls give on
    x[:, a]: the same block loop, fold order and constant expressions.  A > 256: the centring kernel's per-agent
    constants take more than one pass of its loop strided by the block size."""
    from madrl_b200.postproc import center_advantages, moments, moments_agents
    blocks = pe.csrc_default("MADRL_MOM_BLOCKS", "postproc.cu")
    rows = blocks * 256 + 7 if A <= 2 else 777
    x, y = pe.agent_columns(rows, A, A)
    xt, yt = cu(x), cu(y)
    cols = [(xt[:, a].contiguous(), yt[:, a].contiguous()) for a in range(A)]
    assert torch.equal(moments_agents(xt, yt), torch.stack([moments(xa, ya) for xa, ya in cols]))
    for center, positive in pe.CENTRE_MODES:
        got = center_advantages(xt, center, positive, per_agent=True)
        want = torch.stack([center_advantages(xa, center, positive) for xa, _ in cols], dim=1)
        assert torch.equal(got, want), (center, positive)


# ---------------------------------------------------------------- frame stack

@pytest.mark.parametrize("bf16", [False, True], ids=["f32", "bf16"])
def test_frame_stack_every_buffer_size(bf16):
    """B = 1..8 over E*A*D = 3219 values (13 blocks, a tail); three chained calls: done on a call's first step, on
    every step, never; bit for bit ObservationBuffer's."""
    from madrl_b200.postproc import FrameStack
    E, A, D = 37, 3, 29
    dt = torch.bfloat16 if bf16 else torch.float32
    obs0, calls = pe.frame_stack_calls(E, A, D, 5, bf16)
    for B in range(1, 9):
        fs = FrameStack(E, A, D, B, DEV, dtype=dt)
        fs.reset(obs_dev(obs0, bf16))
        outs = [fs.rollout(obs_dev(o, bf16), cu(d)).float().cpu().numpy() for o, d in calls]
        pe.check_frame_stack(obs0, calls, outs, B)


# ---------------------------------------------------------------- standardiser

def test_standardizer_across_both_inv_std_paths():
    """Running estimates set so that the updated variance v' lands on 0, subnormals, 1e-300, float32 1e-30 and its
    neighbours, 1, float32 1e30 and its neighbours and 1e300, on the reward path (not centred, scaled) and the
    centred observation path; one step is within a float32 ulp of the float64 (x - m') / (sqrt(v') + eps) and
    equal to it rounded to float32 but for a few near-ties.  bfloat16 observations give the float32 result rounded
    to nearest even; pure scaling without the estimate; the terminal-observation pass with done at t = 0 and on
    every step."""
    from madrl_b200.postproc import Standardizer
    eps, alpha = pe.STD_EPS, pe.STD_ALPHA
    x, m, v, vt = pe.std_reward_case()
    n = x.size
    for enable in (True, False):
        sd = Standardizer(n, 1, 1, DEV, scale_reward=0.5, enable_rewnorm=enable, rew_alpha=alpha, eps=eps)
        sd.rew_mean.copy_(cu(m).view(n, 1))
        sd.rew_var.copy_(cu(v).view(n, 1))
        r = cu(x).view(1, n, 1).clone()
        sd.rew(r)
        got = r.cpu().numpy().ravel()
        if enable:
            assert np.array_equal(sd.rew_mean.cpu().numpy().ravel(), m)
            assert np.array_equal(sd.rew_var.cpu().numpy().ravel(), vt)
            off = pe.check_standardized(got, 0.5 * x.astype(np.float64) / (np.sqrt(vt) + eps))
        else:                                                                   # pure scaling
            assert np.array_equal(got, (0.5 * x.astype(np.float64)).astype(np.float32))
            assert np.array_equal(sd.rew_var.cpu().numpy().ravel(), v)
    x, m, v, m1, v1 = pe.std_obs_case()
    n_obs = x.size
    assert all(pe.std_target_classes(v1).values())
    outs = {}
    for dt in (torch.float32, torch.bfloat16):
        so = Standardizer(n_obs, 1, 1, DEV, enable_obsnorm=True, obs_alpha=alpha, eps=eps)
        so.obs_mean.copy_(cu(m).view(n_obs, 1, 1))
        so.obs_var.copy_(cu(v).view(n_obs, 1, 1))
        xo = cu(x).to(dt).view(1, n_obs, 1, 1).clone()                          # x is bfloat16-representable
        so.obs(xo)
        assert np.array_equal(so.obs_mean.cpu().numpy().ravel(), m1)
        assert np.array_equal(so.obs_var.cpu().numpy().ravel(), v1)
        outs[dt] = xo.ravel()
    off += pe.check_standardized(outs[torch.float32].cpu().numpy(), (x.astype(np.float64) - m1) / (np.sqrt(v1) + eps))
    assert torch.equal(outs[torch.bfloat16], outs[torch.float32].to(torch.bfloat16))
    print("standardiser: %d of %d outputs are the other float32 neighbour of the float64 value" % (off, n + n_obs))
    assert off <= 2, off
    obs, term, done = pe.terminal_case(4, 7, 40, 3)
    T, E, P = obs.shape
    st = Standardizer(E, 1, P, DEV, enable_obsnorm=True, obs_alpha=0.05)
    xt, tm = cu(obs).view(T, E, 1, P).clone(), cu(term).view(T, E, 1, P).clone()
    st.obs(xt, cu(done), tm)
    pe.check_terminal(xt.view(T, E, P).cpu().numpy(), tm.view(T, E, P).cpu().numpy(), obs, term, done, 0.05,
                      st.obs_mean.view(E, P).cpu().numpy())


# ---------------------------------------------------------------- GAE and episode statistics

@pytest.mark.parametrize("T", [1, 17])
def test_gae_edges(T):
    """E*A = 903 (4 blocks, a tail); done at t = 0, at T-1, on every step, never; with and without last_value;
    (gamma, lambda) in {(0.99, 0.95), (1, 1), (0, 0.5)}."""
    from madrl_b200.postproc import gae
    E, A = 301, 3
    rew, val, last, done = pe.gae_case(T, E, A, T)
    for discount, lam in pe.GAE_PARAMS:
        for lv in (None, last):
            adv, ret = gae(cu(rew), cu(val), cu(done), discount, lam, cu(lv))
            pe.check_gae(adv.cpu().numpy(), ret.cpu().numpy(), rew, val, done, discount, lam, lv)


@pytest.mark.parametrize("E,A,kind", [(131, 32, "len1"), (131, 3, "boundary"), (140, 5, "span3")])
def test_episode_stats_edges(E, A, kind):
    """E > 128 (two blocks); max_traj_len = 1; episodes ending exactly at a call boundary, done and max_traj_len on
    the same step; one episode across three calls."""
    from madrl_b200.postproc import EpisodeStats
    mtl, calls = pe.episode_stats_calls(E, A, kind, 1)
    es = EpisodeStats(E, A, DEV, discount=0.9, max_traj_len=mtl)
    outs = []
    for rew, done in calls:
        s = es.rollout(cu(rew), cu(done))
        outs.append([s["episode_reward"].cpu().numpy(), s["episode_disc_return"].cpu().numpy(),
                     s["episode_length"].cpu().numpy(), s["end"].cpu().numpy().astype(np.uint8)])
    assert pe.check_episode_stats(outs, calls, 0.9, mtl) > 0


# ---------------------------------------------------------------- path packing

@pytest.mark.parametrize("itemsize", [4, 2], ids=["u32", "u16"])
def test_path_packing_word_counts(itemsize):
    """Observation rows of D in {1..5, 31, 32, 33} words (one thread per row up to 4, one warp beyond), 4-byte and
    bfloat16, with and without the obs_before shift; T = 1, episodes of one step, E > 128; bit for bit to_paths."""
    from madrl_b200.postproc import pack_paths
    for k, D in enumerate(pe.PACK_WORDS):
        for shifted in (False, True):
            T, E, A, p_done = pe.PACK_SHAPES[(k + shifted) % len(pe.PACK_SHAPES)]
            c = pe.pack_case(T, E, A, D, p_done, itemsize, 10 * D + shifted)
            if itemsize == 4:
                obs, ob = cu(c["obs"].view(np.int32)), cu(c["obs_before"].view(np.int32))
            else:
                obs, ob = [cu(c[key].view(np.int16)).view(torch.bfloat16) for key in ("obs", "obs_before")]
            pp = pack_paths(obs, cu(c["act"]), cu(c["rew"]), cu(c["done"]), dict(k=cu(c["info"])),
                            obs_before=ob if shifted else None)
            words = pp.observations.view(torch.int32 if itemsize == 4 else torch.int16).cpu().numpy()
            paths = list(zip(*[getattr(pp, f).tolist() for f in ("env", "agent", "terminated", "offset", "length",
                                                                   "info_offset")]))
            pe.check_packed(c, shifted, paths, words.view(c["obs"].dtype), pp.actions.cpu().numpy(),
                            pp.rewards.cpu().numpy(), pp.env_infos["k"].cpu().numpy())
