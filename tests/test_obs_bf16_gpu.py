"""bfloat16 observations on the GPU (obs_dtype=torch.bfloat16, madrl_*_set_obs_format): against an fp32
engine with the same config, seed and actions, the state, rewards, dones and infos are identical and the
observations are the fp32 ones converted with `.to(torch.bfloat16)`, bit for bit, through every entry
point; the post-processing wrappers take the bf16 tensors."""
import os

import numpy as np
import pytest
import torch

from conftest import ROOT

pytestmark = pytest.mark.gpu

C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
          catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)
CONV = dict(n_evaders=3, n_pursuers=3, obs_range=4, surround=False, n_catch=1, reward_mech='global', flatten=False)


def pool16():
    return np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))


def small_map():
    m = np.zeros((1, 5, 5), dtype=np.int32)
    m[0, 2, 2] = -1
    return m


def make(case, obs_dtype, E=48, **kw):
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    kw = dict(dict(seed=5, device="cuda", obs_dtype=obs_dtype), **kw)
    if case == "ww_c2":
        return BatchedMAWaterWorld(E, 5, 5, n_poison=10, **kw)
    if case == "ww_c4":
        return BatchedMAWaterWorld(E, 20, 50, n_poison=50, **kw)
    if case == "ww_global_nospeed":
        return BatchedMAWaterWorld(E, 3, 4, n_poison=2, n_sensors=7, n_coop=1, radius=0.05, reward_mech='global',
                                   speed_features=False, addid=False, obstacle_loc=None, **kw)
    if case == "pe_c3":
        return BatchedPursuitEvade(E, pool16(), **C3, **kw)
    if case == "pe_conv":
        return BatchedPursuitEvade(E, small_map(), **CONV, **kw)
    return BatchedHostageWorld(E, 10, 16, 16, 4, 2, **kw)


def actions(eng, T, seed=0):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    shape = (T, eng.n_envs, eng._n_acting) + eng._act_tail
    if eng._act_dtype == torch.int32:
        return torch.randint(0, 5, shape, dtype=torch.int32, device="cuda", generator=g)
    return torch.randn(shape, device="cuda", generator=g) * 0.5


def same_obs(o32, o16):
    assert o16.dtype == torch.bfloat16 and o32.dtype == torch.float32
    assert torch.equal(o32.to(torch.bfloat16).view(torch.int16), o16.view(torch.int16))


def same_rest(ra, rb):
    for x, y in zip(ra, rb):
        assert torch.equal(x, y)


def same_state(a, b):
    torch.cuda.synchronize()
    assert torch.equal(a._blob, b._blob), "state blobs differ"


CASES = ["ww_c2", "ww_c4", "ww_global_nospeed", "pe_c3", "pe_conv", "hw_c5"]


@pytest.mark.parametrize("case", CASES)
def test_device_entry_points(case):
    a, b = make(case, torch.float32, max_path_length=7), make(case, torch.bfloat16, max_path_length=7)
    assert b.obs_dtype == torch.bfloat16 and b.dtype == torch.float32
    same_obs(a.reset(), b.reset())
    same_state(a, b)
    # step (no auto-reset)
    act = actions(a, 1, seed=1)[0]
    sa, sb = a.step(act), b.step(act)
    same_obs(sa[0], sb[0])
    assert torch.equal(sa[1], sb[1]) and torch.equal(sa[2], sb[2])
    # rollout with auto-reset across done steps, terminal observations kept on the side
    T = 23
    act = actions(a, T, seed=2)
    ta = torch.full((T, a.n_envs, a._n_acting, a.obs_dim), -7.0, device="cuda")
    tb = torch.full_like(ta, -7.0, dtype=torch.bfloat16)
    a.set_terminal_obs(ta)
    b.set_terminal_obs(tb)
    ra, rb = a.rollout(act, auto_reset=True), b.rollout(act, auto_reset=True)
    a.set_terminal_obs(None)
    b.set_terminal_obs(None)
    same_obs(ra[0], rb[0])
    same_rest(ra[1:], rb[1:])
    assert int(ra[2].sum()) >= a.n_envs * (T // 7 - 1)
    same_obs(ta, tb)
    same_state(a, b)
    # rollout without auto-reset, then a masked reset
    act = actions(a, 5, seed=3)
    ra, rb = a.rollout(act, auto_reset=False), b.rollout(act, auto_reset=False)
    same_obs(ra[0], rb[0])
    same_rest(ra[1:], rb[1:])
    mask = torch.arange(a.n_envs, device="cuda") % 3 == 0
    same_obs(a.reset(mask=mask), b.reset(mask=mask))
    same_state(a, b)


@pytest.mark.parametrize("case", ["ww_c2", "pe_c3", "hw_c5"])
def test_host_entry_points(case):
    a, b = make(case, torch.float32, max_path_length=6), make(case, torch.bfloat16, max_path_length=6)
    a.reset(), b.reset()
    T, E, A, D = 13, a.n_envs, a._n_acting, a.obs_dim
    act = actions(a, T, seed=4).cpu()
    for obs_last in (False, True):
        oshape = (E, A, D) if obs_last else (T, E, A, D)
        info = (T, E) + a._info_tail
        ha = (torch.empty(oshape), torch.empty((T, E, A)), torch.empty((T, E), dtype=torch.uint8),
              torch.empty(info, dtype=torch.int32))
        hb = (torch.empty(oshape, dtype=torch.bfloat16), torch.empty((T, E, A)), torch.empty((T, E), dtype=torch.uint8),
              torch.empty(info, dtype=torch.int32))
        a.rollout_host(act, *ha, obs_last=obs_last)
        b.rollout_host(act, *hb, obs_last=obs_last)
        same_obs(ha[0], hb[0])
        same_rest(ha[1:], hb[1:])
        same_state(a, b)
    with pytest.raises(TypeError):
        b.rollout_host(act, *ha)   # float32 obs buffer on a bf16 engine


@pytest.mark.parametrize("case", ["ww_c2", "pe_c3", "pe_conv"])
def test_heuristic_rollout_reads_widened_obs0(case):
    """A bf16 rollout_heuristic equals the fp32 one whose obs0 is the bf16 obs0 widened to fp32."""
    a, b = make(case, torch.float32, max_path_length=9), make(case, torch.bfloat16, max_path_length=9)
    a.reset()
    ob = b.reset()
    ra = a.rollout_heuristic(20, ob.float())
    rb = b.rollout_heuristic(20, ob)
    assert torch.equal(ra[0], rb[0])
    same_obs(ra[1], rb[1])
    same_rest(ra[2:], rb[2:])
    same_state(a, b)


@pytest.mark.parametrize("case", ["pe_c3", "pe_conv"])
def test_pursuit_bf16_heuristic_chained_equals_long(case):
    a, b = make(case, torch.bfloat16, max_path_length=9), make(case, torch.bfloat16, max_path_length=9)
    oa, ob = a.reset(), b.reset()
    long_ = a.rollout_heuristic(24, oa)
    first = b.rollout_heuristic(10, ob)
    second = b.rollout_heuristic(14, first[1][-1].contiguous())
    for x, y, z in zip(first, second, long_):
        assert torch.equal(torch.cat([x, y]).view(torch.int16) if x.dtype == torch.bfloat16 else torch.cat([x, y]),
                           z.view(torch.int16) if z.dtype == torch.bfloat16 else z)
    same_state(a, b)


@pytest.mark.parametrize("case", ["ww_c2", "pe_c3", "hw_c5"])
def test_sharded_batch_equals_unsharded(case):
    from madrl_b200.dist import make_sharded
    from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade
    E = 48
    whole = make(case, torch.bfloat16, E=E, max_path_length=5)
    cls = {"ww": BatchedMAWaterWorld, "pe": BatchedPursuitEvade, "hw": BatchedHostageWorld}[case[:2]]
    args = {"ww_c2": (5, 5), "pe_c3": (pool16(),), "hw_c5": (10, 16, 16, 4, 2)}[case]
    kw = dict(C3) if case == "pe_c3" else (dict(n_poison=10) if case == "ww_c2" else {})
    shards = [make_sharded(cls, E, *args, rank=r, world=2, seed=5, device="cuda", max_path_length=5,
                           obs_dtype=torch.bfloat16, **kw) for r in range(2)]
    T = 12
    act = actions(whole, T, seed=6)
    ow = whole.reset()
    os_ = [s.reset() for s in shards]
    assert torch.equal(torch.cat(os_, 0).view(torch.int16), ow.view(torch.int16))
    rw = whole.rollout(act)
    rs = [s.rollout(act[:, lo:hi].contiguous()) for s, (lo, hi) in zip(shards, ((0, E // 2), (E // 2, E)))]
    for i in range(4):
        x = torch.cat([r[i] for r in rs], 1)
        y = rw[i]
        if x.dtype == torch.bfloat16:
            x, y = x.view(torch.int16), y.view(torch.int16)
        assert torch.equal(x, y)


def test_bad_obs_dtype_is_rejected():
    from madrl_b200 import BatchedMAWaterWorld
    with pytest.raises(ValueError):
        BatchedMAWaterWorld(4, 5, 5, device="cuda", obs_dtype=torch.float16)
    with pytest.raises(ValueError):
        BatchedMAWaterWorld(4, 5, 5, device="cuda", dtype=torch.float64, obs_dtype=torch.bfloat16)


def test_postproc_passes_on_bf16_observations():
    """FrameStack, both Standardizer paths and pack_paths on a bf16 engine's tensors equal the fp32 passes
    on the same observations widened to fp32, rounded to bfloat16."""
    from madrl_b200.postproc import FrameStack, Standardizer, pack_paths
    E, T, A, mpl = 24, 30, 5, 7
    b = make("ww_c2", torch.bfloat16, E=E, max_path_length=mpl)
    ob0 = b.reset().clone()
    act = actions(b, T, seed=8)
    term = torch.zeros((T, E, A, b.obs_dim), dtype=torch.bfloat16, device="cuda")
    b.set_terminal_obs(term)
    obs, rew, done, info = b.rollout(act, auto_reset=True)
    b.set_terminal_obs(None)
    assert int(done.sum()) >= E * (T // mpl)
    wide, wide0, wterm = obs.float(), ob0.float(), term.float()

    def rounded_equal(x32, x16):
        assert x16.dtype == torch.bfloat16
        assert torch.equal(x32.to(torch.bfloat16).view(torch.int16), x16.view(torch.int16))

    f32, f16 = FrameStack(E, A, b.obs_dim, 4, "cuda"), FrameStack(E, A, b.obs_dim, 4, "cuda", dtype=torch.bfloat16)
    rounded_equal(f32.reset(wide0), f16.reset(ob0))
    for sl in (slice(0, 13), slice(13, T)):       # two calls exercise the carry
        rounded_equal(f32.rollout(wide[sl], done[sl]), f16.rollout(obs[sl], done[sl]))
    # Standardizer: plain path, then the terminal-observation path
    for terminal in (False, True):
        s32 = Standardizer(E, A, b.obs_dim, "cuda", enable_obsnorm=True, obs_alpha=0.05)
        s16 = Standardizer(E, A, b.obs_dim, "cuda", enable_obsnorm=True, obs_alpha=0.05)
        x32, x16 = wide.clone(), obs.clone()
        if terminal:
            t32, t16 = wterm.clone(), term.clone()
            s32.obs(x32, done, t32)
            s16.obs(x16, done, t16)
            rounded_equal(t32, t16)
        else:
            s32.obs(x32)
            s16.obs(x16)
        rounded_equal(x32, x16)
        assert torch.equal(s32.obs_mean, s16.obs_mean) and torch.equal(s32.obs_var, s16.obs_var)
    # path packing: 2-byte rows of odd length (D = 213)
    assert b.obs_dim % 2 == 1
    infos = dict(evcatches=info[..., 0].contiguous())
    p32 = pack_paths(wide, act, rew, done, infos, obs_before=wide0)
    p16 = pack_paths(obs, act, rew, done, infos, obs_before=ob0)
    rounded_equal(p32.observations, p16.observations)
    for k in ("actions", "rewards", "offset", "length", "env", "agent", "terminated", "info_offset"):
        assert torch.equal(getattr(p32, k), getattr(p16, k)), k
    rounded_equal(pack_paths(wide, act, rew, done).observations, pack_paths(obs, act, rew, done).observations)
