"""Waterworld's writer-warp observation path against the one-warp kernel (needs a GPU).

madrl_ww_set_obs_writer(OFF) keeps the one-warp kernel; the default (AUTO) and ON take the writer-warp kernel where
it can run (csrc/waterworld.cu, ww_use_writer).  Both must compute the same bits: observations, rewards, dones,
infos, terminal observations and the state record, on the headline shape (C2, 4 096 envs, T = 256, auto-resets
every few steps), with envs whose paths end at different steps within a group of adjacent envs, with a partial
last group (4 092 envs), and on the launches that must fall back: a step stride that is not 16-byte aligned
(4 093 envs) and an observation base that is not.  Also through rollout_host (madrl_ww_rollout_host2).
"""
import pytest
import torch

from madrl_b200 import BatchedMAWaterWorld, _lib

pytestmark = pytest.mark.gpu

C2 = dict(n_pursuers=5, n_evaders=5)
MPL, SEED = 7, 5


def bits(x):
    return x.view(torch.int32) if x.dtype == torch.float32 else x


def make(E, mode):
    eng = BatchedMAWaterWorld(E, **C2, device="cuda", seed=SEED, max_path_length=MPL)
    if mode is not None:
        eng.set_obs_writer(mode)
    return eng


def actions(T, E, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    return torch.randn(T, E, 5, 2, device="cuda", generator=g) * 0.7


def run(eng, act, obs_offset=0, desync=False):
    """reset (and a masked reset of every other env after a first rollout), then one auto-reset rollout with
    terminal observations into an obs tensor `obs_offset` floats into its allocation."""
    T, E = act.shape[:2]
    eng.reset()
    if desync:
        eng.rollout(act[:3], auto_reset=True)
        eng.reset(mask=(torch.arange(E, device="cuda") % 2).to(torch.uint8))
    flat = torch.empty(obs_offset + T * E * 5 * eng.obs_dim, device="cuda")
    obs = flat[obs_offset:].view(T, E, 5, eng.obs_dim)
    out = (obs, torch.empty(T, E, 5, device="cuda"), torch.empty(T, E, dtype=torch.uint8, device="cuda"),
           torch.empty(T, E, 2, dtype=torch.int32, device="cuda"))
    term = torch.full((T, E, 5, eng.obs_dim), -3.0, device="cuda")
    eng.set_terminal_obs(term)
    outs = eng.rollout(act, auto_reset=True, out=out) + (term,)
    eng.set_terminal_obs(None)
    torch.cuda.synchronize()
    return outs, {k: v.clone() for k, v in eng.state.items()}


def assert_same(a, b):
    (got, got_state), (want, want_state) = a, b
    for k, (x, y) in enumerate(zip(got, want)):
        assert x.shape == y.shape and torch.equal(bits(x), bits(y)), k
    for k in want_state:
        assert torch.equal(bits(got_state[k]), bits(want_state[k])), k


def test_headline_default_equals_one_warp_kernel():
    E, T = 4096, 256
    act = actions(T, E, 1)
    eng = make(E, None)
    assert _lib.lib().madrl_ww_default_blocks_per_sm(eng._h, T) == 16   # the default takes the writer path
    got = run(eng, act)
    assert int(got[0][2].sum()) >= E * (T // MPL)
    del eng
    assert_same(got, run(make(E, _lib.WW_OBS_WRITER_OFF), act))


@pytest.mark.parametrize("E,offset,desync", [(4096, 0, True), (4092, 0, False), (4093, 0, False), (4096, 1, False)],
                         ids=["desync", "partial_group", "odd_stride", "misaligned_base"])
def test_writer_equals_one_warp_kernel(E, offset, desync):
    act = actions(64, E, 2)
    got = run(make(E, _lib.WW_OBS_WRITER_ON), act, offset, desync)
    if desync:
        done = got[0][2]
        assert (done[:, 0::2] != done[:, 1::2]).any()
    assert_same(got, run(make(E, _lib.WW_OBS_WRITER_OFF), act, offset, desync))


def test_rollout_host_writer_equals_one_warp_kernel():
    E, T = 4096, 40
    act = actions(T, E, 3).cpu()
    res = []
    for mode in (_lib.WW_OBS_WRITER_ON, _lib.WW_OBS_WRITER_OFF):
        eng = make(E, mode)
        eng.reset()
        bufs = (torch.empty(T, E, 5, eng.obs_dim).pin_memory(), torch.empty(T, E, 5).pin_memory(),
                torch.empty(T, E, dtype=torch.uint8).pin_memory(), torch.empty(T, E, 2, dtype=torch.int32).pin_memory())
        eng.rollout_host(act.pin_memory(), *bufs, auto_reset=True)
        res.append((bufs, {k: v.clone() for k, v in eng.state.items()}))
    assert int(res[0][0][2].sum()) >= E * (T // MPL)
    assert_same(*res)
