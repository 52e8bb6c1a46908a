"""The frame kernels (csrc/render.cu) on the GPU against the NumPy oracle (oracle/render_oracle.py), bit for bit:
Waterworld C2 / C4 and Hostage C5 at 800 x 800 after a few hundred steps, a float64 engine, Pursuit C3 and the
dispatch-edge maps; ids that repeat and include the last env; the state untouched; out= reuse and CUDA-graph
capture; argument checks; the drop-in render()."""
import numpy as np
import pytest
import torch

import env_dispatch_edges as D
from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade, _lib
from madrl_b200.closed_loop import PolicyRollout
from madrl_b200.hostage import ContinuousHostageWorld
from madrl_b200.pursuit import PursuitEvade
from madrl_b200.waterworld import MAWaterWorld
from oracle import render_oracle as R

pytestmark = pytest.mark.gpu

WW_SHAPES = {"c2": dict(n_pursuers=5, n_evaders=5, n_poison=10), "c4": dict(n_pursuers=20, n_evaders=50, n_poison=50)}
HW_C5 = (10, 16, 16, 4, 2)
PE_C3 = dict(n_evaders=30, n_pursuers=8, obs_range=7, surround=True, n_catch=2, flatten=True, reward_mech='local',
             catchr=0.1, term_pursuit=5.0, sample_maps=True, include_id=True)


def stepped(eng, T, seed=0):
    """`eng` after T random steps with auto-reset."""
    g = torch.Generator(device=eng.device).manual_seed(seed)
    E, A = eng.n_envs, eng._n_acting
    if eng._act_dtype == torch.int32:
        act = torch.randint(0, 5, (T, E, A), generator=g, device=eng.device, dtype=torch.int32)
    else:
        act = torch.randn((T, E, A, 2), generator=g, device=eng.device, dtype=eng._act_dtype)
    eng.reset()
    eng.rollout(act, auto_reset=True)
    torch.cuda.synchronize()
    return eng


def ww_want(eng, ids, S):
    return R.ww_frames(eng.state, ids, S, eng.cfg, eng.n_pursuers, eng.n_evaders)


def hw_want(eng, ids, S):
    return R.hw_frames(eng.state, ids, S, eng.cfg)


def pe_want(eng, ids, cell):
    return R.pe_frames(eng.state, eng.map_pool, ids, eng.obs_range, cell)


def assert_frames(got, want):
    got = got.cpu().numpy()
    assert got.shape == want.shape
    bad = np.argwhere((got != want).any(axis=-1))
    assert bad.size == 0, "%d pixels differ, first (frame, row, col) %s" % (len(bad), bad[:5].tolist())


@pytest.mark.parametrize("shape", ["c2", "c4"])
def test_waterworld_frames(shape):
    eng = stepped(BatchedMAWaterWorld(40, seed=5, **WW_SHAPES[shape]), 300)
    ids = [0, 39, 7, 39, 0]
    assert_frames(eng.render_frames(ids), ww_want(eng, ids, 800))


def test_waterworld_random_obstacle_float64_odd_size():
    eng = stepped(BatchedMAWaterWorld(9, 3, 4, n_poison=2, n_sensors=7, radius=0.05, sensor_range=0.45,
                                      obstacle_loc=None, seed=2, dtype=torch.float64), 120)
    ids = torch.tensor([8, 3, 8], dtype=torch.int64)
    for S in (800, 257, 37, 1):
        assert_frames(eng.render_frames(ids, screen_size=S), ww_want(eng, [8, 3, 8], S))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float64])
def test_hostage_frames(dtype):
    eng = stepped(BatchedHostageWorld(24, *HW_C5, seed=6, dtype=dtype), 250)
    st = eng.state   # a closed gate and saved hostages in some envs, whatever the episodes reached
    st["flags"][::2] &= ~1
    st["flags"][1::2] |= 1
    st["saved"][::3, ::2] = 1
    ids = [23, 0, 1, 23, 12]
    assert_frames(eng.render_frames(ids), hw_want(eng, ids, 800))
    assert_frames(eng.render_frames(ids, screen_size=257), hw_want(eng, ids, 257))


@pytest.mark.parametrize("cell", [16, 7])
def test_pursuit_c3(cell):
    eng = stepped(BatchedPursuitEvade(48, D.pool16(), seed=4, **PE_C3), 60)
    ids = [47, 0, 47, 5]
    assert_frames(eng.render_frames(ids, cell=cell), pe_want(eng, ids, cell))


@pytest.mark.parametrize("name", ["e2_c1_conv", "e2_rc7_flat", "e1_c1_flat", "e2_c2_flat"])
def test_pursuit_dispatch_edge_maps(name):
    case = D.P_BY_NAME[name]
    eng = stepped(BatchedPursuitEvade(case.E, case.maps(), seed=8, **case.cfg), case.T)
    ids = list(range(case.E)) + [case.E - 1]
    for cell in (16, 3):
        assert_frames(eng.render_frames(ids, cell=cell), pe_want(eng, ids, cell))


@pytest.mark.parametrize("family", ["ww", "hw", "pe"])
def test_state_untouched_out_reused_and_bad_ids_zero(family):
    eng = {"ww": lambda: BatchedMAWaterWorld(16, 5, 5, seed=1),
           "hw": lambda: BatchedHostageWorld(16, *HW_C5, seed=1),
           "pe": lambda: BatchedPursuitEvade(16, D.pool16(), seed=1, **PE_C3)}[family]()
    stepped(eng, 40)
    draw = (lambda ids, out=None: eng.render_frames(ids, cell=9, out=out)) if family == "pe" else \
        (lambda ids, out=None: eng.render_frames(ids, screen_size=200, out=out))
    before = eng._blob.clone()
    first = draw([15, 2])
    out = torch.full_like(first, 7)
    again = draw(torch.tensor([15, 2], dtype=torch.int32, device=eng.device), out=out)
    torch.cuda.synchronize()
    assert again.data_ptr() == out.data_ptr() and torch.equal(again, first)
    assert torch.equal(eng._blob, before)
    # CUDA ids are not read back on the host: an id outside the range gets an all-zero frame
    odd = draw(torch.tensor([-1, 2, 16], dtype=torch.int32, device=eng.device))
    assert int(odd[0].max()) == 0 and int(odd[2].max()) == 0 and torch.equal(odd[1], first[1])
    assert int(first.min()) >= (102 if family != "pe" else 0)


def test_capture_after_policy_rollout():
    eng = BatchedMAWaterWorld(32, 5, 5, seed=9)
    obs0 = eng.reset()
    pol = lambda obs, state: (torch.tanh(obs[..., :2] * 3), {}, state)
    ro = PolicyRollout(eng, pol, 4)
    ro(obs0)
    ids = torch.tensor([31, 0, 17], dtype=torch.int32, device=eng.device)
    frames = torch.empty((3, 800, 800, 3), dtype=torch.uint8, device=eng.device)
    eng.render_frames(ids, out=frames)   # first call at this shape: builds the direction table
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        eng.render_frames(ids, out=frames)
    for _ in range(2):
        r = ro(obs0)
        obs0 = r.obs[-1]
        g.replay()
        torch.cuda.synchronize()
        assert_frames(frames, ww_want(eng, [31, 0, 17], 800))


def test_bad_arguments_raise_before_the_abi():
    ww = BatchedMAWaterWorld(4, 2, 2, n_poison=2, seed=0)
    pe = BatchedPursuitEvade(4, D.pool16(), seed=0, **PE_C3)
    for bad in ([4], [-1], [], [[0, 1]], [0.5]):
        with pytest.raises((ValueError, TypeError)):
            ww.render_frames(bad)
        with pytest.raises((ValueError, TypeError)):
            pe.render_frames(bad)
    for S in (0, -3, 32769):
        with pytest.raises(ValueError):
            ww.render_frames([0], screen_size=S)
    for c in (0, 2049):   # 16 x 2049 pixels > 32768
        with pytest.raises(ValueError):
            pe.render_frames([0], cell=c)
    with pytest.raises(ValueError):
        ww.render_frames([0, 1], screen_size=8, out=torch.empty((1, 8, 8, 3), dtype=torch.uint8, device=ww.device))
    with pytest.raises(TypeError):
        ww.render_frames([0], screen_size=8, out=torch.empty((1, 8, 8, 3), dtype=torch.int32, device=ww.device))
    # the C ABI refuses on its own what the Python layer would have caught
    L, ids = _lib.lib(), torch.zeros(1, dtype=torch.int32, device=ww.device)
    out = torch.empty((1, 8, 8, 3), dtype=torch.uint8, device=ww.device)
    dirs = torch.zeros((2, 30), dtype=torch.float64, device=ww.device)
    assert L.madrl_ww_render(ww._h, 0, _lib._ptr(ids), 8, _lib._ptr(dirs), _lib._ptr(out), None) == -1
    assert L.madrl_ww_render(ww._h, 1, _lib._ptr(ids), 0, _lib._ptr(dirs), _lib._ptr(out), None) == -1
    assert L.madrl_ww_render(ww._h, 1, _lib._ptr(ids), 8, None, _lib._ptr(out), None) == -1
    assert L.madrl_ww_render(ww._h, 1, _lib._ptr(ids), 40000, _lib._ptr(dirs), _lib._ptr(out), None) == -1
    assert b"screen_size" in L.madrl_last_error()
    assert L.madrl_pursuit_render(pe._h, 1, _lib._ptr(ids), 4096, _lib._ptr(out), None) == -1
    assert b"pixels a side" in L.madrl_last_error()


def test_drop_in_render_is_env_zero():
    ww = MAWaterWorld(5, 5)
    ww.reset()
    for _ in range(20):
        ww.step(np.random.RandomState(0).randn(5, 2))
    f = ww.render()
    assert isinstance(f, np.ndarray) and f.shape == (800, 800, 3) and f.dtype == np.uint8
    assert np.array_equal(f, ww._engine.render_frames([0])[0].cpu().numpy())
    hw = ContinuousHostageWorld(*HW_C5)
    hw.reset()
    f = hw.render(screen_size=300)
    assert f is not None and np.array_equal(f, hw._engine.render_frames([0], screen_size=300)[0].cpu().numpy())
    pe = PursuitEvade(D.pool16(), n_evaders=5, n_pursuers=3)
    pe.reset()
    f = pe.render()
    assert f.shape == (16 * 16, 16 * 16, 3)
    assert np.array_equal(f, pe_want(pe._engine, [0], 16)[0])
