"""The frame kernels' source (csrc/render.cu) on the warp emulator (tests/emu) against the NumPy oracle, bit for bit,
with the shared-memory race checker on, at the scenes of tests/render_edges.py: primitives stacked across the
256-primitive chunks, coordinates on, off and far off the frame's edges, and non-finite ones.  The library is the one
tests/test_emulated_render.py builds.  (The emulator compiles the kernels as host code, so contraction of the sensor
end points is checked on the GPU only.)"""
import numpy as np
import pytest

import render_edges as RE
from emu import driver
from oracle import render_oracle as R
from test_emulated_render import TAG, hw_state, lib, render, ww_state  # noqa: F401  (lib: the library fixture)

pytestmark = driver.needs_cxx


@pytest.mark.parametrize("fp64", [False, True])
def test_waterworld_chunks(lib, fp64):
    S = 64
    eng = driver.EmuWaterworld(2, fp64=fp64, defines=TAG, **RE.chunk_ww_kw(S))
    st = ww_state(eng)
    for e in range(2):
        RE.chunk_scene_ww(st, e, S, seed=e + 7)
    assert RE.check_chunk_scene(RE.ww_prims(st, 0, S, eng.cfg, eng.n_pursuers, eng.n_evaders), S) > 256
    want = R.ww_frames(st, [1, 0], S, eng.cfg, eng.n_pursuers, eng.n_evaders)
    RE.assert_frames_equal(render(eng, [1, 0], S, R.sensor_dirs(eng.cfg.n_sensors)), want)


@pytest.mark.parametrize("fp64", [False, True])
def test_hostage_chunks(lib, fp64):
    S = 64
    args, kw = RE.chunk_hw_args(S)
    eng = driver.EmuHostage(2, *args, fp64=fp64, defines=TAG, **kw)
    st = hw_state(eng)
    for e in range(2):
        RE.chunk_scene_hw(st, e, S, seed=e + 3, gate_closed=e == 0)
    assert RE.check_chunk_scene(RE.hw_prims(st, 0, S, eng.cfg), S) > 256
    RE.assert_frames_equal(render(eng, [0, 1], S, R.sensor_dirs(eng.cfg.n_sensors)), R.hw_frames(st, [0, 1], S, eng.cfg))


@pytest.mark.parametrize("sensor_range", [0.6, 0.0, -0.35])
@pytest.mark.parametrize("fp64", [False, True])
def test_waterworld_off_frame_and_non_finite(lib, fp64, sensor_range):
    n_pat = len(RE.NON_FINITE)
    E = n_pat + 3
    eng = driver.EmuWaterworld(E, 6, 5, n_poison=5, n_sensors=8, radius=0.05, obstacle_radius=0.1,
                               sensor_range=sensor_range, fp64=fp64, defines=TAG)
    st = ww_state(eng)
    dirs = R.sensor_dirs(8)
    for S in (37, 40):
        for e in range(E - 1):
            RE.off_frame_scene_ww(st, e, S, seed=e)
        RE.edge_lines_ww(st, E - 1, S)
        for k in range(n_pat):
            RE.non_finite_ww(st, k, k, eng.n_pursuers)
        ids = list(range(E))
        RE.assert_frames_equal(render(eng, ids, S, dirs), R.ww_frames(st, ids, S, eng.cfg, 6, 5), "S=%d" % S)


@pytest.mark.parametrize("fp64", [False, True])
def test_hostage_off_frame_and_non_finite(lib, fp64):
    n_pat = len(RE.NON_FINITE)
    E = n_pat + 2
    eng = driver.EmuHostage(E, 6, 5, 5, 1, 1, n_sensors=8, radius=0.05, sensor_range=0.6, fp64=fp64, defines=TAG)
    st = hw_state(eng)
    dirs = R.sensor_dirs(8)
    S = 37
    for e in range(E):
        RE.off_frame_scene_hw(st, e, S, seed=e, gate_closed=e % 2 == 0)
    for k in range(n_pat):
        RE.non_finite_hw(st, k, k, 6)
    ids = list(range(E))
    RE.assert_frames_equal(render(eng, ids, S, dirs), R.hw_frames(st, ids, S, eng.cfg))
