"""The constructed frame scenes of tests/render_edges.py check themselves on the CPU: the end points a fused
multiply-add would move really move, the chunk scenes really reach past 256 primitives in a tile, and the oracle's row
bands and non-finite rule agree with its whole frames.  Where OpenCV is installed, the oracle's primitives are pinned
against it on a 32768 x 32768 frame."""
import numpy as np
import pytest

import render_edges as RE
from oracle import render_oracle as R

try:
    import cv2
except ImportError:
    cv2 = None


class _Cfg(object):
    def __init__(self, **kw):
        self.__dict__.update(kw)


def ww_state(E, Np, Ne, Npo, dtype=np.float64):
    n = Np + Ne + Npo
    return dict(pos_x=np.zeros((E, n), dtype), pos_y=np.zeros((E, n), dtype), obst_x=np.zeros(E, dtype),
                obst_y=np.zeros(E, dtype))


def hw_state(E, Ng, Nh, Nb, dtype=np.float64):
    n = Ng + Nh + Nb
    return dict(pos_x=np.zeros((E, n), dtype), pos_y=np.zeros((E, n), dtype), key=np.zeros((E, 2), dtype),
                bomb=np.zeros((E, 2), dtype), saved=np.zeros((E, Nh), np.uint8), flags=np.zeros(E, np.int32))


def test_fused_sensor_ends_move_a_pixel():
    S, K, r = 800, 30, 0.2
    dirs = R.sensor_dirs(K)
    for row in (0, 1):
        pts = RE.fma_points_f64(S, r, dirs[row], 64)
        assert len(pts) == 64
        for j, p in pts:
            d = dirs[row, j]
            a, b = int(RE.unfused_end(p, r, d) * S), int(RE.fused_end(p, r, d) * S)
            assert abs(a - b) == 1 and 99 <= min(a, b) < 700
            # the line to the moved end point has other pixels
            c = int(0.5 * S)
            ends = [(a, c), (b, c)] if row == 0 else [(c, a), (c, b)]
            px = (int(p * S), c) if row == 0 else (c, int(p * S))
            assert set(R.line_pixels(S, S, *px, *ends[0])) != set(R.line_pixels(S, S, *px, *ends[1]))
    for p in (0.4375001, 0.61):
        hits = RE.fma_points_f32(S, p, dirs[0], 4)
        assert len(hits) == 4
        p = float(np.float32(p))
        for j, r32 in hits:
            assert 0 < r32 < 1
            assert int(RE.unfused_end(p, r32, dirs[0, j]) * S) != int(RE.fused_end(p, r32, dirs[0, j]) * S)


@pytest.mark.parametrize("S", [64, 97])
def test_chunk_scenes_reach_past_one_chunk(S):
    kw = RE.chunk_ww_kw(S)
    st = ww_state(1, 32, 112, 112)
    RE.chunk_scene_ww(st, 0, S, seed=1)
    cfg = _Cfg(n_sensors=64, radius=kw["radius"], obstacle_radius=kw["obstacle_radius"],
               sensor_range=kw["sensor_range"])
    prims = RE.ww_prims(st, 0, S, cfg, 32, 112)
    assert len(prims) == 2305 and RE.check_chunk_scene(prims, S) > 1000
    args, kw = RE.chunk_hw_args(S)
    st = hw_state(1, 32, 112, 112)
    RE.chunk_scene_hw(st, 0, S, seed=1)
    cfg = _Cfg(n_sensors=64, n_good=32, n_bad=112, radius=kw["radius"], bomb_radius=kw["bomb_radius"],
               sensor_range=kw["sensor_range"])
    prims = RE.hw_prims(st, 0, S, cfg)
    assert len(prims) == 2307 and RE.check_chunk_scene(prims, S) > 1000


def test_max_sensor_range_is_the_last_double_below_the_bound():
    for S in (1, 37, 800, 32767, 32768):
        r = RE.max_sensor_range(S)
        assert r * S < 2.0 ** 29 and not float(np.nextafter(r, np.inf)) * S < 2.0 ** 29


@pytest.mark.parametrize("S", [1, 5, 37, 100])
def test_bands_equal_the_whole_frame(S):
    rs = np.random.RandomState(S)
    dirs = R.sensor_dirs(7)
    st = ww_state(3, 6, 5, 5)
    for e in range(2):
        RE.off_frame_scene_ww(st, e, S, seed=e)
    RE.edge_lines_ww(st, 2, S)
    hs = hw_state(2, 6, 5, 5)
    for e in range(2):
        RE.off_frame_scene_hw(hs, e, S, seed=e + 3, gate_closed=e == 0)
    bands = [(0, S)] + [(a, min(a + b, S)) for b in (1, 3, 16) for a in range(0, S, b)]
    for e in range(3):
        args = (st["pos_x"][e], st["pos_y"][e], (st["obst_x"][e], st["obst_y"][e]), 6, 5, S, 0.05, 0.2, 0.6, dirs)
        whole = R.ww_frame(*args)
        for y0, y1 in bands:
            assert np.array_equal(R.ww_frame(*args, rows=(y0, y1)), whole[y0:y1]), (e, y0, y1)
    for e in range(2):
        fixed = np.concatenate([hs["key"][e], hs["bomb"][e]])
        args = (hs["pos_x"][e], hs["pos_y"][e], fixed, hs["saved"][e], hs["flags"][e], 6, 5, S, 0.05, 0.1, 0.6, dirs)
        whole = R.hw_frame(*args)
        for y0, y1 in bands:
            assert np.array_equal(R.hw_frame(*args, rows=(y0, y1)), whole[y0:y1]), (e, y0, y1)
    building = rs.rand(4, 3) < 0.3
    for cell in (1, 3, 8):
        args = (building, [0, 3], [2, 1], [3, 1, 0], [2, 1, 0], 0b010, 3, cell)
        whole = R.pe_frame(*args)
        for y0, y1 in [(0, 3 * cell), (1, 2), (cell - 1, 2 * cell + 1), (3 * cell - 1, 3 * cell)]:
            assert np.array_equal(R.pe_frame(*args, rows=(y0, y1)), whole[y0:y1]), (cell, y0, y1)


def test_non_finite_objects_contribute_no_primitive():
    S, dirs = 64, R.sensor_dirs(5)
    st = ww_state(1, 3, 3, 3)
    rs = np.random.RandomState(0)
    st["pos_x"][0], st["pos_y"][0] = rs.rand(9), rs.rand(9)
    st["obst_x"][0], st["obst_y"][0] = 0.4, 0.6
    frame = lambda g: R.ww_frame(g["pos_x"][0], g["pos_y"][0], (g["obst_x"][0], g["obst_y"][0]), 3, 3, S, 0.05, 0.2,
                                 0.3, dirs)
    for k in range(len(RE.NON_FINITE)):
        g = {n: v.copy() for n, v in st.items()}
        RE.non_finite_ww(g, 0, k, 3)
        prims = R.ww_prims(g["pos_x"][0], g["pos_y"][0], (g["obst_x"][0], g["obst_y"][0]), 3, 3, S, 0.05, 0.2, 0.3,
                           dirs)
        gone = [p for p, q in enumerate(prims) if q is None]
        assert gone == [0] + list(range(1, 7)) + [3 * 6 + 1, len(prims) - 1], k   # obstacle, pursuer 0, evader, poison
        # the frame is the one drawn without those objects: moved far off the frame instead
        h = {n: v.copy() for n, v in st.items()}
        for i in (0, 3, 8):
            h["pos_x"][0, i] = 1e6
        h["obst_x"][0] = 1e6
        assert np.array_equal(frame(g), frame(h)), k


@pytest.mark.skipif(cv2 is None, reason="OpenCV is not installed")
def test_primitives_equal_opencv_on_the_largest_frame():
    """A few lines with ends up to +-2^30 and circles up to r = 32768, on one 32768 x 32768 single-channel frame."""
    S = 32768
    img = np.zeros((S, S), np.uint8)
    lines = [(0, 0, S - 1, S - 1), (-(1 << 30), 5, 1 << 30, S - 7), (S // 2, S // 2, S // 2 + (1 << 30), S // 2 + (1 << 29)),
             (-5, -(1 << 30), S + 5, 1 << 30)]
    for p in lines:
        img[:] = 0
        cv2.line(img, p[:2], p[2:], 255, 1, cv2.LINE_8)
        ys, xs = np.nonzero(img)
        assert set(zip(xs.tolist(), ys.tolist())) == set(R.line_pixels(S, S, *p)), p
    for cx, cy, r in ((S // 2 - 3, S // 2 + 5, S // 2 + 7), (-100, S - 1, S)):
        img[:] = 0
        cv2.circle(img, (cx, cy), r, 255, -1, cv2.LINE_8)
        got = np.zeros((S, S, 1), np.uint8)
        R.fill_circle(got, cx, cy, r, 255)
        assert np.array_equal(got[..., 0], img), (cx, cy, r)
