"""The frame oracle (oracle/render_oracle.py) on the CPU: its primitives against the installed OpenCV, and its
Waterworld and Hostage frames against the frames the reference's own render drew (tests/golden/render_*.npz,
made by oracle/make_render_golden.py)."""
import json
import os

import numpy as np
import pytest

from oracle import render_oracle as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

try:
    import cv2
except ImportError:   # the golden tests below need no cv2
    cv2 = None
needs_cv2 = pytest.mark.skipif(cv2 is None, reason="OpenCV is not installed")
COLOR = (17, 200, 255)


def test_add_weighted_table_is_the_kernels_integer_form():
    """csrc/render.cu blends with round(102 + 0.6 v) in integers: 102 + (6 v + 5) div 10."""
    v = np.arange(256)
    assert np.array_equal(R.add_weighted_lut(), 102 + (6 * v + 5) // 10)


@needs_cv2
def test_add_weighted_every_value():
    v = np.repeat(np.arange(256, dtype=np.uint8)[:, None, None], 3, axis=2)
    got = cv2.addWeighted(np.full_like(v, 255), 0.4, v, 0.6, 0)
    assert np.array_equal(got[:, 0, 0], R.add_weighted_lut())
    assert np.array_equal(R.blend_background(v), got)


@needs_cv2
@pytest.mark.parametrize("seed", range(4))
def test_filled_circle(seed):
    rs = np.random.RandomState(seed)
    for it in range(1000):
        H, W = rs.randint(1, 80, 2)
        r = 0 if it % 10 == 0 else int(rs.choice([rs.randint(1, 8), rs.randint(1, 60), rs.randint(60, 200)]))
        cx, cy = (int(c) for c in rs.randint(-r - 10, np.array([W, H]) + r + 10))
        if it % 7 == 0:   # centres on the frame's edges
            cx, cy = int(rs.choice([0, W - 1, W, -1])), int(rs.choice([0, H - 1, H, -1]))
        want = np.zeros((H, W, 3), np.uint8)
        cv2.circle(want, (cx, cy), r, COLOR, -1, cv2.LINE_8)
        got = np.zeros_like(want)
        R.fill_circle(got, cx, cy, r, COLOR)
        assert np.array_equal(got, want), (H, W, cx, cy, r)


@needs_cv2
@pytest.mark.parametrize("seed", range(4))
def test_clipped_line(seed):
    rs = np.random.RandomState(100 + seed)
    for it in range(1500):
        H, W = (int(v) for v in rs.randint(1, 90, 2))
        span = int(rs.choice([10, 100, 3000, 200000]))
        p = [int(v) for v in rs.randint(-span, span + 90, 4)]
        if it % 5 == 0:   # end points on and just past the frame's edges
            k = rs.randint(4)
            p[k] = int(rs.choice([0, W - 1, W, -1] if k % 2 == 0 else [0, H - 1, H, -1]))
        if it % 11 == 0:   # a point, or a line along an edge
            p[2:] = p[:2] if it % 2 else [p[0], int(rs.choice([0, H - 1]))]
        want = np.zeros((H, W, 3), np.uint8)
        cv2.line(want, tuple(p[:2]), tuple(p[2:]), COLOR, 1, cv2.LINE_8)
        got = np.zeros_like(want)
        R.draw_line(got, *p, COLOR)
        assert np.array_equal(got, want), (H, W, p)


def _golden(name, ragged):
    z = np.load(os.path.join(GOLDEN, name))
    meta = json.loads(str(z["meta"]))
    off = {k: np.concatenate([[0], np.cumsum(z[k + "_len"])]) for k in ragged}
    foff = np.concatenate([[0], np.cumsum(z["size"].astype(np.int64) ** 2 * 3)])
    for i in range(len(z["size"])):
        row = {k: z[k][i] for k in z.files if k not in ragged and k not in ("frames", "meta") and not k.endswith("_len")}
        row.update({k: z[k][off[k][i]:off[k][i + 1]] for k in ragged})
        S = int(row["size"])
        row["frame"] = z["frames"][foff[i]:foff[i + 1]].reshape(S, S, 3)
        yield meta[int(row["case"])], row


def test_golden_covers_what_it_claims():
    ww = list(_golden("render_ww.npz", ("pos",)))
    hw = list(_golden("render_hw.npz", ("pos", "saved")))
    assert {r["size"] for _, r in ww} >= {800, 257, 37} and {r["size"] for _, r in hw} >= {800, 257, 37}
    assert {int(r["gate"]) for _, r in hw} == {0, 1}
    assert any(r["saved"].any() and not r["gate"] for _, r in hw)
    for _, r in ww + hw:   # the background blend lifts every channel to at least 102
        assert r["frame"].min() >= 102


def test_waterworld_frames_equal_the_references():
    n = 0
    for m, r in _golden("render_ww.npz", ("pos",)):
        got = R.ww_frame(r["pos"][:, 0], r["pos"][:, 1], r["obst"], m["n_pursuers"], m["n_evaders"], int(r["size"]),
                         m["radius"], m["obstacle_radius"], m["sensor_range"], R.sensor_dirs(m["n_sensors"]))
        assert np.array_equal(got, r["frame"]), (m, int(r["size"]))
        n += 1
    assert n >= 8


def test_hostage_frames_equal_the_references():
    n = 0
    for m, r in _golden("render_hw.npz", ("pos", "saved")):
        got = R.hw_frame(r["pos"][:, 0], r["pos"][:, 1], r["fixed"], r["saved"], r["gate"], m["n_good"], m["n_bad"],
                         int(r["size"]), m["radius"], m["bomb_radius"], m["sensor_range"], R.sensor_dirs(m["n_sensors"]))
        assert np.array_equal(got, r["frame"]), (m, int(r["size"]))
        n += 1
    assert n >= 8


def test_pursuit_frame_rule():
    """The integer rule on a hand-checked 3 x 2 map: a building, a window blended twice, markers, a gone evader."""
    building = np.zeros((3, 2), bool)
    building[2, 1] = True
    img = R.pe_frame(building, [0, 0], [0, 0], [0, 2, 1], [1, 1, 1], gone=0b100, obs_range=3, cell=4)
    assert img.shape == (8, 12, 3)
    twice = ((((255 + 255 + 1) >> 1) + 255 + 1) >> 1, (((255 + 152 + 1) >> 1) + 152 + 1) >> 1,
             (((255 + 72 + 1) >> 1) + 72 + 1) >> 1)
    assert tuple(img[0, 0]) == twice and tuple(img[7, 7]) == twice          # cells (0, 0) and (1, 1): both windows
    assert tuple(img[0, 8]) == (255, 255, 255)                              # cell (2, 0): outside them
    assert tuple(img[4, 8]) == (64, 64, 64) and tuple(img[5, 9]) == (0, 0, 255)    # building (2, 1), an evader on it
    assert tuple(img[1, 1]) == (255, 0, 0) and tuple(img[2, 2]) == (255, 0, 0)     # pursuers at (0, 0)
    assert tuple(img[0, 0]) != (255, 0, 0) and tuple(img[3, 3]) == twice          # marker is [1, 3)^2
    assert tuple(img[5, 1]) == (0, 0, 255) and tuple(img[5, 5]) == twice          # evader at (0, 1), gone one at (1, 1)
