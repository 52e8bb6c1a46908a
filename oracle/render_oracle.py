"""CPU oracle of the frame kernels (madrl_b200/csrc/render.cu) -- TEST INFRASTRUCTURE, integer NumPy.

A rasteriser of the rules in DESIGN §4.10: the reference's Waterworld and Hostage ``render`` bodies
(``waterworld.py:438-479``, ``hostage.py:431-478``) drawn with OpenCV's 8-connected primitives instead of
the anti-aliased ones, and the integer Pursuit picture.  The primitives restate what ``cv2.circle(..., -1,
LINE_8)``, ``cv2.line(..., 1, LINE_8)`` and ``cv2.addWeighted`` draw; ``tests/test_render_cpu.py`` pins them
against the installed ``cv2`` and pins the frames against the reference's own render output
(``tests/golden/render_*.npz``, made by ``oracle/make_render_golden.py``).

Frames are ``uint8 [H, W, 3]`` RGB.  Only ``tests/`` and ``scripts/`` import this module.
"""
import math

import numpy as np

# RGB colours (the reference passes BGR tuples to cv2 and Waterworld flips the frame to RGB)
WW_OBSTACLE, WW_PURSUER, WW_EVADER, WW_POISON = (0, 128, 128), (0, 0, 255), (0, 255, 0), (255, 0, 0)
HW_GATE, HW_KEY, HW_BOMB, HW_HOSTAGE, HW_CRIMINAL, HW_RESCUER = (
    (200, 128, 128), (255, 0, 0), (255, 0, 0), (0, 120, 255), (200, 50, 50), (0, 0, 255))
SENSOR_LINE = (0, 0, 0)
PE_FREE, PE_BUILDING, PE_WINDOW, PE_PURSUER, PE_EVADER = (255, 255, 255), (64, 64, 64), (255, 152, 72), \
    (255, 0, 0), (0, 0, 255)


def sensor_dirs(n_sensors):
    """float64 [2, K]: the cos row and the sin row of the reference's sensor angles (waterworld.py:29-30,
    hostage.py's CircAgent), the table the frame kernels are given."""
    ang = np.linspace(0., 2. * np.pi, n_sensors + 1)[:-1]
    return np.ascontiguousarray(np.stack([np.cos(ang), np.sin(ang)]))


def to_px(x, size):
    """int(float64(x) * size), truncated toward zero (NumPy's astype(int))."""
    return int(np.float64(x) * size)


# ------------------------------------------------------------------------------------------ primitives
def circle_half_widths(r):
    """Half-width of the filled circle of radius r in each row offset 0..r (-1: row not drawn).

    OpenCV's filled LINE_8 circle walks the first octant from (dx, dy) = (r, 0), dy += 1 per step, while
    dx >= dy; dx drops by one when dx^2 + dy^2 > r^2, which keeps dx = isqrt(r^2 - dy^2).  Each step fills rows
    +-dy over |x| <= dx and rows +-dx over |x| <= dy."""
    h = np.full(r + 1, -1, np.int64)
    dy = 0
    while dy <= r:
        dx = math.isqrt(r * r - dy * dy)
        if dx < dy:
            break
        h[dy] = max(h[dy], dx)
        h[dx] = max(h[dx], dy)
        dy += 1
    return h


def fill_circle(img, cx, cy, r, color, y0=0):
    """`img` holds the frame's rows y0 .. y0 + len(img) - 1 (all of it when y0 = 0 and it is H rows)."""
    H, W = img.shape[:2]
    h = circle_half_widths(r)
    for oy in range(max(-r, y0 - cy), min(r, y0 + H - 1 - cy) + 1):
        y, w = cy + oy, h[abs(oy)]
        if w >= 0:
            x0, x1 = max(cx - w, 0), min(cx + w, W - 1)
            if x0 <= x1:
                img[y - y0, x0:x1 + 1] = color


def clip_line(W, H, x1, y1, x2, y2):
    """OpenCV's clipLine on the rectangle [0, W-1] x [0, H-1]: the segment's end points moved onto the
    rectangle's edges (y edges first, then x edges; each move truncates a float64 quotient), or None."""
    right, bottom = W - 1, H - 1
    code = lambda x, y: (x < 0) + (x > right) * 2 + (y < 0) * 4 + (y > bottom) * 8
    c1, c2 = code(x1, y1), code(x2, y2)
    if (c1 & c2) == 0 and (c1 | c2) != 0:
        if c1 & 12:
            a = 0 if c1 < 8 else bottom
            x1 += int(float(a - y1) * (x2 - x1) / (y2 - y1))
            y1 = a
            c1 = (x1 < 0) + (x1 > right) * 2
        if c2 & 12:
            a = 0 if c2 < 8 else bottom
            x2 += int(float(a - y2) * (x2 - x1) / (y2 - y1))
            y2 = a
            c2 = (x2 < 0) + (x2 > right) * 2
        if (c1 & c2) == 0 and (c1 | c2) != 0:
            if c1:
                a = 0 if c1 == 1 else right
                y1 += int(float(a - x1) * (y2 - y1) / (x2 - x1))
                x1 = a
                c1 = 0
            if c2:
                a = 0 if c2 == 1 else right
                y2 += int(float(a - x2) * (y2 - y1) / (x2 - x1))
                x2 = a
                c2 = 0
    return (x1, y1, x2, y2) if (c1 | c2) == 0 else None


def line_pixels(W, H, x1, y1, x2, y2):
    """The (x, y) pixels of OpenCV's 8-connected one-pixel line: clipped, walked from its left end point
    along the major axis; the minor coordinate advances after a step whose error term is negative."""
    c = clip_line(W, H, x1, y1, x2, y2)
    if c is None:
        return []
    x1, y1, x2, y2 = c
    if x2 < x1:
        x1, y1, x2, y2 = x2, y2, x1, y1
    dx, dy = x2 - x1, abs(y2 - y1)
    sy = -1 if y2 < y1 else 1
    vert = dy > dx
    major, minor = (dy, dx) if vert else (dx, dy)
    err, px, py, out = major - 2 * minor, x1, y1, []
    for _ in range(major + 1):
        out.append((px, py))
        step_minor = err < 0
        err += -2 * minor + (2 * major if step_minor else 0)
        if vert:
            py += sy
            px += 1 if step_minor else 0
        else:
            px += 1
            py += sy if step_minor else 0
    return out


def draw_line(img, x1, y1, x2, y2, color):
    H, W = img.shape[:2]
    for x, y in line_pixels(W, H, x1, y1, x2, y2):
        img[y, x] = color


def add_weighted_lut():
    """uint8 [256]: cv2.addWeighted(255, 0.4, v, 0.6, 0) -- float32 products and sums, rounded to nearest even."""
    v = np.arange(256, dtype=np.float32)
    t = np.float32(255) * np.float32(0.4) + v * np.float32(0.6)
    return np.clip(np.rint(t), 0, 255).astype(np.uint8)


def blend_background(img):
    return add_weighted_lut()[img]


# ------------------------------------------------------------------------------------------ frames
# A frame is built as its primitives in painter's order -- ("circle", cx, cy, r, color), ("pixels", xs, ys, color)
# for a line walked once into its pixels, or None for a primitive that draws nothing -- then painted.  The list is
# indexed as the kernels index their primitives, and painting it in row bands lets a 32768 x 32768 frame be checked
# without holding it whole.
def _finite(*v):
    return all(math.isfinite(float(x)) for x in v)


def circle_prim(x, y, size, r, color):
    """A filled circle at the stored coordinate (x, y); None if a coordinate is not finite (such an object
    draws nothing, DESIGN §4.10)."""
    return ("circle", to_px(x, size), to_px(y, size), r, color) if _finite(x, y) else None


def line_prim(W, H, x1, y1, x2, y2, color):
    a = np.array(line_pixels(W, H, x1, y1, x2, y2), np.int64).reshape(-1, 2)
    return ("pixels", a[:, 0], a[:, 1], color)


def paint(prims, W, H, rows=None):
    """The RGB frame [H, W, 3] the primitives draw, background blend included; `rows` = (y0, y1): only its rows
    y0 .. y1 - 1, as a [y1 - y0, W, 3] band."""
    y0, y1 = (0, H) if rows is None else rows
    img = np.full((y1 - y0, W, 3), 255, np.uint8)
    for q in prims:
        if q is None:
            continue
        if q[0] == "circle":
            fill_circle(img, q[1], q[2], q[3], q[4], y0=y0)
        else:
            xs, ys, color = q[1], q[2], q[3]
            m = (ys >= y0) & (ys < y1)
            img[ys[m] - y0, xs[m]] = color
    return blend_background(img)


def _sensor_prims(x, y, sensor_range, dirs, size, body_r, body_color):
    """A pursuer / rescuer: each sensor line, then its body (the reference redraws the body after every line,
    which leaves the body over all of them)."""
    K = dirs.shape[1]
    if not _finite(x, y):
        return [None] * (K + 1)
    p = (to_px(x, size), to_px(y, size))
    out = []
    for k in range(K):
        ex = int((np.float64(x) + sensor_range * dirs[0, k]) * size)
        ey = int((np.float64(y) + sensor_range * dirs[1, k]) * size)
        out.append(line_prim(size, size, p[0], p[1], ex, ey, SENSOR_LINE))
    return out + [circle_prim(x, y, size, int(body_r * size), body_color)]


def ww_prims(px, py, obst, Np, Ne, size, radius, obstacle_radius, sensor_range, dirs):
    """The primitives of ww_frame, in the kernels' order: the obstacle, each pursuer's lines and body, evaders,
    poison."""
    out = [circle_prim(obst[0], obst[1], size, int(obstacle_radius * size), WW_OBSTACLE)]
    for i in range(Np):
        out += _sensor_prims(px[i], py[i], sensor_range, dirs, size, radius, WW_PURSUER)
    for i in range(Np, Np + Ne):
        out.append(circle_prim(px[i], py[i], size, int(radius * 2 * size), WW_EVADER))
    for i in range(Np + Ne, len(px)):
        out.append(circle_prim(px[i], py[i], size, int(radius * 3 / 4 * size), WW_POISON))
    return out


def ww_frame(px, py, obst, Np, Ne, size, radius, obstacle_radius, sensor_range, dirs, rows=None):
    """The reference MAWaterWorld.render frame of one env: px, py [n_obj] (pursuers, evaders, poisons),
    obst [2]; RGB uint8 [size, size, 3] (`rows`: a band of it, as paint)."""
    return paint(ww_prims(px, py, obst, Np, Ne, size, radius, obstacle_radius, sensor_range, dirs), size, size, rows)


def hw_prims(px, py, fixed, saved, flags, n_good, n_bad, size, radius, bomb_radius, sensor_range, dirs):
    """The primitives of hw_frame, in the kernels' order: gate line and key (None while the gate is open), bomb,
    hostages (None once saved), criminals, each rescuer's lines and body."""
    out = [None, None]
    if not int(flags) & 1:
        out = [line_prim(size, size, 0, int(0.5 * size), int(1 * size), int(0.5 * size), HW_GATE),
               circle_prim(fixed[0], fixed[1], size, int(radius * size), HW_KEY)]
    out.append(circle_prim(fixed[2], fixed[3], size, int(bomb_radius * size), HW_BOMB))
    for j in range(len(saved)):
        i = n_good + n_bad + j
        out.append(None if saved[j] else circle_prim(px[i], py[i], size, int(radius * 2 * size), HW_HOSTAGE))
    for i in range(n_good, n_good + n_bad):
        out.append(circle_prim(px[i], py[i], size, int(radius * size), HW_CRIMINAL))
    for i in range(n_good):
        out += _sensor_prims(px[i], py[i], sensor_range, dirs, size, radius, HW_RESCUER)
    return out


def hw_frame(px, py, fixed, saved, flags, n_good, n_bad, size, radius, bomb_radius, sensor_range, dirs, rows=None):
    """The reference ContinuousHostageWorld.render frame of one env: px, py [n_obj] (rescuers, criminals,
    hostages), fixed [4] = key x, y, bomb x, y, saved [n_hostages], flags (bit 0: gate open); RGB (`rows`: a
    band, as paint)."""
    return paint(hw_prims(px, py, fixed, saved, flags, n_good, n_bad, size, radius, bomb_radius, sensor_range, dirs),
                 size, size, rows)


def pe_frame(building, pur_x, pur_y, ev_x, ev_y, gone, obs_range, cell, rows=None):
    """The Pursuit frame of one env: building bool [xs, ys]; pursuer and evader cells; gone = the evaders_gone
    bits (set for evaders removed and for those a random_opponents episode never spawned); RGB uint8
    [ys * cell, xs * cell, 3], pixel (row, col) in cell (col // cell, row // cell).  `rows` = (y0, y1): only
    rows y0 .. y1 - 1."""
    xs, ys = building.shape
    y0, y1 = (0, ys * cell) if rows is None else rows
    grid = np.where(building.T[..., None], np.array(PE_BUILDING, np.int64), np.array(PE_FREE, np.int64))
    off = (obs_range - 1) // 2
    win = np.array(PE_WINDOW, np.int64)
    for x, y in zip(pur_x, pur_y):
        wx0, wy0 = max(int(x) - off, 0), max(int(y) - off, 0)
        wx1, wy1 = min(int(x) - off + obs_range, xs), min(int(y) - off + obs_range, ys)
        grid[wy0:wy1, wx0:wx1] = (grid[wy0:wy1, wx0:wx1] + win + 1) >> 1
    img = grid.astype(np.uint8)[np.arange(y0, y1) // cell][:, np.arange(xs * cell) // cell]
    lo, hi = cell // 4, cell - cell // 4

    def mark(x, y, color):
        r0, r1 = max(int(y) * cell + lo, y0), min(int(y) * cell + hi, y1)
        if r0 < r1:
            img[r0 - y0:r1 - y0, int(x) * cell + lo:int(x) * cell + hi] = color

    for x, y in zip(pur_x, pur_y):
        mark(x, y, PE_PURSUER)
    for j, (x, y) in enumerate(zip(ev_x, ev_y)):
        if not (int(gone) >> j) & 1:
            mark(x, y, PE_EVADER)
    return img


# ------------------------------------------------------------------------------------------ engine state
def ww_frames(state, env_ids, size, cfg, Np, Ne, rows=None):
    """Frames of the listed envs of a BatchedMAWaterWorld state dict (tensors or arrays); `cfg` its
    madrl_ww_config; `rows`: a band of each, as paint."""
    g = {k: np.asarray(v.cpu() if hasattr(v, "cpu") else v) for k, v in state.items()}
    dirs = sensor_dirs(cfg.n_sensors)
    return np.stack([ww_frame(g["pos_x"][e], g["pos_y"][e], (g["obst_x"][e], g["obst_y"][e]), Np, Ne, size,
                              cfg.radius, cfg.obstacle_radius, cfg.sensor_range, dirs, rows) for e in env_ids])


def hw_frames(state, env_ids, size, cfg, rows=None):
    """Frames of the listed envs of a BatchedHostageWorld state dict; `cfg` its madrl_hostage_config."""
    g = {k: np.asarray(v.cpu() if hasattr(v, "cpu") else v) for k, v in state.items()}
    dirs = sensor_dirs(cfg.n_sensors)
    fixed = np.concatenate([g["key"], g["bomb"]], axis=1)
    return np.stack([hw_frame(g["pos_x"][e], g["pos_y"][e], fixed[e], g["saved"][e], g["flags"][e], cfg.n_good,
                              cfg.n_bad, size, cfg.radius, cfg.bomb_radius, cfg.sensor_range, dirs, rows)
                     for e in env_ids])


def pe_frames(state, map_pool, env_ids, obs_range, cell, rows=None):
    """Frames of the listed envs of a BatchedPursuitEvade state dict; map_pool int32 [n_maps, xs, ys]."""
    g = {k: np.asarray(v.cpu() if hasattr(v, "cpu") else v) for k, v in state.items()}
    return np.stack([pe_frame(map_pool[g["map_id"][e]] == -1, g["pursuer_x"][e], g["pursuer_y"][e],
                              g["evader_x"][e], g["evader_y"][e], int(g["gone"][e]), obs_range, cell, rows)
                     for e in env_ids])
