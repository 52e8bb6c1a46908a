"""Constructed scenes for the frame kernels (csrc/render.cu) at the edges that stepped envs never reach, shared by
tests/test_render_edges_gpu.py, tests/test_render_edges_cpu.py and tests/test_emulated_render_edges.py.

A scene is written through a state dict of views -- BatchedMAWaterWorld.state / BatchedHostageWorld.state on the
GPU, the emulator's views on the CPU -- so the same builder serves both, and the NumPy oracle
(oracle/render_oracle.py) draws what it wrote.  Coordinates are in frame units: pixel p of an S-pixel frame is
p / S."""
from fractions import Fraction

import numpy as np
import torch

from oracle import render_oracle as R

TILE = 32          # the tiles kernel's tile edge
CHUNK = 256        # primitives the tiles kernel builds per pass
INF, NAN = float("inf"), float("nan")
# the non-finite patterns an object's (x, y) can take
NON_FINITE = [(NAN, 0.5), (0.5, NAN), (NAN, NAN), (INF, 0.5), (0.5, -INF), (-INF, INF), (INF, NAN)]


def put(dst, src):
    """Write `src` into the view `dst` (a torch tensor or a NumPy array) in the view's dtype."""
    if isinstance(dst, torch.Tensor):
        dst[...] = torch.as_tensor(np.asarray(src, np.float64), device=dst.device).to(dst.dtype)
    else:
        dst[...] = np.asarray(src, np.float64).astype(dst.dtype)


def assert_frames_equal(got, want, what=""):
    """Every pixel of every frame; the (frame, row, column) of the first differences on failure.  Torch tensors are
    compared where they live (the other side is moved there)."""
    if isinstance(got, torch.Tensor) or isinstance(want, torch.Tensor):
        dev = got.device if isinstance(got, torch.Tensor) else want.device
        got, want = (torch.as_tensor(np.asarray(t)).to(dev) if not isinstance(t, torch.Tensor) else t
                     for t in (got, want))
        assert tuple(got.shape) == tuple(want.shape), (what, tuple(got.shape), tuple(want.shape))
        bad = (got != want).any(dim=-1).nonzero()
        n, first = int(bad.shape[0]), bad[:5].tolist()
    else:
        assert got.shape == want.shape, (what, got.shape, want.shape)
        bad = np.argwhere((got != want).any(axis=-1))
        n, first = len(bad), bad[:5].tolist()
    assert n == 0, "%s: %d pixels differ, first (frame, row, col) %s" % (what, n, first)


# ------------------------------------------------------------------------------------------ primitive boxes
def prim_box(q):
    """(x0, x1, y0, y1), inclusive, of an oracle primitive's pixels (circles: the bounding square); None if it
    draws nothing."""
    if q is None:
        return None
    if q[0] == "circle":
        _, cx, cy, r, _ = q
        return cx - r, cx + r, cy - r, cy + r
    if len(q[1]) == 0:
        return None
    return int(q[1].min()), int(q[1].max()), int(q[2].min()), int(q[2].max())


def tile_chunks(prims, S):
    """{tile (tx, ty): [primitive indices whose box meets it]} over the S x S frame's 32 x 32 tiles."""
    out = {}
    for p, q in enumerate(prims):
        b = prim_box(q)
        if b is None:
            continue
        x0, x1, y0, y1 = max(b[0], 0), min(b[1], S - 1), max(b[2], 0), min(b[3], S - 1)
        for ty in range(y0 // TILE, y1 // TILE + 1) if y0 <= y1 else ():
            for tx in range(x0 // TILE, x1 // TILE + 1) if x0 <= x1 else ():
                out.setdefault((tx, ty), []).append(p)
    return out


def check_chunk_scene(prims, S):
    """The chunk scene does what it is for: some tile meets more than 256 primitives, and at every chunk boundary
    of the primitive list one tile meets primitives of different colours on both sides of it.  Returns the most
    primitives one tile meets."""
    tiles = tile_chunks(prims, S)
    most = max(len(v) for v in tiles.values())
    assert most > CHUNK, most
    colour = lambda p: prims[p][-1]
    for b in range(CHUNK, len(prims), CHUNK):
        sides = [({colour(p) for p in v if b - CHUNK <= p < b}, {colour(p) for p in v if b <= p < b + CHUNK})
                 for v in tiles.values()]
        assert any(lo and hi and len(lo | hi) > 1 for lo, hi in sides), b
    return most


# ------------------------------------------------------------------------------------------ configs
def chunk_ww_kw(S):
    """Waterworld with 32 pursuers of 64 sensors and 224 evaders and poison: 1 + 32 * 65 + 224 = 2305 primitives,
    ten chunks; radii and sensor range of a few pixels at S."""
    return dict(n_pursuers=32, n_evaders=112, n_poison=112, n_sensors=64, radius=4.6 / S, obstacle_radius=9.3 / S,
                sensor_range=11.0 / S)


def chunk_hw_args(S):
    """Hostage with 32 rescuers of 64 sensors, 112 criminals and 112 hostages: 3 + 224 + 32 * 65 = 2307
    primitives."""
    return (32, 112, 112, 2, 2), dict(n_sensors=64, radius=4.6 / S, bomb_radius=6.2 / S, sensor_range=11.0 / S)


# ------------------------------------------------------------------------------------------ scenes
def _stack_points(rs, n, S, centre):
    """n points stacked on three spots a few pixels apart around pixel `centre` (a tile corner), each jittered
    by up to 2.5 pixels."""
    spots = np.array([[-1.5, -1.2], [2.7, -0.4], [0.4, 3.1]]) + centre
    k = rs.randint(0, 3, n)
    return (spots[k] + rs.uniform(-2.5, 2.5, (n, 2))) / S


def chunk_scene_ww(st, e, S, seed):
    """Every object of env e stacked on three spots around the frame's first tile corner (32, 32) in pixels, so
    that the four tiles around it meet nearly all 2305 primitives, in every chunk, with colours overlapping."""
    rs = np.random.RandomState(seed)
    n = st["pos_x"].shape[1]
    c = min(TILE, S // 2)
    xy = _stack_points(rs, n, S, c)
    put(st["pos_x"][e], xy[:, 0])
    put(st["pos_y"][e], xy[:, 1])
    put(st["obst_x"][e:e + 1], (c + 0.5) / S)
    put(st["obst_y"][e:e + 1], (c - 3.3) / S)


def chunk_scene_hw(st, e, S, seed, gate_closed=True):
    rs = np.random.RandomState(seed)
    n = st["pos_x"].shape[1]
    c = min(TILE, S // 2)
    xy = _stack_points(rs, n, S, c)
    put(st["pos_x"][e], xy[:, 0])
    put(st["pos_y"][e], xy[:, 1])
    put(st["key"][e], [(c - 2.2) / S, (c + 1.7) / S])
    put(st["bomb"][e], [(c + 1.4) / S, (c - 0.6) / S])
    st["saved"][e] = 0
    st["saved"][e, ::5] = 1
    st["flags"][e:e + 1] = 0 if gate_closed else 1


def edge_coords(S):
    """Coordinates at the frame's edges, in frame units: centres in (-1, 0) px (truncation and floor differ),
    exactly 0, S - 1 and S px, coordinate 1.0, just past each side, far off (|x| up to 1e6) and beyond the 2^30
    pixel clamp."""
    big = 2.0 ** 31 / S
    return [-0.5 / S, -0.999 / S, -1e-9, 0.0, (S - 1) / S, (S - 0.5) / S, 1.0, (S + 0.5) / S, -3.0 / S,
            (S + 3.0) / S, 0.5, 0.37, 1e6, -1e6, big, -big, 1e12, -1e12]


def off_frame_positions(S, n, seed):
    """n (x, y) positions, pairs of edge_coords in an order the seed shuffles: across the envs of a scene they pair
    every edge coordinate with the others, so circles hang off each side and corner and lines clip at each."""
    rs = np.random.RandomState(seed)
    c = edge_coords(S)
    pts = [(c[i], c[j]) for i in range(len(c)) for j in range(len(c))]
    pts = [pts[i] for i in rs.permutation(len(pts))]
    return np.array(pts[:n], np.float64)


def off_frame_scene_ww(st, e, S, seed):
    n = st["pos_x"].shape[1]
    xy = off_frame_positions(S, n + 1, seed)
    put(st["pos_x"][e], xy[:n, 0])
    put(st["pos_y"][e], xy[:n, 1])
    put(st["obst_x"][e:e + 1], xy[n, 0])
    put(st["obst_y"][e:e + 1], xy[n, 1])


def off_frame_scene_hw(st, e, S, seed, gate_closed=True):
    n = st["pos_x"].shape[1]
    xy = off_frame_positions(S, n + 2, seed)
    put(st["pos_x"][e], xy[:n, 0])
    put(st["pos_y"][e], xy[:n, 1])
    put(st["key"][e], xy[n])
    put(st["bomb"][e], xy[n + 1])
    st["saved"][e] = 0
    st["flags"][e:e + 1] = 0 if gate_closed else 1


def edge_lines_ww(st, e, S):
    """Pursuers whose sensor lines run along each edge, clip at each edge and corner, or start on a corner."""
    n = st["pos_x"].shape[1]
    pts = [(0.0, 0.0), ((S - 1) / S, 0.0), (0.0, (S - 1) / S), ((S - 1) / S, (S - 1) / S), (1.0, 1.0),
           (0.5, 0.0), (0.0, 0.5), ((S - 1) / S, 0.5), (0.5, (S - 1) / S), (-0.5 / S, 0.5), (0.5, -0.5 / S),
           (0.5, 0.5), (0.1, 0.9), (0.9, 0.1)]
    xy = np.array([pts[i % len(pts)] for i in range(n)])
    put(st["pos_x"][e], xy[:, 0])
    put(st["pos_y"][e], xy[:, 1])
    put(st["obst_x"][e:e + 1], 0.5)
    put(st["obst_y"][e:e + 1], 1.0)


def non_finite_ww(st, e, k, Np):
    """Non-finite pattern k of NON_FINITE written over pursuer 0, the first evader, the last poison and the obstacle
    of env e (its other objects as they were).  Such an object draws nothing."""
    x, y = NON_FINITE[k % len(NON_FINITE)]
    for i in (0, Np, st["pos_x"].shape[1] - 1):
        put(st["pos_x"][e, i:i + 1], x)
        put(st["pos_y"][e, i:i + 1], y)
    put(st["obst_x"][e:e + 1], x)
    put(st["obst_y"][e:e + 1], y)


def non_finite_hw(st, e, k, Ng):
    """The same over rescuer 0, the first criminal, the last hostage, the key and the bomb."""
    x, y = NON_FINITE[k % len(NON_FINITE)]
    for i in (0, Ng, st["pos_x"].shape[1] - 1):
        put(st["pos_x"][e, i:i + 1], x)
        put(st["pos_y"][e, i:i + 1], y)
    put(st["key"][e], [x, y])
    put(st["bomb"][e], [y, x])


# ------------------------------------------------------------------------------------------ no contraction
def fused_end(p, r, d):
    """float64 p + r d rounded once, as a fused multiply-add would give it (float(Fraction) rounds correctly)."""
    return float(Fraction(p) + Fraction(r) * Fraction(d))


def unfused_end(p, r, d):
    """float64 p + r d with the product rounded first: what the kernels and the oracle compute."""
    return float(np.float64(p) + np.float64(r) * np.float64(d))


def _steps(x, u, to=np.float64):
    """x moved u representable values of type `to` up (u > 0) or down."""
    x = to(x)
    for _ in range(abs(u)):
        x = np.nextafter(x, to(np.inf) if u > 0 else to(-np.inf))
    return float(x)


def fma_points_f64(S, r, dirs_row, want, lo=100, hi=700):
    """Up to `want` (j, p) with p a float64 position whose sensor-j end coordinate p + r dirs_row[j] lands in an
    other pixel when the product and the sum are fused: trunc(S * fused) != trunc(S * unfused).  The end pixel
    lies in [lo, hi)."""
    out = []
    for k in range(lo, hi, 7):
        for j in range(len(dirs_row)):
            d = dirs_row[j]
            if abs(d) < 1e-3:
                continue
            p0 = k / S - r * d
            for u in (0, 1, -1, 2, -2, 3, -3) + tuple(range(4, 41)) + tuple(range(-4, -41, -1)):
                p = _steps(p0, u)
                if int(unfused_end(p, r, d) * S) != int(fused_end(p, r, d) * S):
                    out.append((j, p))
                    break
            if len(out) >= want:
                return out
    return out


def fma_points_f32(S, p, dirs_row, want, lo=100, hi=700):
    """Up to `want` (j, r) for a float32 position p: a sensor_range r (a double in (0, 1)) whose sensor-j end
    coordinate lands in an other pixel when fused, as fma_points_f64."""
    p = float(np.float32(p))
    out = []
    for j in range(len(dirs_row)):
        d = dirs_row[j]
        if abs(d) < 1e-3:
            continue
        for k in range(lo, hi, 13):
            r0 = (k / S - p) / d
            if not 0.05 < r0 < 0.9:
                continue
            hit = None
            for u in range(-60, 61):
                r = _steps(r0, u)
                if int(unfused_end(p, r, d) * S) != int(fused_end(p, r, d) * S):
                    hit = (j, r)
                    break
            if hit:
                out.append(hit)
                break
        if len(out) >= want:
            break
    return out


def max_sensor_range(S):
    """The largest double r with r * S < 2^29 in float64, the largest sensor_range the frame kernels take at S."""
    bound = float(1 << 29)
    r = bound / S
    while not r * S < bound:
        r = float(np.nextafter(r, -np.inf))
    while float(np.nextafter(r, np.inf)) * S < bound:
        r = float(np.nextafter(r, np.inf))
    return r


# ------------------------------------------------------------------------------------------ oracle helpers
def _host(st):
    return {k: np.asarray(v.cpu() if hasattr(v, "cpu") else v) for k, v in st.items()}


def ww_prims(st, e, S, cfg, Np, Ne):
    """The oracle's primitives of env e of a Waterworld state dict, in the kernels' order."""
    g = _host(st)
    return R.ww_prims(g["pos_x"][e], g["pos_y"][e], (g["obst_x"][e], g["obst_y"][e]), Np, Ne, S, cfg.radius,
                      cfg.obstacle_radius, cfg.sensor_range, R.sensor_dirs(cfg.n_sensors))


def hw_prims(st, e, S, cfg):
    """The same for a Hostage state dict."""
    g = _host(st)
    fixed = np.concatenate([g["key"][e], g["bomb"][e]])
    return R.hw_prims(g["pos_x"][e], g["pos_y"][e], fixed, g["saved"][e], g["flags"][e], cfg.n_good, cfg.n_bad, S,
                      cfg.radius, cfg.bomb_radius, cfg.sensor_range, R.sensor_dirs(cfg.n_sensors))
