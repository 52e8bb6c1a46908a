"""The frame kernels (csrc/render.cu) on the GPU at the edges that stepped scenes never reach, against the NumPy
oracle (oracle/render_oracle.py), every pixel of every frame: more work items than one grid of blocks, the largest
frames, painter's order across the 256-primitive chunks, coordinates on and off the frame's edges and non-finite
ones, sensor end points a fused multiply-add would move, the sensor_range bound and int64 ids outside the range.
Scenes come from tests/render_edges.py."""
import numpy as np
import pytest
import torch

import render_edges as RE
from madrl_b200 import BatchedHostageWorld, BatchedMAWaterWorld, BatchedPursuitEvade, _lib
from oracle import render_oracle as R

pytestmark = pytest.mark.gpu

FAMILIES = [("ww", torch.float32), ("ww", torch.float64), ("hw", torch.float32), ("hw", torch.float64)]
FAM_IDS = ["ww_f32", "ww_f64", "hw_f32", "hw_f64"]
GRID = 1 << 20   # blocks of one launch; more work items loop


def ww(E, dtype, **kw):
    kw.setdefault("n_pursuers", 2)
    kw.setdefault("n_evaders", 2)
    return BatchedMAWaterWorld(E, dtype=dtype, **kw)


def hw(E, dtype, args=(2, 2, 2, 1, 1), **kw):
    return BatchedHostageWorld(E, *args, dtype=dtype, **kw)


def want_frames(eng, fam, ids, S, rows=None):
    if fam == "ww":
        return R.ww_frames(eng.state, ids, S, eng.cfg, eng.n_pursuers, eng.n_evaders, rows)
    return R.hw_frames(eng.state, ids, S, eng.cfg, rows)


def cycling_ids(n, E):
    """int64 CUDA ids cycling over every env, with -1, E and +-2^32 + k mixed in before and after item 2^20."""
    ids = torch.arange(n, dtype=torch.int64) % E
    bad = {3: -1, 5: E, 7: (1 << 32) + 1, 11: -(1 << 32) + 2, n - 1: (1 << 32), n - 2: -1, n - 4: E,
           n - 6: (1 << 33) + E - 1, n // 2: -(1 << 32)}
    for i, v in bad.items():
        ids[i] = v
    return ids.cuda()


def check_gathered(out, ids, table, E, chunk=1 << 15):
    """out [n, ...] against table [E, ...] gathered by id, zero frames for ids outside [0, E), on the device."""
    tab = torch.cat([torch.as_tensor(table).cuda(), torch.zeros_like(torch.as_tensor(table[:1])).cuda()])
    idx = torch.where((ids >= 0) & (ids < E), ids, torch.full_like(ids, E))
    for c0 in range(0, out.shape[0], chunk):
        RE.assert_frames_equal(out[c0:c0 + chunk], tab[idx[c0:c0 + chunk]], "frames %d.." % c0)


def s1_colours_ww(eng):
    """Envs whose single pixel shows, in turn, poison, evader, pursuer, obstacle and background: each env moves
    the objects drawn later off the frame."""
    st = eng.state
    RE.put(st["pos_x"], 0.3)
    RE.put(st["pos_y"], 0.6)
    RE.put(st["obst_x"], 0.2)
    RE.put(st["obst_y"], 0.9)
    Np, Ne = eng.n_pursuers, eng.n_evaders
    for e in range(eng.n_envs):
        k = e % 5
        if k >= 1:
            RE.put(st["pos_x"][e, Np + Ne:], 2.0)
        if k >= 2:
            RE.put(st["pos_x"][e, Np:Np + Ne], -1.5)
        if k >= 3:
            RE.put(st["pos_y"][e, :Np], 7.0)
        if k >= 4:
            RE.put(st["obst_x"][e:e + 1], float("nan"))


def s1_colours_hw(eng):
    st = eng.state
    RE.put(st["pos_x"], 0.3)
    RE.put(st["pos_y"], 0.6)
    RE.put(st["key"], 0.4)
    RE.put(st["bomb"], 0.7)
    Ng, Nb = eng.n_good, eng.n_bad
    st["saved"][:] = 0
    for e in range(eng.n_envs):
        k = e % 5
        st["flags"][e] = 1 if k >= 4 else 0
        if k >= 4:
            RE.put(st["bomb"][e], 5.0)
        if k >= 1:
            RE.put(st["pos_x"][e, :Ng], -2.0)
        if k >= 2:
            RE.put(st["pos_y"][e, Ng:Ng + Nb], 3.0)
        if k >= 3:
            st["saved"][e] = 1


def random_scene(eng, fam, seed):
    rs = np.random.RandomState(seed)
    st = eng.state
    RE.put(st["pos_x"], rs.uniform(-0.1, 1.1, tuple(st["pos_x"].shape)))
    RE.put(st["pos_y"], rs.uniform(-0.1, 1.1, tuple(st["pos_y"].shape)))
    if fam == "ww":
        RE.put(st["obst_x"], rs.rand(eng.n_envs))
        RE.put(st["obst_y"], rs.rand(eng.n_envs))
    else:
        RE.put(st["key"], rs.rand(eng.n_envs, 2))
        RE.put(st["bomb"], rs.rand(eng.n_envs, 2))
        st["flags"][:] = torch.arange(eng.n_envs, device=eng.device, dtype=torch.int32) % 2
        st["saved"][:] = 0
        st["saved"][::3, 0] = 1


# ------------------------------------------------------------------------------------------ past one grid
@pytest.mark.parametrize("S,n", [(1, GRID + 37), (33, GRID // 4 + 13)], ids=["S1", "S33"])
@pytest.mark.parametrize("fam,dtype", FAMILIES, ids=FAM_IDS)
def test_tiles_past_one_grid(fam, dtype, S, n):
    """n frames of S x S: n * tiles > 2^20 work items, so the grid-stride loop runs; every frame checked."""
    E = 7
    kw = dict(n_sensors=5, radius=0.1, sensor_range=0.4)
    eng = ww(E, dtype, n_poison=2, obstacle_radius=0.15, **kw) if fam == "ww" else hw(E, dtype, **kw)
    if S == 1:
        (s1_colours_ww if fam == "ww" else s1_colours_hw)(eng)
    else:
        random_scene(eng, fam, 11)
    table = want_frames(eng, fam, range(E), S)
    if S == 1:
        assert len({tuple(f[0, 0]) for f in table}) == 5   # five envs, five different pixels
    assert n * ((S + 31) // 32) ** 2 > GRID
    ids = cycling_ids(n, E)
    out = torch.full((n, S, S, 3), 0x5A, dtype=torch.uint8, device=eng.device)
    eng.render_frames(ids, screen_size=S, out=out)
    check_gathered(out, ids, table, E)
    del out
    torch.cuda.empty_cache()


@pytest.mark.parametrize("xs,ys,cell,n", [(2, 2, 1, GRID + 29), (3, 3, 10, GRID // 4 + 5)], ids=["2x2c1", "3x3c10"])
def test_pursuit_past_one_grid(xs, ys, cell, n):
    E = 5
    maps = np.zeros((2, xs, ys), np.int32)
    maps[1, 0, ys - 1] = -1
    eng = BatchedPursuitEvade(E, maps, n_evaders=2, n_pursuers=2, obs_range=3, sample_maps=True, seed=3)
    eng.reset()
    st = eng.state
    rs = np.random.RandomState(4)
    for k in ("pursuer_x", "evader_x"):
        st[k][:] = torch.as_tensor(rs.randint(0, xs, tuple(st[k].shape)), device=eng.device).to(st[k].dtype)
    for k in ("pursuer_y", "evader_y"):
        st[k][:] = torch.as_tensor(rs.randint(0, ys, tuple(st[k].shape)), device=eng.device).to(st[k].dtype)
    st["map_id"][:] = torch.arange(E, device=eng.device, dtype=torch.int32) % 2
    st["gone"][:] = torch.arange(E, device=eng.device, dtype=st["gone"].dtype) % 3
    table = R.pe_frames(eng.state, eng.map_pool, range(E), eng.obs_range, cell)
    assert len({f.tobytes() for f in table}) == E
    assert n * -(-xs * ys * cell * cell // 256) > GRID
    ids = cycling_ids(n, E)
    out = torch.full((n, ys * cell, xs * cell, 3), 0x5A, dtype=torch.uint8, device=eng.device)
    eng.render_frames(ids, cell=cell, out=out)
    check_gathered(out, ids, table, E)
    del out
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ largest frames
def big_scene(eng, fam, S):
    """Sensor lines that cross the whole frame: pursuers / rescuers on a corner, on the right edge (x = S) and just
    off the left one, 64 sensors each (near-diagonal ones among them) and sensor_range 1.5."""
    st = eng.state
    pts = [(0.0, 0.0), (1.0, 0.5), (-0.3 / S, 0.37)]
    n = st["pos_x"].shape[1]
    xy = np.array([pts[i % len(pts)] for i in range(n)], np.float64)
    Na = eng.n_pursuers if fam == "ww" else eng.n_good
    xy[Na:] = np.random.RandomState(S).rand(n - Na, 2)
    RE.put(st["pos_x"][0], xy[:, 0])
    RE.put(st["pos_y"][0], xy[:, 1])
    if fam == "ww":
        RE.put(st["obst_x"][0:0 + 1], 0.75)
        RE.put(st["obst_y"][0:0 + 1], 0.2)
    else:
        RE.put(st["key"][0], [0.6, 0.45])
        RE.put(st["bomb"][0], [0.2, 0.8])
        st["flags"][0] = 0
        st["saved"][0] = 0


def compare_in_bands(out, prims, W, H, band=4096):
    for y0 in range(0, H, band):
        y1 = min(y0 + band, H)
        want = R.paint(prims, W, H, (y0, y1))
        RE.assert_frames_equal(out[:, y0:y1], want[None], "rows %d..%d" % (y0, y1))


@pytest.mark.parametrize("fam,dtype,S", [f + (S,) for f, S in zip(FAMILIES, (32768, 32767, 32767, 32768))],
                         ids=["%s_%d" % (n, S) for n, S in zip(FAM_IDS, (32768, 32767, 32767, 32768))])
def test_largest_frames(fam, dtype, S):
    """One 3.2 GB frame per call, checked in bands of 4096 rows (the oracle walks each line once)."""
    kw = dict(n_sensors=64, sensor_range=1.5)
    if fam == "ww":
        eng = ww(1, dtype, n_pursuers=3, n_evaders=3, n_poison=3, **kw)
        prims_of = lambda: RE.ww_prims(eng.state, 0, S, eng.cfg, eng.n_pursuers, eng.n_evaders)
    else:
        eng = hw(1, dtype, args=(3, 3, 3, 1, 1), **kw)
        prims_of = lambda: RE.hw_prims(eng.state, 0, S, eng.cfg)
    big_scene(eng, fam, S)
    out = eng.render_frames([0], screen_size=S)
    prims = prims_of()
    assert sum(q is not None and q[0] == "pixels" and len(q[1]) >= S for q in prims) >= 8   # lines across it
    compare_in_bands(out, prims, S, S)
    del out
    torch.cuda.empty_cache()


@pytest.mark.parametrize("xs,ys,cell", [(255, 16, 128), (16, 16, 2048)], ids=["255x16c128", "16x16c2048"])
def test_pursuit_largest_frames(xs, ys, cell):
    maps = np.zeros((1, xs, ys), np.int32)
    maps[0, ::7, ::3] = -1
    maps[0, 0, 0] = maps[0, xs - 1, ys - 1] = 0
    eng = BatchedPursuitEvade(1, maps, n_evaders=3, n_pursuers=3, obs_range=5, seed=2)
    eng.reset()
    st = eng.state
    put = lambda k, v: st[k].copy_(torch.as_tensor([v], dtype=st[k].dtype, device=eng.device))
    put("pursuer_x", [0, xs - 1, xs // 2])
    put("pursuer_y", [0, ys - 1, 1])
    put("evader_x", [xs - 1, 0, xs // 2])
    put("evader_y", [ys - 1, ys - 1, 1])
    st["gone"][:] = 0
    out = eng.render_frames([0], cell=cell)
    H, W = ys * cell, xs * cell
    for y0 in range(0, H, 4096):
        y1 = min(y0 + 4096, H)
        want = R.pe_frames(eng.state, eng.map_pool, [0], eng.obs_range, cell, (y0, y1))
        RE.assert_frames_equal(out[:, y0:y1], want, "rows %d..%d" % (y0, y1))
    del out
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------ painter's order
@pytest.mark.parametrize("S", [64, 97])
@pytest.mark.parametrize("fam,dtype", FAMILIES, ids=FAM_IDS)
def test_painters_order_across_chunks(fam, dtype, S):
    E = 3
    if fam == "ww":
        eng = ww(E, dtype, **RE.chunk_ww_kw(S))
        for e in range(E):
            RE.chunk_scene_ww(eng.state, e, S, seed=e)
        prims = RE.ww_prims(eng.state, 1, S, eng.cfg, eng.n_pursuers, eng.n_evaders)
    else:
        args, kw = RE.chunk_hw_args(S)
        eng = hw(E, dtype, args=args, **kw)
        for e in range(E):
            RE.chunk_scene_hw(eng.state, e, S, seed=e, gate_closed=e != 2)
        prims = RE.hw_prims(eng.state, 1, S, eng.cfg)
    assert len(prims) > 2300
    RE.check_chunk_scene(prims, S)
    ids = [2, 0, 1, 2]
    RE.assert_frames_equal(eng.render_frames(ids, screen_size=S), want_frames(eng, fam, ids, S))


# ------------------------------------------------------------------------------------------ off the frame
@pytest.mark.parametrize("sensor_range", [0.6, 0.0, -0.35])
@pytest.mark.parametrize("fam,dtype", FAMILIES, ids=FAM_IDS)
def test_coordinates_off_the_frame(fam, dtype, sensor_range):
    """Positions at and past the edges, far off and beyond the clamp (every env a different mix), pursuers
    whose lines run along the edges and clip at them, zero-length and negative sensor lines."""
    E = 12
    kw = dict(n_sensors=8, radius=0.02, sensor_range=sensor_range)
    if fam == "ww":
        eng = ww(E, dtype, n_pursuers=14, n_evaders=12, n_poison=12, obstacle_radius=0.1, **kw)
        for e in range(E - 1):
            RE.off_frame_scene_ww(eng.state, e, 800, seed=e)
        RE.edge_lines_ww(eng.state, E - 1, 800)
    else:
        eng = hw(E, dtype, args=(14, 12, 12, 1, 1), bomb_radius=0.05, **kw)
        for e in range(E):
            RE.off_frame_scene_hw(eng.state, e, 800, seed=e, gate_closed=e % 2 == 0)
    ids = list(range(E))
    for S in (800, 37):
        if S != 800:   # the same coordinates in pixels of this frame
            for e in range(E - 1 if fam == "ww" else E):
                (RE.off_frame_scene_ww if fam == "ww" else RE.off_frame_scene_hw)(eng.state, e, S, seed=e)
        RE.assert_frames_equal(eng.render_frames(ids, screen_size=S), want_frames(eng, fam, ids, S), "S=%d" % S)


@pytest.mark.parametrize("fam,dtype", FAMILIES, ids=FAM_IDS)
def test_non_finite_objects_draw_nothing(fam, dtype):
    """Every pattern of NaN and +-inf in x, y or both, over one object of each kind; the rest of the frame is
    the oracle's (which draws no primitive for such an object)."""
    n_pat = len(RE.NON_FINITE)
    E = n_pat + 1
    if fam == "ww":
        eng = ww(E, dtype, n_pursuers=3, n_evaders=3, n_poison=3, n_sensors=9, radius=0.04)
    else:
        eng = hw(E, dtype, args=(3, 3, 3, 1, 1), n_sensors=9, radius=0.04)
    random_scene(eng, fam, 5)
    if fam == "hw":
        eng.state["flags"][:] = 0   # key and gate drawn
    before = want_frames(eng, fam, [E - 1], 400)
    for k in range(n_pat):
        if fam == "ww":
            RE.non_finite_ww(eng.state, k, k, eng.n_pursuers)
        else:
            RE.non_finite_hw(eng.state, k, k, eng.n_good)
    ids = list(range(E))
    got = eng.render_frames(ids, screen_size=400)
    RE.assert_frames_equal(got, want_frames(eng, fam, ids, 400))
    RE.assert_frames_equal(got[E - 1:], before, "untouched env")


# ------------------------------------------------------------------------------------------ no contraction
def _place_points(eng, fam, xs, ys):
    """Pursuers / rescuers at (xs[i], ys[i]), one env per 32 of them; every other object off the frame."""
    st = eng.state
    Na = eng.n_pursuers if fam == "ww" else eng.n_good
    RE.put(st["pos_x"], -5.0)
    RE.put(st["pos_y"], -5.0)
    for i, (x, y) in enumerate(zip(xs, ys)):
        RE.put(st["pos_x"][i // Na, i % Na], x)
        RE.put(st["pos_y"][i // Na, i % Na], y)
    if fam == "ww":
        RE.put(st["obst_x"], -5.0)
    else:
        RE.put(st["key"], -5.0)
        RE.put(st["bomb"], -5.0)
        st["flags"][:] = 1


@pytest.mark.parametrize("fam", ["ww", "hw"])
def test_sensor_ends_not_contracted_float64(fam):
    """float64 positions whose sensor end pixel a fused multiply-add would move (found with exact rationals)."""
    S, K, rng = 800, 30, 0.2
    dirs = R.sensor_dirs(K)
    px = RE.fma_points_f64(S, rng, dirs[0], 64)
    py = RE.fma_points_f64(S, rng, dirs[1], 64, lo=130)
    assert len(px) == 64 and len(py) == 64
    E = 2
    kw = dict(n_sensors=K, sensor_range=rng, radius=0.005)
    eng = ww(E, torch.float64, n_pursuers=32, **kw) if fam == "ww" else hw(E, torch.float64, args=(32, 2, 2, 1, 1),
                                                                           **kw)
    _place_points(eng, fam, [p for _, p in px], [p for _, p in py])
    RE.assert_frames_equal(eng.render_frames([0, 1], screen_size=S), want_frames(eng, fam, [0, 1], S))


@pytest.mark.parametrize("fam", ["ww", "hw"])
def test_sensor_ends_not_contracted_float32(fam):
    """float32 positions with a sensor_range built so that a fused multiply-add would move a sensor end pixel:
    one engine per point."""
    S, K = 800, 30
    dirs = R.sensor_dirs(K)
    hits = [(0.4375001, h) for h in RE.fma_points_f32(S, 0.4375001, dirs[0], 4)] + \
           [(0.61, h) for h in RE.fma_points_f32(S, 0.61, dirs[0], 4)]
    assert len(hits) == 8
    for p, (j, r) in hits:
        kw = dict(n_sensors=K, sensor_range=r, radius=0.005)
        eng = ww(1, torch.float32, **kw) if fam == "ww" else hw(1, torch.float32, **kw)
        _place_points(eng, fam, [p], [0.5])
        RE.assert_frames_equal(eng.render_frames([0], screen_size=S), want_frames(eng, fam, [0], S), (p, j, r))


# ------------------------------------------------------------------------------------------ bounds and ids
@pytest.mark.parametrize("fam", ["ww", "hw"])
@pytest.mark.parametrize("S", [800, 37])
def test_sensor_range_bound(fam, S):
    """The largest sensor_range with |r| S < 2^29 draws the oracle's frame (lines towards +-2^29 px, untouched by
    the 2^30 clamp); the next double up, its negative, NaN and +-inf are refused by the Python layer and the C
    ABI alike."""
    top = RE.max_sensor_range(S)
    make = lambda r: ww(2, torch.float32, sensor_range=r) if fam == "ww" else hw(2, torch.float32, sensor_range=r)
    for r in (top, -top):
        eng = make(r)
        eng.reset()
        RE.put(eng.state["pos_x"][0], np.linspace(0.05, 0.95, eng.state["pos_x"].shape[1]))
        RE.assert_frames_equal(eng.render_frames([0, 1], screen_size=S), want_frames(eng, fam, [0, 1], S), r)
    L = _lib.lib()
    up = float(np.nextafter(top, np.inf))
    for r in (up, -up, float("nan"), float("inf"), -float("inf")):
        eng = make(r)
        with pytest.raises(ValueError):
            eng.render_frames([0], screen_size=S)
        ids = torch.zeros(1, dtype=torch.int32, device=eng.device)
        out = torch.empty((1, S, S, 3), dtype=torch.uint8, device=eng.device)
        dirs = torch.as_tensor(R.sensor_dirs(eng.cfg.n_sensors), device=eng.device)
        fn = L.madrl_ww_render if fam == "ww" else L.madrl_hostage_render
        assert fn(eng._h, 1, _lib._ptr(ids), S, _lib._ptr(dirs), _lib._ptr(out), None) == -1
        assert b"sensor_range" in L.madrl_last_error()


def test_radius_bound():
    """A radius of 2^29 pixels is refused; one below it is not."""
    L = _lib.lib()
    S = 1024
    ids = torch.zeros(1, dtype=torch.int32, device="cuda")
    out = torch.empty((1, S, S, 3), dtype=torch.uint8, device="cuda")
    for r, rc in ((float(1 << 19), -1), (float(np.nextafter(float(1 << 19), 0)), 0)):
        eng = ww(1, torch.float32, obstacle_radius=r)   # not reset: no spawn could clear such an obstacle
        RE.put(eng.state["obst_x"], -1e7)
        dirs = torch.as_tensor(R.sensor_dirs(eng.cfg.n_sensors), device=eng.device)
        assert L.madrl_ww_render(eng._h, 1, _lib._ptr(ids), S, _lib._ptr(dirs), _lib._ptr(out), None) == rc, r
    torch.cuda.synchronize()


@pytest.mark.parametrize("family", ["ww", "hw", "pe"])
def test_int64_ids_outside_the_range_draw_zero(family):
    """int64 CUDA ids are mapped before the int32 cast: 2^32 + 2 is not env 2, nor -2^32 + 1 env 1."""
    E = 4
    if family == "pe":
        eng = BatchedPursuitEvade(E, np.zeros((1, 6, 5), np.int32), n_evaders=2, n_pursuers=2, obs_range=3, seed=1)
        draw = lambda ids: eng.render_frames(ids, cell=5)
    else:
        eng = ww(E, torch.float32) if family == "ww" else hw(E, torch.float32)
        draw = lambda ids: eng.render_frames(ids, screen_size=64)
    eng.reset()
    good = draw([2, 1, 3])
    ids = torch.tensor([(1 << 32) + 2, -(1 << 32) + 1, 2, (1 << 31), -(1 << 31) - 1, (1 << 32) + 3, 1],
                       dtype=torch.int64, device=eng.device)
    got = draw(ids)
    torch.cuda.synchronize()
    for i in (0, 1, 3, 4, 5):
        assert int(got[i].max()) == 0, i
    assert torch.equal(got[2], good[0]) and torch.equal(got[6], good[1])
