"""Float32-exact scenes for Waterworld's and Hostage's rollout kernels (ww_kernel in csrc/waterworld.cu, hw_kernel in
csrc/hostage.cu), shared by tests/test_exact_ties_gpu.py (on the device) and tests/test_emulated_exact_ties.py (in
the warp emulator of tests/emu).

The float32 teacher-forced tests (tests/teacher_forced.py) skip every observation element whose comparisons lie
within 3e-7 of a threshold, exact ties included.  These scenes sit exactly there: objects that coincide with a
pursuer (projections of -0.0 and +0.0), objects at exactly the sensor range and the pursuer's radius off a ray,
argmin ties between objects of one class (across the 32-object chunk boundaries too, and -0.0 against +0.0),
collisions, obstacle rebounds and respawn draws at exactly the squared threshold and at the next float32-exact
sum of two squares above it, and pursuers landing exactly on a wall.  Each scene is a hand-placed pre-step state
on a coarse dyadic grid, stepped once with zero actions and a sensor table of few-bit vectors (`SENSORS`, sensor 0 =
(1, 0)) that the tests write into the engine and hand to the float64 oracle widened.  `validate_*` recomputes every
quantity the oracle compares, in exact rational arithmetic, and asserts that each one is exact in float32 (then
no rounding and no FMA contraction can move it), or -- for the quantities of objects far from the decision, and
of respawn draws -- that it lies farther from its threshold than float32 rounding could move it.  On such a state
the kernel must decide every comparison as the reference does, so the tests compare everything bit for bit.

`build_ww(scene, n_obj, K, env_id)` / `build_hw(...)` pad a scene with parked objects (outside the unit square,
still, out of every range) up to the object count of the instantiation under test, place a scene's tie pair
across a chunk boundary when the padding makes one, and return the engine state and the oracle for that env."""
from fractions import Fraction as Fr

import numpy as np

from oracle.hostage_oracle import HostageOracle
from oracle.philox import Stream
from oracle.waterworld_oracle import WaterworldOracle
from ww_writer_edges import STAGE_MAX_FLOATS

SEED = 23
F32 = np.float32
D6 = 2.0 ** -6
# few-bit sensor vectors: sensor 0 = (1, 0); the ones with both components negative project a coincident object
# (relative position (+0, +0)) to -0.0, the others to +0.0.  The table is cycled up to K sensors.
SENSORS = np.array([[1, 0], [0, 1], [-1, 0], [0, -1], [-0.5, -0.75], [0.75, -0.5], [-0.75, 0.5], [0.5, 0.75],
                    [-1, -0.25], [0.75, 0.5], [-0.25, -1], [1, 0.25]], np.float64)


def sensor_table(K):
    """[K, 2] float32: SENSORS cycled."""
    return SENSORS[np.arange(K) % len(SENSORS)].astype(F32)


def f32(x):
    return np.asarray(x, np.float64).astype(F32)


def up(x, n=1):
    for _ in range(n):
        x = np.nextafter(F32(x), F32(np.inf))
    return float(x)


def dn(x, n=1):
    for _ in range(n):
        x = np.nextafter(F32(x), F32(-np.inf))
    return float(x)


def exact(v):
    """Whether the rational v is a float32 value."""
    return Fr(float(F32(float(v)))) == v


def next_sum_of_squares_above(t, grid=2.0 ** -16, span=64):
    """(dx, dy) on `grid` with dx^2 + dy^2 the smallest float32-exact sum of two float32-exact squares above t
    (a float32), dx nearest sqrt(t)."""
    best = None
    x0 = int(round(np.sqrt(t) / grid))
    for a in range(x0 - span, x0 + span):
        for b in range(0, span):
            dx, dy = a * grid, b * grid
            s = Fr(dx) ** 2 + Fr(dy) ** 2
            if s > Fr(float(t)) and exact(Fr(dx) ** 2) and exact(Fr(dy) ** 2) and exact(s):
                if best is None or s < best[0]:
                    best = (s, dx, dy)
    assert best is not None, t
    return best[1], best[2]


# ------------------------------------------------------------------------------------------------ Waterworld
# dyadic constants: radius r_p = 2^-6 (evaders 2r, poisons 3r/4), range 1/4, obstacle radius 1/8
WW_CFG = dict(n_pursuers=8, radius=D6, sensor_range=0.25, obstacle_radius=0.125, n_coop=2, ev_speed=2.0 ** -7,
              poison_speed=2.0 ** -7, action_scale=2.0 ** -7, poison_reward=-1.0, food_reward=1.0,
              encounter_reward=0.0625, control_penalty=-0.5, reward_mech="local")
# the product's defaults where they are thresholds (range 0.2, radius 0.015, obstacle radius 0.2): rounded to
# float32 they lie on one side of the double threshold, which an operand equal to the float32 value exposes
WW_DEFAULT = dict(WW_CFG, radius=0.015, sensor_range=0.2, obstacle_radius=0.2)
# radii a hair below the dyadic ones: every threshold then lies just below a float32-exact value (the dyadic
# distance, or its square), which rounds to that value.  A float32 operand equal to it must get the reference's
# verdict (beyond), which rounding the threshold to nearest, or searching the squared collision thresholds with a
# float32 sqrt against the rounded radius, turns into "within".
EPS_R, EPS_O = 2.0 ** -58, 2.0 ** -50
WW_ROUNDED = dict(WW_CFG, radius=D6 - EPS_R, obstacle_radius=0.125 - EPS_O)


def sq_thresholds(R):
    """(the largest float32 t with the double sqrt(t) <= R, the same with a float32 sqrt against float32(R)):
    what the squared collision thresholds are, and what a float32 search would make them."""
    t = F32(R * R)
    while np.sqrt(np.float64(t)) <= R:
        t = np.nextafter(t, F32(np.inf))
    while np.sqrt(np.float64(t)) > R:
        t = np.nextafter(t, F32(-np.inf))
    r, u = F32(R), F32(R * R)
    while np.sqrt(u) <= r:
        u = np.nextafter(u, F32(np.inf))
    while np.sqrt(u) > r:
        u = np.nextafter(u, F32(-np.inf))
    return float(t), float(u)


def in_window(R, R0):
    """R0 (dyadic) is just beyond the radius R in double, but a float32 search would count R0^2 within."""
    new, old = sq_thresholds(R)
    return R < R0 and new < R0 * R0 <= old


# r_p off the ray exactly, and the nearest offsets either side whose squares stay exact next to (1/16)^2
RAY = (("ray_exact", D6), ("ray_above", D6 + 2.0 ** -15), ("ray_below", D6 - 2.0 ** -15))
WW_NP2 = dict(WW_CFG, n_pursuers=2)
PARK = [(0.0625 + 0.125 * i, 0.9375) for i in range(8)]    # pursuers a scene does not use: a row along the top


class WWScene(object):
    """px/pv [Np, 2], ex/ev, ox/ov lists of (x, y, vx, vy), obst (x, y); `tie`: ("ev" | "po", B) puts the scene's
    first two objects of that class at object indices B - 1 and B when the padded count reaches past B;
    `counter(env_id) -> (counter, obst)`: a Philox counter and obstacle placed on the draws (respawn scenes)."""

    def __init__(self, name, cfg, pursuers, ev=(), po=(), obst=(0.5, 0.5), tie=None, counter=None):
        self.name, self.cfg, self.tie, self.counter = name, cfg, tie, counter
        p = list(pursuers) + [(x, y, 0.0, 0.0) for x, y in PARK[len(pursuers):cfg["n_pursuers"]]]
        assert len(p) == cfg["n_pursuers"], name
        self.p, self.ev, self.po, self.obst = np.array(p, float), list(ev), list(po), obst

    def __repr__(self):
        return self.name


def ww_r(cfg):
    r = cfg["radius"]
    return r, 2 * r, r * 3 / 4


def _sq_pair(R, above):
    """(dx, dy) with dx^2 + dy^2 = R^2 exactly (above = False; R dyadic) or the next exact sum above it."""
    return next_sum_of_squares_above(F32(R * R)) if above else (R, 0.0)


def _ww_scenes():
    c, r = WW_CFG, D6
    S = []
    # -- coincidences: two pursuers pushed into each corner (clipped, velocity zeroed), both at (+-0, +-0) of the
    #    other; a pursuer on an evader, on a poison, on the obstacle centre.  The evader and the poison carry
    #    velocities so that the speed features say which object a sensor took.
    v = 2.0 ** -7
    S.append(WWScene("corners", c, [(0, 0, -v, -v), (0, 0, -v, 0), (1, 0, v, -v), (1, 0, 0, -v),
                                    (0, 1, -v, v), (0, 1, -v, 0), (1, 1, v, v), (1, 1, v, 0)]))
    S.append(WWScene("on_objects", c, [(0.25, 0.25, 0, 0), (0.75, 0.25, 0, 0), (0.5 - 2 * v, 0.5, 2 * v, 0)],
                     ev=[(0.25, 0.25, v, -v)], po=[(0.75, 0.25, -v, v)]))
    # -- range: an object at exactly the range along sensor 0 and the nearest float32 positions either side of
    #    it, for a dyadic range and for the default 0.2 (float32(0.2) > 0.2: the reference does not sense it)
    for cfg, nm in ((c, "range_dyadic"), (WW_DEFAULT, "range_default")):
        rng = cfg["sensor_range"]
        rows = (0.125, 0.5, 0.875)
        xs = (float(F32(rng)), up(rng), dn(rng))
        S.append(WWScene(nm, cfg, [(0, y, 0, 0) for y in rows],
                         ev=[(x, y, 0, v) for x, y in zip(xs, rows)], po=[(xs[0], 0.3125, 0, v)]))
    # -- the ray: an object exactly r_p off sensor 0's ray, and at the nearest float32-exact squares either side
    #    (1/16 along the ray keeps |rel|^2 exact)
    for nm, dy in RAY:
        S.append(WWScene(nm, c, [(0.25, 0.25, 0, 0), (0.25, 0.75, 0, 0)],
                         ev=[(0.3125, 0.25 + dy, v, 0)], po=[(0.3125, 0.75 - dy, 0, -v)]))
    # -- argmin ties of equal sv: the lower index must win (its velocity shows in the speed feature); +0 vs -0
    d = 2.0 ** -8
    S.append(WWScene("tie_chunk0", c, [(0.25, 0.5, 0, 0), (0.6875, 0.5, 0, 0), (0.625, 0.125, 0, 0),
                                       (0.625 + 0.125, 0.125 + d, 0, 0), (0.625 + 0.125, 0.125 - d, 0, 0)],
                     ev=[(0.375, 0.5 + d, v, 0), (0.375, 0.5 - d, -v, 0)],
                     po=[(0.8125, 0.5 - d, 0, v), (0.8125, 0.5 + d, 0, -v)]))
    # pursuer 0 sits on evader 0 (sv = -0.0 on the negative sensors) with evader 1 at sv = +0.0 on sensor
    # (-0.5, -0.75); pursuer 1 has the +0.0 one first and the coincident one second
    zx, zy = 0.75 * d, -0.5 * d
    S.append(WWScene("tie_signed_zero", c, [(0.25, 0.25, 0, 0), (0.75, 0.75, 0, 0)],
                     ev=[(0.25, 0.25, v, 0), (0.25 + zx, 0.25 + zy, -v, v), (0.75 + zx, 0.75 + zy, 0, v),
                         (0.75, 0.75, v, -v)]))
    for cls in ("ev", "po"):
        for B in (32, 64, 128):
            objs = [(0.375, 0.5 + d, v, 0), (0.375, 0.5 - d, -v, 0)]
            S.append(WWScene("tie_%s_b%d" % (cls, B), c, [(0.25, 0.5, 0, 0)], tie=(cls, B),
                             **{cls: objs, ("po" if cls == "ev" else "ev"): []}))
    # -- collisions at d2 = R^2 (a hit) and at the next exact sum of squares above (no hit).  Evader 0: two
    #    pursuers at R (caught with n_coop = 2); evader 1: one at R, one just beyond (touched, not caught);
    #    poison 0 at R_po (caught), poison 1 just beyond.
    rp, re, rpo = ww_r(c)
    ax, ay = _sq_pair(rp + re, True)
    bx, by = _sq_pair(rp + rpo, True)
    S.append(WWScene("collide", c, [(0.25 - (rp + re), 0.25, 0, 0), (0.25, 0.25 + (rp + re), 0, 0),
                                    (0.75 - (rp + re), 0.25, 0, 0), (0.75 + ax, 0.25 + ay, 0, 0),
                                    (0.25, 0.75 - (rp + rpo), 0, 0), (0.75 - bx, 0.75 - by, 0, 0)],
                     ev=[(0.25, 0.25, v, 0), (0.75, 0.25, 0, v)], po=[(0.25, 0.75, 0, -v), (0.75, 0.75, -v, 0)]))
    # -- obstacle rebound at d2 = (r + R_obst)^2 (rebounds) and just beyond (does not), per class
    Ro = c["obstacle_radius"]
    pr, er, orr = rp + Ro, re + Ro, rpo + Ro
    qx, qy = _sq_pair(pr, True)
    S.append(WWScene("rebound", c, [(0.5 - pr - v, 0.5, v, 0), (0.5 + qx, 0.5 + qy + v, 0, -v)],
                     ev=[(0.5, 0.5 + er, v, v), (0.5 + _sq_pair(er, True)[1], 0.5 - _sq_pair(er, True)[0], -v, v)],
                     po=[(0.5 + orr, 0.5, v, -v), (0.5 - _sq_pair(orr, True)[0], 0.5 - _sq_pair(orr, True)[1], v, v)]))
    # -- the respawn rejection loop: a caught evader's first draw lands at exactly 2 r_e + R_obst from the obstacle
    #    (rejected: `<=`), or at the next exact sum of squares beyond it (accepted)
    for nm, above in (("respawn_on", False), ("respawn_above", True)):
        S.append(WWScene(nm, c, [(0.25 - (rp + re), 0.0625, 0, 0), (0.25 + (rp + re), 0.0625, 0, 0)],
                         ev=[(0.25, 0.0625, 0, 0)], counter=_respawn_counter(2 * re + Ro, above)))
    # -- the same thresholds a hair below the dyadic distances (WW_ROUNDED): objects at exactly the dyadic catch,
    #    rebound and respawn distances and r_p off a ray are beyond them in the reference
    q = WW_ROUNDED
    qp, qe, qpo = ww_r(q)
    Rc, Rpc = 3 * r, 1.75 * r
    Rrp, Rre, Rrpo, Rsp = r + 0.125, 2 * r + 0.125, 0.75 * r + 0.125, 4 * r + 0.125
    for R, R0 in ((qp + qe, Rc), (qp + qpo, Rpc), (qp + q["obstacle_radius"], Rrp), (qe + q["obstacle_radius"], Rre),
                  (qpo + q["obstacle_radius"], Rrpo), (2 * qe + q["obstacle_radius"], Rsp)):
        assert in_window(R, R0), (R, R0)
    S.append(WWScene("collide_rounded", q, [(0.25 - Rc, 0.25, 0, 0), (0.25, 0.25 + Rc, 0, 0), (0.75 - Rpc, 0.25, 0, 0)],
                     ev=[(0.25, 0.25, v, 0)], po=[(0.75, 0.25, 0, v)]))
    S.append(WWScene("rebound_rounded", q, [(0.5 - Rrp - v, 0.5, v, 0)],
                     ev=[(0.5, 0.5 + Rre, v, v)], po=[(0.5 + Rrpo, 0.5, v, -v)]))
    S.append(WWScene("respawn_rounded", q, [(0.25 - 2.5 * r, 0.0625, 0, 0), (0.25 + 2.5 * r, 0.0625, 0, 0)],
                     ev=[(0.25, 0.0625, 0, 0)], counter=_respawn_counter(Rsp, False)))
    S.append(WWScene("ray_rounded", q, [(0.25, 0.25, 0, 0), (0.25, 0.75, 0, 0)],
                     ev=[(0.3125, 0.25 + r, v, 0)], po=[(0.3125, 0.75 - r, 0, -v)]))
    # -- two pursuers (the writer-warp kernel stages a whole env-step of them at every sensor layout): both in a
    #    corner, an evader and a poison on them and one of each at sv = +0.0 on sensor (-0.5, -0.75), in both orders
    S.append(WWScene("np2_corner_ties", WW_NP2, [(1, 1, v, v), (1, 1, 0, v)],
                     ev=[(1, 1, -v, 0), (1 - zx, 1 - zy, 0, -v)], po=[(1 - zx, 1 - zy, v, 0), (1, 1, 0, v)]))
    S.append(WWScene("np2_range_ray", dict(WW_DEFAULT, n_pursuers=2), [(0, 0.125, 0, 0), (0.25, 0.75, 0, 0)],
                     ev=[(float(F32(0.2)), 0.125, 0, v), (dn(0.2), 0.125 + 2 * d, 0, -v)],
                     po=[(0.3125, 0.75 - r, 0, -v)]))
    # -- walls: pursuers landing exactly on 0 and 1 keep their velocity; an evader and a poison end a step with one
    #    coordinate exactly on a wall and the other outside (no bounce)
    S.append(WWScene("walls", c, [(v, 0.5, -v, 0), (1 - v, 0.25, v, v), (0.5, v, 0, -v), (0.25, 1 - 2 * v, v, 2 * v)],
                     ev=[(v, -2 * v, -v, -v), (1 + v, 1 - v, v, v)], po=[(-v, 1 + v, v, v), (1 - v, 2 * v, v, -2 * v)]))
    return S


def _respawn_counter(R, above):
    """counter(env_id) -> (counter, obstacle): the obstacle placed R (dyadic) left of the first draw pair of the
    env's stream at `counter`, or R left and the next exact square sum beyond (`above`)."""
    def f(env_id, counter=4000):
        st = Stream(SEED, env_id, counter=counter)
        x0, y0 = st.rand(2)
        dx, dy = _sq_pair(R, above)
        return counter, (x0 - dx, y0 - dy)
    return f


WW_SCENES = _ww_scenes()


def build_ww(scene, n_obj, K, env_id):
    """-> (cfg for the engine and oracle, state dict as Batched*.state names it (float64 values), oracle pre-state)."""
    cfg = dict(scene.cfg)
    Np = cfg["n_pursuers"]
    ev, po = list(scene.ev), list(scene.po)
    pads = n_obj - Np - len(ev) - len(po)
    assert pads >= 2, (scene, n_obj)
    pre_e = pre_p = 0
    if scene.tie is not None:
        cls, B = scene.tie
        B = max([b for b in (32, 64, 128) if b <= B and b < n_obj - 1] or [0])
        if B:
            if cls == "ev":
                pre_e = B - 1 - Np
            else:
                pre_e, pre_p = 1, B - 1 - Np - 1 - len(ev)
    park = lambda i: (3.0 + 0.0625 * i, 0.5, 0.0, 0.0)   # outside the square, still, x out of every range
    if not ev:
        pre_e = max(pre_e, 1)
    post_p = pads - pre_e - pre_p
    assert post_p >= (0 if po else 1), (scene, n_obj)
    k = iter(range(1000))
    ev = [park(next(k)) for _ in range(pre_e)] + ev
    po = [park(next(k)) for _ in range(pre_p)] + po + [park(next(k)) for _ in range(post_p)]
    cfg.update(n_evaders=len(ev), n_poison=len(po), n_sensors=K)
    P = np.array([tuple(p) for p in scene.p] + ev + po, float)
    counter, obst = 0, scene.obst
    if scene.counter is not None:
        counter, obst = scene.counter(env_id)
    state = dict(pos_x=P[:, 0], pos_y=P[:, 1], vel_x=P[:, 2], vel_y=P[:, 3], obst_x=obst[0], obst_y=obst[1],
                 timestep=0, rng_counter=counter)
    Ne = len(ev)
    pre = dict(px=P[:Np, :2], pv=P[:Np, 2:], ex=P[Np:Np + Ne, :2], ev=P[Np:Np + Ne, 2:], ox=P[Np + Ne:, :2],
               ov=P[Np + Ne:, 2:], obst=np.array([obst], float), t=0, counter=counter)
    return cfg, state, pre


class TermwiseTable(np.ndarray):
    """A sensor table whose `dot` sums the two products term by term, sx * x + sy * y, as the kernels do.  The
    values are the reference's (every quantity here is exact); only a zero's sign can differ: NumPy's dot sums
    from +0.0, so where both products are -0.0 (an object exactly at the pursuer, or a relative velocity of
    zero, on a sensor with no positive component) the reference has +0.0 and the term-by-term sum -0.0."""

    def dot(self, b):
        a = np.asarray(self)
        return a[:, 0:1] * b[0:1] + a[:, 1:2] * b[1:2]


def termwise(S):
    return np.asarray(S, np.float64).view(TermwiseTable)


def ww_oracle(cfg, pre, env_id):
    o = WaterworldOracle(rng=Stream(SEED, env_id, counter=pre["counter"]),
                         **{k: v for k, v in cfg.items() if k != "n_envs"})
    o.S = termwise(sensor_table(cfg["n_sensors"]))
    o.set_state(pre)
    return o


# ------------------------------------------------------------------------------------------------ exactness
MARGIN = 2.0 ** -16   # float32 rounding of these sums of products of values below 4 moves them far less


class Inexact(AssertionError):
    pass


def _need(v, what):
    if not exact(v):
        raise Inexact("%s = %r is not exact in float32" % (what, float(v)))


def _need_or_far(parts, v, thr, what):
    """v (rational, computed from `parts`) against thr: every part exact in float32, or v farther from thr than
    float32 rounding can move it."""
    if abs(float(v) - float(thr)) > MARGIN:
        return
    for x in parts + [v]:
        _need(x, what)


def _fr(x):
    return Fr(float(x))


def _check_sense(S, me, mv, objs, vel, rng, r2, what, lim):
    """Every sensor's sv and ray distance of every object within `lim` of `me` (per coordinate), and (vel) the
    relative speed."""
    for j, o in enumerate(objs):
        if max(abs(float(o[0]) - float(me[0])), abs(float(o[1]) - float(me[1]))) > lim:
            continue
        rx, ry = _fr(o[0]) - _fr(me[0]), _fr(o[1]) - _fr(me[1])
        _need(rx, what + " rel x")
        _need(ry, what + " rel y")
        for sx, sy in S:
            sx, sy = _fr(sx), _fr(sy)
            sv = sx * rx + sy * ry
            q = rx * rx + ry * ry - sv * sv
            if sv < -MARGIN or sv > Fr(rng) + MARGIN or q > Fr(r2) + MARGIN:
                continue        # rejected whatever the rounding
            for x in (sx * rx, sy * ry, sv):
                _need(x, what + " sv")
            _need_or_far([rx * rx, ry * ry, rx * rx + ry * ry, sv * sv], q, r2, what + " |rel|^2 - sv^2")
            if vel is not None:
                wx, wy = _fr(vel[j][0]) - _fr(mv[0]), _fr(vel[j][1]) - _fr(mv[1])
                for x in (wx, wy, sx * wx, sy * wy, sx * wx + sy * wy):
                    _need(x, what + " relative speed")


def _check_d2(a, b, R, what):
    dx, dy = _fr(a[0]) - _fr(b[0]), _fr(a[1]) - _fr(b[1])
    _need_or_far([dx, dy, dx * dx, dy * dy], dx * dx + dy * dy, Fr(R) ** 2, what + " d2")


def _moved(x, v, what, lo=0.0):
    for a in range(2):
        _need(_fr(x[a]) + _fr(v[a]), what + " moved")
    return np.clip(np.asarray(x, float) + v, lo, 1)


def validate_ww(cfg, pre, S, env_id):
    """Raises Inexact unless every quantity the oracle compares in this step is exact in float32 (or, for a
    quantity far from its threshold, decisively on one side of it)."""
    S = S[:min(len(S), len(SENSORS))]
    rp, re, rpo = ww_r(cfg)
    Ro, rng = cfg["obstacle_radius"], cfg["sensor_range"]
    obst = pre["obst"][0]
    px = [_moved(x, v, "pursuer %d" % i) for i, (x, v) in enumerate(zip(pre["px"], pre["pv"]))]
    lim = rng + rp + MARGIN
    for i, me in enumerate(px):
        mv = pre["pv"][i]
        _check_sense(S, me, mv, [obst], None, rng, rp * rp, "obstacle", lim)
        for nm, X, V in (("evader", pre["ex"], pre["ev"]), ("poison", pre["ox"], pre["ov"]), ("pursuer", px, pre["pv"])):
            _check_sense(S, me, mv, X, V, rng, rp * rp, nm, lim)
        for X, R, nm in ((pre["ex"], rp + re, "catch"), (pre["ox"], rp + rpo, "poison catch")):
            for x in X:
                _check_d2(me, x, R, nm)
        _check_d2(me, obst, rp + Ro, "pursuer rebound")
    for X, V, R, nm in ((pre["ex"], pre["ev"], re + Ro, "evader"), (pre["ox"], pre["ov"], rpo + Ro, "poison")):
        for x, v in zip(X, V):
            _check_d2(x, obst, R, nm + " rebound")
            _moved(x, v, nm, -np.inf)
    # the respawn draws (24-bit uniforms, as pairs) against the obstacle's keep-out discs
    o = ww_oracle(cfg, pre, env_id)
    o.step(np.zeros((cfg["n_pursuers"], 2)))
    st = Stream(SEED, env_id, counter=pre["counter"])
    while st.counter < o.np_random.counter:
        x = st.rand(2)
        for R in (2 * re + Ro, 2 * rpo + Ro):
            _check_d2(x, obst, R, "respawn draw")


# ------------------------------------------------------------------------------------------------ Hostage
# dyadic constants: radius r = 2^-6 (hostages 2r), range 1/4, bomb radius 1/16, key radius 1/32
HW_CFG = dict(radius=D6, sensor_range=0.25, bad_speed=2.0 ** -7, action_scale=2.0 ** -7, save_reward=4.0,
              hit_reward=-1.0, encounter_reward=0.0625, not_saved_reward=-2, bomb_reward=-4.0, bomb_radius=0.0625,
              key_radius=0.03125, control_penalty=-0.125, reward_mech="local", key_loc=np.array([[0.875, 0.0625]]))
HW_DEFAULT = dict(HW_CFG, radius=0.015, sensor_range=0.2)
HW_NR = 6
HW_ROUNDED = dict(HW_CFG, radius=D6 - EPS_R, bomb_radius=0.0625 - EPS_O, key_radius=0.03125 - EPS_O)
HPARK = [(0.0625 + 0.1875 * i, 0.9375) for i in range(HW_NR)]


class HWScene(object):
    """r: rescuers (x, y, vx, vy); c: criminals (x, y, vx, vy); h: hostages (x, y); key, bomb (x, y);
    gate: whether the gate is open before the step; `tie`: ("c", B) as WWScene's."""

    def __init__(self, name, cfg, rescuers, c=(), h=(), key=(0.875, 0.0625), bomb=(0.0625, 0.0625), gate=True,
                 tie=None, n_coop_save=2):
        self.name, self.cfg, self.tie, self.gate, self.key, self.bomb = name, cfg, tie, gate, key, bomb
        self.n_coop_save = n_coop_save
        r = list(rescuers) + [(x, y, 0.0, 0.0) for x, y in HPARK[len(rescuers):]]
        assert len(r) == HW_NR, name
        self.r, self.c, self.h = np.array(r, float), list(c), list(h)

    def __repr__(self):
        return self.name


def _hw_scenes():
    c, r, v, d = HW_CFG, D6, 2.0 ** -7, 2.0 ** -8
    S = []
    # a rescuer on a criminal (hit, respawn), on a hostage (saved with n_coop_save = 1), on the bomb, on the key
    S.append(HWScene("on_objects", dict(c), [(0.25, 0.25, 0, 0), (0.5, 0.25, 0, 0), (0.25, 0.5, 0, 0)],
                     c=[(0.25, 0.25, v, 0)], h=[(0.5, 0.25)], bomb=(0.25, 0.5), n_coop_save=1))
    S.append(HWScene("on_key", dict(c), [(0.625, 0.625, 0, 0), (0.875, 0.875, 0, 0)], c=[(0.625, 0.625, 0, v)],
                     key=(0.875, 0.875), gate=False))
    for cfg, nm in ((c, "range_dyadic"), (HW_DEFAULT, "range_default")):
        rng = cfg["sensor_range"]
        rows = (0.125, 0.5, 0.875)
        xs = (float(F32(rng)), up(rng), dn(rng))
        S.append(HWScene(nm, cfg, [(0, y, 0, 0) for y in rows], c=[(x, y, 0, v) for x, y in zip(xs, rows)],
                         h=[(xs[0], 0.3125)], bomb=(0.5, 0.625)))
    for nm, dy in RAY:
        S.append(HWScene(nm, dict(c), [(0.25, 0.25, 0, 0), (0.25, 0.75, 0, 0)], c=[(0.3125, 0.25 + dy, v, 0)],
                         h=[(0.3125, 0.75 - dy)]))
    S.append(HWScene("tie_chunk0", dict(c), [(0.25, 0.5, 0, 0)], c=[(0.375, 0.5 + d, v, 0), (0.375, 0.5 - d, -v, 0)],
                     h=[(0.375, 0.25 + d), (0.375, 0.25 - d)]))
    for B in (32, 64, 128):
        S.append(HWScene("tie_c_b%d" % B, dict(c), [(0.25, 0.5, 0, 0)], tie=("c", B),
                         c=[(0.375, 0.5 + d, v, 0), (0.375, 0.5 - d, -v, 0)]))
    # a criminal at exactly 2r (hit) and at the next exact square sum beyond; a hostage at exactly 3r with two
    # rescuers (saved, n_coop_save = 2) and one at 3r with the second rescuer just beyond; the bomb just beyond
    cx, cy = _sq_pair(2 * r, True)
    hx, hy = _sq_pair(3 * r, True)
    bx, by = _sq_pair(r + c["bomb_radius"], True)
    S.append(HWScene("collide", dict(c), [(0.25 - 2 * r, 0.25, 0, 0), (0.75 - cx, 0.25 - cy, 0, 0),
                                          (0.25, 0.625 - 3 * r, 0, 0), (0.25, 0.625 + 3 * r, 0, 0),
                                          (0.75 - 3 * r, 0.625, 0, 0), (0.75 + hx, 0.625 + hy, 0, 0)],
                     c=[(0.25, 0.25, v, 0), (0.75, 0.25, 0, v)], h=[(0.25, 0.625), (0.75, 0.625)],
                     bomb=(0.0625 + 0.0, 0.0625)))
    S.append(HWScene("collide_bomb", dict(c), [(0.5 + bx, 0.125 + by, 0, 0)], c=[(0.875, 0.875, 0, 0)],
                     bomb=(0.5, 0.125)))
    # the thresholds a hair below the dyadic distances: a criminal at exactly 2r, a hostage at exactly 3r from both
    # rescuers, the bomb at exactly r + bomb radius, an object exactly r off a ray, all beyond in the reference
    q = HW_ROUNDED
    qr = q["radius"]
    for R, R0 in ((qr + qr, 2 * r), (qr + qr * 2, 3 * r), (qr + q["bomb_radius"], r + 0.0625),
                  (qr + q["key_radius"], r + 0.03125)):
        assert in_window(R, R0), (R, R0)
    S.append(HWScene("collide_rounded", q, [(0.25 - 2 * r, 0.25, 0, 0), (0.25, 0.625 - 3 * r, 0, 0),
                                            (0.25, 0.625 + 3 * r, 0, 0), (0.75 - r - 0.0625, 0.5, 0, 0),
                                            (0.3125 - 0.0625, 0.875 - r, 0, 0)],
                     c=[(0.25, 0.25, v, 0), (0.3125, 0.875, 0, v)], h=[(0.25, 0.625)], bomb=(0.75, 0.5)))
    S.append(HWScene("key_rounded", q, [(0.75, 0.75, 0, 0), (0.875, 0.625, 0, 0)], c=[(0.875, 0.625 + 0.125, v, 0)],
                     key=(0.75 + r + 0.03125, 0.75), gate=False))
    S.append(HWScene("walls", dict(c), [(v, 0.5, -v, 0), (1 - v, 0.25, v, v), (0.5, v, 0, -v)],
                     c=[(v, -2 * v, -v, -v), (1 + v, 1 - v, v, v)]))
    return S


HW_SCENES = _hw_scenes()


def build_hw(scene, n_obj, K, env_id):
    """-> (args, kw, state dict as BatchedHostageWorld.state names it, oracle pre-state); n_obj counts the
    criminals and hostages."""
    cr, ho = list(scene.c), list(scene.h)
    pads = n_obj - len(cr) - len(ho)
    assert pads >= 2, (scene, n_obj)
    pre_c = 0
    if scene.tie is not None:
        B = max([b for b in (32, 64, 128) if b <= scene.tie[1] and b < n_obj - 1] or [0])
        pre_c = B - 1 if B else 0
    park = lambda i: (3.0 + 0.0625 * i, 0.5)
    k = iter(range(1000))
    if not cr:
        pre_c = max(pre_c, 1)
    cr = [park(next(k)) + (0.0, 0.0) for _ in range(pre_c)] + cr
    ho = ho + [park(next(k)) for _ in range(pads - pre_c)]
    Nc, Nh = len(cr), len(ho)
    args = (HW_NR, Nh, Nc, scene.n_coop_save, 1)
    kw = dict(scene.cfg, n_sensors=K, key_loc=np.array([scene.key], float))
    R, C, H = scene.r, np.array(cr, float), np.array(ho, float)
    pos = np.concatenate([R[:, :2], C[:, :2], H])
    vel = np.concatenate([R[:, 2:], C[:, 2:], np.zeros_like(H)])
    flags = 4 | (1 if scene.gate else 0)
    state = dict(pos_x=pos[:, 0], pos_y=pos[:, 1], vel_x=vel[:, 0], vel_y=vel[:, 1], key=np.array(scene.key, float),
                 bomb=np.array(scene.bomb, float), saved=np.zeros(Nh, np.uint8), flags=flags, timestep=0,
                 rng_counter=0)
    pre = dict(rx=R[:, :2], rv=R[:, 2:], cx=C[:, :2], cv=C[:, 2:], hx=H, bomb=np.array([scene.bomb], float),
               key=np.array([scene.key], float), saved=np.zeros(Nh, bool), gate_open=scene.gate, bombed=False, t=0,
               counter=0)
    return args, kw, state, pre


def hw_oracle(args, kw, pre, env_id):
    o = HostageOracle(*args, rng=Stream(SEED, env_id, counter=pre["counter"]), **kw)
    o.S = termwise(sensor_table(kw["n_sensors"]))
    o.set_state(pre)
    return o


def validate_hw(args, kw, pre, S):
    S = S[:min(len(S), len(SENSORS))]
    r, rng = kw["radius"], kw["sensor_range"]
    lo = 0.0 if pre["gate_open"] else 0.5 + r      # a closed gate clips the rescuers to [0.5 + r, 1]
    rx = [_moved(x, v, "rescuer %d" % i, lo) for i, (x, v) in enumerate(zip(pre["rx"], pre["rv"]))]
    lim = rng + r + MARGIN
    for i, me in enumerate(rx):
        mv = pre["rv"][i]
        for nm, X, V in (("criminal", pre["cx"], pre["cv"]), ("hostage", pre["hx"], None), ("key", pre["key"], None),
                         ("bomb", pre["bomb"], None)):
            _check_sense(S, me, mv, X, V, rng, r * r, nm, lim)
        for X, R, nm in ((pre["cx"], 2 * r, "hit"), (pre["hx"], 3 * r, "save"),
                         (pre["bomb"], r + kw["bomb_radius"], "bomb"), (pre["key"], r + kw["key_radius"], "key")):
            for x in X:
                _check_d2(me, x, R, nm)
    for x, v in zip(pre["cx"], pre["cv"]):
        _moved(x, v, "criminal", -np.inf)


# ------------------------------------------------------------------------------------------------ expectations
# the instantiation layouts: OPL -> objects (Waterworld: all; Hostage: criminals + hostages), (KCH, KC) -> K
WW_N = {1: 32, 2: 64, 4: 128, 8: 256}
HW_N = {1: 32, 2: 64, 4: 128, 8: 250}
K_OF = {(1, 30): 30, (1, 0): 19, (2, 0): 64}


def writer_runs(scene, opl, K):
    """Whether set_obs_writer(ON) takes the writer-warp kernel for `scene`: at most 32 objects and a whole env-step
    of float32 rows staged (8 pursuers only at K = 19, 2 pursuers at every K), with ww_envs envs."""
    return opl == 1 and scene.cfg["n_pursuers"] * (7 * K + 3) <= STAGE_MAX_FLOATS


def ww_envs(scene, K):
    """Envs of the Waterworld engine a scene runs in: the fewest that make the observation step stride E Np D a
    multiple of 16 bytes, which the writer-warp kernel needs.  Env 0 is the scene; the others are copies of it,
    with their own Philox streams, and are not checked."""
    E = 1
    while E * scene.cfg["n_pursuers"] * (7 * K + 3) % 4:
        E += 1
    return E
ENV = 0           # every scene runs as env 0 of its engine
_valid = set()


def ww_expect(scene, n_obj, K):
    """-> (engine cfg, state to write, expected dict) for `scene` padded to n_obj objects and K sensors."""
    cfg, state, pre = build_ww(scene, n_obj, K, ENV)
    if scene.name not in _valid:
        validate_ww(cfg, pre, sensor_table(K), ENV)
        _valid.add(scene.name)
    o = ww_oracle(cfg, pre, ENV)
    obs, rew, done, info = o.step(np.zeros((cfg["n_pursuers"], 2)))
    ref = ww_oracle(cfg, pre, ENV)
    ref.S = np.asarray(ref.S)
    assert np.array_equal(np.array(ref.step(np.zeros((cfg["n_pursuers"], 2)))[0]), np.array(obs)), scene
    pos = np.concatenate([o.px, o.ex, o.ox])
    vel = np.concatenate([o.pv, o.ev, o.ov])
    return cfg, state, dict(obs=np.array(obs), rew=np.asarray(rew, float), done=bool(done),
                            info=[info["evcatches"], info["pocatches"]], pos=pos, vel=vel,
                            counter=o.np_random.counter, S=sensor_table(K))


def hw_expect(scene, n_obj, K):
    args, kw, state, pre = build_hw(scene, n_obj, K, ENV)
    if scene.name not in _valid:
        validate_hw(args, kw, pre, sensor_table(K))
        _valid.add(scene.name)
    o = hw_oracle(args, kw, pre, ENV)
    obs, rew, done, info = o.step(np.zeros((args[0], 2)))
    ref = hw_oracle(args, kw, pre, ENV)
    ref.S = np.asarray(ref.S)
    assert np.array_equal(np.array(ref.step(np.zeros((args[0], 2)))[0]), np.array(obs)), scene
    return args, kw, state, dict(obs=np.array(obs), rew=np.asarray(rew, float), done=bool(done),
                                 info=[info["ho_saved"], info["cr_encs"]], pos=np.concatenate([o.rx, o.cx, o.hx]),
                                 vel=np.concatenate([o.rv, o.cv, np.zeros_like(o.hx)]),
                                 counter=o.np_random.counter, saved=o.saved.copy(),
                                 flags=4 | int(o.gate_open) | 2 * int(o.bombed), S=sensor_table(K))


def bf16_bits(x):
    """float32 -> bfloat16 bit patterns, rounded to nearest even (no NaNs here)."""
    b = np.ascontiguousarray(x, F32).view(np.uint32).astype(np.uint64)
    return ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)


def want_obs_bits(want, kind):
    """The expected observation bits: float64 ('f64'), float32 ('f32') or bfloat16 ('bf16') of the oracle's."""
    if kind == "f64":
        return np.asarray(want, np.float64).view(np.uint64)
    w = np.asarray(want, np.float64).astype(F32)
    return bf16_bits(w) if kind == "bf16" else w.view(np.uint32)


def obs_bits(obs, kind):
    return np.ascontiguousarray(obs).view({"f64": np.uint64, "f32": np.uint32, "bf16": np.uint16}[kind])


def check_obs(where, got, exp, kind):
    """Observation rows bit for bit, signed zeros included (the oracle's zeros carry the term-by-term sign,
    see TermwiseTable)."""
    g, w = obs_bits(got, kind), want_obs_bits(exp["obs"], kind)
    bad = np.argwhere(g != w)
    assert bad.size == 0, (where, "obs", [(tuple(i), obs_val(got, kind, i), float(exp["obs"][tuple(i)]))
                                          for i in bad[:6]])


def obs_val(x, kind, i):
    v = np.asarray(x)[tuple(i)]
    if kind == "bf16":
        return float((np.uint32(v) << 16).view(F32)) if np.isscalar(v) else None
    return float(v)


def check_step(where, exp, rew, done, info, kind):
    real = np.float64 if kind == "f64" else F32
    assert np.array_equal(np.asarray(rew, np.float64), exp["rew"].astype(real).astype(np.float64)), \
        (where, "rew", rew, exp["rew"])
    assert bool(done) == exp["done"], (where, "done")
    assert list(np.asarray(info).tolist()) == exp["info"], (where, "info", info, exp["info"])


def check_state(where, exp, pos, vel, counter, kind):
    real = np.float64 if kind == "f64" else F32
    for nm, got, want in (("pos", pos, exp["pos"]), ("vel", vel, exp["vel"])):
        want = want.astype(real)
        bad = np.argwhere(np.asarray(got, real) != want)
        assert bad.size == 0, (where, nm, [(tuple(i), got[tuple(i)], want[tuple(i)]) for i in bad[:6]])
    assert int(counter) == exp["counter"], (where, "counter", int(counter), exp["counter"])


def ww_heuristic(obs, S, norm):
    """heuristics/waterworld.py's action of every row of obs [Np, D] (float64), with the sensor table S [K, 2]
    the rows were sensed with; norm "agent" divides each row by its own norm, "env" all rows by one."""
    o = np.asarray(obs, np.float64)
    K, S = len(S), np.asarray(S, np.float64)
    a = -(o[:, :K] @ S) + (o[:, K:2 * K] @ S) * np.where(o[:, 7 * K] > 0, 1.5, 1.0)[:, None] \
        - (o[:, 3 * K:4 * K] @ S) * np.where(o[:, 7 * K + 1] > 0, 1.5, 1.0)[:, None] + (o[:, 5 * K:6 * K] @ S) / 2
    n = np.linalg.norm(a, axis=1, keepdims=True) if norm == "agent" else np.linalg.norm(a)
    return np.where(n > 0, a / np.where(n > 0, n, 1), 0.0)
