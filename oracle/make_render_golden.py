"""Generate the render golden vectors from the REAL reference (run in the build container).

    python -m oracle.make_render_golden

Steps the unmodified reference MAWaterWorld and ContinuousHostageWorld (via ``oracle/refshim.py``) and calls
their own ``render`` on several states, with a ``cv2`` shim in ``sys.modules``: ``CV_AA`` (gone from OpenCV 3
and later) is mapped to ``LINE_8``, ``imshow`` keeps the image it is shown instead of opening a window and
``waitKey`` returns at once.  Every other call is the installed OpenCV's.  For each state it stores the frame
the reference drew (RGB: Waterworld's return value; Hostage returns nothing, so the image it showed, flipped
from BGR) and the state it drew from, in ``tests/golden/render_ww.npz`` and ``tests/golden/render_hw.npz``.
"""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(ROOT, "tests", "golden")
sys.path.insert(0, ROOT)

from oracle.refshim import load_reference  # noqa: E402

WW_CASES = [
    # (ctor kwargs, seed, steps between frames, frame sizes)
    (dict(n_pursuers=5, n_evaders=5), 1, (0, 40, 200), (800, 257)),
    (dict(n_pursuers=20, n_evaders=50, n_poison=50), 2, (0, 30), (800,)),
    (dict(n_pursuers=3, n_evaders=4, n_poison=2, n_sensors=7, radius=0.05, sensor_range=0.45,
          obstacle_loc=None), 3, (0, 25), (800, 37)),
]
HW_CASES = [
    # (ctor args, ctor kwargs, seed, steps between frames, frame sizes); the gate opens at once with the key in the
    # rescuers' spawn band and a large key radius
    ((10, 16, 16, 4, 2), dict(), 4, (0, 40, 200), (800, 257)),
    ((3, 4, 5, 1, 1), dict(key_loc=np.array([[0.5, 0.75]]), key_radius=0.5, sensor_range=0.35), 5, (0, 30),
     (800, 37)),
]


class _Shown(object):
    img = None


def _install_cv2_shim():
    import cv2 as real
    shim = types.ModuleType("cv2")
    shim.__dict__.update({k: getattr(real, k) for k in dir(real) if not k.startswith("__")})
    shim.CV_AA = real.LINE_8

    def imshow(name, img):
        _Shown.img = np.array(img)

    shim.imshow = imshow
    shim.waitKey = lambda *a, **k: -1
    sys.modules["cv2"] = shim


def _frames(env, steps, sizes, act, snap):
    rows = []
    for n in steps:
        for _ in range(n):
            if env.step(act(env))[2]:
                env.reset()
        for size in sizes:
            _Shown.img = None
            ret = env.render(screen_size=size)
            frame = ret if ret is not None else _Shown.img[..., ::-1]
            rows.append(dict(snap(env), size=size, frame=np.ascontiguousarray(frame)))
    return rows


def gen_waterworld(MAWaterWorld):
    rows, meta = [], []
    for case, (kw, seed, steps, sizes) in enumerate(WW_CASES):
        env = MAWaterWorld(**kw)
        env.seed(seed)
        env.reset()
        rs = np.random.RandomState(seed)
        snap = lambda env: dict(
            case=case, pos=np.array([a.position for a in list(env._pursuers) + list(env._evaders) +
                                     list(env._poisons)]).reshape(-1, 2),
            obst=np.array(env.obstaclesx_No_2).reshape(2))
        rows += _frames(env, steps, sizes, lambda env: rs.randn(env.n_pursuers, 2), snap)
        meta.append(dict(n_pursuers=env.n_pursuers, n_evaders=env.n_evaders, n_poison=env.n_poison,
                         n_sensors=env.n_sensors, radius=env.radius, obstacle_radius=env.obstacle_radius,
                         sensor_range=float(env.sensor_range[0])))
    _save(os.path.join(GOLDEN, "render_ww.npz"), rows, meta, ("pos",))


def gen_hostage(ContinuousHostageWorld):
    rows, meta = [], []
    for case, (args, kw, seed, steps, sizes) in enumerate(HW_CASES):
        env = ContinuousHostageWorld(*args, **kw)
        env.seed(seed)
        env.reset()
        rs = np.random.RandomState(seed)
        snap = lambda env: dict(
            case=case, pos=np.array([a.position for a in list(env._rescuers) + list(env._criminals) +
                                     list(env._hostages)]).reshape(-1, 2),
            fixed=np.concatenate([np.asarray(env.key_loc).reshape(2), np.asarray(env.bomb_loc).reshape(2)]),
            saved=np.array(env.curr_host_saved_mask, dtype=np.uint8), gate=int(bool(env._gate_open)))
        case_rows = _frames(env, steps, sizes, lambda env: rs.randn(env.n_good, 2), snap)
        # a saved hostage is not drawn: mark some saved on a closed gate, whatever the episode reached
        env._gate_open = False
        env.curr_host_saved_mask[::2] = True
        case_rows += _frames(env, (0,), sizes, None, snap)
        rows += case_rows
        meta.append(dict(n_good=env.n_good, n_bad=env.n_bad, n_hostages=env.n_hostages, n_sensors=env.n_sensors,
                         radius=env.radius, bomb_radius=env.bomb_radius, sensor_range=float(env.sensor_range[0])))
    _save(os.path.join(GOLDEN, "render_hw.npz"), rows, meta, ("pos", "saved"))


def _save(path, rows, meta, ragged):
    """One array per state field; the fields named in `ragged` (whose length depends on the case) and the frames
    (whose size does) are concatenated, with `<field>_len` per row; `meta`: each case's configuration."""
    flat = []
    for r in rows:
        r = dict(r)
        for k in ragged:
            r[k + "_len"] = r[k].shape[0]
        flat.append(r)
    out = {k: np.array([r[k] for r in flat]) for k in flat[0] if k != "frame" and k not in ragged}
    for k in ragged:
        out[k] = np.concatenate([r[k] for r in flat])
    out["frames"] = np.concatenate([r["frame"].ravel() for r in flat])
    out["meta"] = json.dumps(meta)
    np.savez_compressed(path, **out)


def main():
    _install_cv2_shim()
    MAWaterWorld, _, ContinuousHostageWorld = load_reference()
    gen_waterworld(MAWaterWorld)
    gen_hostage(ContinuousHostageWorld)


if __name__ == "__main__":
    main()
