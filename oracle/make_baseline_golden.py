"""Writes tests/golden/linear_baseline_ref.npz: the REAL rllab LinearFeatureBaseline
(rllab/rllab/baselines/linear_feature_baseline.py, loaded by oracle.baseline_oracle.load_reference_baseline)
fitted and evaluated on scripted rollouts cut into rllab paths.

Cases (each: obs [T,E,A,D] float32, obs_before [E,A,D], done [T,E], returns [T,E,A] float32):
  ragged         several paths per env of different lengths, obs_before given
  rank_deficient constant observation columns (as Pursuit's walls / ids), so F^T F is singular
  beyond_clip    observations well past +-10, no obs_before
Stored per case: the inputs, the reference's feature matrix and predictions in path order, its coefficients.
Run:  python -m oracle.make_baseline_golden
"""
import os

import numpy as np

from oracle import baseline_oracle as bo
from oracle.refshim import REFERENCE_ROOT

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "linear_baseline_ref.npz")


def cases():
    rs = np.random.RandomState(20261015)
    out = {}
    T, E, A, D = 23, 3, 2, 5
    done = np.zeros((T, E), np.uint8)
    done[[4, 11, 12, 19], 0] = 1
    done[[0, 9], 1] = 1
    done[[21], 2] = 1
    out["ragged"] = dict(obs=(rs.randn(T, E, A, D) * 3).astype(np.float32),
                         obs_before=(rs.randn(E, A, D) * 3).astype(np.float32), done=done,
                         returns=(rs.randn(T, E, A) * 5 + 2).astype(np.float32))
    T, E, A, D = 16, 2, 3, 6
    obs = rs.randn(T, E, A, D).astype(np.float32)
    obs[..., 1] = 0.0
    obs[..., 4] = 1.0
    done = np.zeros((T, E), np.uint8)
    done[[5, 13], 0] = 1
    done[[7], 1] = 1
    out["rank_deficient"] = dict(obs=obs, obs_before=np.ones((E, A, D), np.float32), done=done,
                                 returns=rs.randn(T, E, A).astype(np.float32))
    T, E, A, D = 14, 2, 2, 4
    done = np.zeros((T, E), np.uint8)
    done[[6], 0] = 1
    out["beyond_clip"] = dict(obs=(rs.randn(T, E, A, D) * 15).astype(np.float32), obs_before=None, done=done,
                              returns=(rs.randn(T, E, A) * 20).astype(np.float32))
    return out


def main():
    Ref = bo.load_reference_baseline(REFERENCE_ROOT)
    arrays = {}
    for name, c in cases().items():
        T, E, A, D = c["obs"].shape
        src = bo.source_rows(c["obs"], c["obs_before"]).reshape(-1, D)
        rows, lens = bo.path_rows(c["done"], A)
        y = c["returns"].astype(np.float64).reshape(-1)
        paths, p = [], 0
        for L in lens:
            r = rows[p:p + L]
            paths.append(dict(observations=src[r], rewards=y[r], returns=y[r]))
            p += L
        b = Ref(env_spec=None)
        assert b.predict(paths[0]) is not None and not np.any(b.predict(paths[0]))   # zeros before fit
        b.fit(paths)
        arrays[name + "/featmat"] = np.concatenate([b._features(q) for q in paths])
        arrays[name + "/coeffs"] = b.get_param_values()
        arrays[name + "/pred"] = np.concatenate([b.predict(q) for q in paths])
        for k in ("obs", "obs_before", "done", "returns"):
            if c[k] is not None:
                arrays[name + "/" + k] = c[k]
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
