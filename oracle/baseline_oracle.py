"""NumPy restatement of rllab's LinearFeatureBaseline (rllab/rllab/baselines/linear_feature_baseline.py) over
time-major rollout arrays -- the oracle of madrl_b200.postproc.LinearFeatureBaseline and of the
madrl_lfb_* kernels (csrc/baseline.cu).

Rows are the (t, e, a) rows of a rollout in that order.  Row t's observation is the one action t was taken in
(``obs_before`` for t = 0 and ``obs[t-1]`` afterwards when ``obs_before`` is given, else ``obs[t]``); its time
index is its position in its path (paths cut at ``done``), plus ``t0[e]`` on env e's first path.  The features
are ``_features`` (:19-23) evaluated on float64 observations: a float32 observation is widened before it is
squared, as the reference does with the float64 observations of its own envs.
"""
import importlib.util
import os
import sys
import types

import numpy as np


def source_rows(obs, obs_before=None):
    """[T,E,A,D] float64: the observation each action was taken in."""
    obs = np.asarray(obs, dtype=np.float64)
    if obs_before is None:
        return obs
    return np.concatenate([np.asarray(obs_before, dtype=np.float64)[None], obs[:-1]])


def time_index(done, t0=None):
    """[T,E] int64: position of step t in its path (cut after every done step), + t0[e] on the first path."""
    done = np.asarray(done).astype(bool)
    T, E = done.shape
    idx = np.zeros((T, E), np.int64)
    for e in range(E):
        i = 0 if t0 is None else int(t0[e])
        for t in range(T):
            idx[t, e] = i
            i = 0 if done[t, e] else i + 1
    return idx


def features(obs, done, obs_before=None, t0=None):
    """F [T*E*A, 2D+4] float64, rows in (t, e, a) order."""
    o = np.clip(source_rows(obs, obs_before), -10, 10)
    T, E, A, D = o.shape
    o = o.reshape(-1, D)
    al = np.repeat(time_index(done, t0).reshape(-1), A).reshape(-1, 1) / 100.0
    return np.concatenate([o, o ** 2, al, al ** 2, al ** 3, np.ones((o.shape[0], 1))], axis=1)


def normal_equations(F, y):
    """[F y]^T [F y], float64 [Df+1, Df+1], its blocks formed by the reference's own expressions
    (featmat.T.dot(featmat), featmat.T.dot(returns), :31-33)."""
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    Df = F.shape[1]
    G = np.empty((Df + 1, Df + 1))
    G[:Df, :Df] = F.T.dot(F)
    G[:Df, Df] = G[Df, :Df] = F.T.dot(y)
    G[Df, Df] = y.dot(y)
    return G


def fit(F, y, reg_coeff=1e-5):
    """fit() (:25-37): lstsq on the regularised normal equations, reg x 10 (at most 5 tries) while NaN."""
    y = np.asarray(y, dtype=np.float64).reshape(-1)
    reg = reg_coeff
    for _ in range(5):
        c = np.linalg.lstsq(F.T.dot(F) + reg * np.identity(F.shape[1]), F.T.dot(y), rcond=None)[0]
        if not np.any(np.isnan(c)):
            break
        reg *= 10
    return c


def objective(F, y, c, reg_coeff=1e-5):
    """rllab's regularised least-squares objective ||F c - y||^2 + reg ||c||^2 (what fit() minimises)."""
    r = F.dot(c) - np.asarray(y, dtype=np.float64).reshape(-1)
    return float(r.dot(r) + reg_coeff * np.dot(c, c))


def path_rows(done, A):
    """Rollout row index (t*E + e)*A + a of every row in path order (env, episode, agent; the order of
    ``to_paths`` / ``pack_paths``), and the path lengths."""
    done = np.asarray(done).astype(bool)
    T, E = done.shape
    rows, lens = [], []
    for e in range(E):
        ends = list(np.nonzero(done[:, e])[0] + 1)
        if not ends or ends[-1] != T:
            ends.append(T)
        s = 0
        for end in ends:
            for a in range(A):
                rows.extend((t * E + e) * A + a for t in range(s, end))
                lens.append(end - s)
            s = end
    return np.array(rows, np.int64), np.array(lens, np.int64)


def load_reference_baseline(reference_root):
    """The real ``LinearFeatureBaseline`` class, loaded from its file with ``rllab.baselines.base``,
    ``rllab.misc.overrides`` and ``rllab.misc.autoargs`` stubbed (the way oracle.refshim.load_rllab_numeric
    stubs theano); sys.modules is restored afterwards."""
    path = os.path.join(reference_root, "rllab", "rllab", "baselines", "linear_feature_baseline.py")
    if not os.path.exists(path):
        raise RuntimeError("reference file not found: %s" % path)
    saved = dict(sys.modules)
    try:
        def module(name, **attrs):
            m = types.ModuleType(name)
            m.__dict__.update(attrs)
            sys.modules[name] = m
            return m
        for name in ("rllab", "rllab.baselines", "rllab.misc"):
            module(name)
        module("rllab.baselines.base", Baseline=type("Baseline", (object,), {}))
        module("rllab.misc.overrides", overrides=lambda f: f)
        module("rllab.misc.autoargs", arg=lambda *a, **k: (lambda f: f), inherit=lambda *a, **k: (lambda f: f))
        spec = importlib.util.spec_from_file_location("_ref_linear_feature_baseline", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        return mod.LinearFeatureBaseline
    finally:
        for k in list(sys.modules):
            if k not in saved:
                del sys.modules[k]
        sys.modules.update(saved)


# ---------------------------------------------------------------- the obvious PyTorch implementation
# Features built per chunk of rows in float64 on the device, G.addmm_(F^T, F) (cuBLAS DGEMM) and F @ c: the
# comparison point of scripts/linear_baseline_rate.py and the full-size GPU test.

def torch_time_index(done, t0=None):
    """[T,E] int64 on done's device (a loop over T of vector ops)."""
    import torch
    T, E = done.shape
    idx = torch.empty((T, E), dtype=torch.int64, device=done.device)
    cur = torch.zeros(E, dtype=torch.int64, device=done.device) if t0 is None else t0.long()
    for t in range(T):
        idx[t] = cur
        cur = torch.where(done[t].bool(), torch.zeros_like(cur), cur + 1)
    return idx


def torch_feature_chunks(obs, done, obs_before=None, t0=None, chunk=1 << 16):
    """Yields (row slice, F [rows, 2D+4] float64) over the (t, e, a) rows of a device rollout."""
    import torch
    T, E, A, D = obs.shape
    flat = obs.reshape(T * E * A, D)
    first = obs_before.reshape(E * A, D) if obs_before is not None else None
    al = (torch_time_index(done, t0).unsqueeze(-1).expand(T, E, A).reshape(-1).double() / 100.0).unsqueeze(1)
    n, EA = T * E * A, E * A
    for r0 in range(0, n, chunk):
        r1 = min(n, r0 + chunk)
        if first is None:
            src = flat[r0:r1]
        elif r0 >= EA:
            src = flat[r0 - EA:r1 - EA]
        else:
            src = torch.cat([first[r0:min(r1, EA)], flat[0:max(0, r1 - EA)]])
        o = src.double().clamp_(-10, 10)
        a = al[r0:r1]
        yield slice(r0, r1), torch.cat([o, o * o, a, a * a, a ** 3, torch.ones_like(a)], dim=1)


def torch_normal_equations(obs, done, returns, obs_before=None, t0=None, chunk=1 << 16, pairwise=False):
    """G.addmm_ over the chunks; pairwise=True keeps every chunk's Gram and sums them pairwise (a more
    accurate float64 reference for the tests: no summation chain longer than one chunk)."""
    import torch
    D = obs.shape[3]
    y = returns.reshape(-1, 1).double()
    G = torch.zeros((2 * D + 5, 2 * D + 5), dtype=torch.float64, device=obs.device)
    parts = []
    for sl, F in torch_feature_chunks(obs, done, obs_before, t0, chunk):
        Fy = torch.cat([F, y[sl]], dim=1)
        if pairwise:
            parts.append(Fy.T @ Fy)
        else:
            G.addmm_(Fy.T, Fy)
    if not pairwise:
        return G
    while len(parts) > 1:
        parts = [parts[i] + parts[i + 1] if i + 1 < len(parts) else parts[i] for i in range(0, len(parts), 2)]
    return parts[0]


def torch_predict(obs, done, coef, obs_before=None, t0=None, chunk=1 << 16):
    import torch
    T, E, A, _ = obs.shape
    out = torch.empty(T * E * A, dtype=torch.float32, device=obs.device)
    for sl, F in torch_feature_chunks(obs, done, obs_before, t0, chunk):
        out[sl] = (F @ coef).float()
    return out.view(T, E, A)
