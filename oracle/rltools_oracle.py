"""CPU oracle (TEST INFRASTRUCTURE) of rltools' sample processing: a NumPy restatement of ``Sampler.process``
(rltools/rltools/samplers/__init__.py:35-88), ``nn.Standardizer`` (rltools/rltools/nn.py:533-592), rltools'
``LinearFeatureBaseline`` (rltools/rltools/baselines/linear.py) and the fields ``sample()`` logs
(samplers/serial.py), over rollout tensors cut into paths by oracle/recurrent_oracle.py's ``rollout_paths``.
tests/test_rltools_samples_cpu.py pins it to tests/golden/rltools_samples_ref.npz, which
oracle/make_rltools_golden.py writes with the reference's own Sampler.process and linear.py; the device tests
compare with it.
"""
import numpy as np
import scipy.linalg

from oracle.recurrent_oracle import rollout_paths

F32 = np.float32


class Standardizer(object):
    """nn.Standardizer on float32 state (the TensorFlow variables' dtype): ``update`` mixes in float64 where NumPy
    promotes (``a`` and ``a * mean`` are float32, the batch mean float64) and rounds at the assign; ``stdev`` is
    float32; ``standardize`` divides by ``f32(stdev + eps)`` in float64."""

    def __init__(self, shape, eps=1e-6):
        shape = (shape,) if isinstance(shape, int) else tuple(shape)
        self._eps, self._shape = eps, shape
        self.count = np.zeros((1,), F32)
        self.mean = np.zeros((1,) + shape, F32)
        self.meansq = np.ones((1,) + shape, F32)

    def get_count(self, **kwargs):
        return self.count.copy()

    def get_mean(self, **kwargs):
        return self.mean.copy()

    def get_meansq(self, **kwargs):
        return self.meansq.copy()

    def get_stdev(self, **kwargs):
        return np.sqrt(self.meansq - np.square(self.mean) + F32(self._eps)).astype(F32)

    def update(self, points_N_D, **kwargs):
        assert points_N_D.ndim >= 2 and points_N_D.shape[1:] == self._shape
        num = points_N_D.shape[0]
        count = self.get_count()
        a = count / (count + num)
        self.mean = np.asarray(a * self.get_mean() + (1. - a) * points_N_D.mean(axis=0, keepdims=True), F32)
        self.meansq = np.asarray(a * self.get_meansq() + (1. - a) * (points_N_D ** 2).mean(axis=0, keepdims=True),
                                 F32)
        self.count = np.asarray(count + num, F32)

    def standardize(self, x_B_D, centered=True, **kwargs):
        mu = 0.
        if centered:
            mu = self.get_mean()
        return (x_B_D - mu) / (self.get_stdev() + self._eps)


class NoOpStandardizer(object):
    def __init__(self, shape, eps=1e-6):
        pass

    def update(self, points_N_D, **kwargs):
        pass

    def standardize(self, x_B_D, **kwargs):
        return x_B_D


def discount(r_N_T, gamma):
    """rltools/util.py:56-80 on a zero-padded [N, T] matrix: cumsum(gamma^t r)[::-1] / gamma^t."""
    f = np.power(gamma, np.arange(r_N_T.shape[1]))
    return np.cumsum((r_N_T * f[None])[:, ::-1], axis=1)[:, ::-1] / f[None]


def _padded(arrays, fill):
    out = np.full((len(arrays), max(len(a) for a in arrays)), fill, np.float64)
    for i, a in enumerate(arrays):
        out[i, :len(a)] = a
    return out


class Baseline(object):
    """rltools' LinearFeatureBaseline on per-path features."""

    def __init__(self, obs_dim, enable_obsnorm, reg_coeff=1e-5):
        self.w, self.reg = None, reg_coeff
        self.obsnorm = (Standardizer if enable_obsnorm else NoOpStandardizer)(obs_dim)

    def features(self, paths):
        o = np.concatenate([p["observations"] for p in paths])
        t = np.concatenate([np.arange(len(p["rewards"]), dtype=float) for p in paths])[:, None] / 100.
        return np.concatenate([self.obsnorm.standardize(o), t, t ** 2, np.ones((len(o), 1))], axis=1)

    def predict(self, paths):
        F = self.features(paths)
        return F.dot(self.w if self.w is not None else np.zeros(F.shape[1]))

    def normal_equations(self, paths, q):
        F = self.features(paths)
        Fy = np.concatenate([F, q[:, None]], axis=1)
        return Fy.T.dot(Fy)

    def fit(self, paths, q):
        F = self.features(paths)
        self.w = scipy.linalg.solve(F.T.dot(F) + self.reg * np.eye(F.shape[1]), F.T.dot(q), assume_a="pos")


def process(paths, baseline, rewnorm, gamma, lam):
    """Sampler.process on one batch of paths; baseline None = ZeroBaseline.  -> dict of per-path lists (adv, q,
    simplev, v: the values used) and v_r, tv_r, fallback."""
    lens = [len(p["rewards"]) for p in paths]
    r = rewnorm.standardize(_padded([p["rewards"] for p in paths], 0.), centered=False)
    qz = discount(r, gamma)
    q = [qz[i, :l] for i, l in enumerate(lens)]
    qs = np.concatenate(q)
    simplev_row = np.nanmean(_padded(q, np.nan), axis=0)
    simplev = [simplev_row[:l] for l in lens]
    v = baseline.predict(paths) if baseline is not None else np.zeros(len(qs))
    var_q = np.var(qs)
    tv_r = 1. - np.var(qs - np.concatenate(simplev)) / (var_q + 1e-8)
    v_r = 1. - np.var(qs - v) / (var_q + 1e-8)
    vl = np.split(v, np.cumsum(lens)[:-1])
    if v_r < 0:
        vl = simplev
    vz = np.concatenate([_padded(vl, 0.), np.zeros((len(paths), 1))], axis=1)
    delta = r + gamma * vz[:, 1:] - vz[:, :-1]
    adv = discount(delta, gamma * lam)
    out = dict(adv=[adv[i, :l] for i, l in enumerate(lens)], q=q, simplev=simplev, v=vl, v_r=v_r, tv_r=tv_r,
               fallback=bool(v_r < 0), simplev_bins=simplev_row)
    if baseline is not None:
        baseline.fit(paths, qs)
    return out


def batches(obs, rew, done, obs_before, mode):
    """The path lists of one rollout: [paths] (decentralized, centralized) or one list per agent (concurrent).
    Observations and rewards float64 (float32-representable), as the reference envs emit them."""
    T, E, A = np.shape(rew)
    acts = np.zeros((T, E, A, 1), np.float32)
    paths = rollout_paths(obs, acts, rew, done, obs_before=obs_before, mode=mode)
    return paths if mode == "concurrent" else [paths]


def to_rollout(values, done, A, mode):
    """Per-path arrays (in `batches` order, one list per batch) -> [T,E,A] float64 (centralized: [T,E,1])."""
    done = np.asarray(done).astype(bool)
    T, E = done.shape
    out = np.full((T, E, 1 if mode == "centralized" else A), np.nan)
    idx = [0] * len(values)
    for e in range(E):
        ends = list(np.nonzero(done[:, e])[0] + 1)
        if not ends or ends[-1] != T:
            ends.append(T)
        s = 0
        for end in ends:
            for a in range(out.shape[2]):
                b = a if mode == "concurrent" else 0
                out[s:end, e, a] = values[b][idx[b]]
                idx[b] += 1
            s = end
    return out


def sample_fields(paths_per_batch):
    """serial.py's logged fields: per batch ret, batch, avglen, maxlen, minlen, ravg; averaged over batches
    (concurrent control) where the reference averages."""
    f = []
    for paths in paths_per_batch:
        lens = [len(p["rewards"]) for p in paths]
        f.append(dict(ret=_padded([p["rewards"] for p in paths], 0.).sum(axis=1).mean(), batch=len(paths),
                      avglen=int(np.mean(lens)), maxlen=int(np.max(lens)), minlen=int(np.min(lens)),
                      ravg=np.concatenate([p["rewards"] for p in paths]).mean()))
    if len(f) == 1:
        return f[0]
    return dict(ret=np.mean([x["ret"] for x in f]), batch=np.mean([x["batch"] for x in f]), avglen=f[-1]["avglen"],
                maxlen=f[-1]["maxlen"], minlen=f[-1]["minlen"], ravg=np.mean([x["ravg"] for x in f]))


def golden_case(z, name):
    """A case of tests/golden/rltools_samples_ref.npz: (settings dict, list of rollout dicts)."""
    g, lam, obsnorm, rewnorm = z[name + "/settings"]
    rollouts, k = [], 0
    while "%s/r%d/obs" % (name, k) in z.files:
        pre = "%s/r%d/" % (name, k)
        rollouts.append({f[len(pre):]: z[f] for f in z.files if f.startswith(pre)})
        k += 1
    return dict(discount=float(g), gae_lambda=float(lam), obsnorm=bool(obsnorm), rewnorm=bool(rewnorm)), rollouts


def replay(settings, rollouts, mode):
    """The golden's training-loop order on the oracle: rollout 0 is the extra batch, each later one is processed.
    Yields (k, per-batch `process` results (None for the extra batch), baselines, rewnorm) after each rollout."""
    pm = "decentralized" if mode == "zero" else mode
    A, D = rollouts[0]["obs"].shape[2:]
    nb, od = (A if pm == "concurrent" else 1), (A * D if pm == "centralized" else D)
    bls = [None if mode == "zero" else Baseline(od, settings["obsnorm"]) for _ in range(nb)]
    rewnorm = (Standardizer if settings["rewnorm"] else NoOpStandardizer)(1)
    for k, it in enumerate(rollouts):
        rew = it["rew_cent"] if pm == "centralized" else it["rew"]
        bs = batches(it["obs"], rew, it["done"], it.get("obs_before"), pm)
        res = None
        if k == 0:
            for bl, ps in zip(bls, bs):
                if bl is not None:
                    bl.obsnorm.update(np.concatenate([p["observations"] for p in ps]))
                rewnorm.update(np.concatenate([p["rewards"] for p in ps])[:, None])
        else:
            res = [process(ps, bl, rewnorm, settings["discount"], settings["gae_lambda"]) for bl, ps in zip(bls, bs)]
            for ps in bs:
                rewnorm.update(np.concatenate([p["rewards"] for p in ps])[:, None])
        yield k, res, bls, rewnorm


# ---------------------------------------------------------------- the obvious PyTorch implementation
# Sampler.process on the device with PyTorch only: float64 features materialised, a backward loop over time for q
# and the advantages, scatter_add bins, a DGEMM Gram and torch.linalg.cholesky.  The comparison point of
# scripts/rltools_samples_rate.py and the full-size GPU test.

def torch_index(done):
    """The time index (position in the path) of every (t, e) of done [T,E] (cuda), int64."""
    import torch
    T = done.shape[0]
    ar = torch.arange(T, device=done.device).unsqueeze(1)
    ends = torch.cummax(torch.where(done.bool(), ar + 1, torch.zeros_like(ar)), dim=0).values
    start = torch.cat([torch.zeros_like(ends[:1]), ends[:-1]])
    return ar - start


def torch_discount(x, done, gamma):
    """Per-path discounted sums of x [T,E,A] float64 (paths end at done and at the rollout's end)."""
    import torch
    out = torch.empty_like(x)
    run = torch.zeros_like(x[0])
    for t in range(x.shape[0] - 1, -1, -1):
        run = torch.where(done[t].bool().unsqueeze(-1), torch.zeros_like(run), run)
        run = x[t] + gamma * run
        out[t] = run
    return out


def torch_features(obs, obs_before, done, norm):
    """rltools' features [T,E,A,D+3] float64 of the action rows; norm [G,2,D] (G = 1 or A) or None."""
    import torch
    seen = obs if obs_before is None else torch.cat([obs_before.unsqueeze(0), obs[:-1]])
    o = seen.double()
    if norm is not None:
        o = (o - norm[:, 0]) / norm[:, 1]
    i = torch_index(done).double().unsqueeze(-1).expand(o.shape[:3]).unsqueeze(-1) / 100.
    return torch.cat([o, i, i * i, torch.ones_like(i)], -1)


def torch_process_samples(obs, obs_before, done, rew, gamma, lam, denom, w, norm, per_agent, reg=1e-5):
    """Sampler.process in PyTorch on the mode's view (obs [T,E,A,D], rew [T,E,A]); w [Df] or [A, Df] (None: zero
    baseline), denom the reward normaliser's f32(stdev + eps) (None: off).  -> dict(q, adv, values, simplev, v_r,
    tv_r (tensors [G]), fallback, w) with the new coefficients fitted to q."""
    import torch
    T, E, A = rew.shape
    r = rew.double() / (denom.double() if denom is not None else 1.0)
    q = torch_discount(r, done, gamma)
    F = torch_features(obs, obs_before, done, norm) if w is not None else None
    v = torch.zeros_like(q) if w is None else (F * (w if w.dim() == 2 else w.unsqueeze(0))).sum(-1)
    G = A if per_agent else 1
    idx = torch_index(done).unsqueeze(-1).expand(T, E, A)
    grp = torch.arange(A, device=q.device).expand(T, E, A) if per_agent else torch.zeros_like(idx)
    L = int(idx.max()) + 1
    key = (grp * L + idx).reshape(-1)
    sums = torch.zeros(G * L, dtype=torch.float64, device=q.device).scatter_add_(0, key, q.reshape(-1))
    cnt = torch.zeros(G * L, dtype=torch.float64, device=q.device).scatter_add_(0, key, torch.ones_like(q).reshape(-1))
    simplev = (sums / cnt.clamp(min=1))[key].view(T, E, A)
    dims = (0, 1) if per_agent else (0, 1, 2)
    var_q = q.var(dim=dims, correction=0)
    v_r = 1 - (q - v).var(dim=dims, correction=0) / (var_q + 1e-8)
    tv_r = 1 - (q - simplev).var(dim=dims, correction=0) / (var_q + 1e-8)
    fb = v_r < 0
    vals = torch.where(fb, simplev, v) if per_agent else (simplev if bool(fb) else v)
    nxt = torch.cat([vals[1:], torch.zeros_like(vals[:1])])
    nxt = torch.where(done.bool().unsqueeze(-1), torch.zeros_like(nxt), nxt)
    adv = torch_discount(r + gamma * nxt - vals, done, gamma * lam)
    w_new = None
    if w is not None:
        Fq = torch.cat([F, q.unsqueeze(-1)], -1)
        Fq = Fq.permute(2, 0, 1, 3).reshape(A, T * E, -1) if per_agent else Fq.reshape(1, T * E * A, -1)
        Gm = Fq.transpose(1, 2) @ Fq
        Df = Gm.shape[-1] - 1
        M = Gm[:, :Df, :Df] + reg * torch.eye(Df, dtype=Gm.dtype, device=Gm.device)
        w_new = torch.cholesky_solve(Gm[:, :Df, Df:], torch.linalg.cholesky(M)).squeeze(-1)
        w_new = w_new if per_agent else w_new[0]
    return dict(q=q, adv=adv, values=vals, simplev=simplev, v_r=v_r, tv_r=tv_r, fallback=fb, w=w_new)
