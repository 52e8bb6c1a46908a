"""CPU oracle (TEST INFRASTRUCTURE) of the recurrent branch of rllab's ``BaseSampler.process_samples``
(rllab/rllab/sampler/base.py:48-68, :105-180; concurrent control: per agent, batch_ma_sampler.py:124-181): a NumPy
restatement of the padding (``tensor_utils.pad_tensor_n``), the per-path GAE / returns, the centring, the sampler's
return statistics and rllab's LinearFeatureBaseline on per-path features.  tests/test_recurrent_samples_cpu.py pins
it to tests/golden/recurrent_samples_ref.npz, which oracle/make_recurrent_golden.py writes with the real rllab
pieces; the kernel tests compare with it.
"""
import numpy as np

from oracle.postproc_oracle import discount_cumsum, explained_variance_1d


def pad_tensor_n(xs, max_len):                          # tensor_utils.py:29-33
    out = np.zeros((len(xs), max_len) + np.shape(xs[0])[1:], dtype=np.asarray(xs[0]).dtype)
    for i, x in enumerate(xs):
        out[i, :len(x)] = x
    return out


def rollout_paths(obs, actions, rew, done, infos=None, agent_infos=None, obs_before=None, mode="decentralized"):
    """rllab paths of a rollout [T,E,A,...] (observations float64, the observation each action was taken in when
    obs_before [E,A,D] is given; rewards float64): decentralized -> one list in (env, episode, agent) order;
    concurrent -> A lists, agent a's paths in (env, episode) order; centralized -> one list in (env, episode) order
    of the agents' observations, actions and agent_infos side by side, with agent 0's reward."""
    obs = np.asarray(obs, np.float64)
    if obs_before is not None:
        obs = np.concatenate([np.asarray(obs_before, np.float64)[None], obs[:-1]])
    done = np.asarray(done).astype(bool)
    rew = np.asarray(rew, np.float64)
    T, E, A = rew.shape
    infos, agent_infos = dict(infos or {}), dict(agent_infos or {})
    side = lambda x: np.asarray(x).reshape(len(x), -1)                  # noqa: E731  (one row per step)
    per_agent = {}
    for e in range(E):
        ends = list(np.nonzero(done[:, e])[0] + 1)
        if not ends or ends[-1] != T:
            ends.append(T)
        s = 0
        for end in ends:
            env_infos = {k: v[s:end, e] for k, v in infos.items()}
            if mode == "centralized":
                per_agent.setdefault(0, []).append(dict(
                    observations=side(obs[s:end, e]), actions=side(np.asarray(actions)[s:end, e]),
                    rewards=rew[s:end, e, 0], env_infos=env_infos,
                    agent_infos={k: side(np.asarray(v)[s:end, e]) for k, v in agent_infos.items()}))
            else:
                for a in range(A):
                    per_agent.setdefault(a, []).append(dict(
                        observations=obs[s:end, e, a], actions=np.asarray(actions)[s:end, e, a],
                        rewards=rew[s:end, e, a], env_infos=env_infos,
                        agent_infos={k: np.asarray(v)[s:end, e, a] for k, v in agent_infos.items()}))
            s = end
    if mode == "concurrent":
        return [per_agent[a] for a in range(A)]
    if mode == "centralized":
        return per_agent[0]
    n = len(per_agent[0])
    return [per_agent[a][j] for j in range(n) for a in range(A)]


class PathBaseline(object):
    """rllab's LinearFeatureBaseline restated on per-path features (linear_feature_baseline.py:19-43)."""

    def __init__(self, reg_coeff=1e-5):
        self.coeffs, self.reg_coeff = None, reg_coeff

    @staticmethod
    def features(path):
        o = np.clip(path["observations"], -10, 10)
        al = np.arange(len(path["rewards"])).reshape(-1, 1) / 100.0
        return np.concatenate([o, o ** 2, al, al ** 2, al ** 3, np.ones((len(al), 1))], axis=1)

    def predict(self, path):
        if self.coeffs is None:
            return np.zeros(len(path["rewards"]))
        return self.features(path).dot(self.coeffs)

    def fit(self, paths):
        F = np.concatenate([self.features(p) for p in paths])
        y = np.concatenate([p["returns"] for p in paths])
        reg = self.reg_coeff
        for _ in range(5):
            self.coeffs = np.linalg.lstsq(F.T.dot(F) + reg * np.identity(F.shape[1]), F.T.dot(y), rcond=None)[0]
            if not np.any(np.isnan(self.coeffs)):
                break
            reg *= 10


def process_samples_recurrent(paths, baseline, discount, gae_lambda, center_adv=True):
    """base.py:48-68, :105-161 and the statistics of :170-180 (entropy aside) on one list of paths ->
    (samples_data, stats).  No positive_adv: the recurrent branch never applies it."""
    bl, rets = [], []
    for path in paths:
        b = np.append(baseline.predict(path), 0)
        deltas = path["rewards"] + discount * b[1:] - b[:-1]
        path["advantages"] = discount_cumsum(deltas, discount * gae_lambda)
        path["returns"] = discount_cumsum(path["rewards"], discount)
        bl.append(b[:-1])
        rets.append(path["returns"])
    ev = explained_variance_1d(np.concatenate(bl), np.concatenate(rets))
    L = max(len(p["advantages"]) for p in paths)
    adv = [p["advantages"] for p in paths]
    if center_adv:
        raw = np.concatenate(adv)
        adv = [(a - np.mean(raw)) / (np.std(raw) + 1e-8) for a in adv]
    pad = lambda key: pad_tensor_n([p[key] for p in paths], L)          # noqa: E731
    data = dict(observations=pad("observations"), actions=pad("actions"), rewards=pad("rewards"),
                returns=pad("returns"), advantages=pad_tensor_n(adv, L),
                valids=pad_tensor_n([np.ones_like(p["returns"]) for p in paths], L),
                env_infos={k: pad_tensor_n([p["env_infos"][k] for p in paths], L) for k in paths[0]["env_infos"]},
                agent_infos={k: pad_tensor_n([p["agent_infos"][k] for p in paths], L)
                             for k in paths[0]["agent_infos"]})
    baseline.fit(paths)
    undisc = [sum(p["rewards"]) for p in paths]
    stats = dict(AverageDiscountedReturn=np.mean([p["returns"][0] for p in paths]), AverageReturn=np.mean(undisc),
                 ExplainedVariance=ev, NumTrajs=len(paths), StdReturn=np.std(undisc), MaxReturn=np.max(undisc),
                 MinReturn=np.min(undisc))
    return data, stats


# ---------------------------------------------------------------- the obvious PyTorch implementation
# A gather of the source rows through a [P, L] index into a zero-filled tensor: the comparison point of
# scripts/recurrent_samples_rate.py and of the full-size GPU test.

def torch_pad(x, rec, L, per_agent=True, first=None):
    """x [T,E,A,...] (per agent) or [T,E,...] (per env) on the device, rec int [P, 4] = (env, agent, start,
    length) -> [P, L, ...]: row (p, i) = x[start + i, env, agent] for i < length, zeros after."""
    import torch
    T, E = x.shape[:2]
    A = x.shape[2] if per_agent else 1
    tail = tuple(x.shape[3:] if per_agent else x.shape[2:])
    flat = x.reshape(T * E * A, -1)
    if first is not None:
        flat = torch.cat([first.reshape(E * A, -1), flat[:(T - 1) * E * A]])
    rec = rec.long()
    i = torch.arange(L, device=x.device).unsqueeze(0)
    valid = i < rec[:, 3:4]
    row = ((rec[:, 2:3] + i) * E + rec[:, 0:1]) * A + (rec[:, 1:2] if per_agent else 0)
    out = torch.zeros((rec.shape[0], L, flat.shape[1]), dtype=x.dtype, device=x.device)
    out[valid] = flat[row[valid]]
    return out.view((rec.shape[0], L) + tail)
