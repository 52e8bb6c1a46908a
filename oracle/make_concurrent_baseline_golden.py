"""Writes tests/golden/linear_baseline_concurrent_ref.npz: the non-recurrent concurrent branch of rllab's
BatchMASampler.process_samples (rllab/sandbox/rocky/tf/samplers/batch_ma_sampler.py:64-123) and its baseline fit
(:184-188), run with the REAL rllab pieces on scripted rollouts cut into per-agent paths, for two consecutive
iterations:
  LinearFeatureBaseline       rllab/rllab/baselines/linear_feature_baseline.py (oracle.baseline_oracle loader)
  special.discount_cumsum, special.explained_variance_1d, util.center_advantages,
  util.shift_advantages_to_positive                           (oracle.refshim.load_rllab_numeric)

Two flavours of the baseline list:
  independent  A distinct LinearFeatureBaseline instances;
  shared       ONE instance listed A times, as runners/rurllab.py:275-276 builds it.

Cases (each iteration: obs [T,E,A,D] float32, obs_before [E,A,D], done [T,E], rew [T,E,A] float32; rllab's
sampler starts fresh paths every iteration, so the time index starts at 0 in each):
  ragged       3 agents, several paths per env of different lengths; agent 1 has constant observation columns
  beyond_clip  4 agents, observations and rewards well past +-10, positive_adv as well
Stored per case: the inputs and settings; per iteration and agent the reference's feature matrix (path order);
per flavour, iteration and agent its predictions, processed advantages and returns (path order), the explained
variances [A] and the coefficients after each agent's fit [A, Df].
Run:  python -m oracle.make_concurrent_baseline_golden
"""
import os

import numpy as np

from oracle import baseline_oracle as bo
from oracle.refshim import REFERENCE_ROOT, load_rllab_numeric

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "linear_baseline_concurrent_ref.npz")
FLAVOURS = ("independent", "shared")


def _iteration(rs, T, E, A, D, done_steps, scale, rew_scale, const_agent=None):
    done = np.zeros((T, E), np.uint8)
    for e, steps in enumerate(done_steps):
        done[list(steps), e] = 1
    obs = (rs.randn(T, E, A, D) * scale).astype(np.float32)
    obs_before = (rs.randn(E, A, D) * scale).astype(np.float32)
    if const_agent is not None:
        obs[:, :, const_agent, 0] = obs_before[:, const_agent, 0] = 0.0
        obs[:, :, const_agent, 2] = obs_before[:, const_agent, 2] = 1.0
    return dict(obs=obs, obs_before=obs_before, done=done,
                rew=(rs.randn(T, E, A) * rew_scale + 0.5).astype(np.float32))


def cases():
    rs = np.random.RandomState(20261016)
    return {
        "ragged": dict(discount=0.99, gae_lambda=0.97, center_adv=True, positive_adv=False, iterations=[
            _iteration(rs, 17, 3, 3, 4, [(3, 9, 10), (0, 12), (15,)], 3.0, 2.0, const_agent=1),
            _iteration(rs, 17, 3, 3, 4, [(5,), (2, 7, 13), ()], 3.0, 2.0, const_agent=1)]),
        "beyond_clip": dict(discount=0.95, gae_lambda=1.0, center_adv=True, positive_adv=True, iterations=[
            _iteration(rs, 12, 2, 4, 3, [(4,), (8, 9)], 15.0, 20.0),
            _iteration(rs, 12, 2, 4, 3, [(), (1, 6)], 15.0, 20.0)]),
    }


def agent_paths(it, a):
    """Agent a's paths in (env, episode) order: observation rows (the observation each action was taken in)
    and float64 rewards."""
    src = bo.source_rows(it["obs"], it["obs_before"])
    T, E = it["done"].shape
    rows, lens = bo.path_rows(it["done"], 1)
    rew = it["rew"].astype(np.float64)
    paths, p = [], 0
    for L in lens:
        te = rows[p:p + L]
        t, e = te // E, te % E
        paths.append(dict(observations=src[t, e, a], rewards=rew[t, e, a]))
        p += L
    return paths


def process_concurrent(baselines, paths, settings, util, special):
    """batch_ma_sampler.py:64-123 (non-recurrent) and :184-188, per agent in order."""
    discount, gae_lambda = settings["discount"], settings["gae_lambda"]
    out = []
    for ps, baseline in zip(paths, baselines):
        all_path_baselines = [baseline.predict(path) for path in ps]
        bl, returns = [], []
        for idx, path in enumerate(ps):
            path_baselines = np.append(all_path_baselines[idx], 0)
            deltas = path["rewards"] + discount * path_baselines[1:] - path_baselines[:-1]
            path["advantages"] = special.discount_cumsum(deltas, discount * gae_lambda)
            path["returns"] = special.discount_cumsum(path["rewards"], discount)
            bl.append(path_baselines[:-1])
            returns.append(path["returns"])
        ev = special.explained_variance_1d(np.concatenate(bl), np.concatenate(returns))
        advantages = np.concatenate([path["advantages"] for path in ps])
        if settings["center_adv"]:
            advantages = util.center_advantages(advantages)
        if settings["positive_adv"]:
            advantages = util.shift_advantages_to_positive(advantages)
        baseline.fit(ps)
        out.append(dict(pred=np.concatenate(bl), adv=advantages, ret=np.concatenate(returns), ev=ev,
                        coeffs=np.array(baseline.get_param_values())))
    return out


def main():
    Ref = bo.load_reference_baseline(REFERENCE_ROOT)
    util, special = load_rllab_numeric()
    arrays = {}
    for name, case in cases().items():
        A = case["iterations"][0]["obs"].shape[2]
        arrays[name + "/settings"] = np.array([case["discount"], case["gae_lambda"], case["center_adv"],
                                               case["positive_adv"]], np.float64)
        for n, it in enumerate(case["iterations"]):
            for k in ("obs", "obs_before", "done", "rew"):
                arrays["%s/it%d/%s" % (name, n, k)] = it[k]
            ref = Ref(env_spec=None)
            for a in range(A):
                arrays["%s/it%d/featmat%d" % (name, n, a)] = np.concatenate([ref._features(p)
                                                                             for p in agent_paths(it, a)])
        for flavour in FLAVOURS:
            if flavour == "independent":
                baselines = [Ref(env_spec=None) for _ in range(A)]
            else:
                one = Ref(env_spec=None)
                baselines = [one for _ in range(A)]
            for n, it in enumerate(case["iterations"]):
                res = process_concurrent(baselines, [agent_paths(it, a) for a in range(A)], case, util, special)
                key = "%s/%s/it%d/" % (name, flavour, n)
                for a, r in enumerate(res):
                    for k in ("pred", "adv", "ret"):
                        arrays[key + "%s%d" % (k, a)] = r[k]
                arrays[key + "ev"] = np.array([r["ev"] for r in res], np.float64)
                arrays[key + "coeffs"] = np.stack([r["coeffs"] for r in res])
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
