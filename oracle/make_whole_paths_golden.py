"""Writes tests/golden/whole_paths_ref.npz: rllab's sample processing of the batch that the whole-path selection rule
(oracle/whole_paths_oracle.py, DESIGN §4.9) takes from scripted continuing done / reward streams, run with the REAL
rllab code:
  BaseSampler.process_samples   rllab/rllab/sampler/base.py:48-180, the non-recurrent and the recurrent branch, with
                                a stub algo whose policy's distribution has zero entropy; logger.record_tabular is
                                patched to capture the statistics (oracle.refshim.load_rllab_callers loader)
  LinearFeatureBaseline         rllab/rllab/baselines/linear_feature_baseline.py (oracle.baseline_oracle loader)
The paths are those of the flat batch, in its env-major (env, episode, agent) order, with the observation each
action was taken in.  One fresh baseline per branch and case, two iterations on the same batch (the second predicts
with the first's fit).

Cases (streams [S, E], A = 2 agents, D = 3):
  ragged   6 envs, paths ending at random or at the horizon 7, length-1 paths, batch_size 23; launches of 4 steps
  exact    4 envs, batch_size equal to the count at a step where paths end (the threshold crossed at a path end)
  late     5 envs, four end every 2 steps and one runs 17 steps: it finishes two launches after t*
Run:  python -m oracle.make_whole_paths_golden
"""
import os
import types

import numpy as np

from oracle import baseline_oracle as bo
from oracle import refshim
from oracle import whole_paths_oracle as wo
from oracle.recurrent_oracle import rollout_paths

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "whole_paths_ref.npz")
STATS = ("AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "StdReturn", "MaxReturn",
         "MinReturn")


def _stream(rs, S, E, mpl, p_end):
    done = np.zeros((S, E), np.uint8)
    for e in range(E):
        n = 0
        for t in range(S):
            n += 1
            if n == mpl or rs.rand() < p_end:
                done[t, e], n = 1, 0
    return done


def cases():
    rs = np.random.RandomState(20261018)
    ragged = _stream(rs, 24, 6, 7, 0.25)
    ragged[0, 2] = 1                                     # a length-1 path at the start
    exact = _stream(rs, 30, 4, 6, 0.3)
    last, count, counts = np.full(4, -1), 0, []
    for t in range(30):
        d = exact[t].astype(bool)
        count += int(np.sum(t - last[d]))
        last[d] = t
        counts.append(count)
    t_cross = next(t for t in range(8, 30) if exact[t].any())
    late = np.zeros((30, 5), np.uint8)
    late[1::2, :4] = 1
    late[[16], 4] = 1
    out = {}
    for name, done, bs, chunk in (("ragged", ragged, 23, 4), ("exact", exact, counts[t_cross], 3),
                                  ("late", late, 12, 5)):
        S, E = done.shape
        A, D = 2, 3
        out[name] = dict(done=done, batch_size=np.int64(bs), chunk=np.int64(chunk),
                         policy_obs=(rs.randn(S, E, A, D) * 3).astype(np.float32),
                         obs0=(rs.randn(E, A, D) * 3).astype(np.float32),
                         rew=(rs.randn(S, E, A) * 2 + 0.3).astype(np.float32),
                         actions=rs.randn(S, E, A, 2).astype(np.float32),
                         mean=rs.randn(S, E, A, 2).astype(np.float32))
    return out


def main():
    refshim.load_rllab_callers()
    import rllab.sampler.base as base
    Ref = bo.load_reference_baseline(refshim.REFERENCE_ROOT)
    captured = {}
    saved = base.logger.record_tabular, base.logger.log
    base.logger.record_tabular = lambda key, val: captured.__setitem__(key, val)
    base.logger.log = lambda *a, **k: None

    class ZeroEntropy(object):
        def entropy(self, agent_infos):
            return np.zeros(next(iter(agent_infos.values())).shape[:-1])

    arrays = {}
    try:
        for name, c in cases().items():
            for k, v in c.items():
                arrays["%s/%s" % (name, k)] = v
            t_star, end = wo.select(c["done"], int(c["batch_size"]))
            ps = wo.path_start(c["done"], end)
            arrays[name + "/t_star"], arrays[name + "/end"], arrays[name + "/path_start"] = np.int64(t_star), end, ps
            flat = lambda x, first=None: wo.gather(x, end, first)[:, None]     # noqa: E731  [N, 1, ...]
            obs, done = flat(c["policy_obs"], c["obs0"]), flat(c["done"])[:, 0:1]
            paths = rollout_paths(obs, flat(c["actions"]), flat(c["rew"]), done, None, {"mean": flat(c["mean"])})
            for recurrent in (False, True):
                bl = Ref(env_spec=None)
                for it in range(2):
                    algo = types.SimpleNamespace(baseline=bl, discount=0.99, gae_lambda=0.95, center_adv=True,
                                                 positive_adv=False,
                                                 policy=types.SimpleNamespace(recurrent=recurrent,
                                                                              distribution=ZeroEntropy()))
                    captured.clear()
                    ps_ = [dict(p, observations=np.array(p["observations"]), rewards=np.array(p["rewards"]))
                           for p in paths]
                    sd = base.BaseSampler(algo).process_samples(it, ps_)
                    key = "%s/%s/it%d/" % (name, "recurrent" if recurrent else "flat", it)
                    for k in ("observations", "advantages", "returns") + (("valids",) if recurrent else ()):
                        arrays[key + k] = np.asarray(sd[k])
                    arrays[key + "stats"] = np.array([captured[k] for k in STATS], np.float64)
                    arrays[key + "coeffs"] = np.array(bl.get_param_values())
    finally:
        base.logger.record_tabular, base.logger.log = saved
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
