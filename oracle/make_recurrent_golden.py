"""Writes tests/golden/recurrent_samples_ref.npz: the recurrent branch of rllab's sampler post-processing, run with
the REAL rllab code on scripted rollouts cut into paths, for two consecutive iterations (the second predicts with
the baseline fitted on the first):
  BaseSampler.process_samples   rllab/rllab/sampler/base.py:48-180, with a stub algo whose policy has
                                recurrent=True and a distribution of zero entropy; logger.record_tabular is
                                patched to capture the statistics (oracle.refshim.load_rllab_callers loader)
  LinearFeatureBaseline         rllab/rllab/baselines/linear_feature_baseline.py (oracle.baseline_oracle loader)

Control modes (path construction: oracle.recurrent_oracle.rollout_paths):
  decentralized            one call on every agent's paths, (env, episode, agent) order, one baseline;
  concurrent_independent,  batch_ma_sampler.py imports TensorFlow and cannot be loaded here; its recurrent branch
  concurrent_shared        (:124-181) is, line for line, base.py:105-161 on one agent's paths, so process_samples
                           is called once per agent on that agent's paths, with A baseline objects (independent)
                           or one object listed A times (shared, as runners/rurllab.py:275-276 builds it);
  centralized              one call on the agents' observations, actions and agent_infos side by side, with agent
                           0's reward (the rollout's rewards are equal across agents there: `rew_cent`).

Cases:
  ragged    4 envs x 2 agents, D = 5, obs_before given: episodes of several lengths, a length-1 path at t = 0
            (done at t = 0) and at the end, done at t = T-1, an env with no done; float32 actions [.., 2],
            a 2-column int32 info, agent_infos `mean` [.., 2]; center_adv and positive_adv (which the branch ignores)
  bf16_int  3 envs x 3 agents, D = 3, bfloat16-representable observations, no obs_before, int32 Pursuit-style
            actions [T,E,A], a 2-column float32 info, agent_infos `prob` [.., 5]; center_adv off
Run:  python -m oracle.make_recurrent_golden
"""
import os
import types

import numpy as np

from oracle import baseline_oracle as bo
from oracle import refshim
from oracle.recurrent_oracle import rollout_paths

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "recurrent_samples_ref.npz")
STATS = ("AverageDiscountedReturn", "AverageReturn", "ExplainedVariance", "NumTrajs", "StdReturn", "MaxReturn",
         "MinReturn")
RUNS = ("decentralized", "concurrent_independent", "concurrent_shared", "centralized")


def _bf16(x):
    u = np.asarray(x, np.float32).view(np.uint32).astype(np.uint64)
    return (((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16).astype(np.uint32).view(np.float32)


def _iteration(rs, T, E, A, D, cuts, bf16, with_before, int_actions, ai_width):
    done = np.zeros((T, E), np.uint8)
    for e, steps in enumerate(cuts):
        done[list(steps), e] = 1
    cvt = _bf16 if bf16 else (lambda x: x)
    obs = cvt((rs.randn(T, E, A, D) * 6).astype(np.float32))
    rew = (rs.randn(T, E, A) * 2 + 0.3).astype(np.float32)
    it = dict(obs=obs, done=done, rew=rew, rew_cent=np.repeat(rew[..., :1], A, axis=2),
              actions=(rs.randint(0, 5, (T, E, A)).astype(np.int32) if int_actions else
                       rs.randn(T, E, A, 2).astype(np.float32)),
              info=(rs.randint(0, 9, (T, E, 2)).astype(np.int32) if not int_actions else
                    rs.randn(T, E, 2).astype(np.float32)),
              agent_info=rs.randn(T, E, A, ai_width).astype(np.float32))
    if with_before:
        it["obs_before"] = cvt((rs.randn(E, A, D) * 6).astype(np.float32))
    return it


def cases():
    rs = np.random.RandomState(20261017)
    ragged = dict(discount=0.99, gae_lambda=0.95, center_adv=True, positive_adv=True, info_key="k",
                  agent_info_key="mean")
    ragged["iterations"] = [
        _iteration(rs, 9, 4, 2, 5, [(0, 4), (2, 8), (), (3, 5, 6)], False, True, False, 2),
        _iteration(rs, 9, 4, 2, 5, [(), (0,), (1, 7), (8,)], False, True, False, 2)]
    bf16_int = dict(discount=0.95, gae_lambda=1.0, center_adv=False, positive_adv=False, info_key="pos",
                    agent_info_key="prob")
    bf16_int["iterations"] = [
        _iteration(rs, 7, 3, 3, 3, [(2,), (6,), ()], True, False, True, 5),
        _iteration(rs, 7, 3, 3, 3, [(0, 1), (), (3,)], True, False, True, 5)]
    return dict(ragged=ragged, bf16_int=bf16_int)


def run_paths(case, it, run):
    """The path lists of one run: [paths] or, for the concurrent runs, one list per agent."""
    mode = run.split("_")[0]
    return rollout_paths(it["obs"], it["actions"], it["rew_cent"] if mode == "centralized" else it["rew"],
                         it["done"], {case["info_key"]: it["info"]}, {case["agent_info_key"]: it["agent_info"]},
                         it.get("obs_before"), mode)


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
            return np.zeros(next(iter(agent_infos.values())).shape[:2])

    def process(paths, baseline, case):
        algo = types.SimpleNamespace(baseline=baseline, discount=case["discount"], gae_lambda=case["gae_lambda"],
                                     center_adv=case["center_adv"], positive_adv=case["positive_adv"],
                                     policy=types.SimpleNamespace(recurrent=True, distribution=ZeroEntropy()))
        captured.clear()
        sd = base.BaseSampler(algo).process_samples(0, paths)
        out = {k: sd[k] for k in ("observations", "actions", "rewards", "returns", "advantages", "valids")}
        out["env_infos." + case["info_key"]] = sd["env_infos"][case["info_key"]]
        out["agent_infos." + case["agent_info_key"]] = sd["agent_infos"][case["agent_info_key"]]
        out["stats"] = np.array([captured[k] for k in STATS], np.float64)
        out["undisc"] = np.array([sum(p["rewards"]) for p in paths], np.float64)
        out["coeffs"] = np.array(baseline.get_param_values())
        return out

    arrays = {}
    try:
        for name, case in cases().items():
            arrays[name + "/settings"] = np.array([case["discount"], case["gae_lambda"], case["center_adv"],
                                                   case["positive_adv"]], np.float64)
            A = case["iterations"][0]["obs"].shape[2]
            one = Ref(env_spec=None)
            baselines = dict(decentralized=[Ref(env_spec=None)], centralized=[Ref(env_spec=None)],
                             concurrent_independent=[Ref(env_spec=None) for _ in range(A)],
                             concurrent_shared=[one] * A)
            for n, it in enumerate(case["iterations"]):
                for k, v in it.items():
                    arrays["%s/it%d/%s" % (name, n, k)] = v
                for run in RUNS:
                    paths = run_paths(case, it, run)
                    groups = paths if run.startswith("concurrent") else [paths]
                    for a, (ps, bl) in enumerate(zip(groups, baselines[run])):
                        key = "%s/%s/it%d/" % (name, run, n) + ("a%d/" % a if run.startswith("concurrent") else "")
                        for k, v in process(ps, bl, case).items():
                            arrays[key + k] = v
    finally:
        base.logger.record_tabular, base.logger.log = saved
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
