"""Writes tests/golden/eval_ww_heuristic.npz: rltools' evaluate_policy statistics (rltools/rltools/util.py:141-231)
of the reference's Waterworld heuristic, computed by the REFERENCE's own code:

  * the real ``MAWaterWorld`` (oracle.refshim.load_reference) with reward_mech='global', as the pipelines run it, and
    the counter-based stream of oracle/philox.py injected as its ``np_random`` (one stream per env id, continued
    across that env's episodes, as the engine's in-place resets continue it);
  * stepped by the real ``decrollout`` (rltools/rltools/samplers/__init__.py:145-189, loaded by
    oracle.refshim.load_rltools_samplers) with the real ``WaterworldHeuristicPolicy`` (heuristics/waterworld.py),
    which therefore sees each env's Np observations as one batch: one norm per env;
  * statistics from the real ``TrajBatch`` and ``discount`` (util.py:56-80, executed from the source text as
    oracle/make_rltools_golden.py does: util.py as a whole does not parse on Python 3), in util.py:219-231's
    decentralized branch, over each env's first K episodes in record order k * E + e (what the engine evaluates).

The gevent workers of evaluate_policy are not run: they only decide which trajectories are kept.
Run:  python -m oracle.make_eval_golden
"""
import json
import os
import sys

import numpy as np

from oracle import refshim
from oracle.eval_oracle import waterworld_env_action
from oracle.philox import Stream

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "eval_ww_heuristic.npz")
CASE = dict(config=dict(n_pursuers=5, n_evaders=5, reward_mech='global'), seed=31, env_id_base=500, E=3, K=3,
            max_traj_len=50, discount=0.99, n_trajs=8)


def load():
    """(MAWaterWorld, decrollout, WaterworldHeuristicPolicy, TrajBatch, discount) from the reference files."""
    root = os.path.join(refshim.REFERENCE_ROOT, "rltools", "rltools")
    MAWaterWorld = refshim.load_reference()[0]
    with open(os.path.join(root, "util.py")) as f:
        lines = f.readlines()
    ns = dict(np=np)
    src = "".join(lines[55:80])                                   # lines 56-80, 1-based
    assert src.startswith("def discount(")
    exec(compile(src, os.path.join(root, "util.py"), "exec"), ns)
    samplers = refshim.load_rltools_samplers()
    WPol = refshim.load_reference_heuristics()[0]
    return MAWaterWorld, samplers.decrollout, WPol, sys.modules["rltools.trajutil"].TrajBatch, ns["discount"]


def main():
    MAWaterWorld, decrollout, WPol, TrajBatch, discount = load()
    c = CASE
    E, K, L = c["E"], c["K"], c["max_traj_len"]
    per_env, min_norm = [], np.inf
    for e in range(E):
        env = MAWaterWorld(**c["config"])
        env.np_random = Stream(c["seed"], c["env_id_base"] + e)
        pol = WPol(env.agents[0].observation_space, env.agents[0].action_space)
        pol.reset = lambda dones=None: None                        # rltools' Policy.reset: nothing to reset here
        eps = []
        for _ in range(K):
            trajs = decrollout(env, pol, L, env.agents[0].action_space)
            eps.append(trajs)
            for t in range(len(trajs[0].obs_T_Do)):                # the joint norm of every decision taken
                n = waterworld_env_action(np.array([tr.obs_T_Do[t] for tr in trajs]))[1]
                if n > 0:
                    min_norm = min(min_norm, n)
        per_env.append(eps)
    assert min_norm > 1e-6, "a decision normalises a rounding residue: pick another seed"
    episodes = [per_env[e][k] for k in range(K) for e in range(E)][:c["n_trajs"]]
    A = len(episodes[0])
    rets, stds, discs, infos = [], [], [], []
    for a in range(A):                                            # util.py:219-231, decentralized
        tb = TrajBatch.FromTrajs([ep[a] for ep in episodes])
        r_B_T = tb.r.padded(fill=0.)
        rets.append(r_B_T.sum(axis=1).mean())
        stds.append(r_B_T.sum(axis=1).std())
        discs.append(discount(r_B_T, c["discount"]).mean())
        infos.append({k: np.mean(v) for k, v in tb.info})
    keys = sorted(infos[0])
    np.savez_compressed(
        OUT, case=json.dumps(c), ret=np.array(rets), retstd=np.array(stds), disc_ret=np.array(discs),
        info_keys=np.array(keys), info=np.array([[d[k] for k in keys] for d in infos]),
        ep_ret=np.array([[ep[a].r_T.sum() for a in range(A)] for ep in episodes]),
        ep_len=np.array([len(ep[0].r_T) for ep in episodes], np.int32),
        ep_info=np.array([[np.sum(ep[0].info_D[k]) for k in ("evcatches", "pocatches")] for ep in episodes], np.int64),
        min_norm=min_norm)
    print("wrote", OUT, "ret", np.round(rets, 4), "lengths", [len(ep[0].r_T) for ep in episodes],
          "catches", [[int(np.sum(ep[0].info_D[k])) for k in ("evcatches", "pocatches")] for ep in episodes],
          "min joint norm %.3g" % min_norm)


if __name__ == "__main__":
    main()
