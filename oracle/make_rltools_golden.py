"""Writes tests/golden/rltools_samples_ref.npz: rltools' sample processing run with the REFERENCE's own code on
scripted rollouts cut into paths, over an iteration-0 extra batch and two iterations, in rltools' training-loop
order (rltools/rltools/algos/policyopt.py:45-70, concurrent :199-231):
  extra batch       baseline.update_obsnorm and rewnorm.update (per agent, in agent order, when concurrent)
  each iteration    Sampler.process (rltools/rltools/samplers/__init__.py:35-88) per batch, then rewnorm.update
                    with each batch's rewards in batch order

Executed from reference source: ``Sampler.process`` and ``Trajectory`` / ``TrajBatch`` (oracle.refshim's
load_rltools_samplers), ``rltools.util.discount`` and ``safezip`` (util.py lines 56-80 and 90-92, executed from the source text:
the file as a whole does not parse on Python 3), ``baselines/linear.py`` (TensorFlow stubbed; its module-level ``scipy`` is a
proxy whose ``linalg.solve`` translates ``sym_pos=True`` to ``assume_a="pos"``, which SciPy 1.18 requires) and
``baselines/zero.py``.  NOT executed from reference source: ``nn.Standardizer``, which needs TensorFlow; the
oracle's float32 NumPy restatement (oracle/rltools_oracle.py: ``Standardizer``) stands in for it, for the
baselines' obsnorm and the sampler's rewnorm alike.

Observations and rewards are fed as float64 arrays of float32-representable values, as the reference envs emit
them.  Control modes (paths: oracle.recurrent_oracle.rollout_paths): decentralized (one batch, one baseline),
concurrent (one batch and one independent baseline per agent, one shared rewnorm), centralized (the agents'
observations side by side, agent 0's reward), and ``zero`` (decentralized with ZeroBaseline).

Cases:
  ragged  T 9, E 4, A 2, D 5, obs_before, obsnorm and rewnorm on; length-1 paths at t = 0 and t = T-1, an env
          with no done; rewards follow the observations, so the second iteration's fit predicts well (v_r > 0)
  plain   T 7, E 3, A 3, D 3, bfloat16-representable observations, no obs_before, obsnorm and rewnorm off; rewards
          independent of the observations, so the second iteration falls back to the time baseline (v_r < 0)
Every v_r of a fitted baseline is asserted to lie more than 1e-3 from 0, so that no decision rests on rounding.
Run:  python -m oracle.make_rltools_golden
"""
import importlib.util
import os
import sys
import types

import numpy as np
import scipy.linalg

from oracle import refshim
from oracle import rltools_oracle as ro
from oracle.make_recurrent_golden import _bf16

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "rltools_samples_ref.npz")
MODES = ("decentralized", "concurrent", "centralized", "zero")


def _rollout(rs, T, E, A, D, cuts, bf16, with_before, coupled):
    done = np.zeros((T, E), np.uint8)
    for e, steps in enumerate(cuts):
        done[list(steps), e] = 1
    cvt = _bf16 if bf16 else (lambda x: x)
    obs = cvt((rs.randn(T, E, A, D) * 2 + 0.5).astype(np.float32))
    it = dict(obs=obs, done=done)
    if with_before:
        it["obs_before"] = cvt((rs.randn(E, A, D) * 2 + 0.5).astype(np.float32))
    if coupled:         # the reward of a step follows the observation its action was taken in
        seen = np.concatenate([it["obs_before"][None], obs[:-1]]) if with_before else obs
        rew = seen[..., 0] * 1.5 - seen[..., 1] + rs.randn(T, E, A) * 0.05 + 0.3
    else:
        rew = rs.randn(T, E, A) * 2 + 0.3
    rew = rew.astype(np.float32)
    it["rew"] = rew
    it["rew_cent"] = np.repeat(rew[..., :1], A, axis=2)
    return it


def cases():
    rs = np.random.RandomState(20261016)
    ragged = dict(discount=0.99, gae_lambda=0.95, obsnorm=True, rewnorm=True)
    cut = [(0, 4), (2, 8), (), (3, 5, 6)]
    ragged["rollouts"] = [_rollout(rs, 9, 4, 2, 5, c, False, True, True)
                          for c in (cut, cut, [(), (0,), (1, 7), (8,)])]
    plain = dict(discount=0.95, gae_lambda=1.0, obsnorm=False, rewnorm=False)
    plain["rollouts"] = [_rollout(rs, 7, 3, 3, 3, c, True, False, False)
                         for c in ([(2,), (6,), ()], [(2,), (6,), ()], [(0, 1), (), (3,)])]
    return dict(ragged=ragged, plain=plain)


def load_reference():
    """(Sampler, TrajBatch, Trajectory, LinearFeatureBaseline, ZeroBaseline) from the reference files."""
    root = os.path.join(refshim.REFERENCE_ROOT, "rltools", "rltools")
    refshim.install()
    rl = sys.modules["rltools"]
    rl.nn = refshim._module("rltools.nn", Standardizer=ro.Standardizer, NoOpStandardizer=ro.NoOpStandardizer)
    with open(os.path.join(root, "util.py")) as f:
        lines = f.readlines()
    ns = dict(np=np)
    for first, last, fn in ((56, 80, "discount"), (90, 92, "safezip")):    # 1-based, inclusive
        src = "".join(lines[first - 1:last])
        assert src.startswith("def %s(" % fn)
        exec(compile(src, os.path.join(root, "util.py"), "exec"), ns)
        setattr(sys.modules["rltools.util"], fn, ns[fn])
    samplers = refshim.load_rltools_samplers()

    class _Scope(object):
        def __init__(self, *a, **k):
            pass

        def __enter__(self):
            return self

        def __exit__(self, *a):
            return False

    refshim._module("tensorflow", variable_scope=_Scope)

    def load(name, rel):
        spec = importlib.util.spec_from_file_location(name, os.path.join(root, rel))
        mod = importlib.util.module_from_spec(spec)
        sys.modules[name] = mod
        spec.loader.exec_module(mod)
        return mod

    rl.baselines = load("rltools.baselines", "baselines/__init__.py")
    linear = load("_ref_rltools_linear", "baselines/linear.py")
    zero = load("_ref_rltools_zero", "baselines/zero.py")

    def solve(a, b, sym_pos=False, **kw):
        return scipy.linalg.solve(a, b, assume_a="pos" if sym_pos else kw.pop("assume_a", "gen"), **kw)

    linear.scipy = types.SimpleNamespace(linalg=types.SimpleNamespace(solve=solve))
    tj = sys.modules["rltools.trajutil"]
    return samplers.Sampler, tj.TrajBatch, tj.Trajectory, linear.LinearFeatureBaseline, zero.ZeroBaseline


def main():
    Sampler, TrajBatch, Trajectory, Linear, Zero = load_reference()

    def trajbatch(paths):
        return TrajBatch.FromTrajs([Trajectory(p["observations"], np.zeros((len(p["rewards"]), 1)),
                                               np.zeros((len(p["rewards"]), 1)), p["rewards"], {}) for p in paths])

    arrays = {}
    for name, case in cases().items():
        arrays[name + "/settings"] = np.array([case["discount"], case["gae_lambda"], case["obsnorm"],
                                               case["rewnorm"]], np.float64)
        for k, it in enumerate(case["rollouts"]):
            for key, v in it.items():
                arrays["%s/r%d/%s" % (name, k, key)] = v
        A = case["rollouts"][0]["obs"].shape[2]
        D = case["rollouts"][0]["obs"].shape[3]
        for mode in MODES:
            pm = "decentralized" if mode == "zero" else mode
            nb, od = (A if pm == "concurrent" else 1), (A * D if pm == "centralized" else D)
            space = types.SimpleNamespace(shape=(od,))
            bls = [Zero(space) if mode == "zero" else Linear(space, case["obsnorm"]) for _ in range(nb)]
            sampler = Sampler.__new__(Sampler)
            sampler.algo = types.SimpleNamespace(discount=case["discount"])
            sampler.rewnorm = (ro.Standardizer if case["rewnorm"] else ro.NoOpStandardizer)(1)
            for k, it in enumerate(case["rollouts"]):
                rew = it["rew_cent"] if pm == "centralized" else it["rew"]
                tbs = [trajbatch(ps) for ps in ro.batches(it["obs"], rew, it["done"], it.get("obs_before"), pm)]
                key = "%s/%s/r%d/" % (name, mode, k)
                if k == 0:                                          # the extra batch (policyopt.py:49-54)
                    for bl, tb in zip(bls, tbs):
                        if mode != "zero":
                            bl.update_obsnorm(tb.obs.stacked, None)
                        sampler.rewnorm.update(tb.r.stacked[:, None])
                else:
                    for b, (bl, tb) in enumerate(zip(bls, tbs)):
                        vals, _ = sampler.process(None, k, tb, case["discount"], case["gae_lambda"], bl)
                        fitted = mode != "zero" and not (k == 1)
                        if fitted:
                            assert abs(vals["v_r"]) > 1e-3, (name, mode, k, vals["v_r"])
                        sub = key + ("a%d/" % b if pm == "concurrent" else "")
                        arrays[sub + "adv"] = np.concatenate(vals["advantage"].arrays)
                        arrays[sub + "q"] = vals["qval"].stacked
                        arrays[sub + "stats"] = np.array([vals["v_r"], vals["tv_r"], vals["v_r"] < 0], np.float64)
                        if mode != "zero":
                            arrays[sub + "w"] = np.asarray(bl.w_Df, np.float64)
                    for tb in tbs:                                 # policyopt.py:69-70, :229-231
                        sampler.rewnorm.update(tb.r.stacked[:, None])
                for b, bl in enumerate(bls):
                    if mode != "zero" and case["obsnorm"]:
                        sub = key + ("a%d/" % b if pm == "concurrent" else "")
                        on = bl.obsnorm
                        arrays[sub + "obsnorm"] = np.concatenate([on.count, on.mean.ravel(), on.meansq.ravel()])
                if case["rewnorm"]:
                    rn = sampler.rewnorm
                    arrays[key + "rewnorm"] = np.concatenate([rn.count, rn.mean.ravel(), rn.meansq.ravel()])
    fb = [bool(v[2]) for k, v in arrays.items() if k.endswith("/stats") and "/zero/" not in k and "/r2/" in k]
    assert any(fb) and not all(fb), fb
    np.savez_compressed(OUT, **arrays)
    print("wrote", OUT)


if __name__ == "__main__":
    main()
