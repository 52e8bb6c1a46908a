"""The oracle's evader controllers against the real reference (tests/golden/pe_evaders.npz, oracle/make_evaders_golden.py):
SingleActionPolicy(4) with surround capture, SingleActionPolicy(1) with n_catch capture, and a table replayed by
original evader index under random_opponents, over several episodes -- observations, rewards, dones, removed counts
and model_state (taken before the step's removals) step by step.  tests/test_pursuit_evaders_gpu.py holds the engine
to the oracle."""
import os

import numpy as np
import pytest

from oracle.philox import Stream
from oracle.pursuit_evaders_oracle import PursuitEvadersOracle

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "pe_evaders.npz")
MAPS = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
SEED = 5
RUNS = {
    "stay_surround": dict(n_evaders=6, n_pursuers=24, obs_range=5, surround=True, sample_maps=True, reward_mech='local'),
    "right_ncatch": dict(n_evaders=5, n_pursuers=6, obs_range=3, surround=False, n_catch=1, sample_maps=True,
                         reward_mech='global'),
    "table_random_opp": dict(n_evaders=8, n_pursuers=6, obs_range=5, surround=False, n_catch=1, sample_maps=True,
                             random_opponents=True, max_opponents=9, reward_mech='local'),
}


@pytest.mark.parametrize("name", sorted(RUNS))
def test_oracle_evader_controllers_match_reference(name):
    g = np.load(GOLDEN)
    r = {k.split("/", 1)[1]: g[k] for k in g.files if k.startswith(name + "/")}
    o = PursuitEvadersOracle(MAPS, rng=Stream(SEED, 0), **RUNS[name])
    ep = 0
    assert np.array_equal(np.array(o.reset()), r["obs0"][0])
    assert np.array_equal(o.model_state, r["model_state0"][0])
    for t in range(len(r["act"])):
        ev = int(r["a"]) if str(r["kind"]) == "fixed" else r["table"][t]
        obs, rew, done, info = o.step(r["act"][t], ev)
        assert np.array_equal(np.array(obs), r["obs"][t]), t
        assert np.array_equal(np.asarray(rew, np.float64), r["rew"][t]), t
        assert done == bool(r["done"][t]) and info["removed"] == r["removed"][t], t
        assert np.array_equal(o.model_state, r["model_state"][t]), t
        if done:
            ep += 1
            assert np.array_equal(np.array(o.reset()), r["obs0"][ep])
            assert np.array_equal(o.model_state, r["model_state0"][ep])
    assert ep + 1 == len(r["starts"])


def test_oracle_fed_random_controller_actions_equals_random_oracle():
    """The random controller's own actions, read off the stream before each step, given as evader actions: the same
    trajectory and stream position as the unchanged PursuitOracle (the counter rule)."""
    from oracle.pursuit_oracle import PursuitOracle
    cfg = RUNS["table_random_opp"]
    base = PursuitOracle(MAPS, rng=Stream(SEED, 3), **cfg)
    o = PursuitEvadersOracle(MAPS, rng=Stream(SEED, 3), **cfg)
    assert np.array_equal(np.array(base.reset()), np.array(o.reset()))
    act = np.random.RandomState(1).randint(0, 5, size=(60, cfg["n_pursuers"]))
    for t in range(len(act)):
        s = Stream(SEED, 3, 0, o.rng.counter)
        ev = np.full(cfg["n_evaders"], 7)
        for j in np.flatnonzero(~o.gone):
            ev[j] = s.randint(5)
        want, got = base.step(act[t]), o.step(act[t], ev)
        assert np.array_equal(np.array(want[0]), np.array(got[0])) and want[2:] == got[2:], t
        assert np.array_equal(want[1], got[1]) and np.array_equal(base.model_state, o.model_state), t
        assert base.rng.counter == o.rng.counter, t
        if want[2]:
            assert np.array_equal(np.array(base.reset()), np.array(o.reset()))
