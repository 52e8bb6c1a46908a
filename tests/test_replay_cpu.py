"""oracle/replay_oracle.py against tests/golden/replay_pool_ref.npz, which rllab's own DDPG.train and MAReplayPool
wrote on a scripted env (oracle/make_replay_golden.py): horizon cuts dropped and kept, a termination exactly at the
horizon, env-terminal events, and a pool of 13 slots that wraps several times.  Fed the run's engine-shaped rollout,
the oracle's ring arrays and counters equal the reference's bit for bit (rewards: the float32 rounding of the
reference's float64), and at every recorded pool state the reference's random_batch accepts exactly the slots
[0, size - 1) that the device sampler draws from."""
import os

import numpy as np
import pytest

from conftest import GOLDEN_DIR
from oracle import replay_oracle as ro

GOLDEN = np.load(os.path.join(GOLDEN_DIR, "replay_pool_ref.npz"))
CASES = ("cuts", "cuts_kept", "at_limit", "events")


def f32(x):
    """float32 of float64 values that must be float32-representable."""
    y = x.astype(np.float32)
    assert np.array_equal(y.astype(np.float64), x)
    return y


@pytest.mark.parametrize("case", CASES)
def test_oracle_pool_equals_the_reference_loop(case):
    g = {k.split("__", 1)[1]: v for k, v in GOLDEN.items() if k.startswith(case + "__")}
    mpl, limit, include, M = (int(x) for x in g["config"])
    orc = ro.ReplayOracle(M, g["observations"].shape[1], g["actions"].shape[1], scale_reward=0.01,
                          include_horizon_terminal_transitions=bool(include))
    zero = np.zeros(1, np.int32)
    orc.add(f32(g["obs"]), f32(g["act"]), f32(g["rew"]), g["done"], f32(g["obs_before"]), f32(g["term"]), zero, zero,
            mpl, limit)
    for name in ("observations", "next_observations", "actions"):
        assert np.array_equal(getattr(orc, name), f32(g[name])), name
    assert np.array_equal(orc.rewards, g["rewards"].astype(np.float32))
    assert np.array_equal(orc.terminals, g["terminals"])
    assert [orc.top, orc.bottom, orc.size] == g["ring"].tolist()
    assert g["done"].sum() > 0 and g["terminals"].any() == (case != "cuts")


@pytest.mark.parametrize("case", CASES)
def test_reference_random_batch_accepts_all_but_the_newest_slot(case):
    states, slots, counts = (GOLDEN["%s__%s" % (case, k)] for k in ("acc_state", "acc_slots", "acc_count"))
    M = int(GOLDEN[case + "__config"][3])
    assert len(states) > 10 and (states[:, 1] == M).any() and (states[:, 1] < M).any()   # before and after full
    got = np.split(slots, np.cumsum(counts)[:-1])
    for (bottom, size), acc in zip(states, got):
        assert np.array_equal(acc, np.arange(size - 1)), (bottom, size)
        assert np.array_equal(acc, ro.accepted_candidates(bottom, size, M))


def test_sample_indices_stay_in_range():
    for size in (1, 2, 3, 40, 500000):
        idx = ro.sample_indices(7, 123, 5000, size)
        assert idx.min() >= 0 and idx.max() < max(size - 1, 1)
    u = np.array([0, 1, 2 ** 63, 2 ** 64 - 1], np.uint64)
    assert ro.mulhi64(u, 2 ** 64 - 1).tolist() == [(int(x) * (2 ** 64 - 1)) >> 64 for x in u]


@pytest.mark.parametrize("mode", ["centralized", "concurrent"])
def test_oracle_refuses_other_control_modes(mode):
    with pytest.raises(NotImplementedError):
        ro.ReplayOracle(10, 3, 2, mode=mode)
