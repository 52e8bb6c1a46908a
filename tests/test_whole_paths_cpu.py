"""The whole-path selection rule (oracle/whole_paths_oracle.py, DESIGN §4.9) against the selection stored with the
real rllab processing in tests/golden/whole_paths_ref.npz (oracle/make_whole_paths_golden.py), and the rule's
properties on the golden's streams."""
import os

import numpy as np
import pytest

from oracle import whole_paths_oracle as wo

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "whole_paths_ref.npz")
CASES = ("ragged", "exact", "late")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("case", CASES)
def test_selection_matches_golden(golden, case):
    done, bs = golden[case + "/done"], int(golden[case + "/batch_size"])
    t_star, end = wo.select(done, bs)
    assert t_star == int(golden[case + "/t_star"])
    np.testing.assert_array_equal(end, golden[case + "/end"])
    ps = wo.path_start(done, end)
    np.testing.assert_array_equal(ps, golden[case + "/path_start"])
    A = golden[case + "/rew"].shape[2]
    # rllab's batch holds every kept path once per agent, each ending at a done, and at least batch_size env-steps
    assert len(golden[case + "/recurrent/it0/valids"]) == (len(ps) - 1) * A
    assert ps[-1] >= bs and wo.gather(done, end)[ps[1:] - 1].all()
    # the count of finished env-steps before t* is short of batch_size: t* is the first crossing
    assert wo.select(done[:t_star], bs) is None


def test_threshold_at_a_path_end_keeps_nothing_after_it(golden):
    done = golden["exact/done"]
    t_star, end = wo.select(done, int(golden["exact/batch_size"]))
    ended = np.nonzero(done[t_star])[0]
    assert len(ended) and (end[ended] == t_star).all() and (end >= t_star).all()


def test_in_flight_path_finishes_launches_later(golden):
    t_star, end = wo.select(golden["late/done"], int(golden["late/batch_size"]))
    assert end[4] - t_star >= 2 * int(golden["late/chunk"])
