"""rltools' sample processing without a GPU: the NumPy oracle (oracle/rltools_oracle.py) against the golden the
reference's own Sampler.process and LinearFeatureBaseline wrote (oracle/make_rltools_golden.py), and the argument
checks of the Python entry points that run before any pointer reaches the library."""
import os

import numpy as np
import pytest
import torch

from oracle import rltools_oracle as ro

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "rltools_samples_ref.npz")
CASES = ("ragged", "plain")
MODES = ("decentralized", "concurrent", "centralized", "zero")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case", CASES)
def test_oracle_reproduces_the_reference(golden, case, mode):
    settings, rollouts = ro.golden_case(golden, case)
    for k, res, bls, rewnorm in ro.replay(settings, rollouts, mode):
        key = "%s/%s/r%d/" % (case, mode, k)
        for b, bl in enumerate(bls):
            sub = key + ("a%d/" % b if mode == "concurrent" else "")
            if res is not None:
                r = res[b]
                np.testing.assert_allclose(np.concatenate(r["q"]), golden[sub + "q"], rtol=1e-12, atol=1e-12)
                np.testing.assert_allclose(np.concatenate(r["adv"]), golden[sub + "adv"], rtol=1e-12, atol=1e-12)
                st = golden[sub + "stats"]
                assert abs(r["v_r"] - st[0]) < 1e-12 and abs(r["tv_r"] - st[1]) < 1e-12
                assert r["fallback"] == bool(st[2])
                if bl is not None:
                    np.testing.assert_allclose(bl.w, golden[sub + "w"], rtol=1e-9, atol=1e-12)
            if bl is not None and settings["obsnorm"]:
                on = bl.obsnorm
                assert np.array_equal(np.concatenate([on.count, on.mean.ravel(), on.meansq.ravel()]),
                                      golden[sub + "obsnorm"].astype(np.float32))
        if settings["rewnorm"]:
            assert np.array_equal(np.concatenate([rewnorm.count, rewnorm.mean.ravel(), rewnorm.meansq.ravel()]),
                                  golden[key + "rewnorm"].astype(np.float32))


def test_golden_covers_both_sides_of_the_fallback(golden):
    fb = [bool(golden[k][2]) for k in golden.files if k.endswith("/stats") and "/r2/" in k and "/zero/" not in k]
    assert any(fb) and not all(fb)


def test_argument_checks_before_the_library():
    from madrl_b200 import rltools_sampler as rs
    T, E, A, D = 4, 3, 2, 5
    rew = torch.zeros(T, E, A)
    done = torch.zeros(T, E, dtype=torch.uint8)
    with pytest.raises(TypeError, match="q"):
        rs.time_baseline(rew.double(), done)
    with pytest.raises(ValueError, match="done"):
        rs.time_baseline(rew, done[:-1])
    with pytest.raises(ValueError, match="t0"):
        rs.time_baseline(rew, done, t0=torch.zeros(E + 1, dtype=torch.int32))
    with pytest.raises(ValueError, match="cuda"):
        rs.time_baseline(rew, done)
    with pytest.raises(ValueError, match="mode"):
        rs.process_samples(None, torch.zeros(T, E, A, D), done, rew, 0.99, 1.0, mode="bogus")
    with pytest.raises(ValueError, match="rew"):
        rs.process_samples(None, torch.zeros(T, E, A, D), done, rew[:, :, :1], 0.99, 1.0)
    with pytest.raises(TypeError, match="obs"):
        rs.process_samples(None, torch.zeros(T, E, A, D, dtype=torch.float64), done, rew, 0.99, 1.0)
    with pytest.raises(ValueError, match="done"):
        rs.sample_fields(rew, done.t())
    with pytest.raises(ValueError, match="n_agents"):
        rs.RunningStandardizer(D, "cpu", n_agents=0)
    st = rs.RunningStandardizer(D, "cpu")
    with pytest.raises(ValueError, match="x"):
        st.update(torch.zeros(7, D + 1))
    with pytest.raises(TypeError, match="x"):
        st.update(torch.zeros(7, D, dtype=torch.float64))
    with pytest.raises(ValueError, match="CUDA device"):
        st.update(torch.zeros(7, D))                   # host tensors never reach the kernels
    with pytest.raises(ValueError, match="count"):
        st.set_param_values(np.zeros(2), np.zeros(D), np.ones(D))
    with pytest.raises(ValueError, match="n_agents"):
        rs.RunningStandardizer(1, "cpu", 2).update_per_agent(torch.zeros(7, 2, 1))


def test_baseline_state_round_trip_includes_the_obsnorm():
    from madrl_b200 import rltools_sampler as rs
    a = rs.LinearFeatureBaseline(4, "cpu", True, n_agents=2)
    a.set_param_values((np.arange(14.).reshape(2, 7), (np.array([3., 5.], np.float32),
                                                       np.full((2, 4), 0.25, np.float32),
                                                       np.full((2, 4), 2.0, np.float32))))
    b = rs.LinearFeatureBaseline(4, "cpu", True, n_agents=2)
    b.set_param_values(a.get_param_values())
    (ca, na), (cb, nb) = a.get_param_values(), b.get_param_values()
    assert np.array_equal(ca, cb) and all(np.array_equal(x, y) for x, y in zip(na, nb))
    assert torch.equal(a.obsnorm.norm_table, b.obsnorm.norm_table)
    with pytest.raises(ValueError, match="obsnorm"):
        rs.LinearFeatureBaseline(4, "cpu", False, n_agents=2).set_param_values(a.get_param_values())
