"""Waterworld's default launch geometry (needs a GPU).

Unless set_launch says otherwise, an open-loop Waterworld rollout with float32 observations and whole-step
staging keeps at most 16 one-warp blocks per SM when it is at least 16 steps long and 16 x SMs warps split
its envs into rounds whose last is at least 4/5 full (csrc/waterworld.cu, ww_default_blocks_per_sm, which
madrl_ww_default_blocks_per_sm reports and the launch uses).  The test checks that rule on this card's SM
count, and that bench.py's headline batch (C2, 4 096 envs), which it caps, computes bit for bit what an
explicit 16-block launch and a launch with as many blocks as fit (one warp per env on an H100) compute.
"""
import pytest
import torch

from madrl_b200 import BatchedMAWaterWorld, _lib

pytestmark = pytest.mark.gpu

C2 = dict(n_pursuers=5, n_evaders=5)
C4 = dict(n_pursuers=20, n_evaders=50, n_poison=50)
T, MPL, SEED = 16, 5, 21


def n_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def default_cap(eng, T):
    v = _lib.lib().madrl_ww_default_blocks_per_sm(eng._h, T)
    assert v >= 0
    return v


def expected_cap(E, T):
    g = 16 * n_sms()
    rounds = -(-E // g)
    return 16 if T >= 16 and rounds >= 2 and 5 * (E - (rounds - 1) * g) >= 4 * g else 0


@pytest.mark.parametrize("per_sm", [10, 16.5, 20, 25, 29, 31, 40, 46, 62])
def test_default_cap_rule(per_sm):
    E = int(per_sm * n_sms())
    eng = BatchedMAWaterWorld(E, **C2, device="cuda", seed=0)
    for t in (1, 15, 16, 256):
        assert default_cap(eng, t) == expected_cap(E, t), (E, t)
    assert default_cap(BatchedMAWaterWorld(E, **C2, device="cuda", obs_dtype=torch.bfloat16), 256) == 0
    assert default_cap(BatchedMAWaterWorld(E, **C4, device="cuda"), 256) == 0   # ring staging


def bits(x):
    return x.view(torch.int32) if x.dtype == torch.float32 else x


def run(E, bps):
    eng = BatchedMAWaterWorld(E, **C2, device="cuda", seed=SEED, max_path_length=MPL)
    if bps is not None:
        eng.set_launch(blocks_per_sm=bps)
    obs0 = eng.reset()
    g = torch.Generator(device="cuda")
    g.manual_seed(3)
    act = torch.randn(T, E, 5, 2, device="cuda", generator=g) * 0.7
    outs = (obs0,) + tuple(eng.rollout(act, auto_reset=True))
    torch.cuda.synchronize()
    return eng, outs, {k: v.clone() for k, v in eng.state.items()}


def test_capped_default_launch_equals_explicit_launches():
    E = 4096
    assert E > 16 * n_sms()   # the capped launch steps several envs on some warps
    eng, got, got_state = run(E, None)
    assert default_cap(eng, T) == 16
    assert int(got[3].sum()) >= E * (T // MPL)   # auto-resets happened
    for bps in (16, 32):
        _, want, want_state = run(E, bps)
        for k, (a, b) in enumerate(zip(got, want)):
            assert a.shape == b.shape and torch.equal(bits(a), bits(b)), (bps, k)
        for k in want_state:
            assert torch.equal(bits(got_state[k]), bits(want_state[k])), (bps, k)
