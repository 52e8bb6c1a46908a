"""Waterworld's float32 sensing of a pursuer that sits exactly on another one, in the warp emulator of tests/emu.

Pursuers are clipped to [0, 1], so two of them can share a corner.  The coincident pursuer's relative position is
(+0, +0), and a sensor's projection onto it is sx * 0 + sy * 0: +0.0, or -0.0 for the sensors with both components
negative.  The reference's test is `sensorvals < 0`, which a zero of either sign passes, so every sensor senses the
other pursuer at distance 0 and its relative speed 0, the sign of each zero being that of the projection.  The other
objects are placed beyond sensor range, so these two rows of the corner pursuers are known exactly.  Both the
one-warp kernel and the writer-warp kernel (set_obs_writer ON) run."""
import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)
from emu import driver
from madrl_b200 import _lib as L

pytestmark = driver.needs_cxx

E, NP, NE, NPO, K = 4, 5, 5, 10, 30
CORNER = (0, 1)   # the pursuers driven into (1, 1)


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


@pytest.mark.parametrize("writer", [L.WW_OBS_WRITER_OFF, L.WW_OBS_WRITER_ON], ids=["one_warp", "writer"])
def test_coincident_pursuers_are_sensed_at_signed_zero(writer):
    from emu.driver import EmuWaterworld
    eng = EmuWaterworld(E, n_pursuers=NP, n_evaders=NE, n_poison=NPO, n_sensors=K, seed=7, fp64=False)
    assert eng.lib.madrl_ww_set_obs_writer(eng._h, writer) == 0
    eng.reset()
    Ly, N = eng.layout, int(eng.layout.n_obj)
    objs = eng.view(Ly.objs, np.float32, (E, 4, N))
    objs[:, 2:4] = 0.0                                   # nothing moves this step
    objs[:, 0, :NP] = [1.0, 1.0, 0.5, 0.3, 0.7]          # pursuers 0 and 1 share the corner, 2-4 far from it
    objs[:, 1, :NP] = [1.0, 1.0, 0.2, 0.5, 0.1]
    others = np.arange(N - NP, dtype=np.float32)
    objs[:, 0, NP:] = 0.05 + 0.02 * others               # evaders and poisons along the bottom-left edge
    objs[:, 1, NP:] = 0.05
    obst = eng.view(Ly.obst, np.float32, (E, 2))
    obst[:] = 0.5

    obs = eng.rollout(np.zeros((1, E, NP, 2), np.float32), auto_reset=False)[0][0]

    s = eng.view(Ly.sensors, np.float32, (2, K))
    zero = np.float32(0.0)
    proj = s[0] * zero + s[1] * zero                     # the projection onto (+0, +0): -0.0 where both are negative
    assert np.signbit(proj).sum() > 0, "no sensor points into the negative quadrant"
    want = np.concatenate([proj, proj]).view(np.uint32)   # distance 0 and relative speed 0, with the projection's sign
    for e in range(E):
        for p in CORNER:
            got = obs[e, p, 5 * K:7 * K].view(np.uint32)
            assert np.array_equal(got, want), (e, p, obs[e, p, 5 * K:7 * K], proj)
            # nothing else is in range: no evader, poison or obstacle feature
            assert not obs[e, p, :5 * K].any(), (e, p)
