"""Waterworld's writer-warp observation path (madrl_ww_set_obs_writer) in the warp emulator of tests/emu: the
writer-warp kernel (set_obs_writer ON) against the one-warp kernel (OFF) on the same seeded float32 rollouts.
Observations, rewards, dones, infos, terminal observations and the state blob must be byte-identical.  The ring's
mbarriers are the only synchronisation between the env warps and the writer.  The emulated mbarriers (csrc/common.cuh)
make a waiting warp yield until the phase completes, so the writer copies what the env warps staged and they do not
overwrite a slot before it is copied; otherwise the observations differ.  A phase that never completes (a missing
arrival) aborts the launch.  The hazard checker follows __syncwarp / __syncthreads only, so it checks each env
warp's own staging (zero hazards), and the writer's reads of the ring are not recorded.

The emulator has two "SMs" and one resident block each, so with 8 env warps per block 20 envs make three groups:
block 0 steps groups 0 and 2 (a partial one of 4 envs), one after the other through the same ring.  Also the
launches that must fall back to the one-warp kernel (a step stride or observation base that is not 16-byte aligned)
and the argument errors of set_obs_writer.  Every layout of tests/ww_writer_edges.py's case table runs the same way,
and so do the ring geometries the build allows (MADRL_WW_WRITER_SLOTS, MADRL_WW_WRITER_ENVS), with either copy of a
slot: a new geometry or layout passes here, where a missing arrival aborts the launch, before it runs on a GPU."""
import numpy as np
import pytest

from conftest import ROOT  # noqa: F401  (puts the repository on sys.path)
from emu import driver
from emu.driver import Guarded
from emu.driver import ptr as _p
from madrl_b200 import _lib as L
from ww_writer_edges import BY_NAME, CASES, tail_events

pytestmark = driver.needs_cxx

C2 = dict(n_pursuers=5, n_evaders=5)
MPL = 5


@pytest.fixture(autouse=True)
def no_shared_memory_hazards():
    driver.races()
    yield
    assert driver.races() == 0, "shared-memory hazard reported by the emulator (see stderr)"


# the writer warp's two ways of copying a slot out: one bulk store (the default build), 16-byte stores
WRITERS = {"bulk": (), "stores": ("-DMADRL_WW_WRITER_BULK=0",)}


def engines(E, defines=(), cfg=C2):
    from emu.driver import EmuWaterworld
    out = []
    for mode in (L.WW_OBS_WRITER_OFF, L.WW_OBS_WRITER_ON):
        eng = EmuWaterworld(E, seed=17, env_id_base=2, fp64=False, max_path_length=MPL, defines=defines, **cfg)
        assert eng.lib.madrl_ww_set_obs_writer(eng._h, mode) == 0
        out.append(eng)
    return out


def rollout(eng, act, auto_reset=True, term=False, obs_offset=0):
    """One rollout into canary-guarded buffers; `obs_offset` bytes shift the observation base."""
    T, E, A, D = act.shape[0], eng.n_envs, eng.n_agents, eng.obs_dim
    n = T * E * A * D
    o = Guarded((n + 4,), np.float32, np.nan)
    r = Guarded((T, E, A), np.float32, np.nan)
    d = Guarded((T, E), np.uint8, 255)
    i = Guarded((T, E, 2), np.int32, -1)
    tb = Guarded((T, E, A, D), np.float32, -3.0) if term else None
    if term:
        assert eng._f("set_terminal_obs")(eng._h, _p(tb.arr)) == 0
    obs_ptr = o.arr.ctypes.data + obs_offset
    assert eng._f("rollout")(eng._h, T, _p(np.ascontiguousarray(act)), obs_ptr, _p(r.arr), _p(d.arr), _p(i.arr),
                             int(auto_reset), None) == 0
    if term:
        assert eng._f("set_terminal_obs")(eng._h, None) == 0
    obs = o.check("obs").view(np.uint8)[obs_offset:obs_offset + 4 * n]
    return [obs, r.check("rew"), d.check("done"), i.check("info")] + ([tb.check("term")] if term else [])


def compare(engs, act, **kw):
    a, b = (rollout(e, act, **kw) for e in engs)
    for x, y, name in zip(a, b, ("obs", "rew", "done", "info", "term")):
        assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
    assert np.array_equal(engs[0].blob, engs[1].blob), "state blobs differ"
    return a


def desync_sequence(engs, T1=13, T2=11, seed=8):
    """From reset: a T1-step auto-reset rollout, a masked reset of every other env (so that paths end at other steps
    than their neighbours'), a T2-step one, and 3 steps without auto-reset; the writer and the one-warp kernel must
    agree on each -> the outputs of the three rollouts."""
    E, Np = engs[0].n_envs, engs[0].n_agents
    for eng in engs:
        eng.reset()
    rs = np.random.RandomState(seed)
    act = rs.randn(T1, E, Np, 2).astype(np.float32)
    first = compare(engs, act, term=True)
    assert first[2].sum() >= E * (T1 // MPL)
    mask = (np.arange(E) % 2).astype(np.uint8)
    for eng in engs:
        eng.reset(mask)
    second = compare(engs, rs.randn(T2, E, Np, 2).astype(np.float32), term=True)
    assert (second[2][:, :-1] != second[2][:, 1:]).any()
    return first, second, compare(engs, act[:3], auto_reset=False)


@pytest.mark.parametrize("writer", sorted(WRITERS))
@pytest.mark.parametrize("E", [20, 19], ids=["aligned", "odd"])
def test_writer_equals_one_warp_kernel(E, writer):
    """E = 20: 16-byte-aligned step stride (20 * 5 * 213 floats), three groups; E = 19: the launch falls back."""
    desync_sequence(engines(E, WRITERS[writer]))


def assert_events(runs, case):
    """Catches and both kinds of collision (the rows' tail flags) happened."""
    assert sum(int(r[3].sum()) for r in runs) > 0, "no catch"
    assert min(sum(tail_events(r[0].view(np.float32), case)[i] for r in runs) for i in (0, 1)) > 0, "no collision"


@pytest.mark.parametrize("case", CASES, ids=str)
def test_case_table_writer_equals_one_warp_kernel(case):
    """Each layout of the case table at E = 20 (three groups over the two SMs, the last a partial one of 4 envs) and
    odd step counts; stage_over and obj33 fall back to the one-warp kernel."""
    assert case.E(20) == 20
    assert_events(desync_sequence(engines(20, cfg=case.cfg), T1=9, T2=7), case)


# ring geometries of the build: MADRL_WW_WRITER_SLOTS steps in flight, MADRL_WW_WRITER_ENVS env warps per block
GEOMETRIES = {"slots3": ("-DMADRL_WW_WRITER_SLOTS=3",), "envs4": ("-DMADRL_WW_WRITER_ENVS=4",),
              "envs16": ("-DMADRL_WW_WRITER_ENVS=16",)}


@pytest.mark.parametrize("writer", sorted(WRITERS))
@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
@pytest.mark.parametrize("name", ["c2", "k30_plain"])
def test_ring_geometries(name, geometry, writer):
    """Five groups over the two SMs, so that block 0 walks three through its ring.  The last group holds 4 envs for c2
    (a full one with 4 env warps per block) and 2 for k30_plain, whose stride allows any E."""
    case = BY_NAME[name]
    envs = 16 if geometry == "envs16" else (4 if geometry == "envs4" else 8)
    E = 4 * envs + (4 if name == "c2" else 2)
    assert case.E(E) == E
    desync_sequence(engines(E, GEOMETRIES[geometry] + WRITERS[writer], cfg=case.cfg), T1=9, T2=7)


def test_misaligned_observation_base_falls_back():
    engs = engines(20)
    for eng in engs:
        eng.reset()
    compare(engs, np.random.RandomState(9).randn(7, 20, 5, 2).astype(np.float32), term=True, obs_offset=4)


def test_set_obs_writer_arguments():
    from emu.driver import EmuWaterworld
    lib = driver.load()
    f = lib.madrl_ww_set_obs_writer
    assert f.argtypes == list(L.SIGNATURES["madrl_ww_set_obs_writer"][1])
    assert f(None, L.WW_OBS_WRITER_ON) == -1 and b"NULL" in lib.madrl_last_error()
    eng = EmuWaterworld(2, **C2, fp64=True)
    for bad in (-1, 3, 1 << 30):
        assert f(eng._h, bad) == -1 and b"unknown observation writer mode" in lib.madrl_last_error()
    for mode in (L.WW_OBS_WRITER_AUTO, L.WW_OBS_WRITER_OFF, L.WW_OBS_WRITER_ON):
        assert f(eng._h, mode) == 0
