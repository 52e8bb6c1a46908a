"""Cases shared by the edge tests of Waterworld's writer-warp kernel (ww_kernel<..., WRITER = true> in
csrc/waterworld.cu, DESIGN §4.1): tests/test_ww_writer_edges_gpu.py runs them on the device,
tests/test_emulated_obs_writer.py in the warp emulator of tests/emu.

The writer is instantiated for every single-chunk object count (OPL = 1, at most 32 objects), and ww_launch_t
picks its sensor instantiation from K: K = 30 with speed features -> KC = 30, any other K <= 32 -> KC = 0, KCH = 1,
K = 33..64 -> KCH = 2.  ww_use_writer then takes it only when the env-step's Np rows are staged whole
(obs_stage_bytes(Np D) <= kStepStageMaxBytes, i.e. Np D <= 1532 float32 values) and the observation base and step
stride E Np D are 16-byte aligned (E Np D = 0 mod 4).  Each case below fixes one such layout; `writer` says whether
the writer must run, and `e_step` is the smallest E multiple that keeps the stride aligned.  Radii are large
enough that catches and collisions (the rows' tail triples) happen within a few steps, which the tests assert."""
import math
import os
import re

import numpy as np

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "madrl_b200", "csrc")


def _source():
    with open(os.path.join(CSRC, "waterworld.cu")) as f:
        return f.read()


def csrc_define(name, source=None):
    """The default of a `#define name <int>` of csrc/waterworld.cu."""
    return int(re.search(r"#define %s (\d+)" % name, source or _source()).group(1))


WR_ENVS = csrc_define("MADRL_WW_WRITER_ENVS")                                     # env warps per writer block
WR_BLOCKS_PER_SM = csrc_define("MADRL_WW_WRITER_WARPS_PER_SM") // WR_ENVS         # the writer grid's blocks per SM
STAGE_MAX_BYTES = math.prod(int(f) for f in re.search(r"kStepStageMaxBytes = (\d+) \* (\d+);", _source()).groups())
# obs_stage_bytes(n, 4) = round_up(4 n, 16) + 16 <= STAGE_MAX_BYTES
STAGE_MAX_FLOATS = (STAGE_MAX_BYTES - 16) // 4


def obs_dim(cfg):
    return cfg.get("n_sensors", 30) * (7 if cfg.get("speed_features", True) else 4) + 2 + int(cfg.get("addid", True))


class Case(object):
    def __init__(self, name, writer, kch, kc, **cfg):
        self.name, self.writer, self.cfg = name, writer, cfg
        self.Np, self.D = cfg["n_pursuers"], obs_dim(cfg)
        self.n_obj = cfg["n_pursuers"] + cfg["n_evaders"] + cfg.get("n_poison", 10)
        self.e_step = 4 // math.gcd(self.Np * self.D, 4)
        # the instantiation the launch takes (the writer's template arguments when it runs)
        self.kch, self.kc = kch, kc
        assert (cfg.get("n_sensors", 30) + 31) // 32 == kch
        assert kc == (30 if cfg.get("n_sensors", 30) == 30 and cfg.get("speed_features", True) else 0)
        stages = self.Np * self.D <= STAGE_MAX_FLOATS
        assert writer == (stages and self.n_obj <= 32), name

    def E(self, n):
        """The smallest E >= n the stride rule allows."""
        return -(-n // self.e_step) * self.e_step

    def __repr__(self):
        return self.name


# Np / Ne / Npo, K, speed, addid; reward_mech 'global', n_coop 1 and 2 and a random obstacle spread over the cases
CASES = [
    Case("c2", True, 1, 30, n_pursuers=5, n_evaders=5, n_poison=10, radius=0.04, sensor_range=0.3),      # Np D = 1065
    Case("k30_plain", True, 1, 0, n_pursuers=6, n_evaders=8, n_poison=8, n_sensors=30, speed_features=False,
         addid=False, radius=0.04, n_coop=1, reward_mech="global"),                                       # 732
    Case("k17", True, 1, 0, n_pursuers=3, n_evaders=10, n_poison=12, n_sensors=17, radius=0.045, n_coop=1,
         obstacle_loc=None),                                                                              # 366
    Case("k64_plain", True, 2, 0, n_pursuers=5, n_evaders=6, n_poison=6, n_sensors=64, speed_features=False,
         radius=0.05, sensor_range=0.3, reward_mech="global"),                                            # 1295
    Case("k40_32obj", True, 2, 0, n_pursuers=3, n_evaders=20, n_poison=9, n_sensors=40, radius=0.04, n_coop=1,
         obstacle_loc=None),                                                                              # 849
    Case("np1", True, 1, 0, n_pursuers=1, n_evaders=1, n_poison=1, n_sensors=1, radius=0.1, obstacle_radius=0.05,
         n_coop=1, sensor_range=0.4, ev_speed=0.03, poison_speed=0.03),                                   # 10
    Case("np30", True, 1, 0, n_pursuers=30, n_evaders=1, n_poison=1, n_sensors=5, radius=0.04,
         reward_mech="global"),                                                                           # 1140
    Case("stage_max", True, 1, 30, n_pursuers=7, n_evaders=5, n_poison=10, radius=0.04, n_coop=1,
         obstacle_loc=None),                                                                              # 1491
    Case("stage_over", False, 1, 30, n_pursuers=8, n_evaders=5, n_poison=10, radius=0.04),              # 1704: ring
    Case("obj33", False, 2, 0, n_pursuers=3, n_evaders=20, n_poison=10, n_sensors=40, radius=0.04, n_coop=1),  # OPL 2
]
BY_NAME = {c.name: c for c in CASES}
assert BY_NAME["stage_max"].Np * BY_NAME["stage_max"].D <= STAGE_MAX_FLOATS < \
    (BY_NAME["stage_max"].Np + 1) * BY_NAME["stage_max"].D


def writer_kernel(case):
    """The demangled name of the writer-warp kernel a launch of `case` runs (as CUPTI spells it on an H100, and as
    the GPU tests spell the records of madrl_ww_launch_log)."""
    return "void madrl::ww_kernel<float, float, 1, %d, %d, false, 0, false, true>(madrl::WWParams<float, float>)" % (
        case.kch, case.kc)


def is_ww_kernel(name):
    return "ww_kernel<" in name


def is_writer(name):
    """A ww_kernel launch of the writer-warp instantiation (template argument WRITER = true)."""
    m = re.search(r"ww_kernel<([^>]*)>", name)
    return m is not None and m.group(1).replace(" ", "").endswith(",true")


def actions(rs, T, E, Np, std=0.7):
    return (rs.randn(T, E, Np, 2) * std).astype(np.float32)


def tail_events(obs, case):
    """How many rows have the touched-an-evader / touched-a-poison flags of their tail triple set."""
    n_feat = (7 if case.cfg.get("speed_features", True) else 4) * case.cfg.get("n_sensors", 30)
    tail = np.asarray(obs).reshape(-1, case.D)[:, n_feat:n_feat + 2]
    return int((tail[:, 0] != 0).sum()), int((tail[:, 1] != 0).sum())
