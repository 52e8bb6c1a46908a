"""The env kernels where one warp steps several envs per launch (needs a GPU).

`engine_launch` (csrc/engine.cuh) launches min(E, SMs x resident blocks per SM) one-warp blocks; when E is
larger, warp w steps envs w, w + grid, w + 2 grid, ... one after another, reusing its shared memory
(Waterworld's candidate slots and the observation staging its TMA bulk stores read asynchronously,
Pursuit's cell words, stale windows and Philox block cache) for each.  The benchmark's Pursuit C3,
Waterworld C4 and Hostage C5 batches run that way.

Here `set_launch(blocks_per_sm=1)` makes the grid exactly G = SMs, and E = 3G + 5 envs makes warps 0-4 step
four envs and the others three.  Every entry point is then compared with

  * the same envs stepped one env per warp: shard engines of at most G envs whose `env_id_base` is their
    first env, at the default launch.  Outputs, terminal observations, recorded heuristic actions and the
    per-env state must be identical bit for bit; a bfloat16 engine's observations must be the float32
    shards' rounded with `.to(torch.bfloat16)`;
  * the float64 oracles, on envs that were the second, third or fourth env of their warp: fp64 Waterworld
    and Hostage within 1e-9, Pursuit bit-exact, the heuristic policies' actions included.
"""
import numpy as np
import pytest
import torch

from oracle.heuristics_oracle import policy_draw, pursuit_action, waterworld_action
from oracle.hostage_oracle import HostageOracle
from oracle.philox import Stream
from oracle.pursuit_oracle import PursuitOracle
from oracle.waterworld_oracle import WaterworldOracle
from test_heuristics import evader_window
from test_obs_bf16_gpu import C3, CONV, pool16, small_map
from test_waterworld_gpu import CFGS

pytestmark = pytest.mark.gpu

SEED, BASE, MPL = 13, 1000, 7
HW_C5 = (10, 16, 16, 4, 2)
BF16 = torch.bfloat16
BITS = {torch.float64: torch.int64, torch.float32: torch.int32, BF16: torch.int16}


def n_sms():
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def forced_wave():
    """(G, E): the grid of a `set_launch(blocks_per_sm=1)` engine of E = 3G + 5 envs."""
    G = n_sms()
    E = 3 * G + 5
    assert E > 2 * G
    return G, E


class Family(object):
    """One config of one env family: `make(n, env_id_base, obs_dtype)` builds its engine, `oracle(env_id)`
    its float64 oracle (None: not checked against it), `policy(oracle, env_id, prev_obs, actions)` checks
    one step of the in-kernel heuristic (None: the family has none).  `exact`: the oracle's values rounded
    to float32 equal the engine's, instead of being within 1e-9 of them."""

    def __init__(self, make, oracle, exact, policy=None, act_scale=0.7):
        self.make, self.oracle, self.exact, self.policy, self.act_scale = make, oracle, exact, policy, act_scale

    def close(self, want, got):
        want = np.asarray(want, dtype=np.float64).reshape(got.shape)
        if self.exact:
            return np.array_equal(want.astype(np.float32), got)
        return np.abs(want - got).max() < 1e-9


def ww_policy(o, env_id, prev, act):
    for i, a in enumerate(act):
        assert np.abs(waterworld_action(prev[i]) - a).max() < 1e-9, (env_id, i)


def pe_policy(cfg):
    R, flat = cfg['obs_range'], cfg.get('flatten', True)

    def check(o, env_id, prev, act):
        ctr = o.rng.counter   # the env's draw counter when `prev` was produced
        for q, a in enumerate(act):
            win = np.zeros((R, R, 4))
            win[..., 2] = evader_window(prev[q], R, flat)
            assert pursuit_action(win, lambda: policy_draw(SEED, env_id, ctr, q), True) == a, (env_id, q)
    return check


def waterworld(name, prec, mpl=MPL):
    from madrl_b200 import BatchedMAWaterWorld
    cfg, dtype = CFGS[name], torch.float64 if prec == "fp64" else torch.float32
    return Family(lambda n, base, obs_dtype=None: BatchedMAWaterWorld(
                      n, seed=SEED, env_id_base=base, max_path_length=mpl, dtype=dtype, obs_dtype=obs_dtype,
                      device="cuda", **cfg),
                  (lambda env_id: WaterworldOracle(rng=Stream(SEED, env_id), **cfg)) if prec == "fp64" else None,
                  False, ww_policy if cfg.get('speed_features', True) else None)


def pursuit(name):
    from madrl_b200 import BatchedPursuitEvade
    maps, cfg = (pool16(), C3) if name == "c3" else (small_map(), CONV)
    return Family(lambda n, base, obs_dtype=None: BatchedPursuitEvade(
                      n, maps, seed=SEED, env_id_base=base, max_path_length=MPL, obs_dtype=obs_dtype, device="cuda",
                      **cfg),
                  lambda env_id: PursuitOracle(maps, rng=Stream(SEED, env_id), **cfg), True, pe_policy(cfg))


def hostage(prec, mpl=MPL):
    from madrl_b200 import BatchedHostageWorld
    dtype = torch.float64 if prec == "fp64" else torch.float32
    return Family(lambda n, base, obs_dtype=None: BatchedHostageWorld(
                      n, *HW_C5, seed=SEED, env_id_base=base, max_path_length=mpl, dtype=dtype, obs_dtype=obs_dtype,
                      device="cuda"),
                  (lambda env_id: HostageOracle(*HW_C5, rng=Stream(SEED, env_id))) if prec == "fp64" else None,
                  False, act_scale=2.0)


def actions(fam, eng, T, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)
    shape = (T, eng.n_envs, eng._n_acting) + eng._act_tail
    if eng._act_dtype == torch.int32:
        return torch.randint(0, 5, shape, dtype=torch.int32, device="cuda", generator=g)
    return torch.randn(shape, dtype=eng._act_dtype, device="cuda", generator=g) * fam.act_scale


def check(got, refs, parts, dim, what):
    """`got` (the persistent-wave engine's tensor) sliced to each part along the env dimension `dim` equals that
    part's `refs` tensor bit for bit (a float32 one rounded to bfloat16 first when `got` is bfloat16)."""
    for (lo, hi), ref in zip(parts, refs):
        g = got.narrow(dim, lo, hi - lo)
        if g.dtype == BF16 and ref.dtype == torch.float32:
            ref = ref.to(BF16)
        ref = ref.to(g.device)
        assert g.dtype == ref.dtype and g.shape == ref.shape, (what, g.dtype, ref.dtype, g.shape, ref.shape)
        diff = g.view(BITS.get(g.dtype, g.dtype)) != ref.view(BITS.get(ref.dtype, ref.dtype))
        if bool(diff.any()):
            bad = (diff.movedim(dim, 0).reshape(hi - lo, -1).any(1).nonzero()[:, 0] + lo).tolist()
            raise AssertionError("%s differs at envs %s%s" % (what, bad[:10], " ..." if len(bad) > 10 else ""))


class Shards(object):
    """Envs [lo, hi) of each part, stepped by an engine of their own at the default launch: a part no larger
    than one wave gets one warp per env."""

    def __init__(self, fam, parts):
        self.parts = parts
        self.engs = [fam.make(hi - lo, BASE + lo) for lo, hi in parts]

    def _sl(self, x, dim):
        return [x.narrow(dim, lo, hi - lo).contiguous() for lo, hi in self.parts]

    def reset(self, mask=None):
        masks = self._sl(mask, 0) if mask is not None else [None] * len(self.engs)
        return [s.reset(mask=m) for s, m in zip(self.engs, masks)]

    def rollout(self, act, auto_reset, term=False):
        """-> per part (obs, rew, done, info, terminal observations or None)"""
        outs = []
        for s, a in zip(self.engs, self._sl(act, 1)):
            t = None
            if term:
                t = torch.full((a.shape[0], s.n_envs, s._n_acting, s.obs_dim), -7.0, dtype=s.obs_dtype, device="cuda")
                s.set_terminal_obs(t)
            outs.append(s.rollout(a, auto_reset=auto_reset) + (t,))
            s.set_terminal_obs(None)
        return outs

    def rollout_heuristic(self, T, obs0):
        return [s.rollout_heuristic(T, o.to(s.obs_dtype)) for s, o in zip(self.engs, self._sl(obs0, 0))]

    def check_outputs(self, got, refs, names):
        for i, name in enumerate(names):
            check(got[i], [r[i] for r in refs], self.parts, 1, name)

    def check_state(self, eng):
        torch.cuda.synchronize()
        for k, v in eng.state.items():
            if k != "sensors":   # the sensor table is shared by all envs
                check(v, [s.state[k] for s in self.engs], self.parts, 0, "state " + k)


TRAJ = ("obs", "rew", "done", "info")


def run_matrix(fam, obs_dtype=None, host=False):
    """Every entry point on a forced persistent-wave engine, against the shards and (fam.oracle) the oracle."""
    G, E = forced_wave()
    eng = fam.make(E, BASE, obs_dtype)
    eng.set_launch(blocks_per_sm=1)
    ref = Shards(fam, [(lo, min(lo + G, E)) for lo in range(0, E, G)])
    A, D = eng._n_acting, eng.obs_dim
    log = []   # ("reset", mask, obs) / ("steps", act, obs, rew, done, info, auto_reset, terminal obs, policy obs0)

    cur = eng.reset()
    check(cur, ref.reset(), ref.parts, 0, "reset obs")
    ref.check_state(eng)
    log.append(("reset", None, cur))

    # auto-reset across done steps, terminal observations kept on the side
    T = 14
    act = actions(fam, eng, T, 1)
    term = torch.full((T, E, A, D), -7.0, dtype=eng.obs_dtype, device="cuda")
    eng.set_terminal_obs(term)
    out = eng.rollout(act, auto_reset=True)
    eng.set_terminal_obs(None)
    ref.check_outputs(out + (term,), ref.rollout(act, True, term=True), TRAJ + ("terminal obs",))
    assert int(out[2].sum()) >= E * (T // MPL)
    ref.check_state(eng)
    log.append(("steps", act) + out + (True, term, None))

    act = actions(fam, eng, 4, 2)
    out = eng.rollout(act, auto_reset=False)
    ref.check_outputs(out, ref.rollout(act, False), TRAJ)
    ref.check_state(eng)
    log.append(("steps", act) + out + (False, None, None))
    cur = out[0][-1]

    # masked reset: warps alternate between resetting their first env and skipping it, and so do later envs
    e = torch.arange(E, device="cuda")
    mask = (e // G + e) % 2 == 1
    obs = eng.reset(mask=mask)
    check(obs, ref.reset(mask), ref.parts, 0, "masked reset obs")
    ref.check_state(eng)
    log.append(("reset", mask, obs))
    cur = torch.where(mask[:, None, None], obs, cur)

    if fam.policy is not None:
        out = eng.rollout_heuristic(10, cur)
        ref.check_outputs(out, ref.rollout_heuristic(10, cur), ("heuristic actions",) + TRAJ)
        ref.check_state(eng)
        log.append(("steps",) + out + (True, None, cur))

    # chained launches on three grids: the state a warp writes back for an env is read by another warp
    for k, bps in enumerate((1, 2, 0)):
        eng.set_launch(blocks_per_sm=bps)
        act = actions(fam, eng, 3, 10 + k)
        out = eng.rollout(act, auto_reset=True)
        ref.check_outputs(out, ref.rollout(act, True), tuple("%s (blocks_per_sm=%d)" % (n, bps) for n in TRAJ))
        log.append(("steps", act) + out + (True, None, None))
    eng.set_launch(blocks_per_sm=1)
    ref.check_state(eng)

    if host:   # host-buffer rollout cut into chunks of about 3 steps: one launch per chunk
        from madrl_b200 import _lib
        T = 13
        act = actions(fam, eng, T, 20)
        bufs = (torch.empty((T, E, A, D), dtype=eng.obs_dtype), torch.empty((T, E, A), dtype=eng.dtype),
                torch.empty((T, E), dtype=torch.uint8), torch.empty((T, E) + eng._info_tail, dtype=torch.int32))
        _lib.lib().madrl_set_host_chunk_bytes(3 * sum(b[0].numel() * b.element_size() for b in bufs))
        try:
            out = eng.rollout_host(act.cpu(), *bufs)
        finally:
            _lib.lib().madrl_set_host_chunk_bytes(0)
        ref.check_outputs(out, ref.rollout(act, True), tuple("host " + n for n in TRAJ))
        ref.check_state(eng)
        log.append(("steps", act) + out + (True, None, None))

    if fam.oracle is not None and obs_dtype is None:
        replay(fam, log, G, E, eng._info_keys)


def replay(fam, log, G, E, info_keys):
    """Step the oracle of envs that were the second, third and fourth env of their warp through `log`."""
    envs = [k * G + j for k in (1, 2, 3) for j in (0, 1, 4)]
    assert min(envs) >= G and max(envs) < E
    log = [tuple(x.cpu().numpy() if torch.is_tensor(x) else x for x in op) for op in log]
    for e in envs:
        o, ts = fam.oracle(BASE + e), 0
        for k, op in enumerate(log):
            if op[0] == "reset":
                _, mask, obs = op
                if mask is None or mask[e]:
                    oo, ts = o.reset(), 0
                    assert fam.close(oo, obs[e]), (k, e)
                continue
            _, act, obs, rew, done, info, auto, term, obs0 = op
            prev = None if obs0 is None else obs0[e]
            for t in range(act.shape[0]):
                if prev is not None:
                    fam.policy(o, BASE + e, prev, act[t, e])
                    prev = obs[t, e]
                oo, rr, dd, ii = o.step(act[t, e])
                ts += 1
                dd = dd or ts >= MPL
                assert bool(done[t, e]) == dd, (k, t, e)
                assert np.array_equal(np.reshape([ii[key] for key in info_keys], info[t, e].shape), info[t, e]), (k, t, e)
                assert fam.close(rr, rew[t, e]), (k, t, e)
                if dd and auto:
                    if term is not None:
                        assert fam.close(oo, term[t, e]), (k, t, e)
                    oo, ts = o.reset(), 0
                assert fam.close(oo, obs[t, e]), (k, t, e)


@pytest.mark.parametrize("case", ["c2-fp32", "c2-bf16", "c2-fp64", "c4-fp32", "c4-bf16", "c4-fp64",
                                  "k40-fp32", "k40-fp64", "big200-fp32", "big200-fp64",
                                  "global_nospeed_randobst-fp32", "global_nospeed_randobst-fp64"])
def test_waterworld_several_envs_per_warp(case):
    """c2: whole-step staging, 30 sensors known at compile time, 1 object per lane; c4: ring staging, 4 objects
    per lane; k40: 2 sensors per lane; big200: 8 objects per lane; global_nospeed_randobst: 4-row layout,
    runtime sensor count, random obstacle."""
    name, prec = case.rsplit("-", 1)
    run_matrix(waterworld(name, prec), obs_dtype=BF16 if prec == "bf16" else None, host=case == "c4-fp32")


@pytest.mark.parametrize("case", ["c3-fp32", "c3-bf16", "conv-fp32", "conv-bf16"])
def test_pursuit_several_envs_per_warp(case):
    name, prec = case.split("-")
    run_matrix(pursuit(name), obs_dtype=BF16 if prec == "bf16" else None, host=case == "c3-fp32")


@pytest.mark.parametrize("prec", ["fp32", "bf16", "fp64"])
def test_hostage_several_envs_per_warp(prec):
    run_matrix(hostage(prec), obs_dtype=BF16 if prec == "bf16" else None, host=prec == "fp32")


@pytest.mark.parametrize("obs_dtype", [torch.float32, BF16])
@pytest.mark.parametrize("family", ["waterworld_c4", "hostage_c5"])
def test_benchmark_shapes_equal_shards(family, obs_dtype):
    """bench.py's Waterworld C4 (4 096 envs) and Hostage C5 (8 192 envs) batches, at the launch bench.py makes and
    at 16 blocks per SM (several envs per warp whatever the occupancy): the first and last 256 envs equal
    256-env shards bit for bit."""
    fam, E = (waterworld("c4", "fp32", mpl=5), 4096) if family == "waterworld_c4" else (hostage("fp32", mpl=5), 8192)
    assert E > 16 * n_sms() > 2 * n_sms()
    T = 16
    ref = Shards(fam, [(0, 256), (E - 256, E)])
    ref_obs0 = ref.reset()
    for bps in (None, 16):
        eng = fam.make(E, BASE, obs_dtype)
        if bps is not None:
            eng.set_launch(blocks_per_sm=bps)
        check(eng.reset(), ref_obs0, ref.parts, 0, "reset obs")
        act = actions(fam, eng, T, 3)
        if bps is None:
            refs = ref.rollout(act, True, term=True)
        term = torch.full((T, E, eng._n_acting, eng.obs_dim), -7.0, dtype=eng.obs_dtype, device="cuda")
        eng.set_terminal_obs(term)
        out = eng.rollout(act, auto_reset=True)
        eng.set_terminal_obs(None)
        ref.check_outputs(out + (term,), refs, tuple("%s (blocks_per_sm=%s)" % (n, bps) for n in TRAJ + ("terminal obs",)))
        assert int(out[2].sum()) >= E * (T // 5)
        ref.check_state(eng)
        del eng, out, term
        torch.cuda.empty_cache()
