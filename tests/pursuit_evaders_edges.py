"""What the emulated and the GPU tests of Pursuit's evader control share: the random controller's actions of a
step read off the env's stream, and the oracle run under a caller's evader actions."""
import numpy as np

from oracle.philox import Stream
from oracle.pursuit_evaders_oracle import PursuitEvadersOracle

import env_dispatch_edges as D


def pe_oracles(case, maps, seed, base, E):
    """env_dispatch_edges.pe_oracles with an evader action source (PursuitEvadersOracle)."""
    return [PursuitEvadersOracle(maps, rng=Stream(seed, base + e), **case.cfg) for e in range(E)]


def random_evader_actions(seed, env_id_base, counter, gone, n_evaders, fill_seed=0):
    """The actions the random controller takes at the next step: live evader j of env e (original index, live rank
    r) takes draw counter[e] + r of the env's stream.  Entries of gone evaders hold arbitrary moves, which the
    kernel must not read.  -> int32 [E, Ne]."""
    E = len(counter)
    out = np.random.RandomState(fill_seed).randint(0, 4, size=(E, n_evaders)).astype(np.int32)
    for e in range(E):
        s = Stream(seed, env_id_base + e, 0, int(counter[e]))
        g = int(gone[e])
        for j in range(n_evaders):
            if not (g >> j) & 1:
                out[e, j] = s.randint(5)
    return out


def oracle_trajectory(oracles, act, ev, mpl, auto_reset=True):
    """Step the oracles (already reset) through pursuer actions act [T, E, Np] and evader actions ev [T, E, Ne]
    (None: the random controller) with the VecEnvExecutor horizon `mpl` -> (obs, rew, done, removed) as float32 /
    bool / int arrays, the oracles left at the end."""
    T, E = act.shape[:2]
    ts = np.zeros(E, int)
    obs, rew, done, rem = [], [], np.zeros((T, E), bool), np.zeros((T, E), int)
    for t in range(T):
        ot, rt = [], []
        for e, o in enumerate(oracles):
            oo, rr, dd, ii = o.step(act[t, e], None if ev is None else ev[t, e])
            ts[e] += 1
            dd = dd or ts[e] >= mpl
            if dd and auto_reset:
                oo, ts[e] = o.reset(), 0
            done[t, e], rem[t, e] = dd, ii['removed']
            ot.append(np.array([D.f32(x).reshape(-1) for x in oo]))
            rt.append(D.f32(rr))
        obs.append(ot)
        rew.append(rt)
    return np.array(obs), np.array(rew), done, rem
