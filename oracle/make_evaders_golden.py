"""Record the REAL reference PursuitEvade under injected evader controllers -> tests/golden/pe_evaders.npz.

    python oracle/make_evaders_golden.py

Three controllers, each run on one env through `refshim.make_reference_pursuit` (every map, window and spawn draw
from the Philox stream of seed 5, env 0): SingleActionPolicy(4) (stationary), SingleActionPolicy(1) (moving) and a
table controller that replays table[t, j] for the evader of ORIGINAL index j (calls come in live order, pe:238-241, so
the controller maps each call's live rank to its original index).  Every controller consumes one stream draw per
call and ignores it: the engine's counter rule (DESIGN §4.2), under which reset draws are those of the random
controller.  Each run covers several episodes of surround and n_catch capture on maps with buildings next to the
evaders, random_opponents in one of them, and records per step the observations, rewards, dones, removed counts and
the model_state the reference holds after the step.  Only data is written.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import refshim  # noqa: E402
from oracle.philox import Stream  # noqa: E402

SEED, T = 5, 120
MAPS = np.load(os.path.join(ROOT, "maps", "map_pool16.npy"))
RUNS = {
    "stay_surround": (dict(n_evaders=6, n_pursuers=24, obs_range=5, surround=True, sample_maps=True,
                           reward_mech='local'), ("fixed", 4)),
    "right_ncatch": (dict(n_evaders=5, n_pursuers=6, obs_range=3, surround=False, n_catch=1, sample_maps=True,
                          reward_mech='global'), ("fixed", 1)),
    "table_random_opp": (dict(n_evaders=8, n_pursuers=6, obs_range=5, surround=False, n_catch=1, sample_maps=True,
                              random_opponents=True, max_opponents=9, reward_mech='local'), ("table", 0)),
}


class Controller(object):
    """SingleActionPolicy(a) or a table replay by original index; each call consumes one draw of `stream`."""

    def __init__(self, stream, kind, a, table):
        self.stream, self.kind, self.a, self.table = stream, kind, a, table
        self.env, self.t, self.k = None, 0, 0

    def act(self, state):
        self.stream.randint(5)
        if self.kind == "fixed":
            return self.a
        live = [j for j in range(len(self.env.evaders_gone)) if not self.env.evaders_gone[j]][:self.env.n_evaders]
        a = int(self.table[self.t, live[self.k]])
        self.k += 1
        return a

    def next_step(self):
        self.t, self.k = self.t + 1, 0


def run(cfg, kind, a):
    rs = np.random.RandomState(3)
    stream = Stream(SEED, 0)
    n = cfg["n_evaders"]
    table = rs.randint(0, 5, size=(T, n)).astype(np.int32)
    act = rs.randint(0, 5, size=(T, cfg["n_pursuers"])).astype(np.int32)
    env = refshim.make_reference_pursuit(MAPS, stream, **cfg)
    ctl = Controller(stream, kind, a, table)
    env.evader_controller, ctl.env = ctl, env
    rec = dict(obs0=[], obs=[], rew=[], done=[], removed=[], model_state=[], model_state0=[])
    rec["obs0"].append(np.array(env.reset()))
    rec["model_state0"].append(env.model_state.copy())
    starts = [0]
    for t in range(T):
        o, r, d, info = env.step(act[t])
        ctl.next_step()
        rec["obs"].append(np.array(o))
        rec["rew"].append(np.asarray(r, np.float64))
        rec["done"].append(bool(d))
        rec["removed"].append(int(info.get("removed", 0)) if isinstance(info, dict) else 0)
        rec["model_state"].append(env.model_state.copy())
        if d:
            rec["obs0"].append(np.array(env.reset()))
            rec["model_state0"].append(env.model_state.copy())
            starts.append(t + 1)
    out = {k: np.array(v) for k, v in rec.items()}
    out.update(act=act, table=table, starts=np.array(starts), kind=np.array(kind), a=np.array(a))
    return out


def main():
    arrays = {}
    for name, (cfg, (kind, a)) in RUNS.items():
        r = run(cfg, kind, a)
        print(name, "episodes", len(r["starts"]), "removed", int(r["removed"].sum()))
        arrays.update(("%s/%s" % (name, k), v) for k, v in r.items())
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "pe_evaders.npz"), **arrays)


if __name__ == "__main__":
    main()
