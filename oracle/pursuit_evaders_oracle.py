"""CPU oracle of PursuitEvade under a caller's evader controller (TEST INFRASTRUCTURE, NumPy).

``PursuitEvadersOracle`` is ``pursuit_oracle.PursuitOracle`` -- the one restatement of pursuit_evade.py (``pe:``) --
whose ``step`` also takes the evaders' actions: None for the reference's default ``RandomPolicy(5)``, an int for
``SingleActionPolicy(a)``, or a sequence indexed by ORIGINAL evader index (a controller that is called once per live
evader per step, in index order, pe:237-241).  A value outside 0..3 stays.  ``model_state`` is the base class's: the
map and the occupancy after the step's moves and before its removals (pe:244-249), what the reference hands the
controller at the next step.

Each live evader still consumes its stream draw under a caller's controller, and the draw goes unused: the engine's
counter rule (DESIGN §4.2), under which every later reset draw is the random controller's.  Pinned against the real
reference by ``tests/test_pursuit_evaders_golden.py`` (``oracle/make_evaders_golden.py``).
"""
import numpy as np

from .philox import Stream
from .pursuit_oracle import PursuitOracle


class _ControlledDraws(object):
    """The env's stream, except that while `actions` is set, each ``randint(5)`` -- the base class's step draws one
    per live evader, in index order, and nothing else -- consumes its word and returns the next caller action."""

    def __init__(self, rng):
        self.rng = rng
        self.actions = None

    def randint(self, low, high=None, size=None):
        w = self.rng.randint(low, high, size)
        if self.actions is None:
            return w
        a = int(next(self.actions))
        return a if 0 <= a < 4 else 4

    def __getattr__(self, name):   # counter, uniform, ... of the stream itself
        return getattr(self.rng, name)


class PursuitEvadersOracle(PursuitOracle):
    """PursuitOracle with an evader action source; kwargs as PursuitOracle's."""

    def __init__(self, map_pool, rng=None, **kwargs):
        super().__init__(map_pool, rng=_ControlledDraws(rng if rng is not None else Stream(0, 0)), **kwargs)

    def step(self, actions, evader_actions=None):
        if evader_actions is not None:
            live = np.flatnonzero(~self.gone)
            ev = np.broadcast_to(np.asarray(evader_actions), (self.Ne,))
            self.rng.actions = iter(ev[live].tolist())
        try:
            return super().step(actions)
        finally:
            self.rng.actions = None
