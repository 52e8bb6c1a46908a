"""The reference's hand-written policies on the device (SURVEY.md 8f row 4).

Two forms:

* inside the rollout kernels -- ``BatchedMAWaterWorld.rollout_heuristic`` /
  ``BatchedPursuitEvade.rollout_heuristic`` (``madrl_ww_rollout_heuristic`` /
  ``madrl_pursuit_rollout_heuristic``): the policy is evaluated on the features each warp has just computed,
  so a closed-loop rollout of T steps is ONE launch with no action tensor;
* the stand-alone generators below (``madrl_ww_heuristic_actions`` / ``madrl_pursuit_heuristic_actions``,
  csrc/heuristics.cu): one warp per observation row, for callers that step from the host.

``waterworld_heuristic``  heuristics/waterworld.py:11-53 -- flee the obstacle and poison, chase evaders,
close in on allies; observation layout documented at heuristics/waterworld.py:12-22.
``pursuit_heuristic``     heuristics/pursuit.py:18-50 -- walk towards the nearest visible evader, a random
move when none is visible.
"""
import torch

from . import _lib
from ._lib import _ptr


def waterworld_heuristic(obs, n_sensors):
    """obs [..., 7K+2(+1)] float32 / float64 CUDA tensor -> actions [..., 2].

    The reference normalises by the Frobenius norm of the WHOLE batch it is called with
    (heuristics/waterworld.py:46-50); it is called per agent (B = 1) in the reference's own demo,
    so here every agent row is normalised by its own norm."""
    _lib.require_tensor(obs, "obs", (torch.float32, torch.float64), (...,), None, contiguous=False)
    if not obs.is_cuda:
        raise _lib.EngineError("madrl_b200 needs a CUDA tensor (there is no CPU fallback)")
    D = obs.shape[-1]
    o = obs.contiguous().view(-1, D)
    act = torch.empty((o.shape[0], 2), dtype=obs.dtype, device=obs.device)
    with torch.cuda.device(obs.device):
        _lib.check(_lib.lib().madrl_ww_heuristic_actions(int(obs.dtype == torch.float64), o.shape[0], int(n_sensors), D,
                                                        _ptr(o), _ptr(act), _lib.stream(obs.device)))
    return act.view(obs.shape[:-1] + (2,))


def pursuit_heuristic(obs, obs_range=None, generator=None, py2_division=True, fallback=None):
    """obs float32 CUDA tensor, [..., R, R, 4] (flatten=False layout) or [..., 3R^2(+1)] with `obs_range` given
    -> int32 actions [...] (0 left, 1 right, 2 up, 3 down, 4 stay).  `fallback` [...]: the move of the agents
    that see no evader (default: uniform draws from `generator`); `py2_division`: the window centre `xs / 2`
    (heuristics/pursuit.py:23) under Python 2's integer division -- the reference's language."""
    flatten = obs_range is not None
    if flatten:
        R, D, lead = int(obs_range), obs.shape[-1], obs.shape[:-1]
    else:
        R, lead = obs.shape[-2], obs.shape[:-3]
        D = 4 * R * R
        _lib.require_tensor(obs, "obs", obs.dtype, tuple(lead) + (R, R, 4), None, contiguous=False)   # widened below
    n = lead.numel()
    if fallback is not None:
        fallback = _lib.require_tensor(fallback.to(device=obs.device, dtype=torch.int32).contiguous().view(-1),
                                       "fallback", torch.int32, (n,), obs.device)
    if not obs.is_cuda:
        raise _lib.EngineError("madrl_b200 needs a CUDA tensor (there is no CPU fallback)")
    o = obs.to(torch.float32).contiguous().view(-1, D)
    if fallback is None:
        fallback = torch.randint(0, 5, (n,), dtype=torch.int32, device=obs.device, generator=generator)
    act = torch.empty((n,), dtype=torch.int32, device=obs.device)
    lut = torch.empty((128,), dtype=torch.uint8, device=obs.device)
    with torch.cuda.device(obs.device):
        _lib.check(_lib.lib().madrl_pursuit_heuristic_actions(n, R, int(flatten), D, int(bool(py2_division)), _ptr(o),
                                                             _ptr(fallback), _ptr(lut), _ptr(act),
                                                             _lib.stream(obs.device)))
    return act.view(lead)
