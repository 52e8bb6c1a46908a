"""madrl_b200 -- H100-native batched multi-agent environment engine.

Drop-in for the ``reset()/step()`` rollout hot path of sisl/MADRL's ``MAWaterWorld``,
``PursuitEvade`` and ``ContinuousHostageWorld`` (``madrl_environments``): E independent env
instances live in HBM (one struct-of-arrays record per env) and are stepped in lockstep by
hand-written sm_90a CUDA kernels behind the C ABI in ``include/madrl_b200.h``.  There is no CPU
fallback: the classes below raise ``EngineError`` if the CUDA library is missing.
"""
from ._lib import EngineError, launch_count  # noqa: F401
from .core import Agent, AbstractMAEnv, EzPickle  # noqa: F401
from .spaces import Box, Discrete  # noqa: F401
from .waterworld import BatchedMAWaterWorld, MAWaterWorld, Archea  # noqa: F401
from .pursuit import BatchedPursuitEvade, PursuitEvade, DiscreteAgent, RandomPolicy, SingleActionPolicy  # noqa: F401
from .hostage import BatchedHostageWorld, ContinuousHostageWorld, CircAgent  # noqa: F401
from .closed_loop import PolicyRollout  # noqa: F401
from .replay import ReplayPool  # noqa: F401
from .evaluate import evaluate_heuristic, evaluate_policy  # noqa: F401
from .whole_paths import WholePathBatch, WholePathSampler  # noqa: F401

__all__ = [
    "EngineError", "launch_count", "Agent", "AbstractMAEnv", "EzPickle", "Box", "Discrete",
    "BatchedMAWaterWorld", "MAWaterWorld", "Archea", "BatchedPursuitEvade", "PursuitEvade",
    "DiscreteAgent", "RandomPolicy", "SingleActionPolicy", "BatchedHostageWorld", "ContinuousHostageWorld", "CircAgent", "PolicyRollout",
    "ReplayPool", "evaluate_policy", "evaluate_heuristic", "WholePathSampler", "WholePathBatch",
]
