"""art_planner_b200 -- CUDA-native (sm_90a, H100) implementation of art_planner's batchable hot path:
pose validity (ODE box-vs-heightfield torso/feet checks), edge validity over interpolated SE(3) states and
edge cost, behind a C ABI (include/artp.h) and a host-side mirror of the reference's plugin interface."""
from . import synth  # noqa: F401
from .capi import ArtpError  # noqa: F401
from .checker import (GoalStateRegion, MotionCostObjective, MotionValidator, PathLengthObjective,  # noqa: F401
                      PathSimplifier, Planner, PRMRoadmap, SE3FromSE2Sampler, StartState, StateValidityChecker)

__all__ = ["synth", "ArtpError", "StateValidityChecker", "MotionValidator", "PathLengthObjective", "MotionCostObjective", "SE3FromSE2Sampler",
           "StartState", "GoalStateRegion", "PRMRoadmap", "PathSimplifier", "Planner"]
