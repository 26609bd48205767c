"""Shadows the reference's diffusion/respace.py with the CUDA implementation."""
from rohm_b200.diffusion import (SpacedDiffusionPoseNet, SpacedDiffusionTrajNet, _WrappedModel,  # noqa: F401
                                 space_timesteps)
