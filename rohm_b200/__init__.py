"""rohm_b200 -- H100-native implementation of RoHM's iterative diffusion-denoising hot path.

Public Python surface (mirrors the reference's symbols; see rohm_b200/dropin for the import-compatible shims):
    rohm_b200.posenet.PoseNet, rohm_b200.trajnet.TrajNet
    rohm_b200.diffusion.{GaussianDiffusionPoseNet, GaussianDiffusionTrajNet, SpacedDiffusionPoseNet,
                         SpacedDiffusionTrajNet, space_timesteps, create_gaussian_diffusion, ...}
All arithmetic runs in librohm_b200.so (hand-written sm_90a CUDA behind the C ABI of include/rohm_b200.h).
There is no CPU or eager fallback: using the models without the built library and an H100 raises RohmB200Error.
"""
from ._lib import RohmB200Error, LIB_PATH  # noqa: F401

__version__ = "0.1.0"
