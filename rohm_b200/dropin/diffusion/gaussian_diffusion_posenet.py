"""Shadows the reference's diffusion/gaussian_diffusion_posenet.py with the CUDA implementation."""
from rohm_b200.diffusion import (GaussianDiffusionPoseNet, LossType, ModelMeanType, ModelVarType,  # noqa: F401
                                 betas_for_alpha_bar, get_named_beta_schedule)
