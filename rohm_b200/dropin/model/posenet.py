"""Shadows the reference's model/posenet.py with the CUDA implementation."""
from rohm_b200.posenet import PoseNet  # noqa: F401
