"""Shadows the reference's model/trajnet.py with the CUDA implementation."""
from rohm_b200.trajnet import ControlNet, TrajNet  # noqa: F401
