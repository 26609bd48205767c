"""ctypes driver of tests/native_long/liblong_clip_probe.so: attention launches for clips of any length, including the
streaming wgmma kernel (not collected by pytest).  Inputs are prepared with tests/kernel_probe.py's helpers."""
import ctypes as C
import os

import kernel_probe as kp
from helpers import ROOT

LIB_PATH = os.path.join(ROOT, "tests", "native_long", "liblong_clip_probe.so")
ATTN_WGMMA_STREAM = 5  # attention.cuh AttnKernel::kAttnWgmmaStream

_lib = None


def lib():
    """The probe library; a missing one is an error (build() makes it), never a skip."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run __graft_entry__.build()")
        _lib = C.CDLL(LIB_PATH)
        _lib.long_probe_attention.argtypes = [C.POINTER(kp.Attn), C.c_int]
    return _lib


def attention(qkv_hi, qkv_lo, ctx_hi, ctx_lo, B, S, D, H, scale, kind, which, pdl=False, reps=1):
    """launch_attention `reps` times back to back on the default stream; returns 0 or the error code."""
    a = kp.Attn(kp._ptr(qkv_hi), kp._ptr(qkv_lo), qkv_hi.shape[0], kp._ptr(ctx_hi), kp._ptr(ctx_lo), B, S, D, H, scale,
                kind, which, int(pdl))
    return lib().long_probe_attention(C.byref(a), reps)
