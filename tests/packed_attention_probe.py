"""ctypes driver of tests/native_packed/libpacked_attention_probe.so: the wgmma attention kernels (attention.cu) on packed
clips, launched directly on torch device tensors (not collected by pytest)."""
import ctypes as C
import os

from helpers import ROOT

LIB_PATH = os.path.join(ROOT, "tests", "native_packed", "libpacked_attention_probe.so")


class PackedAttn(C.Structure):
    _fields_ = [("qkv_hi", C.c_void_p), ("qkv_lo", C.c_void_p), ("rows", C.c_int64), ("ctx_hi", C.c_void_p),
                ("ctx_lo", C.c_void_p), ("clip_off", C.c_void_p), ("clip_ids", C.c_void_p), ("n", C.c_int), ("S", C.c_int),
                ("D", C.c_int), ("H", C.c_int), ("scale", C.c_float), ("which", C.c_int), ("pdl", C.c_int)]


_lib = None


def lib():
    """The probe library; a missing one is an error (build() makes it), never a skip."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run __graft_entry__.build()")
        _lib = C.CDLL(LIB_PATH)
        _lib.probe_attention_packed.argtypes = [C.POINTER(PackedAttn), C.c_int]
    return _lib


def attention_packed(qkv_hi, qkv_lo, ctx_hi, ctx_lo, clip_off, clip_ids, S, D, H, scale, which, pdl=False, reps=1):
    """launch_attention on packed clips (fp16 pairs, head dim 128): clip c holds rows [clip_off[c], clip_off[c + 1]) and
    the launch runs the clips in clip_ids (int32 device tensors) with the wgmma kernel `which` (kernel_probe.ATTN_*);
    S = their most tokens.  Returns 0 or the error code."""
    a = PackedAttn(qkv_hi.data_ptr(), qkv_lo.data_ptr(), qkv_hi.shape[0], ctx_hi.data_ptr(), ctx_lo.data_ptr(),
                   clip_off.data_ptr(), clip_ids.data_ptr(), clip_ids.numel(), S, D, H, scale, which, int(pdl))
    return lib().probe_attention_packed(C.byref(a), reps)
