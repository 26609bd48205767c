"""ctypes driver of tests/native_groupnorm/libgroup_norm_probe.so: TrajNet's GroupNorm + Mish kernel launched with an
explicit cluster size (not collected by pytest)."""
import ctypes as C
import os

from helpers import ROOT

LIB_PATH = os.path.join(ROOT, "tests", "native_groupnorm", "libgroup_norm_probe.so")

_lib = None


class GnArgs(C.Structure):  # rohm_b200/csrc/groupnorm.cuh GnArgs
    _fields_ = [("part", C.c_void_p), ("splits", C.c_int), ("split_stride", C.c_int64), ("bias", C.c_void_p),
                ("gamma", C.c_void_p), ("beta", C.c_void_p), ("tp", C.c_void_p), ("tp_stride", C.c_int),
                ("r1", C.c_void_p), ("r2", C.c_void_p), ("out", C.c_void_p), ("out_hi", C.c_void_p),
                ("out_lo", C.c_void_p), ("C", C.c_int), ("Tp", C.c_int), ("T", C.c_int), ("groups", C.c_int),
                ("f16", C.c_int)]


def lib():
    """The probe library; a missing one is an error (build() makes it), never a skip."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run __graft_entry__.build()")
        _lib = C.CDLL(LIB_PATH)
        _lib.probe_group_norm.argtypes = [C.POINTER(GnArgs), C.c_int, C.c_int, C.c_int]
        _lib.probe_group_norm_cluster.argtypes = [C.c_int, C.c_int, C.c_int]
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def group_norm(part, splits, split_stride, bias, gamma, beta, tp, tp_stride, r1, r2, out, out_hi, out_lo, C_, Tp, T, B, n,
               f16, groups=8, reps=1):
    """gn_mish_split_kernel over B clips with clusters of n CTAs per (clip, group), `reps` times on the default stream
    (tensors or None); returns 0 or the CUDA error code."""
    p = _ptr
    a = GnArgs(p(part), splits, split_stride, p(bias), p(gamma), p(beta), p(tp), tp_stride, p(r1), p(r2), p(out), p(out_hi),
               p(out_lo), C_, Tp, T, groups, int(f16))
    return lib().probe_group_norm(C.byref(a), B, n, reps)


def group_norm_cluster(T, C_, groups=8):
    """The cluster size the TrajNet engine chooses for groups of T rows of C_ / groups channels."""
    return lib().probe_group_norm_cluster(T, C_, groups)
