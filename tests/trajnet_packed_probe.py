"""ctypes driver of tests/native_trajnet_packed/libtrajnet_packed_probe.so: TrajNet's GEMM epilogue with a packed-clip row
mask and its GroupNorm + Mish kernel with a packed-clip offset table, launched directly on torch device tensors (not
collected by pytest).  Operands, weights and GnArgs come from kernel_probe."""
import ctypes as C
import os

import kernel_probe as kp
from helpers import ROOT

LIB_PATH = os.path.join(ROOT, "tests", "native_trajnet_packed", "libtrajnet_packed_probe.so")


class MaskedGemm(C.Structure):
    _fields_ = [("kind", C.c_int), ("passes", C.c_int), ("block_n", C.c_int), ("a_hi", C.c_void_p), ("a_lo", C.c_void_p),
                ("a_rows", C.c_int64), ("a_cols", C.c_int), ("a_ld", C.c_int), ("kblocks", C.c_int), ("w_hi", C.c_void_p),
                ("w_lo", C.c_void_p), ("w_rows", C.c_int64), ("w_cols", C.c_int), ("bias", C.c_void_p), ("out", C.c_void_p),
                ("ldo", C.c_int), ("acc_scale", C.c_float), ("act", C.c_int), ("M", C.c_int), ("N", C.c_int),
                ("clip_rows", C.c_int), ("clip_valid", C.c_int), ("row_mask", C.c_void_p), ("want_tma_store", C.c_int),
                ("store_rows", C.c_int64), ("tma_store", C.c_int)]


_lib = None


def lib():
    """The probe library; a missing one is an error (build() makes it), never a skip."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run __graft_entry__.build()")
        _lib = C.CDLL(LIB_PATH)
        _lib.probe_gemm_row_mask.argtypes = [C.POINTER(MaskedGemm), C.c_int]
        _lib.probe_group_norm_packed.argtypes = [C.POINTER(kp.GnArgs), C.c_void_p, C.c_int, C.c_int, C.c_int]
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def gemm_row_mask(A, W, M, N, out, bias, act, clip_rows, clip_valid, row_mask, tma_store=False, reps=1):
    """out = act(A W^T + bias) through the masked epilogue (A: kp.Operand, W: kp.Weight with one segment); row_mask: uint8
    device tensor [M] or None (the clip_rows / clip_valid rule).  Returns (rc, the filled MaskedGemm struct)."""
    g = MaskedGemm(A.kind, 3, W.block_n, A.hi.data_ptr(),
                   A.lo.data_ptr(), A.rows, A.cols, A.ld, W.kblocks[0], W.hi.data_ptr(), W.lo.data_ptr(), W.Np, W.Kp,
                   _ptr(bias), out.data_ptr(), out.shape[1], 1.0 / W.scale, act, M, N, clip_rows, clip_valid,
                   _ptr(row_mask), int(tma_store), M, 0)
    rc = lib().probe_gemm_row_mask(C.byref(g), reps)
    return rc, g


def group_norm_packed(part, splits, split_stride, bias, gamma, beta, tp, tp_stride, r1, r2, out, out_hi, out_lo, C_, Tp, T,
                      clip_off, n, f16, groups=8, reps=1):
    """gn_mish_split_kernel over the packed clips of clip_off (int32 device tensor [B + 1]) with clusters of n CTAs per
    (clip, group); Tp / T are the engine's level rows and real rows per clip.  Returns 0 or the CUDA error code."""
    p = _ptr
    a = kp.GnArgs(p(part), splits, split_stride, p(bias), p(gamma), p(beta), p(tp), tp_stride, p(r1), p(r2), p(out),
                  p(out_hi), p(out_lo), C_, Tp, T, groups, int(f16))
    return lib().probe_group_norm_packed(C.byref(a), clip_off.data_ptr(), clip_off.numel() - 1, n, reps)
