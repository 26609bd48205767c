"""ctypes driver of tests/native/libkernel_probe.so: the GEMM (rohm_b200/csrc/gemm.cu) and attention (attention.cu) kernels
launched directly on torch device tensors, plus the operand packing the engines do (not collected by pytest)."""
import ctypes as C
import os

import torch

from helpers import ROOT

LIB_PATH = os.path.join(ROOT, "tests", "native", "libkernel_probe.so")
KIND_TF32, KIND_F16 = 0, 1
ACT_NONE, ACT_GELU, ACT_SILU, ACT_MISH = 0, 1, 2, 3
BLOCK_M = 128
MAX_SEGS = 10
CUDA_ERROR_INVALID_VALUE = 1
# attention.cuh AttnKernel
ATTN_AUTO, ATTN_WGMMA, ATTN_MMA_F16, ATTN_MMA_TF32, ATTN_SIMT = 0, 1, 2, 3, 4


def block_k(kind):
    """gemm_block_k: K elements of one pipeline stage (64 bytes of K per operand row)."""
    return 32 if kind == KIND_F16 else 16


class Seg(C.Structure):
    _fields_ = [("hi", C.c_void_p), ("lo", C.c_void_p), ("rows", C.c_int64), ("cols", C.c_int), ("ld", C.c_int),
                ("row_shift", C.c_int), ("row_mul", C.c_int), ("kblocks", C.c_int)]


class Gemm(C.Structure):
    _fields_ = [("kind", C.c_int), ("passes", C.c_int), ("block_n", C.c_int), ("m_rows", C.c_int), ("n_cols", C.c_int),
                ("num_segs", C.c_int), ("seg", Seg * MAX_SEGS), ("w_hi", C.c_void_p), ("w_lo", C.c_void_p),
                ("w_rows", C.c_int64), ("w_cols", C.c_int), ("bias", C.c_void_p), ("residual", C.c_void_p), ("ldr", C.c_int),
                ("out", C.c_void_p), ("ldo", C.c_int), ("out_hi", C.c_void_p), ("out_lo", C.c_void_p), ("lds", C.c_int),
                ("acc_scale", C.c_float), ("act", C.c_int), ("M", C.c_int), ("N", C.c_int), ("out_row_mul", C.c_int),
                ("out_row_add", C.c_int), ("clip_rows", C.c_int), ("clip_valid", C.c_int), ("gn_stats", C.c_void_p),
                ("gn_groups", C.c_int), ("gn_group_size", C.c_int), ("a_stats", C.c_void_p), ("a_corr", C.c_void_p),
                ("res_stats", C.c_void_p), ("res_gamma", C.c_void_p), ("res_beta", C.c_void_p), ("stats_out", C.c_void_p),
                ("ln_eps", C.c_float), ("k_splits", C.c_int), ("split_row_stride", C.c_int), ("want_tma_store", C.c_int),
                ("store_rows", C.c_int64), ("want_multicast", C.c_int), ("pdl", C.c_int), ("tma_store", C.c_int),
                ("multicast", C.c_int)]


class Attn(C.Structure):
    _fields_ = [("qkv_hi", C.c_void_p), ("qkv_lo", C.c_void_p), ("rows", C.c_int64), ("ctx_hi", C.c_void_p),
                ("ctx_lo", C.c_void_p), ("B", C.c_int), ("S", C.c_int), ("D", C.c_int), ("H", C.c_int), ("scale", C.c_float),
                ("kind", C.c_int), ("which", C.c_int), ("pdl", C.c_int)]


_lib = None


def lib():
    """The probe library; a missing one is an error (build() makes it), never a skip."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run __graft_entry__.build()")
        _lib = C.CDLL(LIB_PATH)
        _lib.probe_gemm.argtypes = [C.POINTER(Gemm)]
        _lib.probe_split.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float]
        _lib.probe_f16_weight_scale.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_float)]
        _lib.probe_attention.argtypes = [C.POINTER(Attn)]
    return _lib


def _ptr(t):
    return None if t is None else t.data_ptr()


def split(kind, x, scale=1.0):
    """The library's operand split of an fp32 device tensor: TF32 pair in fp32 containers, or fp16 pair of x * scale."""
    x = x.contiguous()
    dt = torch.float16 if kind == KIND_F16 else torch.float32
    hi, lo = torch.empty_like(x, dtype=dt), torch.empty_like(x, dtype=dt)
    assert lib().probe_split(kind, x.data_ptr(), hi.data_ptr(), lo.data_ptr(), x.numel(), scale) == 0
    return hi, lo


def pair_value(hi, lo):
    """hi + lo in float64."""
    return hi.double() + lo.double()


class Operand:
    """A row-major A operand [rows, cols] as the kernels read it: a hi/lo pair with a 16-byte row pitch whose padding
    columns hold NaN (the tensor map never reaches them)."""

    def __init__(self, kind, x):
        rows, cols = x.shape
        per16 = 8 if kind == KIND_F16 else 4
        self.kind, self.rows, self.cols = kind, rows, cols
        self.ld = -(-cols // per16) * per16
        full = torch.full((rows, self.ld), float("nan"), device=x.device)
        full[:, :cols] = x
        self.hi, self.lo = split(kind, full)
        self.value = pair_value(self.hi, self.lo)[:, :cols]  # what the kernel multiplies (pad columns excluded)

    def seg(self, kblocks, row_shift=0, row_mul=1):
        return Seg(self.hi.data_ptr(), self.lo.data_ptr(), self.rows, self.cols, self.ld, row_shift, row_mul, kblocks)


class Weight:
    """A K-major weight [N, K_total] packed like the engines do: K segments each padded to whole K blocks, rows padded to
    block_n, fp16 pairs of w * 2^s (f16_weight_scale) or TF32 pairs."""

    def __init__(self, kind, w_parts, block_n):
        """w_parts: list of [N, K_s] fp32 device tensors, one per A segment (a plain linear layer has one)."""
        N = w_parts[0].shape[0]
        bk = block_k(kind)
        self.kind, self.N, self.block_n = kind, N, block_n
        self.kblocks = [-(-p.shape[1] // bk) for p in w_parts]
        self.Kp = bk * sum(self.kblocks)
        self.Np = -(-N // block_n) * block_n
        dev = w_parts[0].device
        packed = torch.zeros(self.Np, self.Kp, device=dev)
        off = 0
        for p, kb in zip(w_parts, self.kblocks):
            packed[:N, off:off + p.shape[1]] = p
            off += kb * bk
        self.scale = 1.0
        if kind == KIND_F16:
            s = C.c_float()
            assert lib().probe_f16_weight_scale(packed.data_ptr(), packed.numel(), C.byref(s)) == 0
            self.scale = s.value
        self.hi, self.lo = split(kind, packed, self.scale)
        full = pair_value(self.hi, self.lo) / self.scale
        self.parts = []  # the weight values the kernel multiplies, per segment, float64 [N, K_s]
        off = 0
        for p, kb in zip(w_parts, self.kblocks):
            self.parts.append(full[:N, off:off + p.shape[1]])
            off += kb * bk


def gemm(kind, w, segs, M, N, *, passes=3, m_rows=None, out=None, ldo=None, out_hi=None, out_lo=None, lds=None,
         bias=None, residual=None, ldr=None, act=ACT_NONE, out_row_mul=1, out_row_add=0, clip_rows=0, clip_valid=0,
         gn_stats=None, gn_groups=0, tma_store=False, store_rows=None, multicast=False, k_splits=0, split_row_stride=0,
         a_stats=None, a_corr=None, res_stats=None, res_gamma=None, res_beta=None, stats_out=None, ln_eps=1e-5,
         pdl=False, n_cols=None):
    """One launch_gemm; returns (rc, the filled Gemm struct).  segs: list of Seg."""
    g = Gemm()
    g.kind, g.passes, g.block_n = kind, passes, w.block_n
    g.m_rows = M if m_rows is None else m_rows
    g.n_cols = N if n_cols is None else n_cols
    g.num_segs = len(segs)
    for i, s in enumerate(segs):
        g.seg[i] = s
    g.w_hi, g.w_lo, g.w_rows, g.w_cols = w.hi.data_ptr(), w.lo.data_ptr(), w.Np, w.Kp
    g.bias, g.residual = _ptr(bias), _ptr(residual)
    g.ldr = ldr if ldr is not None else (residual.shape[1] if residual is not None else 0)
    g.out = _ptr(out)
    g.ldo = ldo if ldo is not None else (out.shape[1] if out is not None else 0)
    g.out_hi, g.out_lo = _ptr(out_hi), _ptr(out_lo)
    g.lds = lds if lds is not None else (out_hi.shape[1] if out_hi is not None else 0)
    g.acc_scale = 1.0 / w.scale
    g.act, g.M, g.N = act, M, N
    g.out_row_mul, g.out_row_add = out_row_mul, out_row_add
    g.clip_rows, g.clip_valid = clip_rows, clip_valid
    g.gn_stats = _ptr(gn_stats)
    g.gn_groups = gn_groups
    g.gn_group_size = N // gn_groups if gn_groups else 0
    g.a_stats, g.a_corr, g.res_stats = _ptr(a_stats), _ptr(a_corr), _ptr(res_stats)
    g.res_gamma, g.res_beta, g.stats_out, g.ln_eps = _ptr(res_gamma), _ptr(res_beta), _ptr(stats_out), ln_eps
    g.k_splits, g.split_row_stride = k_splits, split_row_stride
    g.want_tma_store = int(tma_store)
    g.store_rows = store_rows if store_rows is not None else M
    g.want_multicast = int(multicast)
    g.pdl = int(pdl)
    rc = lib().probe_gemm(C.byref(g))
    return rc, g


def attention(qkv_hi, qkv_lo, ctx_hi, ctx_lo, B, S, D, H, scale, kind, which, pdl=False):
    a = Attn(_ptr(qkv_hi), _ptr(qkv_lo), qkv_hi.shape[0], _ptr(ctx_hi), _ptr(ctx_lo), B, S, D, H, scale, kind, which, int(pdl))
    return lib().probe_attention(C.byref(a))
