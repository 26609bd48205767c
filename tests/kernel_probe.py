"""ctypes driver of tests/native/libkernel_probe.so: the GEMM (rohm_b200/csrc/gemm.cu), attention (attention.cu),
GroupNorm + Mish (groupnorm.cu) and engine (engine_kernels.cu) kernels launched directly on torch device tensors, the operand packing the engines do and
the rotation / trajectory helpers of kin.cuh and repr.cuh one element at a time (not collected by pytest).  The launching functions take `reps`: that many launches back to
back on the default stream."""
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
ATTN_AUTO, ATTN_WGMMA, ATTN_MMA_F16, ATTN_MMA_TF32, ATTN_SIMT, ATTN_WGMMA_STREAM = 0, 1, 2, 3, 4, 5


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
                ("out_row_add", C.c_int), ("clip_rows", C.c_int), ("clip_valid", C.c_int), ("a_stats", C.c_void_p),
                ("a_corr", C.c_void_p), ("res_stats", C.c_void_p), ("res_gamma", C.c_void_p), ("res_beta", C.c_void_p),
                ("stats_out", C.c_void_p), ("ln_eps", C.c_float), ("k_splits", C.c_int), ("split_row_stride", C.c_int),
                ("want_tma_store", C.c_int), ("store_rows", C.c_int64), ("pdl", C.c_int), ("tma_store", C.c_int),
                ("row_mask", C.c_void_p)]


class Attn(C.Structure):
    _fields_ = [("qkv_hi", C.c_void_p), ("qkv_lo", C.c_void_p), ("rows", C.c_int64), ("ctx_hi", C.c_void_p),
                ("ctx_lo", C.c_void_p), ("B", C.c_int), ("S", C.c_int), ("D", C.c_int), ("H", C.c_int), ("scale", C.c_float),
                ("kind", C.c_int), ("which", C.c_int), ("pdl", C.c_int), ("clip_off", C.c_void_p), ("clip_ids", C.c_void_p)]


class GnArgs(C.Structure):  # rohm_b200/csrc/groupnorm.cuh GnArgs
    _fields_ = [("part", C.c_void_p), ("splits", C.c_int), ("split_stride", C.c_int64), ("bias", C.c_void_p),
                ("gamma", C.c_void_p), ("beta", C.c_void_p), ("tp", C.c_void_p), ("tp_stride", C.c_int),
                ("r1", C.c_void_p), ("r2", C.c_void_p), ("out", C.c_void_p), ("out_hi", C.c_void_p),
                ("out_lo", C.c_void_p), ("C", C.c_int), ("Tp", C.c_int), ("T", C.c_int), ("groups", C.c_int),
                ("f16", C.c_int)]


_lib = None


def lib():
    """The probe library; a missing one is an error (build() makes it), never a skip."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FileNotFoundError(f"{LIB_PATH} is missing: run __graft_entry__.build()")
        _lib = C.CDLL(LIB_PATH)
        _lib.probe_gemm.argtypes = [C.POINTER(Gemm), C.c_int]
        _lib.probe_split.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_float]
        _lib.probe_pair_forms.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib.probe_f16_weight_scale.argtypes = [C.c_void_p, C.c_int64, C.POINTER(C.c_float)]
        _lib.probe_attention.argtypes = [C.POINTER(Attn), C.c_int]
        _lib.probe_group_norm.argtypes = [C.POINTER(GnArgs), C.c_int, C.c_int, C.c_int, C.c_void_p]
        _lib.probe_group_norm_clip_slices.argtypes = [C.POINTER(GnArgs), C.c_int, C.c_int, C.POINTER(C.c_int), C.c_void_p,
                                                      C.c_int]
        _lib.probe_group_norm_cluster.argtypes = [C.c_int, C.c_int, C.c_int]
        _lib.probe_layernorm.argtypes = [C.c_int] + [C.c_void_p] * 7 + [C.c_int, C.c_int]
        _lib.probe_fold_ln.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int] + [C.c_void_p] * 3
        _lib.probe_trajnet_time.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int] + [C.c_void_p] * 6 + [
            C.c_int, C.c_void_p, C.c_void_p, C.c_int]
        _lib.probe_sum_split.argtypes = [C.c_void_p, C.c_int, C.c_int64] + [C.c_void_p] * 4 + [
            C.c_int, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_void_p]
        _lib.probe_kin.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
        _lib.probe_clip_of_frame.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int64, C.c_void_p]
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


def pair_forms(x):
    """The operand-pair helpers of rohm_b200/csrc/ptx.cuh on a 1-D fp32 device tensor (length a multiple of 4): fp16 halves
    (hi, lo), each [3, n] with the rows from split_f16, split_f16x2 and split_f16x4, and the TF32 pair (hi, lo), each [n]."""
    x = x.contiguous()
    n = x.numel()
    hi = torch.empty(3, n, dtype=torch.float16, device=x.device)
    lo = torch.empty_like(hi)
    t_hi, t_lo = torch.empty_like(x), torch.empty_like(x)
    assert lib().probe_pair_forms(x.data_ptr(), n, hi.data_ptr(), lo.data_ptr(), t_hi.data_ptr(), t_lo.data_ptr()) == 0
    return hi, lo, t_hi, t_lo


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
         tma_store=False, store_rows=None, k_splits=0, split_row_stride=0,
         a_stats=None, a_corr=None, res_stats=None, res_gamma=None, res_beta=None, stats_out=None, ln_eps=1e-5,
         pdl=False, n_cols=None, row_mask=None, reps=1):
    """launch_gemm, `reps` times; returns (rc, the filled Gemm struct).  segs: list of Seg.  row_mask: uint8 device tensor
    [M] of packed clips' real rows (the others are stored as zeros; it needs clip_rows / clip_valid set) or None."""
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
    g.a_stats, g.a_corr, g.res_stats = _ptr(a_stats), _ptr(a_corr), _ptr(res_stats)
    g.res_gamma, g.res_beta, g.stats_out, g.ln_eps = _ptr(res_gamma), _ptr(res_beta), _ptr(stats_out), ln_eps
    g.k_splits, g.split_row_stride = k_splits, split_row_stride
    g.want_tma_store = int(tma_store)
    g.store_rows = store_rows if store_rows is not None else M
    g.pdl = int(pdl)
    g.row_mask = _ptr(row_mask)
    rc = lib().probe_gemm(C.byref(g), reps)
    return rc, g


def attention(qkv_hi, qkv_lo, ctx_hi, ctx_lo, B, S, D, H, scale, kind, which, pdl=False, reps=1, clip_off=None,
              clip_ids=None):
    """launch_attention for clips of any length, `reps` times; returns 0 or the error code.  Packed clips (int32 device
    tensors, fp16 pairs of head dim 128, wgmma kernels): clip c holds rows [clip_off[c], clip_off[c + 1]) and the launch
    runs the B clips listed in clip_ids, S being their most tokens."""
    a = Attn(_ptr(qkv_hi), _ptr(qkv_lo), qkv_hi.shape[0], _ptr(ctx_hi), _ptr(ctx_lo), B, S, D, H, scale, kind, which, int(pdl),
             _ptr(clip_off), _ptr(clip_ids))
    return lib().probe_attention(C.byref(a), reps)


def group_norm(part, splits, split_stride, bias, gamma, beta, tp, tp_stride, r1, r2, out, out_hi, out_lo, C_, Tp, T, B, n,
               f16, groups=8, reps=1, clip_off=None):
    """gn_mish_split_kernel over B clips with clusters of n CTAs per (clip, group), `reps` times (tensors or None);
    returns 0 or the CUDA error code.  clip_off (int32 device tensor [B + 1]): packed clips, clip b at rows
    [clip_off[b], clip_off[b + 1]) with T real rows at most (the engine's level rows Tp and real rows T per clip)."""
    p = _ptr
    a = GnArgs(p(part), splits, split_stride, p(bias), p(gamma), p(beta), p(tp), tp_stride, p(r1), p(r2), p(out), p(out_hi),
               p(out_lo), C_, Tp, T, groups, int(f16))
    return lib().probe_group_norm(C.byref(a), B, n, reps, p(clip_off))


def group_norm_clip_slices(part, splits, split_stride, bias, gamma, beta, tp, tp_stride, r1, r2, out, out_hi, out_lo, C_, Tp,
                           T, n, f16, clip_off, real_rows, groups=8, reps=1):
    """launch_gn_mish_clip_slices (the batch-invariant engines' instance) over packed clips, n >= 2 CTAs per (clip, group),
    `reps` times; real_rows: the clips' real rows (a list), clip_off as for group_norm.  Returns 0 or the CUDA error code."""
    p = _ptr
    a = GnArgs(p(part), splits, split_stride, p(bias), p(gamma), p(beta), p(tp), tp_stride, p(r1), p(r2), p(out), p(out_hi),
               p(out_lo), C_, Tp, T, groups, int(f16))
    B = len(real_rows)
    rows = (C.c_int * B)(*real_rows)
    return lib().probe_group_norm_clip_slices(C.byref(a), B, n, rows, p(clip_off), reps)


def group_norm_cluster(T, C_, groups=8):
    """The cluster size the TrajNet engine chooses for groups of T rows of C_ / groups channels."""
    return lib().probe_group_norm_cluster(T, C_, groups)


# tests/native/kernel_probe.cu KinOp
OP_ROT6D, OP_ROT6D_BACKWARD, OP_MAT_TO_AA, OP_RODRIGUES, OP_ROUND_TRIP, OP_ROTVEC, OP_HEADING, OP_QROT_Z, OP_TRAJ = range(9)


def _kin(op, a, n_out, b=None, out2=None):
    """One helper over the rows of the fp32 device tensor a ([n, k]) -> fp32 [n, n_out]."""
    a = a.float().contiguous()
    n = a.shape[0]
    out = torch.empty(n, n_out, dtype=torch.float32, device=a.device)
    b = None if b is None else b.float().contiguous()
    assert lib().probe_kin(op, a.data_ptr(), _ptr(b), n, out.data_ptr(), _ptr(out2)) == 0
    return out


def rot6d_to_mat(x):
    """kin::rot6d_to_mat on x [n, 6] -> (R [n, 3, 3], (l1, l2, s) [n, 3])."""
    lls = torch.empty(x.shape[0], 3, dtype=torch.float32, device=x.device)
    return _kin(OP_ROT6D, x, 9, out2=lls).view(-1, 3, 3), lls


def rot6d_backward(x, G):
    """kin::rot6d_backward: x [n, 6], G = dL/dR [n, 3, 3] -> dL/dx [n, 6]."""
    return _kin(OP_ROT6D_BACKWARD, x, 6, b=G.reshape(-1, 9))


def mat_to_aa(R):
    """kin::mat_to_aa: R [n, 3, 3] -> axis-angle [n, 3]."""
    return _kin(OP_MAT_TO_AA, R.reshape(-1, 9), 3)


def rodrigues(r):
    """kin::rodrigues: r [n, 3] -> R [n, 3, 3]."""
    return _kin(OP_RODRIGUES, r, 9).view(-1, 3, 3)


def rot6d_round_trip(x):
    """kin::rodrigues(kin::mat_to_aa(kin::rot6d_to_mat(x))): x [n, 6] -> R [n, 3, 3]."""
    return _kin(OP_ROUND_TRIP, x, 9).view(-1, 3, 3)


def rotvec_to_mat(r):
    """repr::rotvec_to_mat: r [n, 3] -> R [n, 3, 3]."""
    return _kin(OP_ROTVEC, r, 9).view(-1, 3, 3)


def heading_quat(j1, j2, j17, j16):
    """repr::heading_quat on joints [n, 3] each -> (q0, q1, q3) [n, 3]."""
    return _kin(OP_HEADING, torch.cat([j1, j2, j17, j16], dim=1), 3)


def qrot_z(wz, v):
    """repr::qrot_z: wz [n, 2] = (w, z), v [n, 3] -> [n, 3]."""
    return _kin(OP_QROT_Z, wz, 3, b=v)


def traj_channels(q, roots, rots, trs):
    """repr::traj_channels of two frames: q [n, 4] = (w0, z0, w1, z1), roots [n, 2, 3], rots [n, 2, 3, 3], trs [n, 2, 3]
    -> channels [n, 22]."""
    n = q.shape[0]
    return _kin(OP_TRAJ, torch.cat([q, roots.reshape(n, 6), rots.reshape(n, 18), trs.reshape(n, 6)], dim=1), 22)


def clip_of_frame(clip_off, frames):
    """kin::clip_of_frame over int32 device tensors: clip_off [B + 1], frames [n] -> clip ids [n] (int32)."""
    clip_off, frames = clip_off.int().contiguous(), frames.int().contiguous()
    out = torch.empty_like(frames)
    B = clip_off.numel() - 1
    assert lib().probe_clip_of_frame(clip_off.data_ptr(), B, frames.data_ptr(), frames.numel(), out.data_ptr()) == 0
    return out


def layernorm(D, x, res, gamma, beta, out, out_hi, out_lo, rows, f16):
    """layernorm_kernel<D> of x + res (res may be None or `out` itself) over `rows` rows; returns 0 or the error code."""
    return lib().probe_layernorm(D, _ptr(x), _ptr(res), _ptr(gamma), _ptr(beta), _ptr(out), _ptr(out_hi), _ptr(out_lo), rows,
                                 int(f16))


def fold_ln(W, gamma, beta, bias, Wf, c, d):
    """fold_ln_kernel of the [N, K] weight W into Wf, c, d; returns 0 or the error code."""
    N, K = W.shape
    return lib().probe_fold_ln(_ptr(W), _ptr(gamma), _ptr(beta), _ptr(bias), N, K, _ptr(Wf), _ptr(c), _ptr(d))


def trajnet_time(time, ctas_per_clip, time_dim, w1, b1, w3, b3, wcat, bcat, tp, table=None, table_rows=0):
    """trajnet_time_kernel for the int64 timesteps `time` into tp [B, total_out] (total_out = bcat's length); returns 0 or
    the error code."""
    return lib().probe_trajnet_time(_ptr(time), time.numel(), ctas_per_clip, time_dim, _ptr(w1), _ptr(b1), _ptr(w3),
                                    _ptr(b3), _ptr(wcat), _ptr(bcat), bcat.numel(), _ptr(tp), _ptr(table), table_rows)


def sum_split(part, splits, split_stride, bias, out, out_hi, out_lo, C_, Tp, T, rows, f16, row_mask=None):
    """sum_split_kernel over `rows` rows of C_ channels (row_mask: uint8 device tensor of the real rows, or None for
    uniform clips of Tp rows with T real ones); returns 0 or the error code."""
    return lib().probe_sum_split(_ptr(part), splits, split_stride, _ptr(bias), _ptr(out), _ptr(out_hi), _ptr(out_lo), C_, Tp,
                                 T, rows, int(f16), _ptr(row_mask))
