"""CPU model of the hi/lo operand arithmetic of the GEMM (DESIGN.md section 2), shared by the CPU checks of the model
(test_kernel_arithmetic_model.py) and the GPU checks that the kernels compute exactly this (test_gpu_gemm.py,
test_gpu_operand_pairs.py).  The pair models follow the PTX semantics of the conversions in rohm_b200/csrc/ptx.cuh."""
import math

import numpy as np

f16, f32, f64 = np.float16, np.float32, np.float64

F16_MAX = 65504.0
# the fp16 pair of x is finite exactly when |x| < F16_MAX + 65520: beyond, lo = rn_f16(x - 65504) overflows
F16_PAIR_LIMIT = F16_MAX + 65520.0


def split_f16(x):
    """The fp16 operand pair of ptx::split_f16 / split_f16x2 / split_f16x4 (float32 values of the halves):
    hi = rn_f16(x) saturated to +-65504 (NaN stays NaN), lo = rn_f16(x - hi) with no saturation, so the pair is finite
    exactly when |x| < F16_PAIR_LIMIT and +-inf beyond; NaN gives NaN in both halves."""
    x = np.asarray(x, dtype=f32)
    with np.errstate(invalid="ignore", over="ignore"):
        hi = np.where(np.abs(x) > f32(F16_MAX), np.copysign(f32(F16_MAX), x), x).astype(f16)
        lo = (x - hi.astype(f32)).astype(f16)
    return hi.astype(f32), lo.astype(f32)


def split_tf32(x):
    """The TF32 operand pair: hi = ptx::to_tf32(x) (cvt.rna.tf32.f32), lo = x - hi in fp32.  Rounding in integer bit
    operations: the magnitude's bit pattern plus 2^12, low 13 bits cleared -- round half away from zero to 10 mantissa bits,
    with the carry running into the exponent.  So fp32 subnormals round on the same 2^-136 grid as the smallest normal
    binade, and in the top binade |x| >= 2^128 (1 - 2^-12) rounds to hi = +-inf, lo = -+inf (a NaN pair); +-inf gives
    (+-inf, NaN).  Non-finite inputs are not rounded, only their low 13 bits cleared: a NaN keeps the top 10 bits of its
    payload, so one whose payload lies in the low 13 bits becomes hi = +-inf.  lo is NaN for every NaN."""
    x = np.asarray(x, dtype=f32)
    bits = x.view(np.uint32)
    finite = (bits & np.uint32(0x7FFFFFFF)) < np.uint32(0x7F800000)
    hi = (np.where(finite, bits + np.uint32(0x1000), bits) & np.uint32(0xFFFFE000)).view(f32)
    with np.errstate(invalid="ignore", over="ignore"):
        lo = (x - hi).astype(f32)
    return hi, lo


def weight_scale(w):
    """f16_weight_scale: 2^s with max|w| 2^s in [2^13, 2^14)."""
    wmax = float(np.abs(w).max())
    if wmax == 0.0:
        return 1.0
    _, e2 = math.frexp(wmax)
    return math.ldexp(1.0, max(-100, min(100, 14 - e2)))


def gemm_f16x2(a, w):
    """D = A_lo W_hi^T + A_hi W_lo^T (small terms, own accumulator) + A_hi W_hi^T, products exact, fp32 accumulation."""
    s = weight_scale(w)
    ah, al = split_f16(a)
    wh, wl = split_f16((w * f32(s)).astype(f32))
    # fp16 x fp16 products are exact in fp32; the accumulation is modelled in float64 and rounded once per accumulator
    # (the tensor core's fp32 accumulation error is measured on the GPU, not modelled here)
    main = (ah.astype(f64) @ wh.astype(f64).T).astype(f32)
    cross = (al.astype(f64) @ wh.astype(f64).T + ah.astype(f64) @ wl.astype(f64).T).astype(f32)
    return ((main + cross) * f32(1.0 / s)).astype(f32)
