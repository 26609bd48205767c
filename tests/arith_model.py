"""CPU model of the fp16 hi/lo operand arithmetic of the GEMM (DESIGN.md section 2), shared by the CPU checks of the model
(test_kernel_arithmetic_model.py) and the GPU checks that the kernel computes exactly this (test_gpu_gemm.py)."""
import math

import numpy as np

f16, f32, f64 = np.float16, np.float32, np.float64


def split_f16(x):
    """ptx::split_f16: hi = rn_f16(clamp(x, +-65504)), lo = rn_f16(x - hi) (both as float32 values of halves)."""
    x = np.asarray(x, dtype=f32)
    hi = np.clip(x, -65504.0, 65504.0).astype(f16)
    lo = (x - hi.astype(f32)).astype(f16)
    return hi.astype(f32), lo.astype(f32)


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
