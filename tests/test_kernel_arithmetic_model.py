"""CPU models of the arithmetic the CUDA kernels rely on (no GPU, no library calls): the fp16 hi/lo operand pairs with
three products (DESIGN.md section 2) and the branch-free erf GELU whose coefficients live in rohm_b200/csrc/gemm.cu.
These pin the accuracy claims and the constants in the kernel source against float64."""
import math
import os
import re

import numpy as np
from scipy.special import erf

from arith_model import F16_MAX, F16_PAIR_LIMIT, gemm_f16x2, split_f16, split_tf32, weight_scale
from helpers import ROOT

f16, f32, f64 = np.float16, np.float32, np.float64


def test_weight_scale_places_the_largest_weight_in_the_upper_fp16_range():
    rng = np.random.default_rng(0)
    for scale in (1e-6, 3e-3, 0.02, 1.0, 77.0, 4e4):
        w = (rng.standard_normal((64, 48)) * scale).astype(f32)
        s = weight_scale(w)
        top = float(np.abs(w).max()) * s
        assert 2.0 ** 13 <= top < 2.0 ** 14
        assert math.log2(s) == round(math.log2(s))  # a power of two: undone exactly by acc_scale
    assert weight_scale(np.zeros((4, 4), f32)) == 1.0


def test_pair_split_keeps_22_bits_and_degrades_gracefully():
    rng = np.random.default_rng(1)
    x = (rng.standard_normal(200000) * 3).astype(f32)
    hi, lo = split_f16(x)
    rel = np.abs((hi.astype(f64) + lo.astype(f64)) - x.astype(f64)) / np.maximum(np.abs(x.astype(f64)), 1e-30)
    assert rel[np.abs(x) > 0.2].max() < 2.0 ** -21          # both halves in the normal range: 2 x 11 bits
    tiny = (rng.standard_normal(10000) * 1e-4).astype(f32)   # lo halves subnormal: bounded absolute error instead
    hi, lo = split_f16(tiny)
    assert np.abs((hi.astype(f64) + lo.astype(f64)) - tiny.astype(f64)).max() <= 2.0 ** -25
    big = np.array([70000.0, -120000.0, 131000.0], dtype=f32)  # beyond fp16's largest finite value
    hi, lo = split_f16(big)
    assert np.all(np.isfinite(hi)) and np.all(np.isfinite(lo))
    assert np.abs((hi + lo) - big).max() <= 64.0               # still 11+ bits; the pair's range ends at 131024


def _f32_range(lo, hi):
    """Every float32 in [lo, hi] (0 <= lo <= hi), in order."""
    a, b = np.array([lo, hi], dtype=f32).view(np.uint32)
    return np.arange(a, b + 1, dtype=np.uint32).view(f32)


def test_f16_pair_is_finite_exactly_below_131024():
    """hi saturates at 65504 and lo does not: every float32 with |x| < 65504 + 65520 has a finite pair, every larger one
    (and +-inf) a pair of +-inf with the sign of x, never a plausible finite value.  NaN gives NaN in both halves."""
    x = _f32_range(60000.0, 140000.0)
    x = np.concatenate([x, -x, np.array([np.inf, -np.inf, 2e5, -2e5, 1e30, -1e30, 3.4028235e38], dtype=f32)])
    hi, lo = split_f16(x)
    pair = hi.astype(f64) + lo.astype(f64)
    below = np.abs(x) < F16_PAIR_LIMIT
    assert np.isfinite(pair[below]).all() and np.isfinite(hi).all()
    assert (np.abs(hi[np.abs(x) >= F16_MAX]) == F16_MAX).all()
    assert np.isinf(pair[~below]).all() and (np.sign(pair[~below]) == np.sign(x[~below])).all()
    assert np.nextafter(f32(F16_PAIR_LIMIT), f32(0.0)) in x[below] and f32(F16_PAIR_LIMIT) in x[~below]
    # the largest finite pair value: 65504 + 65504
    assert pair[below].max() == 2 * F16_MAX and pair[below].min() == -2 * F16_MAX
    # above the fp16 range the pair still carries 11 significant bits (lo = rn_f16(x - 65504))
    mid = below & (np.abs(x) > F16_MAX)
    assert (np.abs(pair[mid] - x[mid]) <= 2.0 ** -12 * np.abs(x[mid])).all()
    hi, lo = split_f16(np.array([np.nan, -np.nan], dtype=f32))
    assert np.isnan(hi).all() and np.isnan(lo).all()


def test_f16_pair_error_is_2_22_relative_or_2_25_absolute():
    """|hi + lo - x| <= max(2^-22 |x|, 2^-25) for every finite |x| <= 65504: 2 x 11 significant bits while lo is normal,
    an absolute 2^-25 (half the smallest fp16 subnormal) once lo or hi goes subnormal.  Random bit patterns over the whole
    fp32 range, the fp16 subnormal range 2^-24 .. 2^-14 densely, fp32 subnormals, and hi / lo rounding ties."""
    rng = np.random.default_rng(7)
    x = rng.integers(0, 2 ** 32, size=2 ** 20, dtype=np.uint64).astype(np.uint32).view(f32)
    ties = np.array([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 1.0 + 2.0 ** -11 + 2.0 ** -22, 1.0 + 2.0 ** -11 + 3 * 2.0 ** -22,
                     2048.0 + 1.0, 2048.0 + 3.0, 65504.0 - 16.0, 2.0 ** -14 + 2.0 ** -25, 2.0 ** -24 + 2.0 ** -25,
                     2.0 ** -25, 3 * 2.0 ** -25], dtype=f32)
    x = np.concatenate([x, _f32_range(2.0 ** -24, 2.0 ** -14)[::7], _f32_range(1e-45, 1.1754942e-38)[::4099], ties,
                        np.array([0.0, 65504.0, 65519.996], dtype=f32)])
    x = np.concatenate([x, -x])
    x = x[np.isfinite(x) & (np.abs(x) <= F16_MAX)]
    hi, lo = split_f16(x)
    err = np.abs(hi.astype(f64) + lo.astype(f64) - x.astype(f64))
    assert (err <= np.maximum(2.0 ** -22 * np.abs(x.astype(f64)), 2.0 ** -25)).all()
    # hi is x rounded to fp16: |x - hi| <= half an ulp of hi, and lo never exceeds it
    assert (np.abs(lo) <= np.maximum(2.0 ** -11 * np.abs(hi.astype(f64)), 2.0 ** -25)).all()


def test_tf32_model_rounds_half_away_to_11_bits():
    """split_tf32's bit operations against the same rounding done in float64: hi = x rounded half away from zero to a
    multiple of 2^(max(e, -126) - 10), e = floor(log2 |x|) -- the 11 significant bits of TF32 in the normal range, the
    fixed 2^-136 grid of the smallest binade for fp32 subnormals."""
    rng = np.random.default_rng(8)
    x = rng.integers(0, 2 ** 32, size=2 ** 20, dtype=np.uint64).astype(np.uint32).view(f32)
    ties = np.array([1.0 + 2.0 ** -11, 1.0 + 3 * 2.0 ** -11, 2.0 - 2.0 ** -11, 2.0 ** -130 + 2.0 ** -137,
                     2.0 ** -126 - 2.0 ** -137], dtype=f32)
    x = np.concatenate([x, ties, -ties, _f32_range(1e-45, 1.1754942e-38)[::997]])
    x = x[np.isfinite(x) & (np.abs(x) < 2.0 ** 127)]
    hi, lo = split_tf32(x)
    a = np.abs(x.astype(f64))
    e = np.floor(np.log2(np.where(a > 0, a, 1.0)))
    q = np.exp2(np.maximum(e, -126.0) - 10.0)
    want = np.copysign(np.floor(a / q + 0.5) * q, x.astype(f64))
    assert (hi.astype(f64) == want).all()
    assert ((hi.view(np.uint32) & 0x1FFF) == 0).all()


def test_tf32_pair_is_exact_below_the_top_binade():
    """lo = x - hi is exact in fp32, so hi + lo == x for every finite x below 2^127 (fp32 subnormals included).  In the
    top binade |x| >= 2^128 (1 - 2^-12) rounds to hi = +-inf and the pair is NaN (the kernels' behaviour, recorded in
    DESIGN.md section 2); +-inf gives (+-inf, NaN), NaN a NaN lo."""
    rng = np.random.default_rng(9)
    x = rng.integers(0, 2 ** 32, size=2 ** 20, dtype=np.uint64).astype(np.uint32).view(f32)
    x = np.concatenate([x, _f32_range(1e-45, 1.1754942e-38)[::997], np.array([0.0, -0.0], dtype=f32)])
    x = x[np.isfinite(x) & (np.abs(x) < 2.0 ** 127)]
    hi, lo = split_tf32(x)
    assert (hi.astype(f64) + lo.astype(f64) == x.astype(f64)).all()
    top = _f32_range(2.0 ** 127, 3.4028235e38)
    hi, lo = split_tf32(top)
    edge = f32(2.0 ** 128 * (1.0 - 2.0 ** -12))
    fin = top < edge
    assert (hi[fin].astype(f64) + lo[fin].astype(f64) == top[fin].astype(f64)).all()
    assert np.isposinf(hi[~fin]).all() and np.isneginf(lo[~fin]).all() and edge in top[~fin]
    hi, lo = split_tf32(np.array([np.inf, -np.inf, np.nan], dtype=f32))
    assert hi[0] == np.inf and hi[1] == -np.inf and np.isnan(lo).all() and np.isnan(hi[2])
    # NaNs are truncated, not rounded: a payload in the low 13 bits leaves hi = +-inf, but the pair is NaN either way
    hi, lo = split_tf32(np.array([0x7F800001, 0xFF801FFF, 0x7F802000, 0x7FFFFFFF], dtype=np.uint32).view(f32))
    assert hi[0] == np.inf and hi[1] == -np.inf and np.isnan(hi[2:]).all() and np.isnan(lo).all()


def test_three_product_gemm_is_fp32_grade():
    rng = np.random.default_rng(2)
    for K, a_scale, w_scale in ((512, 1.0, 1 / math.sqrt(512)), (1024, 30.0, 0.02), (320, 1e-3, 0.1)):
        a = (rng.standard_normal((96, K)) * a_scale).astype(f32)
        w = (rng.standard_normal((80, K)) * w_scale).astype(f32)
        ref = a.astype(f64) @ w.astype(f64).T
        got = gemm_f16x2(a, w).astype(f64)
        fp32_ref = (a @ w.T).astype(f64)
        bound = np.abs(a.astype(f64)) @ np.abs(w.astype(f64)).T  # sum |a||w|: the natural scale of the rounding error
        # only lo*lo (2^-22 relative per product) is dropped; activations whose lo half is subnormal (|a| < 0.12) add an
        # absolute 2^-25 per element instead (the 1e-3-scaled case)
        floor = 2.0 ** -25 * np.abs(w.astype(f64)).sum(axis=1)[None, :]
        assert (np.abs(got - ref) / (2.0 ** -20 * bound + floor)).max() < 1.0
        if a_scale >= 1.0:
            assert np.abs(got - ref).max() <= 4.0 * np.abs(fp32_ref - ref).max()  # same class as a plain fp32 GEMM
            # a single product (what a one-pass fp16 / TF32 tensor-core GEMM does) is orders of magnitude worse
            ah, _ = split_f16(a)
            wh, _ = split_f16(w)
            one_pass = ah.astype(f64) @ wh.astype(f64).T
            assert np.abs(one_pass - ref).max() > 100.0 * np.abs(got - ref).max()


def _gelu_coefficients():
    src = open(os.path.join(ROOT, "rohm_b200", "csrc", "gemm.cu")).read()
    body = src[src.index("__device__ __forceinline__ float gelu_erf(float x)"):]
    body = body[:body.index("struct EpiParams")]
    q = [float(v) for v in re.findall(r"q = (?:fmaf\(q, u, )?(-?\d\.\d+e[+-]\d+)f", body)]
    clamp = float(re.search(r"fminf\(fabsf\(x\), (\d+\.\d+)f\)", body).group(1))
    assert len(q) == 9, q
    return q, clamp  # highest degree first, as the Horner chain in the kernel evaluates them


def test_branch_free_erf_gelu_constants_match_float64():
    """gelu(x) = max(x, 0) - |x| 2^Q(min(|x|, 6.5)) with the constants compiled into the GEMM epilogue (gemm.cu: gelu_erf),
    evaluated in emulated fp32 against the float64 erf form (nn.GELU's default)."""
    q_coef, clamp = _gelu_coefficients()

    def fma(a, b, c):
        return (a.astype(f64) * b.astype(f64) + np.asarray(c, dtype=f64)).astype(f32)

    x = np.concatenate([np.linspace(-12.0, 12.0, 400001), np.random.default_rng(3).standard_normal(200000) * 3,
                        np.linspace(-500.0, 500.0, 20001)]).astype(f32)
    u = np.minimum(np.abs(x), f32(clamp)).astype(f32)
    q = np.full_like(u, f32(q_coef[0]))
    for c in q_coef[1:]:
        q = fma(q, u, f32(c))
    p = np.exp2(q.astype(f64)).astype(f32)
    gelu = fma(-np.abs(x), p, np.maximum(x, f32(0.0))).astype(f64)
    x64 = x.astype(f64)
    ref = 0.5 * x64 * (1.0 + erf(x64 / math.sqrt(2.0)))
    assert np.abs(gelu - ref).max() < 3e-7  # tools/fit_gelu_erf.py reports 2.5e-7 (fp32 erff formulation: 4.5e-7)
    assert gelu[x > 8.0].tolist() == x64[x > 8.0].tolist() and np.all(np.abs(gelu[x < -8.0]) < 3e-8)  # saturation
    # below -6.5 the tail |x| Phi(-|x|) is taken as |x| 2^Q(6.5): the slope of the extra error gemm.cu documents
    assert 3.4e-11 < float(p[np.abs(x) >= clamp][0]) < 3.6e-11


def test_split_k_partials_added_in_order_stay_fp32_grade():
    """TrajNet's deep-level convolutions (trajnet.cu: pick_split, gemm.cu: GemmParams::k_splits): the K extent is cut into S
    contiguous ranges, every range is accumulated on its own (two accumulators, as above), stored as an fp32 partial and the
    consumer adds bias + partials in split order.  S more fp32 roundings per output: the result stays in the error class of the
    single-pass product, and the order is fixed, so it is deterministic."""
    rng = np.random.default_rng(5)
    for K, S in ((5120, 6), (2560, 3), (1280, 5)):
        a = rng.standard_normal((40, K)).astype(f32)
        w = (rng.standard_normal((64, K)) / math.sqrt(K)).astype(f32)
        bias = rng.standard_normal(64).astype(f32)
        ref = a.astype(f64) @ w.astype(f64).T + bias.astype(f64)
        s = weight_scale(w)
        per = -(-(K // 64) // S) * 64  # ranges of whole 64-column K blocks, ceil(blocks / S) each, the last one shorter
        assert (S - 1) * per < K         # launch_cfg's requirement: no empty range
        acc = bias.astype(f32)[None, :].repeat(40, axis=0)
        for sp in range(S):
            k0, k1 = sp * per, min(K, (sp + 1) * per)
            # one weight scale per matrix (not per range), as the kernel packs it
            ah, al = split_f16(a[:, k0:k1])
            wh, wl = split_f16((w[:, k0:k1] * f32(s)).astype(f32))
            main = (ah.astype(f64) @ wh.astype(f64).T).astype(f32)
            cross = (al.astype(f64) @ wh.astype(f64).T + ah.astype(f64) @ wl.astype(f64).T).astype(f32)
            part = ((main + cross) * f32(1.0 / s)).astype(f32)
            acc = (acc + part).astype(f32)
        single = (gemm_f16x2(a, w) + bias).astype(f32)
        bound = np.abs(a.astype(f64)) @ np.abs(w.astype(f64)).T + np.abs(bias.astype(f64))
        assert (np.abs(acc.astype(f64) - ref) / (2.0 ** -20 * bound)).max() < 1.0
        assert np.abs(acc.astype(f64) - ref).max() <= 4.0 * max(np.abs(single.astype(f64) - ref).max(), 1e-7)


def test_group_statistics_taken_in_the_groupnorm_kernel():
    """gn_mish_split_kernel: per (clip, group) sum and sum of squares of the fp32 values accumulated in double, mean and
    E[x^2] - mean^2 formed in double, mu / rstd cast to fp32 -- against GroupNorm in float64 (torch.nn.GroupNorm(8, C), eps 1e-5)
    for the group shapes of the five pyramid levels, including a large common offset (cancellation in E[x^2] - mean^2)."""
    rng = np.random.default_rng(6)
    for T, gs, offset in ((144, 8, 0.0), (72, 16, 3.0), (36, 32, -50.0), (18, 64, 400.0), (9, 64, 0.0), (144, 4, 1e3)):
        y = (rng.standard_normal((T, gs)) * 2.0 + offset).astype(f32)
        s1 = y.astype(f64).sum()
        s2 = (y.astype(f64) * y.astype(f64)).sum()
        n = float(T * gs)
        mean = s1 / n
        var = max(s2 / n - mean * mean, 0.0)
        mu, rstd = f32(mean), f32(1.0 / math.sqrt(var + 1e-5))
        got = ((y - mu) * rstd).astype(f64)
        y64 = y.astype(f64)
        ref = (y64 - y64.mean()) / np.sqrt(y64.var() + 1e-5)
        assert np.abs(got - ref).max() < 2e-6 * max(1.0, abs(offset) / 2.0)
