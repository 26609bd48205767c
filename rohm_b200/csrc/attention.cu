// The attention kernels declared in attention.cuh and their launchers.
#include "attention.cuh"

#include <cmath>

#include "common.h"
#include "gemm.cuh"
#include "ptx.cuh"

namespace rohm {
namespace {

// Multi-head self-attention, fp32 on CUDA cores (v1): one CTA per (clip, head); K and V of the head live in shared
// memory, each warp owns query rows round-robin.  softmax(Q K^T / sqrt(dh)) V with no mask (posenet.py:63-69).
// qkv: [B*S, 3*D] fp32 (Q | K | V, head h at columns h*DH).  ctx hi/lo: [B*S, D].
// f16 != 0: Q/K/V arrive as fp16 hi/lo pairs (qkv = hi plane, qkv_lo = lo plane; value = hi + lo) and ctx is written as
// fp16 pairs.
__device__ __forceinline__ float4 load_qkv4(const float* qkv, const float* qkv_lo, int f16, int64_t idx) {
  if (!f16) return *reinterpret_cast<const float4*>(qkv + idx);
  const uint2 h = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(qkv) + idx);
  const uint2 l = *reinterpret_cast<const uint2*>(reinterpret_cast<const __half*>(qkv_lo) + idx);
  const __half2 h0 = *reinterpret_cast<const __half2*>(&h.x), h1 = *reinterpret_cast<const __half2*>(&h.y);
  const __half2 l0 = *reinterpret_cast<const __half2*>(&l.x), l1 = *reinterpret_cast<const __half2*>(&l.y);
  return make_float4(__low2float(h0) + __low2float(l0), __high2float(h0) + __high2float(l0),
                     __low2float(h1) + __low2float(l1), __high2float(h1) + __high2float(l1));
}
template <int DH>
__global__ void __launch_bounds__(256) attention_kernel(const float* __restrict__ qkv, const float* __restrict__ qkv_lo,
                                                        float* __restrict__ ctx_hi, float* __restrict__ ctx_lo, int S,
                                                        int D, int H, float scale, int f16) {
  constexpr int KP = DH + 4;  // padded K row: conflict-free float4 reads with one key per lane
  constexpr int NW = 8;
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  extern __shared__ float sm[];
  float* Ks = sm;                      // [S][KP]
  float* Vs = Ks + S * KP;             // [S][DH]
  float* Qs = Vs + S * DH;             // [NW][DH]
  const int Sp = (S + 31) & ~31;
  float* Ps = Qs + NW * DH;            // [NW][Sp]
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t base = static_cast<int64_t>(b) * S;
  const int ld = 3 * D;

  for (int i = threadIdx.x; i < S * (DH / 4); i += blockDim.x) {
    const int s = i / (DH / 4), c = i % (DH / 4);
    const int64_t row = (base + s) * ld + h * DH + c * 4;
    const float4 k = load_qkv4(qkv, qkv_lo, f16, row + D);
    const float4 v = load_qkv4(qkv, qkv_lo, f16, row + 2 * D);
    *reinterpret_cast<float4*>(Ks + s * KP + c * 4) = k;
    *reinterpret_cast<float4*>(Vs + s * DH + c * 4) = v;
  }
  __syncthreads();

  constexpr int MAXJ = 8;  // supports S <= 256
  const int nj = Sp / 32;
  float* q = Qs + warp * DH;
  float* p = Ps + warp * Sp;
  for (int i = warp; i < S; i += NW) {
    const int64_t qrow = (base + i) * ld + h * DH;
    for (int c = lane; c < DH / 4; c += 32) *reinterpret_cast<float4*>(q + c * 4) = load_qkv4(qkv, qkv_lo, f16, qrow + c * 4);
    __syncwarp();
    float sc[MAXJ];
#pragma unroll
    for (int jj = 0; jj < MAXJ; ++jj) sc[jj] = 0.0f;
    for (int d = 0; d < DH; d += 4) {
      const float4 qv = *reinterpret_cast<const float4*>(q + d);
#pragma unroll
      for (int jj = 0; jj < MAXJ; ++jj) {
        if (jj < nj) {
          int j = lane + 32 * jj;
          j = j < S ? j : S - 1;
          const float4 kv = *reinterpret_cast<const float4*>(Ks + j * KP + d);
          sc[jj] = fmaf(qv.x, kv.x, sc[jj]);
          sc[jj] = fmaf(qv.y, kv.y, sc[jj]);
          sc[jj] = fmaf(qv.z, kv.z, sc[jj]);
          sc[jj] = fmaf(qv.w, kv.w, sc[jj]);
        }
      }
    }
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < MAXJ; ++jj) {
      if (jj < nj) {
        sc[jj] = (lane + 32 * jj < S) ? sc[jj] * scale : -INFINITY;
        mx = fmaxf(mx, sc[jj]);
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, off));
    float sum = 0.0f;
#pragma unroll
    for (int jj = 0; jj < MAXJ; ++jj) {
      if (jj < nj) {
        sc[jj] = (lane + 32 * jj < S) ? expf(sc[jj] - mx) : 0.0f;
        sum += sc[jj];
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
    const float inv = 1.0f / sum;
#pragma unroll
    for (int jj = 0; jj < MAXJ; ++jj)
      if (jj < nj) p[lane + 32 * jj] = sc[jj] * inv;
    __syncwarp();
    // P V: lane owns DH/32 consecutive channels
    constexpr int CPL = DH / 32;
    float acc[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) acc[c] = 0.0f;
    for (int j = 0; j < S; ++j) {
      const float pj = p[j];
      const float* vr = Vs + j * DH + lane * CPL;
      if (CPL == 4) {
        const float4 vv = *reinterpret_cast<const float4*>(vr);
        acc[0] = fmaf(pj, vv.x, acc[0]);
        acc[1] = fmaf(pj, vv.y, acc[1]);
        acc[2 % CPL] = fmaf(pj, vv.z, acc[2 % CPL]);
        acc[3 % CPL] = fmaf(pj, vv.w, acc[3 % CPL]);
      } else {
        const float2 vv = *reinterpret_cast<const float2*>(vr);
        acc[0] = fmaf(pj, vv.x, acc[0]);
        acc[1] = fmaf(pj, vv.y, acc[1]);
      }
    }
    const int64_t o = (base + i) * D + h * DH + lane * CPL;
    if (f16) {
#pragma unroll
      for (int c = 0; c < CPL; ++c)
        ptx::split_f16(acc[c], reinterpret_cast<__half*>(ctx_hi)[o + c], reinterpret_cast<__half*>(ctx_lo)[o + c]);
      __syncwarp();
      continue;
    }
    float hh[CPL], ll[CPL];
#pragma unroll
    for (int c = 0; c < CPL; ++c) {
      hh[c] = ptx::to_tf32(acc[c]);
      ll[c] = acc[c] - hh[c];
    }
    if (CPL == 4) {
      *reinterpret_cast<float4*>(ctx_hi + o) = make_float4(hh[0], hh[1], hh[2 % CPL], hh[3 % CPL]);
      *reinterpret_cast<float4*>(ctx_lo + o) = make_float4(ll[0], ll[1], ll[2 % CPL], ll[3 % CPL]);
    } else {
      *reinterpret_cast<float2*>(ctx_hi + o) = make_float2(hh[0], hh[1]);
      *reinterpret_cast<float2*>(ctx_lo + o) = make_float2(ll[0], ll[1]);
    }
    __syncwarp();
  }
}

// ---- tensor-core attention (v2) -------------------------------------------------------------------------------
// One CTA per (clip, head); warp w owns query rows [16w, 16w+16).  S = Q K^T and O = P V run on mma.sync m16n8k8
// TF32 with the same 3-pass hi/lo error compensation as the GEMMs; logits, softmax and P never leave registers
// (the S accumulator fragment is reused as the A fragment of P V by enumerating the 8 keys of a k-step in the
// order the accumulator holds them, so no shuffle or shared-memory round trip is needed).
// K and V of the head are staged once in shared memory with a 132-float row pitch (conflict-free fragment loads);
// Q fragments are read straight from global/L2 (each value is used exactly once).
__device__ __forceinline__ void mma_tf32_16x8x8(float (&c)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  const float h = ptx::to_tf32(x);
  hi = __float_as_uint(h);
  lo = __float_as_uint(x - h);
}

// Same split, but opaque to the optimiser: used inside the rolled P V loop, where hoisting the loop-invariant split of
// the whole P fragment out of the loop would double its register footprint (and spill).
__device__ __forceinline__ void split_tf32_pinned(float x, uint32_t& hi, uint32_t& lo) {
  uint32_t r;
  asm volatile("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  hi = r;
  lo = __float_as_uint(x - __uint_as_float(r));
}

constexpr int kAttnPitch = 132;

template <int DH, int NT>  // NT = number of 8-key tiles (keys padded to 8*NT), rows padded to 16 * warps
__global__ void __launch_bounds__(32 * ((NT + 1) / 2), 1) attention_mma_kernel(const float* __restrict__ qkv,
                                                                          float* __restrict__ ctx_hi,
                                                                          float* __restrict__ ctx_lo, int S, int D,
                                                                          int H, float scale, int f16) {
  extern __shared__ float sm[];
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  float* Ks = sm;                          // [8*NT][kAttnPitch]
  float* Vs = Ks + 8 * NT * kAttnPitch;    // [8*NT][kAttnPitch]
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int64_t base = static_cast<int64_t>(b) * S;
  const int ld = 3 * D;

  for (int i = threadIdx.x; i < 8 * NT * (DH / 4); i += blockDim.x) {
    const int s = i / (DH / 4), c = i % (DH / 4);
    float4 k = make_float4(0.f, 0.f, 0.f, 0.f), v = k;
    if (s < S) {
      const float* row = qkv + (base + s) * ld + h * DH + c * 4;
      k = *reinterpret_cast<const float4*>(row + D);
      v = *reinterpret_cast<const float4*>(row + 2 * D);
    }
    *reinterpret_cast<float4*>(Ks + s * kAttnPitch + c * 4) = k;
    *reinterpret_cast<float4*>(Vs + s * kAttnPitch + c * 4) = v;
  }

  const int r0 = warp * 16;
  const int rowA = min(r0 + g, S - 1), rowB = min(r0 + g + 8, S - 1);
  const float* qA = qkv + (base + rowA) * ld + h * DH;
  const float* qB = qkv + (base + rowB) * ld + h * DH;
  __syncthreads();

  // ---- S = Q K^T ----  (k loop deliberately NOT unrolled: the fully unrolled kernel was instruction-cache bound,
  // ncu: stall_no_instruction 5.1 of 11.3 cycles per issued instruction)
  float acc[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0f;
  // Q fragment of k-step k: a0..a3 = Q[rowA][8k+t], Q[rowB][8k+t], Q[rowA][8k+t+4], Q[rowB][8k+t+4]; prefetched one
  // k-step ahead (each value is used once, straight from L2)
  float qn[4] = {__ldg(qA + t), __ldg(qB + t), __ldg(qA + t + 4), __ldg(qB + t + 4)};
#pragma unroll 1
  for (int k = 0; k < DH / 8; ++k) {
    uint32_t ah[4], al[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) split_tf32(qn[i], ah[i], al[i]);
    if (k + 1 < DH / 8) {
      qn[0] = __ldg(qA + 8 * (k + 1) + t);
      qn[1] = __ldg(qB + 8 * (k + 1) + t);
      qn[2] = __ldg(qA + 8 * (k + 1) + t + 4);
      qn[3] = __ldg(qB + 8 * (k + 1) + t + 4);
    }
    const float* kp = Ks + g * kAttnPitch + 8 * k + t;
    // groups of 4 key tiles: all B fragments of the group are split first, then the three passes are issued pass-major,
    // so consecutive MMAs hit different accumulators (the per-tile order lo*hi, hi*lo, hi*hi would serialise on one)
#pragma unroll
    for (int j0 = 0; j0 < NT; j0 += 4) {
      uint32_t bh[4][2], bl[4][2];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        if (j0 + u < NT) {
          split_tf32(kp[(j0 + u) * 8 * kAttnPitch], bh[u][0], bl[u][0]);
          split_tf32(kp[(j0 + u) * 8 * kAttnPitch + 4], bh[u][1], bl[u][1]);
        }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (j0 + u < NT) mma_tf32_16x8x8(acc[j0 + u], al, bh[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (j0 + u < NT) mma_tf32_16x8x8(acc[j0 + u], ah, bl[u]);
#pragma unroll
      for (int u = 0; u < 4; ++u)
        if (j0 + u < NT) mma_tf32_16x8x8(acc[j0 + u], ah, bh[u]);
    }
  }

  // ---- softmax over keys (rows rowA: elements [0],[1]; rowB: [2],[3]; columns 8j + 2t + {0,1}) ----
  float mxA = -INFINITY, mxB = -INFINITY;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool ok = (8 * j + 2 * t + e) < S;
      acc[j][e] = ok ? acc[j][e] * scale : -INFINITY;
      acc[j][2 + e] = ok ? acc[j][2 + e] * scale : -INFINITY;
      mxA = fmaxf(mxA, acc[j][e]);
      mxB = fmaxf(mxB, acc[j][2 + e]);
    }
  }
  mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 1));
  mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 2));
  mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 1));
  mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 2));
  float sumA = 0.0f, sumB = 0.0f;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      acc[j][e] = expf(acc[j][e] - mxA);      // exp(-inf) = 0 for padded keys
      acc[j][2 + e] = expf(acc[j][2 + e] - mxB);
      sumA += acc[j][e];
      sumB += acc[j][2 + e];
    }
  }
  sumA += __shfl_xor_sync(0xffffffffu, sumA, 1);
  sumA += __shfl_xor_sync(0xffffffffu, sumA, 2);
  sumB += __shfl_xor_sync(0xffffffffu, sumB, 1);
  sumB += __shfl_xor_sync(0xffffffffu, sumB, 2);
  const float invA = 1.0f / sumA, invB = 1.0f / sumB;

  // ---- O = P V ----
  // A fragment of k-step j (keys 8j..8j+7, enumerated as column t -> key 8j+2t, column t+4 -> key 8j+2t+1):
  //   a0 = P[rowA][8j+2t] = acc[j][0], a1 = P[rowB][8j+2t] = acc[j][2], a2 = acc[j][1], a3 = acc[j][3]
  // B fragment for output dims 8n..8n+7:  b0 = V[8j+2t][8n+g], b1 = V[8j+2t+1][8n+g]
  // The loop over the 8-wide output tiles is rolled (P lives in registers and needs static indexing, O does not):
  // each iteration produces and stores one 16 x 8 output tile.
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    acc[j][0] *= invA, acc[j][1] *= invA;
    acc[j][2] *= invB, acc[j][3] *= invB;
  }
  const bool okA = (r0 + g) < S, okB = (r0 + g + 8) < S;
  const int64_t oA = (base + r0 + g) * D + h * DH + 2 * t;
  const int64_t oB = oA + static_cast<int64_t>(8) * D;
  // four 8-wide output tiles per iteration: the hi/lo split of the P fragment is shared by the four tiles and the
  // eight accumulators (main + cross terms per tile) give the tensor pipe independent work
  constexpr int NU = 4;
#pragma unroll 1
  for (int n0 = 0; n0 < DH / 8; n0 += NU) {
    float o[NU][4], os[NU][4];
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      o[u][0] = o[u][1] = o[u][2] = o[u][3] = 0.0f;
      os[u][0] = os[u][1] = os[u][2] = os[u][3] = 0.0f;
    }
    const float* vp = Vs + 2 * t * kAttnPitch + g + 8 * n0;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      uint32_t ah[4], al[4];
      split_tf32_pinned(acc[j][0], ah[0], al[0]);
      split_tf32_pinned(acc[j][2], ah[1], al[1]);
      split_tf32_pinned(acc[j][1], ah[2], al[2]);
      split_tf32_pinned(acc[j][3], ah[3], al[3]);
      uint32_t bh[NU][2], bl[NU][2];
#pragma unroll
      for (int u = 0; u < NU; ++u) {
        split_tf32(vp[8 * j * kAttnPitch + 8 * u], bh[u][0], bl[u][0]);
        split_tf32(vp[(8 * j + 1) * kAttnPitch + 8 * u], bh[u][1], bl[u][1]);
      }
#pragma unroll
      for (int u = 0; u < NU; ++u) mma_tf32_16x8x8(os[u], al, bh[u]);
#pragma unroll
      for (int u = 0; u < NU; ++u) mma_tf32_16x8x8(o[u], ah, bh[u]);
#pragma unroll
      for (int u = 0; u < NU; ++u) mma_tf32_16x8x8(os[u], ah, bl[u]);
    }
    // store ctx as TF32 hi/lo (o[.][0..1] = row rowA, cols 8n+2t,+1; o[.][2..3] = row rowB)
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const int n = n0 + u;
#pragma unroll
      for (int i = 0; i < 4; ++i) o[u][i] += os[u][i];
      if (f16) {
        __half2 hA, lA, hB, lB;
        ptx::split_f16(o[u][0], hA.x, lA.x), ptx::split_f16(o[u][1], hA.y, lA.y);
        ptx::split_f16(o[u][2], hB.x, lB.x), ptx::split_f16(o[u][3], hB.y, lB.y);
        if (okA) {
          *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(ctx_hi) + oA + 8 * n) = hA;
          *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(ctx_lo) + oA + 8 * n) = lA;
        }
        if (okB) {
          *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(ctx_hi) + oB + 8 * n) = hB;
          *reinterpret_cast<__half2*>(reinterpret_cast<__half*>(ctx_lo) + oB + 8 * n) = lB;
        }
        continue;
      }
      if (okA) {
        const float h0 = ptx::to_tf32(o[u][0]), h1 = ptx::to_tf32(o[u][1]);
        *reinterpret_cast<float2*>(ctx_hi + oA + 8 * n) = make_float2(h0, h1);
        *reinterpret_cast<float2*>(ctx_lo + oA + 8 * n) = make_float2(o[u][0] - h0, o[u][1] - h1);
      }
      if (okB) {
        const float h2 = ptx::to_tf32(o[u][2]), h3 = ptx::to_tf32(o[u][3]);
        *reinterpret_cast<float2*>(ctx_hi + oB + 8 * n) = make_float2(h2, h3);
        *reinterpret_cast<float2*>(ctx_lo + oB + 8 * n) = make_float2(o[u][2] - h2, o[u][3] - h3);
      }
    }
  }
}

// ---- tensor-core attention on fp16 hi/lo pairs (ROHM_PRECISION_F16X2) ------------------------------------------------
// Same decomposition (one CTA per (clip, head), warp w owns query rows [16w, 16w+16), logits / softmax / P in
// registers), but Q, K and V arrive already split into fp16 hi/lo halves by the QKV GEMM's epilogue, so the kernel does
// no operand conversion at all: K and V fragments come out of shared memory with ldmatrix (.trans for V), Q fragments
// straight from global/L2, and every product is an mma.sync m16n8k16 -- half the instruction count of the m16n8k8 TF32
// kernel for the same 3-product error compensation.  The S accumulator pair of two adjacent 8-key tiles is exactly the A
// fragment of one 16-key P V step (the usual register reuse), so P is split into hi/lo halves once, in registers.
__device__ __forceinline__ void mma_f16_16x8x16(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem_row) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(ptx::smem_u32(smem_row)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem_row) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(ptx::smem_u32(smem_row)));
}
using ptx::split_f16x2;

template <int DH>
__host__ __device__ constexpr int attn_f16_pitch() { return DH + 8; }  // halves; 16-byte row chunks land on distinct bank groups

// qkv_hi / qkv_lo: [B*S, 3*D] fp16 (Q | K | V, head h at columns h*DH); ctx_hi / ctx_lo: [B*S, D] fp16.
template <int DH, int NK>  // NK = number of 16-key tiles (keys padded to 16*NK); one warp per 16 query rows, <= NK warps
__global__ void __launch_bounds__(32 * NK, 1) attention_f16_kernel(const __half* __restrict__ qkv_hi,
                                                                   const __half* __restrict__ qkv_lo,
                                                                   __half* __restrict__ ctx_hi, __half* __restrict__ ctx_lo,
                                                                   int S, int D, int H, float scale) {
  static_assert(NK % 2 == 0, "key tiles are processed in groups of four 8-key tiles");
  constexpr int P = attn_f16_pitch<DH>();
  constexpr int NT = 2 * NK;  // 8-key tiles
  extern __shared__ __align__(16) unsigned char sm_raw[];
  __half* Kh = reinterpret_cast<__half*>(sm_raw);  // [16*NK][P]
  __half* Kl = Kh + 16 * NK * P;
  __half* Vh = Kl + 16 * NK * P;
  __half* Vl = Vh + 16 * NK * P;
  const int b = blockIdx.x / H, h = blockIdx.x % H;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int g = lane >> 2, t = lane & 3;
  const int64_t base = static_cast<int64_t>(b) * S;
  const int ld = 3 * D;

  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  // K and V of the head -> shared memory with 16-byte cp.async (all copies of a thread in flight at once; key rows past
  // the clip are zero-filled through the src-size operand)
  const int64_t lo_off = qkv_lo - qkv_hi;  // element distance between the hi and lo planes
  for (int i = threadIdx.x; i < 16 * NK * (DH / 8); i += blockDim.x) {
    const int s = i / (DH / 8), c = i % (DH / 8);
    const int sc = s < S ? s : S - 1;
    const uint32_t nbytes = s < S ? 16u : 0u;
    const __half* src = qkv_hi + (base + sc) * ld + h * DH + c * 8 + D;
    const uint32_t dst = ptx::smem_u32(Kh + s * P + c * 8);
    constexpr uint32_t plane = 16 * NK * P * 2;  // bytes between Kh, Kl, Vh, Vl
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(nbytes) : "memory");
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + plane), "l"(src + lo_off), "r"(nbytes) : "memory");
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + 2 * plane), "l"(src + D), "r"(nbytes) : "memory");
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst + 3 * plane), "l"(src + D + lo_off), "r"(nbytes)
                 : "memory");
  }
  asm volatile("cp.async.commit_group;" ::: "memory");

  const int r0 = warp * 16;
  const int rowA = min(r0 + g, S - 1), rowB = min(r0 + g + 8, S - 1);
  // Q fragments come straight from global/L2: one base pointer, the other three addresses are fixed element offsets
  const __half* qA = qkv_hi + (base + rowA) * ld + h * DH + 2 * t;
  const int dB = (rowB - rowA) * ld;
  auto ldq = [](const __half* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); };
  uint32_t qh[4] = {ldq(qA), ldq(qA + dB), ldq(qA + 8), ldq(qA + dB + 8)};
  uint32_t ql[4] = {ldq(qA + lo_off), ldq(qA + lo_off + dB), ldq(qA + lo_off + 8), ldq(qA + lo_off + dB + 8)};
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  __syncthreads();

  // ---- S = Q K^T ----
  float acc[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) acc[j][0] = acc[j][1] = acc[j][2] = acc[j][3] = 0.0f;
  // ldmatrix row address of this lane: matrices 0/1 = K_hi columns +0 / +8, matrices 2/3 = K_lo columns +0 / +8
  const int lm = lane >> 3, lr = lane & 7;
  const __half* kbase = (lm < 2 ? Kh : Kl) + lr * P + (lm & 1) * 8;
#pragma unroll 1
  for (int k = 0; k < DH / 16; ++k) {
    uint32_t ah[4], al[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) ah[i] = qh[i], al[i] = ql[i];
    if (k + 1 < DH / 16) {  // prefetch the next Q fragment (each value is used once, straight from L2)
      const __half* q = qA + 16 * (k + 1);
      qh[0] = ldq(q), qh[1] = ldq(q + dB), qh[2] = ldq(q + 8), qh[3] = ldq(q + dB + 8);
      q += lo_off;
      ql[0] = ldq(q), ql[1] = ldq(q + dB), ql[2] = ldq(q + 8), ql[3] = ldq(q + dB + 8);
    }
    const __half* kp = kbase + 16 * k;
    // groups of 4 key tiles, products issued pass-major so that consecutive MMAs hit different accumulators
#pragma unroll
    for (int j0 = 0; j0 < NT; j0 += 4) {
      uint32_t bf[4][4];  // {b0_hi, b1_hi, b0_lo, b1_lo}
#pragma unroll
      for (int u = 0; u < 4; ++u) ldmatrix_x4(bf[u], kp + (j0 + u) * 8 * P);
#pragma unroll
      for (int u = 0; u < 4; ++u) mma_f16_16x8x16(acc[j0 + u], al, bf[u][0], bf[u][1]);
#pragma unroll
      for (int u = 0; u < 4; ++u) mma_f16_16x8x16(acc[j0 + u], ah, bf[u][2], bf[u][3]);
#pragma unroll
      for (int u = 0; u < 4; ++u) mma_f16_16x8x16(acc[j0 + u], ah, bf[u][0], bf[u][1]);
    }
  }

  // ---- softmax over keys (rows rowA: elements [0],[1]; rowB: [2],[3]; columns 8j + 2t + {0,1}) ----
  float mxA = -INFINITY, mxB = -INFINITY;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool ok = (8 * j + 2 * t + e) < S;
      acc[j][e] = ok ? acc[j][e] * scale : -INFINITY;
      acc[j][2 + e] = ok ? acc[j][2 + e] * scale : -INFINITY;
      mxA = fmaxf(mxA, acc[j][e]);
      mxB = fmaxf(mxB, acc[j][2 + e]);
    }
  }
  mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 1));
  mxA = fmaxf(mxA, __shfl_xor_sync(0xffffffffu, mxA, 2));
  mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 1));
  mxB = fmaxf(mxB, __shfl_xor_sync(0xffffffffu, mxB, 2));
  float sumA = 0.0f, sumB = 0.0f;
#pragma unroll
  for (int j = 0; j < NT; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      acc[j][e] = expf(acc[j][e] - mxA);  // exp(-inf) = 0 for padded keys
      acc[j][2 + e] = expf(acc[j][2 + e] - mxB);
      sumA += acc[j][e];
      sumB += acc[j][2 + e];
    }
  }
  sumA += __shfl_xor_sync(0xffffffffu, sumA, 1);
  sumA += __shfl_xor_sync(0xffffffffu, sumA, 2);
  sumB += __shfl_xor_sync(0xffffffffu, sumB, 1);
  sumB += __shfl_xor_sync(0xffffffffu, sumB, 2);
  const float invA = 1.0f / sumA, invB = 1.0f / sumB;

  // ---- P as A fragments of the 16-key steps: {rowA keys 2t..+1, rowB keys 2t..+1, rowA keys 8+2t.., rowB keys 8+2t..} ----
  uint32_t ph[NK][4], pl[NK][4];
#pragma unroll
  for (int jj = 0; jj < NK; ++jj) {
    split_f16x2(acc[2 * jj][0] * invA, acc[2 * jj][1] * invA, ph[jj][0], pl[jj][0]);
    split_f16x2(acc[2 * jj][2] * invB, acc[2 * jj][3] * invB, ph[jj][1], pl[jj][1]);
    split_f16x2(acc[2 * jj + 1][0] * invA, acc[2 * jj + 1][1] * invA, ph[jj][2], pl[jj][2]);
    split_f16x2(acc[2 * jj + 1][2] * invB, acc[2 * jj + 1][3] * invB, ph[jj][3], pl[jj][3]);
  }

  // ---- O = P V ----  four 8-wide output tiles per (rolled) iteration
  const bool okA = (r0 + g) < S, okB = (r0 + g + 8) < S;
  const int64_t oA = (base + r0 + g) * D + h * DH + 2 * t;
  const int64_t oB = oA + static_cast<int64_t>(8) * D;
  // ldmatrix.trans row address: matrices 0/1 = V_hi keys +0 / +8, matrices 2/3 = V_lo keys +0 / +8
  const __half* vbase = (lm < 2 ? Vh : Vl) + ((lm & 1) * 8 + lr) * P;
  constexpr int NU = 4;
#pragma unroll 1
  for (int n0 = 0; n0 < DH / 8; n0 += NU) {
    float o[NU][4];
#pragma unroll
    for (int u = 0; u < NU; ++u) o[u][0] = o[u][1] = o[u][2] = o[u][3] = 0.0f;
    const __half* vp = vbase + 8 * n0;
#pragma unroll
    for (int jj = 0; jj < NK; ++jj) {
      uint32_t bf[NU][4];  // {b0_hi, b1_hi, b0_lo, b1_lo}
#pragma unroll
      for (int u = 0; u < NU; ++u) ldmatrix_x4_trans(bf[u], vp + 16 * jj * P + 8 * u);
#pragma unroll
      for (int u = 0; u < NU; ++u) mma_f16_16x8x16(o[u], pl[jj], bf[u][0], bf[u][1]);
#pragma unroll
      for (int u = 0; u < NU; ++u) mma_f16_16x8x16(o[u], ph[jj], bf[u][2], bf[u][3]);
#pragma unroll
      for (int u = 0; u < NU; ++u) mma_f16_16x8x16(o[u], ph[jj], bf[u][0], bf[u][1]);
    }
#pragma unroll
    for (int u = 0; u < NU; ++u) {
      const int n = n0 + u;
      uint32_t hA, lA, hB, lB;
      split_f16x2(o[u][0], o[u][1], hA, lA);
      split_f16x2(o[u][2], o[u][3], hB, lB);
      if (okA) {
        *reinterpret_cast<uint32_t*>(ctx_hi + oA + 8 * n) = hA;
        *reinterpret_cast<uint32_t*>(ctx_lo + oA + 8 * n) = lA;
      }
      if (okB) {
        *reinterpret_cast<uint32_t*>(ctx_hi + oB + 8 * n) = hB;
        *reinterpret_cast<uint32_t*>(ctx_lo + oB + 8 * n) = lB;
      }
    }
  }
}

template <int DH>
size_t attention_f16_smem_bytes(int NK) { return sizeof(__half) * 4 * 16 * NK * attn_f16_pitch<DH>(); }

// ---- wgmma attention (ROHM_PRECISION_F16X2, head dim 128, clips of at most 160 tokens) ----------------------------
// One warpgroup per (clip, head, 64 queries).  Q (64 rows) and K / V (160 rows from the clip's first token) arrive by TMA
// as 128B-swizzled hi/lo tiles (V on its own mbarrier).  S = Q K^T (wgmma m64n160k16) stays in registers, the softmax runs
// on the fragments, and the fp16 hi/lo split of P is already the A operand of O = P V (wgmma m64n128k16, V read in place as
// an MN-major B).  Three products each.  Keys past the clip get -inf logits and zeroed V rows.
struct AttnWgParams {
  CUtensorMap q_hi, q_lo;    // Q|K|V planes [rows, 3D] fp16, boxes of 64 columns x 64 rows
  CUtensorMap kv_hi, kv_lo;  // the same planes, boxes of 64 columns x 160 rows
  __half* ctx_hi;
  __half* ctx_lo;
  int S, D, H;
  float scale;
  const int* clip_off;  // packed clips (AttnArgs::clip_off / clip_ids), or null
  const int* clip_ids;
};
constexpr int kAwKeys = 160;                 // padded key count = N of the S product
constexpr int kAwQRows = 64;                 // queries per CTA = M of one wgmma
constexpr int kAwQBuf = kAwQRows * 128;      // bytes of one {plane, 64-wide head-dim chunk} buffer of Q
constexpr int kAwKBuf = kAwKeys * 128;       // the same for K or V
constexpr int kAwSmemBytes = 4 * kAwQBuf + 8 * kAwKBuf + 1024;

__global__ void __launch_bounds__(128, 1) attention_wgmma_kernel(const __grid_constant__ AttnWgParams p) {
  extern __shared__ uint8_t aw_smem_raw[];
  __shared__ uint64_t bar_qk, bar_v;
  const uint32_t raw = ptx::smem_u32(aw_smem_raw);
  uint8_t* const sm = aw_smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint8_t* const Qb = sm;                   // [plane][chunk]
  uint8_t* const Kb = sm + 4 * kAwQBuf;     // [plane][chunk]
  uint8_t* const Vb = Kb + 4 * kAwKBuf;     // [plane][chunk]
  const int qtiles = (p.S + kAwQRows - 1) / kAwQRows;
  const int qt = static_cast<int>(blockIdx.x) % qtiles;
  const int bh = static_cast<int>(blockIdx.x) / qtiles;
  const int h = bh % p.H, b = bh / p.H;
  const int q0 = qt * kAwQRows;
  int S = p.S, row0 = b * p.S;
  if (p.clip_off != nullptr) {  // packed clips: the grid's clip b is clip_ids[b]; tiles past a shorter clip have no work
    const int c = p.clip_ids[b];
    row0 = p.clip_off[c];
    S = p.clip_off[c + 1] - row0;
    if (q0 >= S) return;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&p.q_hi);
    ptx::prefetch_tmap(&p.q_lo);
    ptx::prefetch_tmap(&p.kv_hi);
    ptx::prefetch_tmap(&p.kv_lo);
    ptx::mbar_init(&bar_qk, 1);
    ptx::mbar_init(&bar_v, 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  if (threadIdx.x == 0) {
    ptx::mbar_expect_tx(&bar_qk, 4 * kAwQBuf + 4 * kAwKBuf);
    for (int pl = 0; pl < 2; ++pl)
      for (int c = 0; c < 2; ++c) {
        ptx::tma_load_2d(Qb + (pl * 2 + c) * kAwQBuf, pl ? &p.q_lo : &p.q_hi, &bar_qk, h * 128 + 64 * c, row0 + q0);
        ptx::tma_load_2d(Kb + (pl * 2 + c) * kAwKBuf, pl ? &p.kv_lo : &p.kv_hi, &bar_qk, p.D + h * 128 + 64 * c, row0);
      }
    ptx::mbar_expect_tx(&bar_v, 4 * kAwKBuf);
    for (int pl = 0; pl < 2; ++pl)
      for (int c = 0; c < 2; ++c)
        ptx::tma_load_2d(Vb + (pl * 2 + c) * kAwKBuf, pl ? &p.kv_lo : &p.kv_hi, &bar_v, 2 * p.D + h * 128 + 64 * c, row0);
  }

  // ---- S = Q K^T (64 x 160), three products per k-step ----
  float s[80];
#pragma unroll
  for (int i = 0; i < 80; ++i) s[i] = 0.0f;
  ptx::mbar_wait(&bar_qk, 0);
  ptx::wgmma_fence_regs(s);
  ptx::wgmma_fence();
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int c = k >> 2;
    const uint64_t ko = static_cast<uint64_t>((k & 3) * 2);  // 16 fp16 = 32 bytes inside the 128-byte swizzle span
    const uint64_t qh = ptx::make_desc_kmajor<128>(ptx::smem_u32(Qb + c * kAwQBuf)) + ko;
    const uint64_t ql = ptx::make_desc_kmajor<128>(ptx::smem_u32(Qb + (2 + c) * kAwQBuf)) + ko;
    const uint64_t kh = ptx::make_desc_kmajor<128>(ptx::smem_u32(Kb + c * kAwKBuf)) + ko;
    const uint64_t kl = ptx::make_desc_kmajor<128>(ptx::smem_u32(Kb + (2 + c) * kAwKBuf)) + ko;
    ptx::wgmma_f16(s, ql, kh);
    ptx::wgmma_f16(s, qh, kl);
    ptx::wgmma_f16(s, qh, kh);
  }
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
  ptx::wgmma_fence_regs(s);

  // ---- softmax on the fragments: this thread holds rows r and r + 8 (elements 4j, 4j+1 and 4j+2, 4j+3), keys 8j + c2 + {0,1}
  const int c2 = 2 * (lane & 3);
  float m0 = -INFINITY, m1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < 20; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool valid = 8 * j + c2 + e < S;
      s[4 * j + e] = valid ? s[4 * j + e] : -INFINITY;
      s[4 * j + 2 + e] = valid ? s[4 * j + 2 + e] : -INFINITY;
      m0 = fmaxf(m0, s[4 * j + e]);
      m1 = fmaxf(m1, s[4 * j + 2 + e]);
    }
  }
#pragma unroll
  for (int off = 1; off <= 2; off <<= 1) {
    m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, off));
    m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, off));
  }
  float l0 = 0.0f, l1 = 0.0f;
#pragma unroll
  for (int j = 0; j < 20; ++j) {
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const bool valid = 8 * j + c2 + e < S;
      const float p0 = valid ? expf((s[4 * j + e] - m0) * p.scale) : 0.0f;
      const float p1 = valid ? expf((s[4 * j + 2 + e] - m1) * p.scale) : 0.0f;
      s[4 * j + e] = p0, s[4 * j + 2 + e] = p1;
      l0 += p0, l1 += p1;
    }
  }
#pragma unroll
  for (int off = 1; off <= 2; off <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, off);
    l1 += __shfl_xor_sync(0xffffffffu, l1, off);
  }
  // P as fp16 hi/lo pairs in the A-fragment layout of k-step k (keys 16k..16k+15): {row r, keys 16k + c2}, {row r + 8,
  // same keys}, {row r, keys 16k + 8 + c2}, {row r + 8, same keys} = accumulator elements 8k .. 8k + 7 in order
  uint32_t ph[10][4], plo[10][4];
#pragma unroll
  for (int k = 0; k < 10; ++k)
#pragma unroll
    for (int i = 0; i < 4; ++i) ptx::split_f16x2(s[8 * k + 2 * i], s[8 * k + 2 * i + 1], ph[k][i], plo[k][i]);
#pragma unroll
  for (int k = 0; k < 10; ++k)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(ph[k][i]), "+r"(plo[k][i])::"memory");

  // ---- V: key rows past the clip are zeroed (0 x NaN of a neighbouring clip would otherwise leak into O) ----
  ptx::mbar_wait(&bar_v, 0);
  if (S < kAwKeys) {
    const int n = (kAwKeys - S) * 8;  // 16-byte chunks per buffer
    for (int i = threadIdx.x; i < 4 * n; i += 128) {
      const int buf = i / n, r = i - buf * n;
      *reinterpret_cast<uint4*>(Vb + buf * kAwKBuf + S * 128 + r * 16) = make_uint4(0u, 0u, 0u, 0u);
    }
    ptx::fence_proxy_async();
    __syncthreads();
  }

  // ---- O = P V (64 x 128) ----
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.0f;
  ptx::wgmma_fence_regs(o);
  ptx::wgmma_fence();
#pragma unroll
  for (int k = 0; k < 10; ++k) {
    // 16 keys = two 8-row atoms (SBO 1024 bytes); the two 64-wide head-dim chunks are one buffer apart (LBO)
    const uint64_t vh = ptx::make_desc_mnmajor_sw128(ptx::smem_u32(Vb + k * 2048), kAwKBuf, 1024);
    const uint64_t vl = ptx::make_desc_mnmajor_sw128(ptx::smem_u32(Vb + 2 * kAwKBuf + k * 2048), kAwKBuf, 1024);
    ptx::wgmma_f16_rs_tb(o, plo[k], vh);
    ptx::wgmma_f16_rs_tb(o, ph[k], vl);
    ptx::wgmma_f16_rs_tb(o, ph[k], vh);
  }
  ptx::wgmma_commit();
  ptx::wgmma_wait<0>();
  ptx::wgmma_fence_regs(o);
#pragma unroll
  for (int k = 0; k < 10; ++k)
#pragma unroll
    for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(ph[k][i]), "+r"(plo[k][i])::"memory");

  // ---- normalise, split, store the context rows of this tile ----
  const int ra = q0 + warp * 16 + (lane >> 2), rb = ra + 8;
  const float ia = 1.0f / l0, ib = 1.0f / l1;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = h * 128 + 8 * j + c2;
    uint32_t hi, lo;
    if (ra < S) {
      ptx::split_f16x2(o[4 * j] * ia, o[4 * j + 1] * ia, hi, lo);
      const int64_t off = static_cast<int64_t>(row0 + ra) * p.D + col;
      *reinterpret_cast<uint32_t*>(p.ctx_hi + off) = hi;
      *reinterpret_cast<uint32_t*>(p.ctx_lo + off) = lo;
    }
    if (rb < S) {
      ptx::split_f16x2(o[4 * j + 2] * ib, o[4 * j + 3] * ib, hi, lo);
      const int64_t off = static_cast<int64_t>(row0 + rb) * p.D + col;
      *reinterpret_cast<uint32_t*>(p.ctx_hi + off) = hi;
      *reinterpret_cast<uint32_t*>(p.ctx_lo + off) = lo;
    }
  }
}

// ---- streaming wgmma attention (ROHM_PRECISION_F16X2, head dim 128, any clip length) ---------------------------------
// One warpgroup per (clip, head, 64 queries), like attention_wgmma_kernel, but K and V stream through a two-stage TMA ring
// in blocks of 64 keys (the 64 x 64 boxes of the Q maps) and the softmax is online: per block S_blk = Q K_blk^T (wgmma
// m64n64k16, the same three products in the same order), an fp32 running max m and running sum l, O and l rescaled by
// exp((m_old - m_new) scale), and P split into fp16 hi/lo registers as the A operand of O += P V_blk (V MN-major in place,
// three products).  Shared memory does not grow with the clip.  Keys past the clip get -inf logits and their V rows are
// zeroed before the P V product of the last block.  A stage is refilled as soon as its last reader has finished: the K
// half after the S product, the V half after the P V product.
struct AttnStreamParams {
  CUtensorMap hi, lo;  // Q|K|V planes [rows, 3D] fp16, boxes of 64 columns x 64 rows (AttnWgmmaMaps::q_hi / q_lo)
  __half* ctx_hi;
  __half* ctx_lo;
  int S, D, H;
  float scale;
  const int* clip_off;  // packed clips (AttnArgs::clip_off / clip_ids), or null
  const int* clip_ids;
};
constexpr int kAsBlock = 64;                  // keys per block = queries per CTA
constexpr int kAsBuf = kAsBlock * 128;        // bytes of one {plane, 64-wide head-dim chunk} tile
constexpr int kAsTile = 4 * kAsBuf;           // Q, or one K or V block: two planes x two chunks
constexpr int kAsStages = 2;
constexpr int kAsSmemBytes = (1 + 2 * kAsStages) * kAsTile + 1024;

__global__ void __launch_bounds__(128, 1) attention_wgmma_stream_kernel(const __grid_constant__ AttnStreamParams p) {
  extern __shared__ uint8_t as_smem_raw[];
  __shared__ uint64_t bar_q, bar_k[kAsStages], bar_v[kAsStages];
  const uint32_t raw = ptx::smem_u32(as_smem_raw);
  uint8_t* const sm = as_smem_raw + ((1024u - (raw & 1023u)) & 1023u);
  uint8_t* const Qb = sm;                             // [plane][chunk]
  uint8_t* const Kb = sm + kAsTile;                   // [stage][plane][chunk]
  uint8_t* const Vb = Kb + kAsStages * kAsTile;       // [stage][plane][chunk]
  const int qtiles = (p.S + kAsBlock - 1) / kAsBlock;
  const int qt = static_cast<int>(blockIdx.x) % qtiles;
  const int bh = static_cast<int>(blockIdx.x) / qtiles;
  const int h = bh % p.H, b = bh / p.H;
  const int q0 = qt * kAsBlock;
  int S = p.S, row0 = b * p.S;
  if (p.clip_off != nullptr) {  // packed clips: the grid's clip b is clip_ids[b]; tiles past a shorter clip have no work
    const int c = p.clip_ids[b];
    row0 = p.clip_off[c];
    S = p.clip_off[c + 1] - row0;
    if (q0 >= S) return;
  }
  const int nblk = (S + kAsBlock - 1) / kAsBlock;     // key blocks of the clip, counted from its first token
  const int kcol = p.D + h * 128, vcol = 2 * p.D + h * 128;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&p.hi);
    ptx::prefetch_tmap(&p.lo);
    ptx::mbar_init(&bar_q, 1);
    for (int s = 0; s < kAsStages; ++s) ptx::mbar_init(&bar_k[s], 1), ptx::mbar_init(&bar_v[s], 1);
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  // one 64-row tile of a column range: hi and lo plane, two 64-wide chunks each
  auto load_tile = [&](uint8_t* dst, uint64_t* bar, int col, int row) {
    ptx::mbar_expect_tx(bar, kAsTile);
    for (int pl = 0; pl < 2; ++pl)
      for (int c = 0; c < 2; ++c) ptx::tma_load_2d(dst + (pl * 2 + c) * kAsBuf, pl ? &p.lo : &p.hi, bar, col + 64 * c, row);
  };
  if (threadIdx.x == 0) {
    load_tile(Qb, &bar_q, h * 128, row0 + q0);
    for (int j = 0; j < kAsStages && j < nblk; ++j) {
      load_tile(Kb + j * kAsTile, &bar_k[j], kcol, row0 + j * kAsBlock);
      load_tile(Vb + j * kAsTile, &bar_v[j], vcol, row0 + j * kAsBlock);
    }
  }

  // this thread holds rows r and r + 8 of the tile: accumulator elements 4j, 4j+1 (row r) and 4j+2, 4j+3 (row r + 8),
  // columns 8j + c2 + {0,1}
  const int c2 = 2 * (lane & 3);
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.0f;
  float m0 = -INFINITY, m1 = -INFINITY;  // running max of the raw logits (rows r, r + 8), equal across the quad
  float l0 = 0.0f, l1 = 0.0f;            // running sum of this thread's columns, reduced over the quad at the end
  ptx::mbar_wait(&bar_q, 0);
#pragma unroll 1
  for (int j = 0; j < nblk; ++j) {
    const int st = j % kAsStages;
    const uint32_t phase = (j / kAsStages) & 1;
    uint8_t* const Ks = Kb + st * kAsTile;
    uint8_t* const Vs = Vb + st * kAsTile;
    const int kb = j * kAsBlock;

    // ---- S_blk = Q K_blk^T (64 x 64), three products per k-step ----
    float s[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) s[i] = 0.0f;
    ptx::mbar_wait(&bar_k[st], phase);
    ptx::wgmma_fence_regs(s);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const int c = k >> 2;
      const uint64_t ko = static_cast<uint64_t>((k & 3) * 2);  // 16 fp16 = 32 bytes inside the 128-byte swizzle span
      const uint64_t qh = ptx::make_desc_kmajor<128>(ptx::smem_u32(Qb + c * kAsBuf)) + ko;
      const uint64_t ql = ptx::make_desc_kmajor<128>(ptx::smem_u32(Qb + (2 + c) * kAsBuf)) + ko;
      const uint64_t kh = ptx::make_desc_kmajor<128>(ptx::smem_u32(Ks + c * kAsBuf)) + ko;
      const uint64_t kl = ptx::make_desc_kmajor<128>(ptx::smem_u32(Ks + (2 + c) * kAsBuf)) + ko;
      ptx::wgmma_f16(s, ql, kh);
      ptx::wgmma_f16(s, qh, kl);
      ptx::wgmma_f16(s, qh, kh);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::wgmma_fence_regs(s);
    __syncthreads();  // every warp's share of the S product has read the K stage
    if (threadIdx.x == 0 && j + kAsStages < nblk) load_tile(Ks, &bar_k[st], kcol, row0 + kb + kAsStages * kAsBlock);

    // ---- online softmax: new running max, rescale factor of the old O and l, P of the block ----
    float n0 = m0, n1 = m1;
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool valid = kb + 8 * jj + c2 + e < S;
        s[4 * jj + e] = valid ? s[4 * jj + e] : -INFINITY;
        s[4 * jj + 2 + e] = valid ? s[4 * jj + 2 + e] : -INFINITY;
        n0 = fmaxf(n0, s[4 * jj + e]);
        n1 = fmaxf(n1, s[4 * jj + 2 + e]);
      }
    }
#pragma unroll
    for (int off = 1; off <= 2; off <<= 1) {
      n0 = fmaxf(n0, __shfl_xor_sync(0xffffffffu, n0, off));
      n1 = fmaxf(n1, __shfl_xor_sync(0xffffffffu, n1, off));
    }
    const float a0 = expf((m0 - n0) * p.scale), a1 = expf((m1 - n1) * p.scale);  // 0 on the first block (m = -inf)
    m0 = n0, m1 = n1;
    float b0 = 0.0f, b1 = 0.0f;  // the block's sum first: two roundings of the running sum per block, not sixteen
#pragma unroll
    for (int jj = 0; jj < 8; ++jj) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const bool valid = kb + 8 * jj + c2 + e < S;
        const float p0 = valid ? expf((s[4 * jj + e] - m0) * p.scale) : 0.0f;
        const float p1 = valid ? expf((s[4 * jj + 2 + e] - m1) * p.scale) : 0.0f;
        s[4 * jj + e] = p0, s[4 * jj + 2 + e] = p1;
        b0 += p0, b1 += p1;
      }
    }
    l0 = l0 * a0 + b0, l1 = l1 * a1 + b1;
    // P as fp16 hi/lo pairs in the A-fragment layout of k-step k (keys 16k..16k+15) = accumulator elements 8k..8k+7
    uint32_t ph[4][4], plo[4][4];
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < 4; ++i) ptx::split_f16x2(s[8 * k + 2 * i], s[8 * k + 2 * i + 1], ph[k][i], plo[k][i]);

    // ---- V: key rows past the clip are zeroed (0 x NaN of a neighbouring clip would otherwise leak into O) ----
    ptx::mbar_wait(&bar_v[st], phase);
    if (kb + kAsBlock > S) {
      const int n = (kb + kAsBlock - S) * 8;  // 16-byte chunks per buffer
      for (int i = threadIdx.x; i < 4 * n; i += 128) {
        const int buf = i / n, r = i - buf * n;
        *reinterpret_cast<uint4*>(Vs + buf * kAsBuf + (S - kb) * 128 + r * 16) = make_uint4(0u, 0u, 0u, 0u);
      }
      ptx::fence_proxy_async();
      __syncthreads();
    }

    // ---- O = O exp((m_old - m_new) scale) + P V_blk (64 x 128) ----
    // The block's product gets an accumulator of its own and is folded into O with one rounded fma: accumulating all
    // blocks in the wgmma accumulator would put 12 tensor-core additions per block on the running O (thousands over a
    // long clip), where the fold puts one.
    float ob[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) ob[i] = 0.0f;
    ptx::wgmma_fence_regs(ob);
    ptx::wgmma_fence();
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      // 16 keys = two 8-row atoms (SBO 1024 bytes); the two 64-wide head-dim chunks are one buffer apart (LBO)
      const uint64_t vh = ptx::make_desc_mnmajor_sw128(ptx::smem_u32(Vs + k * 2048), kAsBuf, 1024);
      const uint64_t vl = ptx::make_desc_mnmajor_sw128(ptx::smem_u32(Vs + 2 * kAsBuf + k * 2048), kAsBuf, 1024);
      ptx::wgmma_f16_rs_tb(ob, plo[k], vh);
      ptx::wgmma_f16_rs_tb(ob, ph[k], vl);
      ptx::wgmma_f16_rs_tb(ob, ph[k], vh);
    }
    ptx::wgmma_commit();
    ptx::wgmma_wait<0>();
    ptx::wgmma_fence_regs(ob);
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = fmaf(o[i], (i & 2) ? a1 : a0, ob[i]);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(ph[k][i]), "+r"(plo[k][i])::"memory");
    __syncthreads();  // every warp's share of the P V product has read the V stage
    if (threadIdx.x == 0 && j + kAsStages < nblk) load_tile(Vs, &bar_v[st], vcol, row0 + kb + kAsStages * kAsBlock);
  }

  // ---- normalise, split, store the context rows of this tile ----
#pragma unroll
  for (int off = 1; off <= 2; off <<= 1) {
    l0 += __shfl_xor_sync(0xffffffffu, l0, off);
    l1 += __shfl_xor_sync(0xffffffffu, l1, off);
  }
  const int ra = q0 + warp * 16 + (lane >> 2), rb = ra + 8;
  const float ia = 1.0f / l0, ib = 1.0f / l1;
#pragma unroll
  for (int j = 0; j < 16; ++j) {
    const int col = h * 128 + 8 * j + c2;
    uint32_t hi, lo;
    if (ra < S) {
      ptx::split_f16x2(o[4 * j] * ia, o[4 * j + 1] * ia, hi, lo);
      const int64_t off = static_cast<int64_t>(row0 + ra) * p.D + col;
      *reinterpret_cast<uint32_t*>(p.ctx_hi + off) = hi;
      *reinterpret_cast<uint32_t*>(p.ctx_lo + off) = lo;
    }
    if (rb < S) {
      ptx::split_f16x2(o[4 * j + 2] * ib, o[4 * j + 3] * ib, hi, lo);
      const int64_t off = static_cast<int64_t>(row0 + rb) * p.D + col;
      *reinterpret_cast<uint32_t*>(p.ctx_hi + off) = hi;
      *reinterpret_cast<uint32_t*>(p.ctx_lo + off) = lo;
    }
  }
}

size_t attention_mma_smem_bytes(int NT) { return sizeof(float) * 2 * 8 * NT * kAttnPitch; }

template <int DH, int NT>
cudaError_t launch_attention_mma(const AttnArgs& a, cudaStream_t st, bool pdl) {
  auto kern = attention_mma_kernel<DH, NT>;
  static bool attr_set = false;
  const size_t smem = attention_mma_smem_bytes(NT);
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int warps = (a.S + 15) / 16;
  return launch_chain(kern, dim3(a.B * a.H), dim3(32 * warps), smem, st, pdl, static_cast<const float*>(a.qkv_hi),
                      static_cast<float*>(a.ctx_hi), static_cast<float*>(a.ctx_lo), a.S, a.D, a.H, a.scale,
                      a.kind == kKindF16 ? 1 : 0);
}

template <int DH, int NK>
cudaError_t launch_attention_f16(const AttnArgs& a, cudaStream_t st, bool pdl) {
  const int warps = (a.S + 15) / 16;
  return launch_chain(attention_f16_kernel<DH, NK>, dim3(a.B * a.H), dim3(32 * warps), attention_f16_smem_bytes<DH>(NK), st,
                      pdl, static_cast<const __half*>(a.qkv_hi), static_cast<const __half*>(a.qkv_lo),
                      static_cast<__half*>(a.ctx_hi), static_cast<__half*>(a.ctx_lo), a.S, a.D, a.H, a.scale);
}

}  // namespace

size_t attention_smem_bytes(int S, int DH) {
  const int Sp = (S + 31) & ~31;
  return sizeof(float) * (static_cast<size_t>(S) * (DH + 4) + static_cast<size_t>(S) * DH + 8 * DH + 8 * Sp);
}

int attention_wgmma_maps(AttnWgmmaMaps* maps, const AttnArgs& a) {
  const int D = a.D;
  int rc = make_tile_tmap_f16_sw128(&maps->q_hi, a.qkv_hi, a.rows, 3 * D, 3 * D, kAwQRows);
  if (rc == 0) rc = make_tile_tmap_f16_sw128(&maps->q_lo, a.qkv_lo, a.rows, 3 * D, 3 * D, kAwQRows);
  if (rc == 0) rc = make_tile_tmap_f16_sw128(&maps->kv_hi, a.qkv_hi, a.rows, 3 * D, 3 * D, kAwKeys);
  if (rc == 0) rc = make_tile_tmap_f16_sw128(&maps->kv_lo, a.qkv_lo, a.rows, 3 * D, 3 * D, kAwKeys);
  return rc;
}

cudaError_t attention_init_attributes(int max_tokens, int dh) {
  cudaError_t ea = cudaSuccess;
  auto set = [&](auto kern, size_t bytes) {
    if (ea == cudaSuccess) ea = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
  };
  set(attention_mma_kernel<128, 4>, attention_mma_smem_bytes(4));
  set(attention_mma_kernel<128, 8>, attention_mma_smem_bytes(8));
  set(attention_mma_kernel<128, 12>, attention_mma_smem_bytes(12));
  set(attention_mma_kernel<128, 16>, attention_mma_smem_bytes(16));
  set(attention_mma_kernel<128, 20>, attention_mma_smem_bytes(20));
  set(attention_mma_kernel<64, 8>, attention_mma_smem_bytes(8));
  set(attention_mma_kernel<64, 20>, attention_mma_smem_bytes(20));
  set(attention_f16_kernel<128, 2>, attention_f16_smem_bytes<128>(2));
  set(attention_f16_kernel<128, 4>, attention_f16_smem_bytes<128>(4));
  set(attention_f16_kernel<128, 6>, attention_f16_smem_bytes<128>(6));
  set(attention_f16_kernel<128, 8>, attention_f16_smem_bytes<128>(8));
  set(attention_f16_kernel<128, 10>, attention_f16_smem_bytes<128>(10));
  set(attention_f16_kernel<64, 4>, attention_f16_smem_bytes<64>(4));
  set(attention_f16_kernel<64, 10>, attention_f16_smem_bytes<64>(10));
  set(attention_wgmma_kernel, kAwSmemBytes);
  set(attention_wgmma_stream_kernel, kAsSmemBytes);
  if (dh != 64 && dh != 128) return ea == cudaSuccess ? cudaErrorInvalidValue : ea;
  // the SIMT kernel serves at most 256 tokens whose K and V fit in shared memory; longer clips never reach it
  int simt_tokens = max_tokens < kAttnSimtMaxTokens ? max_tokens : kAttnSimtMaxTokens;
  while (simt_tokens > 1 && attention_smem_bytes(simt_tokens, dh) > kAttnSmemLimit) --simt_tokens;
  if (dh == 128) set(attention_kernel<128>, attention_smem_bytes(simt_tokens, 128));
  else set(attention_kernel<64>, attention_smem_bytes(simt_tokens, 64));
  return ea;
}

cudaError_t launch_attention(const AttnArgs& a, int which, const AttnWgmmaMaps* wg, cudaStream_t st, bool pdl) {
  const bool packed = a.clip_off != nullptr;
  if (a.B <= 0 || a.S <= 0 || a.H <= 0 || a.D % a.H != 0 || (packed ? a.S > a.rows : static_cast<int64_t>(a.B) * a.S > a.rows))
    return cudaErrorInvalidValue;
  if (packed && (a.clip_ids == nullptr || which == kAttnAuto)) return cudaErrorInvalidValue;
  const int dh = a.D / a.H;
  if (dh != 64 && dh != 128) return cudaErrorInvalidValue;
  const bool f16 = a.kind == kKindF16;
  const bool wg_ok = f16 && dh == 128 && a.S <= kAwKeys && wg != nullptr;
  const bool stream_ok = f16 && dh == 128 && wg != nullptr;
  const bool mma_ok = a.S <= kAttnWgmmaMaxTokens;  // register budget of the S / P fragments
  if (which == kAttnAuto)
    which = wg_ok ? kAttnWgmma : (stream_ok && !mma_ok) ? kAttnWgmmaStream : !mma_ok ? kAttnSimt : f16 ? kAttnMmaF16 : kAttnMmaTf32;
  const int S = a.S;
  if (which == kAttnWgmmaStream) {
    if (!stream_ok) return cudaErrorInvalidValue;
    AttnStreamParams prm;
    prm.hi = wg->q_hi, prm.lo = wg->q_lo;
    prm.ctx_hi = static_cast<__half*>(a.ctx_hi), prm.ctx_lo = static_cast<__half*>(a.ctx_lo);
    prm.S = S, prm.D = a.D, prm.H = a.H, prm.scale = a.scale;
    prm.clip_off = a.clip_off, prm.clip_ids = a.clip_ids;
    const int qtiles = (S + kAsBlock - 1) / kAsBlock;
    return launch_chain(attention_wgmma_stream_kernel, dim3(a.B * a.H * qtiles), dim3(128), kAsSmemBytes, st, pdl, prm);
  }
  if (which == kAttnWgmma) {
    if (!wg_ok) return cudaErrorInvalidValue;
    AttnWgParams prm;
    prm.q_hi = wg->q_hi, prm.q_lo = wg->q_lo, prm.kv_hi = wg->kv_hi, prm.kv_lo = wg->kv_lo;
    prm.ctx_hi = static_cast<__half*>(a.ctx_hi), prm.ctx_lo = static_cast<__half*>(a.ctx_lo);
    prm.S = S, prm.D = a.D, prm.H = a.H, prm.scale = a.scale;
    prm.clip_off = a.clip_off, prm.clip_ids = a.clip_ids;
    const int qtiles = (S + kAwQRows - 1) / kAwQRows;
    return launch_chain(attention_wgmma_kernel, dim3(a.B * a.H * qtiles), dim3(128), kAwSmemBytes, st, pdl, prm);
  }
  if (packed) return cudaErrorInvalidValue;  // packed clips run on the wgmma kernels only
  if (which == kAttnMmaF16) {
    if (!f16 || !mma_ok) return cudaErrorInvalidValue;
    const int nk = (S + 15) / 16;
    if (dh == 128 && nk <= 2) return launch_attention_f16<128, 2>(a, st, pdl);
    if (dh == 128 && nk <= 4) return launch_attention_f16<128, 4>(a, st, pdl);
    if (dh == 128 && nk <= 6) return launch_attention_f16<128, 6>(a, st, pdl);
    if (dh == 128 && nk <= 8) return launch_attention_f16<128, 8>(a, st, pdl);
    if (dh == 128) return launch_attention_f16<128, 10>(a, st, pdl);
    if (nk <= 4) return launch_attention_f16<64, 4>(a, st, pdl);
    return launch_attention_f16<64, 10>(a, st, pdl);
  }
  if (which == kAttnMmaTf32) {
    if (f16 || !mma_ok) return cudaErrorInvalidValue;
    const int nt = (S + 7) / 8;
    if (dh == 128 && nt <= 4) return launch_attention_mma<128, 4>(a, st, pdl);
    if (dh == 128 && nt <= 8) return launch_attention_mma<128, 8>(a, st, pdl);
    if (dh == 128 && nt <= 12) return launch_attention_mma<128, 12>(a, st, pdl);
    if (dh == 128 && nt <= 16) return launch_attention_mma<128, 16>(a, st, pdl);
    if (dh == 128) return launch_attention_mma<128, 20>(a, st, pdl);
    if (nt <= 8) return launch_attention_mma<64, 8>(a, st, pdl);
    return launch_attention_mma<64, 20>(a, st, pdl);
  }
  if (which == kAttnSimt) {
    const size_t smem = attention_smem_bytes(S, dh);
    if (S > kAttnSimtMaxTokens || smem > kAttnSmemLimit) return cudaErrorInvalidValue;
    auto kern = dh == 128 ? attention_kernel<128> : attention_kernel<64>;
    return launch_chain(kern, dim3(a.B * a.H), dim3(256), smem, st, pdl, static_cast<const float*>(a.qkv_hi),
                        static_cast<const float*>(a.qkv_lo), static_cast<float*>(a.ctx_hi), static_cast<float*>(a.ctx_lo), S,
                        a.D, a.H, a.scale, f16 ? 1 : 0);
  }
  return cudaErrorInvalidValue;
}

}  // namespace rohm
