// PoseNet denoiser engine: the per-step transformer-encoder forward of RoHM's PoseNet
// (reference model/posenet.py:75-96, model/heads.py:112-176; torch nn.TransformerEncoderLayer post-norm, exact GELU).
//
// Token-major layout: every activation is a row-major [B*S, width] matrix, S = T + 1 tokens per clip (token 0 is the
// timestep embedding), clips contiguous.  All linear layers run on the wgmma GEMM (gemm.cu); operands that feed a
// tensor-core product are kept as hi/lo pairs (fp16 halves by default, TF32 in the tf32 modes) written by the
// producing kernel's epilogue, so no separate conversion pass exists.
//
//   x_t [B,C,1,T] --pack--> A_in --GEMM(+bias+cond_embed+pe)--> X  (token 0 <- time-embedding table gather)
//   8 x { X --GEMM--> Q|K|V --attention (wgmma: S = QK^T, softmax on the fragments, O = PV)--> CTX --GEMM(+bias)--> Y
//         --LN(Y + X)--> X --GEMM(+bias,GELU)--> H --GEMM(+bias)--> Y --LN(Y + X)--> X }
//   X --GEMM--> OUT_tok --unpack(+copy cond[:, :traj])--> out [B,C,1,T]
// One forward = 61 launches, replayed as one CUDA graph with programmatic dependent launch along the chain.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <new>

#include "common.h"
#include "gemm.cuh"
#include "ptx.cuh"

namespace rohm {
namespace {

// ------------------------------------------------------------------------------------------------------------
// small kernels
// ------------------------------------------------------------------------------------------------------------

// [B, C, T] (frames contiguous) -> token rows (b*S + 1 + t) of a [B*S, ld] hi/lo pair.  32x32 smem transpose.
__global__ void pack_tokens_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, int C,
                                   int T, int S, int ld, int f16) {
  __shared__ float tile[32][33];
  // programmatic dependent launch: the embedding GEMM behind this kernel may set itself up (barriers, weight tiles)
  // while it runs; as a dependent (a no-op for a plain launch) nothing is read before the previous kernel has completed
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, t = t0 + tx;
    tile[j][tx] = (c < C && t < T) ? x[(static_cast<int64_t>(b) * C + c) * T + t] : 0.0f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int t = t0 + j, c = c0 + tx;
    if (t < T && c < C) {
      const float v = tile[tx][j];
      const int64_t o = (static_cast<int64_t>(b) * S + 1 + t) * ld + c;
      if (f16) {
        ptx::split_f16(v, reinterpret_cast<__half*>(hi)[o], reinterpret_cast<__half*>(lo)[o]);
      } else {
        const float h = ptx::to_tf32(v);
        hi[o] = h;
        lo[o] = v - h;
      }
    }
  }
}

// Token rows -> [B, C, T]: channels [traj, traj+Cout) from tok[b*S+1+t][c - traj], channels [0, traj) from cond.
__global__ void unpack_tokens_kernel(const float* __restrict__ tok, const float* __restrict__ cond_traj,
                                     float* __restrict__ out, int C, int Cout, int traj, int T, int S, int ldt) {
  __shared__ float tile[32][33];
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();  // the output-head GEMM has completed
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;  // c0 indexes the Cout predicted channels
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int j = ty; j < 32; j += 8) {
    const int t = t0 + j, c = c0 + tx;
    tile[j][tx] = (t < T && c < Cout) ? tok[(static_cast<int64_t>(b) * S + 1 + t) * ldt + c] : 0.0f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, t = t0 + tx;
    if (c < Cout && t < T) out[(static_cast<int64_t>(b) * C + traj + c) * T + t] = tile[tx][j];
  }
  if (blockIdx.y == 0) {  // given trajectory channels are a verbatim copy of the condition (posenet.py:94-95)
    for (int c = ty; c < traj; c += 8) {
      const int t = t0 + tx;
      if (t < T) out[(static_cast<int64_t>(b) * C + c) * T + t] = cond_traj[(static_cast<int64_t>(b) * traj + c) * T + t];
    }
  }
}

// rows[b*S + s][:] = pe[s][:]   (positional rows added to every token incl. the timestep token, posenet.py:90-91)
__global__ void pe_rows_kernel(const float* __restrict__ pe, float* __restrict__ rows, int S, int D, int64_t total4) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int d4 = D / 4;
  const int64_t row = i / d4;
  const int c = static_cast<int>(i - row * d4);
  const int s = static_cast<int>(row % S);
  reinterpret_cast<float4*>(rows)[i] = reinterpret_cast<const float4*>(pe)[static_cast<int64_t>(s) * d4 + c];
}

// TimestepEmbedder (heads.py:132-146): e(t) = W2 silu(W0 pe[t] + b0) + b2 depends on the timestep only, so the whole
// table TE[t] = e(t) + pe[0] (the positional row of token 0) is computed once per weight set at create time (two GEMMs
// over all pe_len timesteps); per step the token row (b, 0) is a gather.
__global__ void time_token_gather_kernel(const int64_t* __restrict__ timesteps, const float* __restrict__ table,
                                         int table_rows, float* __restrict__ X, float* __restrict__ Xh,
                                         float* __restrict__ Xl, int S, int D, int f16, unsigned int* __restrict__ zero_buf,
                                         int zero_n) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();  // the embedding GEMM (which also writes row (b, 0)) has completed
  const int b = blockIdx.x;
  // once per forward: clear the arrival counters of the fused LayerNorm epilogues (GemmParams::ln_count)
  if (b == 0)
    for (int i = threadIdx.x; i < zero_n; i += blockDim.x) zero_buf[i] = 0u;
  int64_t t = timesteps[b];
  // The reference indexes pe[timesteps] and raises on a bad index (heads.py:145).  A kernel cannot raise, so an
  // out-of-range timestep poisons the clip's timestep token with NaN (which attention spreads over the whole clip's
  // output) instead of being clamped to a plausible but wrong embedding.
  const bool bad = t < 0 || t >= table_rows;
  t = bad ? 0 : t;
  const float4* src = reinterpret_cast<const float4*>(table + t * D);
  const int64_t o = static_cast<int64_t>(b) * S * D;
  const float nan = __int_as_float(0x7fc00000);
  for (int i = threadIdx.x; i < D / 4; i += blockDim.x) {
    const float4 v = bad ? make_float4(nan, nan, nan, nan) : src[i];
    reinterpret_cast<float4*>(X + o)[i] = v;
    if (f16) {
      uint2 h, l;
      ptx::split_f16x4(v, h, l);
      reinterpret_cast<uint2*>(reinterpret_cast<__half*>(Xh) + o)[i] = h;
      reinterpret_cast<uint2*>(reinterpret_cast<__half*>(Xl) + o)[i] = l;
    } else {
      float4 h, l;
      h.x = ptx::to_tf32(v.x), h.y = ptx::to_tf32(v.y), h.z = ptx::to_tf32(v.z), h.w = ptx::to_tf32(v.w);
      l.x = v.x - h.x, l.y = v.y - h.y, l.z = v.z - h.z, l.w = v.w - h.w;
      reinterpret_cast<float4*>(Xh + o)[i] = h;
      reinterpret_cast<float4*>(Xl + o)[i] = l;
    }
  }
}

__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
}

// LayerNorm over the last dim (eps 1e-5) of in + res (res = the residual stream, may be null), one warp per row; writes
// fp32 and the hi/lo pair.  `out` may alias `res` (each row is read completely before it is written).
template <int D>
__global__ void __launch_bounds__(256) layernorm_kernel(const float* __restrict__ in, const float* res,
                                                        const float* __restrict__ gamma,
                                                        const float* __restrict__ beta, float* out,
                                                        float* __restrict__ out_hi, float* __restrict__ out_lo,
                                                        int rows, int f16) {
  static_assert(D % 128 == 0, "row must be a multiple of 32 lanes x float4");
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  constexpr int V = D / 128;
  const int row = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= rows) return;
  const float4* src = reinterpret_cast<const float4*>(in + static_cast<int64_t>(row) * D);
  float4 x[V];
#pragma unroll
  for (int i = 0; i < V; ++i) x[i] = src[lane + 32 * i];
  if (res != nullptr) {  // x = sublayer output + residual stream (torch: x + sa_block(x) / x + ff_block(x))
    const float4* rs = reinterpret_cast<const float4*>(res + static_cast<int64_t>(row) * D);
#pragma unroll
    for (int i = 0; i < V; ++i) {
      const float4 r = rs[lane + 32 * i];
      x[i].x += r.x, x[i].y += r.y, x[i].z += r.z, x[i].w += r.w;
    }
  }
  float sum = 0.0f;
#pragma unroll
  for (int i = 0; i < V; ++i) sum += (x[i].x + x[i].y) + (x[i].z + x[i].w);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  const float mean = sum * (1.0f / D);
  float sq = 0.0f;
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float a = x[i].x - mean, b = x[i].y - mean, c = x[i].z - mean, d = x[i].w - mean;
    sq += (a * a + b * b) + (c * c + d * d);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, off);
  const float rstd = rsqrtf(sq * (1.0f / D) + 1e-5f);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  float4* o = reinterpret_cast<float4*>(out + static_cast<int64_t>(row) * D);
  float4* oh = reinterpret_cast<float4*>(out_hi + static_cast<int64_t>(row) * D);
  float4* ol = reinterpret_cast<float4*>(out_lo + static_cast<int64_t>(row) * D);
  uint2* oh16 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out_hi) + static_cast<int64_t>(row) * D);
  uint2* ol16 = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(out_lo) + static_cast<int64_t>(row) * D);
#pragma unroll
  for (int i = 0; i < V; ++i) {
    const float4 g = g4[lane + 32 * i], bb = b4[lane + 32 * i];
    float4 y;
    y.x = (x[i].x - mean) * rstd * g.x + bb.x;
    y.y = (x[i].y - mean) * rstd * g.y + bb.y;
    y.z = (x[i].z - mean) * rstd * g.z + bb.z;
    y.w = (x[i].w - mean) * rstd * g.w + bb.w;
    o[lane + 32 * i] = y;
    if (f16) {
      uint2 h, l;
      ptx::split_f16x4(y, h, l);
      oh16[lane + 32 * i] = h;
      ol16[lane + 32 * i] = l;
    } else {
      float4 h, l;
      h.x = ptx::to_tf32(y.x), h.y = ptx::to_tf32(y.y), h.z = ptx::to_tf32(y.z), h.w = ptx::to_tf32(y.w);
      l.x = y.x - h.x, l.y = y.y - h.y, l.z = y.z - h.z, l.w = y.w - h.w;
      oh[lane + 32 * i] = h;
      ol[lane + 32 * i] = l;
    }
  }
}

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
  const int S = p.S;
  const int qtiles = (S + kAwQRows - 1) / kAwQRows;
  const int qt = static_cast<int>(blockIdx.x) % qtiles;
  const int bh = static_cast<int>(blockIdx.x) / qtiles;
  const int h = bh % p.H, b = bh / p.H;
  const int row0 = b * S, q0 = qt * kAwQRows;
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

size_t attention_mma_smem_bytes(int NT) { return sizeof(float) * 2 * 8 * NT * kAttnPitch; }

size_t attention_smem_bytes(int S, int DH) {
  const int Sp = (S + 31) & ~31;
  return sizeof(float) * (static_cast<size_t>(S) * (DH + 4) + static_cast<size_t>(S) * DH + 8 * DH + 8 * Sp);
}

}  // namespace

// ------------------------------------------------------------------------------------------------------------
// engine
// ------------------------------------------------------------------------------------------------------------
struct PoseNetLayerDev {
  PackedWeight qkv, proj, ff1, ff2;
  float *qkv_b, *proj_b, *ff1_b, *ff2_b, *n1_w, *n1_b, *n2_w, *n2_b;
  // LayerNorm folding: c_n = sum_k gamma_k W[n,k] and d_n = b_n + sum_k beta_k W[n,k] of the GEMMs that consume a
  // normalised input (QKV of layers >= 1: previous layer's norm2; FFN1: this layer's norm1)
  float *qkv_c = nullptr, *qkv_d = nullptr, *ff1_c = nullptr, *ff1_d = nullptr;
};

}  // namespace rohm

using namespace rohm;

struct rohm_posenet {
  rohm_ctx* ctx = nullptr;
  DevicePool pool;
  int D = 0, F = 0, L = 0, H = 0, C = 0, Cout = 0, traj = 0, pe_len = 0, passes = 3;
  int kind = kKindTf32;  // operand element type of every per-step GEMM (kKindF16 in ROHM_PRECISION_F16X2)
  int max_batch = 0, max_frames = 0;
  int64_t max_rows = 0;
  int Kin_p = 0;
  // weights
  PackedWeight w_in, w_cond, w_out;
  float *in_b = nullptr, *cond_b = nullptr, *out_b = nullptr, *pe = nullptr;
  float* time_table = nullptr;  // [pe_len, D]: TimestepEmbedder(t) + pe[0]
  std::vector<PoseNetLayerDev> layers;
  // activations
  float *Ain_h = nullptr, *Ain_l = nullptr;
  float *X = nullptr, *Xh = nullptr, *Xl = nullptr, *Y = nullptr, *QKV = nullptr, *CTXh = nullptr, *CTXl = nullptr;
  float *Hh = nullptr, *Hl = nullptr, *condpe = nullptr, *OUT = nullptr;
  float* cond_traj = nullptr;  // [B, traj, T] copy of cond[:, :traj] taken by set_cond (output channels [0,traj))
  int cond_B = -1, cond_T = -1;
  int launches = 0;
  // CUDA graph of one forward per (B, T): 61 launches become one cudaGraphLaunch; the three nodes that touch caller
  // memory (pack: x_t, time-token gather: timesteps, unpack: out) get their pointers patched before every replay.
  struct FwdGraph {
    int B = 0, T = 0;
    bool with_step = false;  // forward + Philox-fused ancestral update (rohm_posenet_sample_step)
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaGraphNode_t n_pack = nullptr, n_time = nullptr, n_unpack = nullptr, n_step = nullptr;
    cudaKernelNodeParams p_pack{}, p_time{}, p_unpack{}, p_step{};
  };
  std::vector<FwdGraph> graphs;
  bool use_graph = true;
  bool use_pdl = true;
  bool use_tma_store = true;  // ROHM_B200_TMA_STORE=0 falls back to the per-thread store epilogue (developer switch)
  // A-operand TMA multicast across CTA pairs (GemmParams::multicast_a); off by default, ROHM_B200_MULTICAST=1 turns it on.
  bool use_multicast = false;
  // wgmma attention (F16X2, head dim 128, <= 160 tokens per clip; ROHM_B200_TC_ATTENTION=0 selects the mma.sync kernel)
  bool tc_attention = false;
  AttnWgParams attn_wg{};
  // LayerNorm folding (F16X2, d_model 512; ROHM_B200_FUSED_LN=0 keeps the separate layernorm_kernel): the residual stream
  // is stored un-normalised as an fp16 pair plus per-row partial statistics (stats1: after the attention sublayer, stats2:
  // after the feed-forward sublayer), LN(u) is never materialised: see GemmParams::stats_out / a_stats
  bool fused_ln = false;
  float2* stats1 = nullptr;
  float2* stats2 = nullptr;
  float *out_c = nullptr, *out_d = nullptr;  // output head: c_n, d_n of the folded last LayerNorm
  cudaStream_t capture_stream = nullptr;
  ~rohm_posenet() {
    if (capture_stream) cudaStreamDestroy(capture_stream);
    for (auto& g : graphs) {
      if (g.exec) cudaGraphExecDestroy(g.exec);
      if (g.graph) cudaGraphDestroy(g.graph);
    }
  }
  // optional per-kernel event timing (rohm_posenet_profile): category -> list of (start, stop) events
  bool profiling = false;
  std::vector<cudaEvent_t> prof_events;
  std::vector<int> prof_cat;
  // GEMM parameter blocks (tensor maps are built once; only the grid depends on B*S)
  GemmParams g_in{}, g_cond{}, g_out{};
  std::vector<GemmParams> g_qkv, g_proj, g_ff1, g_ff2;
};

enum ProfCat { kCatGemm = 0, kCatAttention = 1, kCatLayerNorm = 2, kCatOther = 3, kNumCats = 4 };

static void prof_begin(rohm_posenet* pn, int cat, cudaStream_t st) {
  if (!pn->profiling) return;
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  pn->prof_events.push_back(a);
  pn->prof_events.push_back(b);
  pn->prof_cat.push_back(cat);
  cudaEventRecord(a, st);
}
static void prof_end(rohm_posenet* pn, cudaStream_t st) {
  if (!pn->profiling) return;
  cudaEventRecord(pn->prof_events.back(), st);
}

static int pick_block_n(int N) {
  if (N % 128 == 0) return 128;
  if (N % 96 == 0) return 96;
  if (N % 64 == 0) return 64;
  if (N <= 32) return 32;
  // ragged N: choose the tile with the least padding, preferring wide tiles
  int best = 128, waste = static_cast<int>(round_up(N, 128)) - N;
  for (int bn : {96, 64}) {
    const int w = static_cast<int>(round_up(N, bn)) - N;
    if (w < waste) best = bn, waste = w;
  }
  return best;
}

// device [N,K] fp32 -> padded hi/lo pair
static __global__ void pack_weight_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo, int N,
                                   int K, int Kp, int f16, float scale) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(N) * K) return;
  const int n = static_cast<int>(i / K), k = static_cast<int>(i % K);
  const float v = w[i];
  const int64_t o = static_cast<int64_t>(n) * Kp + k;
  if (f16) {
    ptx::split_f16(v * scale, reinterpret_cast<__half*>(hi)[o], reinterpret_cast<__half*>(lo)[o]);
  } else {
    const float h = ptx::to_tf32(v);
    hi[o] = h;
    lo[o] = v - h;
  }
}

// LayerNorm folding of a consumer GEMM y = LN(u) W^T + b, LN(u) = (u - mean) rstd gamma + beta:
//   Wf[n,k] = gamma_k W[n,k],  c_n = sum_k Wf[n,k],  d_n = b_n + sum_k beta_k W[n,k]      (one CTA per output row n)
static __global__ void fold_ln_kernel(const float* __restrict__ W, const float* __restrict__ gamma,
                                      const float* __restrict__ beta, const float* __restrict__ bias, int K,
                                      float* __restrict__ Wf, float* __restrict__ c, float* __restrict__ d) {
  const int n = blockIdx.x;
  double sc = 0.0, sd = 0.0;
  for (int k = threadIdx.x; k < K; k += blockDim.x) {
    const float w = W[static_cast<int64_t>(n) * K + k];
    const float wf = gamma[k] * w;
    Wf[static_cast<int64_t>(n) * K + k] = wf;
    sc += static_cast<double>(wf);
    sd += static_cast<double>(beta[k]) * static_cast<double>(w);
  }
  __shared__ double rc[256], rd[256];
  rc[threadIdx.x] = sc, rd[threadIdx.x] = sd;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) rc[threadIdx.x] += rc[threadIdx.x + s], rd[threadIdx.x] += rd[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    c[n] = static_cast<float>(rc[0]);
    d[n] = static_cast<float>(static_cast<double>(bias[n]) + rd[0]);
  }
}

static int pack_weight(rohm_posenet* pn, const float* w, int N, int K, PackedWeight* out, int kind);

// Packs gamma-folded weights of a [N, K] linear layer and produces its c / d vectors (library-owned).
static int pack_folded(rohm_posenet* pn, const float* w, const float* bias, const float* gamma, const float* beta, int N, int K,
                       PackedWeight* out, float** c, float** d) {
  float* wf = nullptr;
  if (cudaMalloc(&wf, static_cast<size_t>(N) * K * sizeof(float)) != cudaSuccess)
    return fail(pn->ctx, ROHM_ERR_CUDA, "folded weight scratch alloc failed");
  *c = pn->pool.floats(N), *d = pn->pool.floats(N);
  int rc = ROHM_OK;
  if (*c == nullptr || *d == nullptr) {
    rc = fail(pn->ctx, ROHM_ERR_CUDA, "alloc failed: %s", cudaGetErrorString(pn->pool.last_error()));
  } else {
    fold_ln_kernel<<<N, 256>>>(w, gamma, beta, bias, K, wf, *c, *d);
    if (cudaGetLastError() != cudaSuccess) rc = fail(pn->ctx, ROHM_ERR_CUDA, "fold_ln_kernel launch failed");
    if (rc == ROHM_OK) rc = pack_weight(pn, wf, N, K, out, pn->kind);
    if (rc == ROHM_OK && cudaDeviceSynchronize() != cudaSuccess) rc = fail(pn->ctx, ROHM_ERR_CUDA, "weight folding failed");
  }
  cudaFree(wf);
  return rc;
}

// kind == kKindF16: the matrix is stored as fp16 hi/lo of w * 2^s, s chosen per matrix so that max |w| 2^s lies in
// [2^13, 2^14): every weight within 2^-13 of the largest keeps a normal-range lo half, and nothing overflows.
static int pack_weight(rohm_posenet* pn, const float* w, int N, int K, PackedWeight* out, int kind) {
  out->N = N, out->K = K;
  out->block_n = pick_block_n(N);
  out->Np = static_cast<int>(round_up(N, out->block_n));
  out->Kp = static_cast<int>(round_up(K, gemm_block_k(kind)));
  out->kind = kind;
  out->scale = 1.0f;
  const int64_t bytes = static_cast<int64_t>(out->Np) * out->Kp * gemm_elem_bytes(kind);
  out->hi = static_cast<float*>(pn->pool.bytes(bytes));
  out->lo = static_cast<float*>(pn->pool.bytes(bytes));
  if (out->hi == nullptr || out->lo == nullptr)
    return fail(pn->ctx, ROHM_ERR_CUDA, "weight alloc failed: %s", cudaGetErrorString(pn->pool.last_error()));
  const int64_t n = static_cast<int64_t>(N) * K;
  if (kind == kKindF16) ROHM_CUDA(pn->ctx, f16_weight_scale(w, n, &out->scale));
  pack_weight_kernel<<<static_cast<unsigned>((n + 255) / 256), 256>>>(w, out->hi, out->lo, N, K, out->Kp,
                                                                     kind == kKindF16 ? 1 : 0, out->scale);
  ROHM_CUDA(pn->ctx, cudaGetLastError());
  return ROHM_OK;
}

static int copy_vec(rohm_posenet* pn, const float* src, int64_t n, float** dst) {
  *dst = pn->pool.floats(n);
  if (*dst == nullptr) return fail(pn->ctx, ROHM_ERR_CUDA, "alloc failed: %s", cudaGetErrorString(pn->pool.last_error()));
  ROHM_CUDA(pn->ctx, cudaMemcpy(*dst, src, static_cast<size_t>(n) * sizeof(float), cudaMemcpyDeviceToDevice));
  return ROHM_OK;
}

// Plain linear layer: A (hi/lo, [rows, K] with pitch lda) x W^T.
static int setup_linear(rohm_posenet* pn, GemmParams* g, const float* a_hi, const float* a_lo, int64_t rows, int K, int lda,
                 const PackedWeight& w, const float* bias) {
  *g = GemmParams{};
  int rc = make_tmap_2d(&g->a_hi[0], a_hi, rows, K, lda, kGemmBlockM, 1, w.kind);
  rc |= make_tmap_2d(&g->a_lo[0], a_lo, rows, K, lda, kGemmBlockM, 1, w.kind);
  rc |= make_tmap_2d(&g->b_hi, w.hi, w.Np, w.Kp, w.Kp, w.block_n, 1, w.kind);
  rc |= make_tmap_2d(&g->b_lo, w.lo, w.Np, w.Kp, w.Kp, w.block_n, 1, w.kind);
  if (rc != 0) return fail(pn->ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d)", rc);
  g->num_segs = 1;
  g->seg_kblocks[0] = w.Kp / gemm_block_k(w.kind);
  g->acc_scale = 1.0f / w.scale;
  g->seg_row_shift[0] = 0;
  g->seg_row_mul[0] = 1;
  g->bias = bias;
  g->N = w.N;
  g->out_row_mul = 1;
  g->out_row_add = 0;
  if (pn->use_multicast && w.kind == kKindF16 && pn->passes == 3 &&
      gemm_enable_multicast(g, a_hi, a_lo, rows, K, lda, w.N, w.block_n, w.kind) != 0)
    return fail(pn->ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled failed (multicast maps)");
  return ROHM_OK;
}

static int run_gemm(rohm_posenet* pn, GemmParams& g, const PackedWeight& w, int rows, cudaStream_t st) {
  g.M = rows;
  prof_begin(pn, kCatGemm, st);
  // programmatic dependent launch: this GEMM's prologue (barrier init, tensor-map prefetch, weight tiles) overlaps the
  // tail of the previous kernel; its griddepcontrol.wait orders all global reads/writes after that kernel
  ROHM_CUDA(pn->ctx, launch_gemm(g, rows, w.N, w.block_n, pn->passes, st, pn->use_pdl && !pn->profiling, w.kind));
  prof_end(pn, st);
  pn->launches++;
  return ROHM_OK;
}

// Kernel launch with the programmatic-dependent-launch attribute (the kernel must call griddepcontrol.wait before it
// touches memory, which every kernel launched through here does).
template <typename... KArgs, typename... Args>
static cudaError_t launch_chain(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, bool pdl,
                                Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

template <int D>
static void launch_ln(const float* in, const float* res, const float* g, const float* b, float* out, float* oh, float* ol,
               int rows, cudaStream_t st, int f16, bool pdl) {
  launch_chain(layernorm_kernel<D>, dim3((rows + 7) / 8), dim3(256), 0, st, pdl, in, res, g, b, out, oh, ol, rows, f16);
}

static int run_ln(rohm_posenet* pn, const float* in, const float* res, const float* g, const float* b, float* out, float* oh,
           float* ol, int rows, cudaStream_t st) {
  prof_begin(pn, kCatLayerNorm, st);
  const int f16 = pn->kind == kKindF16 ? 1 : 0;
  const bool pdl = pn->use_pdl && !pn->profiling;
  switch (pn->D) {
    case 128: launch_ln<128>(in, res, g, b, out, oh, ol, rows, st, f16, pdl); break;
    case 256: launch_ln<256>(in, res, g, b, out, oh, ol, rows, st, f16, pdl); break;
    case 512: launch_ln<512>(in, res, g, b, out, oh, ol, rows, st, f16, pdl); break;
    case 1024: launch_ln<1024>(in, res, g, b, out, oh, ol, rows, st, f16, pdl); break;
    default: return fail(pn->ctx, ROHM_ERR_INVALID, "unsupported d_model %d for LayerNorm", pn->D);
  }
  prof_end(pn, st);
  ROHM_CUDA(pn->ctx, cudaGetLastError());
  pn->launches++;
  return ROHM_OK;
}

template <int DH, int NT>
static cudaError_t launch_attention_mma(rohm_posenet* pn, int B, int S, float scale, cudaStream_t st) {
  auto kern = attention_mma_kernel<DH, NT>;
  static bool attr_set = false;
  const size_t smem = attention_mma_smem_bytes(NT);
  if (!attr_set) {
    cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  const int warps = (S + 15) / 16;
  return launch_chain(kern, dim3(B * pn->H), dim3(32 * warps), smem, st, pn->use_pdl && !pn->profiling, pn->QKV, pn->CTXh,
                      pn->CTXl, S, pn->D, pn->H, scale, pn->kind == kKindF16 ? 1 : 0);
}

static int run_attention_wgmma(rohm_posenet* pn, int B, int S, cudaStream_t st) {
  AttnWgParams prm = pn->attn_wg;
  prm.S = S;
  const int qtiles = (S + kAwQRows - 1) / kAwQRows;
  prof_begin(pn, kCatAttention, st);
  cudaError_t e = launch_chain(attention_wgmma_kernel, dim3(B * pn->H * qtiles), dim3(128), kAwSmemBytes, st,
                               pn->use_pdl && !pn->profiling, prm);
  prof_end(pn, st);
  ROHM_CUDA(pn->ctx, e);
  pn->launches++;
  return ROHM_OK;
}

template <int DH, int NK>
static cudaError_t launch_attention_f16(rohm_posenet* pn, int B, int S, float scale, cudaStream_t st) {
  const int warps = (S + 15) / 16;
  const __half* qh = reinterpret_cast<const __half*>(pn->QKV);
  const __half* ql = qh + pn->max_rows * 3 * pn->D;
  return launch_chain(attention_f16_kernel<DH, NK>, dim3(B * pn->H), dim3(32 * warps), attention_f16_smem_bytes<DH>(NK), st,
                      pn->use_pdl && !pn->profiling, qh, ql, reinterpret_cast<__half*>(pn->CTXh),
                      reinterpret_cast<__half*>(pn->CTXl), S, pn->D, pn->H, scale);
}

static int run_attention(rohm_posenet* pn, int B, int S, cudaStream_t st) {
  const int dh = pn->D / pn->H;
  const float scale = 1.0f / sqrtf(static_cast<float>(dh));
  prof_begin(pn, kCatAttention, st);
  const int nt = (S + 7) / 8;
  cudaError_t e = cudaSuccess;
  bool done = true;
  const bool f16 = pn->kind == kKindF16;
  const float* qkv_lo = reinterpret_cast<const float*>(reinterpret_cast<const __half*>(pn->QKV) + pn->max_rows * 3 * pn->D);
  if (f16) {
    const int nk = (S + 15) / 16;
    if (dh == 128 && nk <= 2) e = launch_attention_f16<128, 2>(pn, B, S, scale, st);
    else if (dh == 128 && nk <= 4) e = launch_attention_f16<128, 4>(pn, B, S, scale, st);
    else if (dh == 128 && nk <= 6) e = launch_attention_f16<128, 6>(pn, B, S, scale, st);
    else if (dh == 128 && nk <= 8) e = launch_attention_f16<128, 8>(pn, B, S, scale, st);
    else if (dh == 128 && nk <= 10) e = launch_attention_f16<128, 10>(pn, B, S, scale, st);
    else if (dh == 64 && nk <= 4) e = launch_attention_f16<64, 4>(pn, B, S, scale, st);
    else if (dh == 64 && nk <= 10) e = launch_attention_f16<64, 10>(pn, B, S, scale, st);
    else done = false;
  }
  // tensor-core path: S <= 160 tokens (register budget of the S/P fragment); wider clips use the SIMT kernel
  else if (dh == 128 && nt <= 4) e = launch_attention_mma<128, 4>(pn, B, S, scale, st);
  else if (dh == 128 && nt <= 8) e = launch_attention_mma<128, 8>(pn, B, S, scale, st);
  else if (dh == 128 && nt <= 12) e = launch_attention_mma<128, 12>(pn, B, S, scale, st);
  else if (dh == 128 && nt <= 16) e = launch_attention_mma<128, 16>(pn, B, S, scale, st);
  else if (dh == 128 && nt <= 20) e = launch_attention_mma<128, 20>(pn, B, S, scale, st);
  else if (dh == 64 && nt <= 8) e = launch_attention_mma<64, 8>(pn, B, S, scale, st);
  else if (dh == 64 && nt <= 20) e = launch_attention_mma<64, 20>(pn, B, S, scale, st);
  else done = false;
  if (!done) {
    const size_t smem = attention_smem_bytes(S, dh);
    if (dh == 128) {
      e = launch_chain(attention_kernel<128>, dim3(B * pn->H), dim3(256), smem, st, pn->use_pdl && !pn->profiling, pn->QKV,
                       qkv_lo, pn->CTXh, pn->CTXl, S, pn->D, pn->H, scale, f16 ? 1 : 0);
    } else if (dh == 64) {
      e = launch_chain(attention_kernel<64>, dim3(B * pn->H), dim3(256), smem, st, pn->use_pdl && !pn->profiling, pn->QKV,
                       qkv_lo, pn->CTXh, pn->CTXl, S, pn->D, pn->H, scale, f16 ? 1 : 0);
    } else {
      return fail(pn->ctx, ROHM_ERR_INVALID, "unsupported head dim %d", dh);
    }
  }
  prof_end(pn, st);
  ROHM_CUDA(pn->ctx, e);
  pn->launches++;
  return ROHM_OK;
}

// TE = (silu(PE W0^T + b0)) W2^T + (b2 + pe[0]) over all pe_len rows, with the engine's own GEMM kernel.
static int build_time_table(rohm_posenet* pn, const rohm_posenet_weights* w) {
  const int D = pn->D, R = pn->pe_len;
  const int64_t n = static_cast<int64_t>(R) * D;
  pn->time_table = pn->pool.floats(n);
  if (pn->time_table == nullptr) return fail(pn->ctx, ROHM_ERR_CUDA, "time table alloc failed");
  DevicePool tmp;  // freed on return
  PackedWeight w0, w2;
  float* pe_h = tmp.floats(n);
  float* pe_l = tmp.floats(n);
  float* h_h = tmp.floats(n);
  float* h_l = tmp.floats(n);
  float* bias2 = tmp.floats(D);
  if (!pe_h || !pe_l || !h_h || !h_l || !bias2) return fail(pn->ctx, ROHM_ERR_CUDA, "time table scratch alloc failed");
  int rc;
  if ((rc = pack_weight(pn, w->t0_w, D, D, &w0, kKindTf32)) != ROHM_OK) return rc;  // small (2 x 2 MB), kept in the pool
  if ((rc = pack_weight(pn, w->t2_w, D, D, &w2, kKindTf32)) != ROHM_OK) return rc;
  ROHM_CUDA(pn->ctx, launch_split_tf32(pn->pe, pe_h, pe_l, n, 0));
  add_vec_kernel<<<(D + 255) / 256, 256>>>(w->t2_b, pn->pe, bias2, D);  // b2 + pe[0]
  ROHM_CUDA(pn->ctx, cudaGetLastError());
  GemmParams g1{}, g2{};
  if ((rc = setup_linear(pn, &g1, pe_h, pe_l, R, D, D, w0, w->t0_b)) != ROHM_OK) return rc;
  g1.act = kActSilu;
  g1.out_hi = h_h, g1.out_lo = h_l, g1.lds = D;
  g1.M = R;
  ROHM_CUDA(pn->ctx, launch_gemm(g1, R, D, w0.block_n, 3, 0));
  if ((rc = setup_linear(pn, &g2, h_h, h_l, R, D, D, w2, bias2)) != ROHM_OK) return rc;
  g2.out = pn->time_table, g2.ldo = D;
  g2.M = R;
  ROHM_CUDA(pn->ctx, launch_gemm(g2, R, D, w2.block_n, 3, 0));
  ROHM_CUDA(pn->ctx, cudaDeviceSynchronize());
  return ROHM_OK;
}

extern "C" int rohm_posenet_create(rohm_ctx* ctx, const rohm_posenet_weights* w, int max_batch, int max_frames,
                                   int precision, rohm_posenet** out) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (w == nullptr || out == nullptr || max_batch <= 0 || max_frames <= 0)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_create: bad arguments");
  if (precision != ROHM_PRECISION_TF32X3 && precision != ROHM_PRECISION_TF32 && precision != ROHM_PRECISION_F16X2)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_create: precision must be 3 (TF32x3), 2 (F16x2) or 1 (TF32)");
  if (w->d_model % 128 != 0 || w->d_model % w->num_heads != 0 || w->ff_size % 64 != 0)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_create: d_model must be a multiple of 128, ff_size of 64");
  const int dh = w->d_model / w->num_heads;
  if (dh != 64 && dh != 128) return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_create: head dim must be 64 or 128");
  if (max_frames + 1 > 256) return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_create: at most 255 frames per clip");
  if (max_frames + 1 > w->pe_len) return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_create: clip longer than pe table");

  rohm_posenet* pn = new (std::nothrow) rohm_posenet();
  if (pn == nullptr) return fail(ctx, ROHM_ERR_INVALID, "out of host memory");
  pn->ctx = ctx;
  pn->D = w->d_model, pn->F = w->ff_size, pn->L = w->num_layers, pn->H = w->num_heads;
  pn->C = w->in_feats, pn->Cout = w->out_feats, pn->traj = w->traj_feats, pn->pe_len = w->pe_len;
  pn->kind = precision == ROHM_PRECISION_F16X2 ? kKindF16 : kKindTf32;
  if (const char* env = getenv("ROHM_B200_TMA_STORE")) pn->use_tma_store = env[0] != '0';
  if (const char* env = getenv("ROHM_B200_MULTICAST")) pn->use_multicast = env[0] != '0';
  pn->passes = precision == ROHM_PRECISION_TF32 ? 1 : 3;
  pn->max_batch = max_batch, pn->max_frames = max_frames;
  pn->max_rows = static_cast<int64_t>(max_batch) * (max_frames + 1);
  pn->Kin_p = static_cast<int>(round_up(pn->C, gemm_block_k(pn->kind)));
  {
    const char* env = getenv("ROHM_B200_TC_ATTENTION");
    pn->tc_attention = pn->kind == kKindF16 && dh == 128 && (env == nullptr || env[0] != '0');
  }
  const int D = pn->D, F = pn->F;
  const int64_t R = pn->max_rows;
  {
    const char* env = getenv("ROHM_B200_FUSED_LN");
    pn->fused_ln = pn->kind == kKindF16 && D == 512 && pn->use_tma_store && (env == nullptr || env[0] != '0');
    if (pn->fused_ln) {
      pn->stats1 = static_cast<float2*>(pn->pool.bytes(R * 8 * static_cast<int64_t>(sizeof(float2))));
      pn->stats2 = static_cast<float2*>(pn->pool.bytes(R * 8 * static_cast<int64_t>(sizeof(float2))));
      if (pn->stats1 == nullptr || pn->stats2 == nullptr) {
        const int rc = fail(ctx, ROHM_ERR_CUDA, "LayerNorm statistics buffers: %s", cudaGetErrorString(pn->pool.last_error()));
        delete pn;
        return rc;
      }
    }
  }

#define TRY(expr)            \
  do {                       \
    int rc__ = (expr);       \
    if (rc__ != ROHM_OK) {   \
      delete pn;             \
      return rc__;           \
    }                        \
  } while (0)

  TRY(pack_weight(pn, w->in_w, D, pn->C, &pn->w_in, pn->kind));
  TRY(pack_weight(pn, w->cond_w, D, pn->C, &pn->w_cond, pn->kind));
  if (pn->fused_ln && pn->L > 0) {  // the head consumes LN2 of the last layer
    const rohm_posenet_layer& last = w->layers[pn->L - 1];
    TRY(pack_folded(pn, w->out_w, w->out_b, last.norm2_w, last.norm2_b, pn->Cout, D, &pn->w_out, &pn->out_c, &pn->out_d));
  } else {
    TRY(pack_weight(pn, w->out_w, pn->Cout, D, &pn->w_out, pn->kind));
  }
  TRY(copy_vec(pn, w->in_b, D, &pn->in_b));
  TRY(copy_vec(pn, w->cond_b, D, &pn->cond_b));
  TRY(copy_vec(pn, w->out_b, pn->Cout, &pn->out_b));
  TRY(copy_vec(pn, w->pe, static_cast<int64_t>(pn->pe_len) * D, &pn->pe));
  TRY(build_time_table(pn, w));
  pn->layers.resize(pn->L);
  for (int l = 0; l < pn->L; ++l) {
    const rohm_posenet_layer& s = w->layers[l];
    PoseNetLayerDev& d = pn->layers[l];
    if (pn->fused_ln && l > 0) {  // QKV consumes LN2 of the previous layer
      const rohm_posenet_layer& prev = w->layers[l - 1];
      TRY(pack_folded(pn, s.in_proj_w, s.in_proj_b, prev.norm2_w, prev.norm2_b, 3 * D, D, &d.qkv, &d.qkv_c, &d.qkv_d));
    } else {
      TRY(pack_weight(pn, s.in_proj_w, 3 * D, D, &d.qkv, pn->kind));
    }
    TRY(pack_weight(pn, s.out_proj_w, D, D, &d.proj, pn->kind));
    if (pn->fused_ln) {  // FFN1 consumes LN1 of this layer
      TRY(pack_folded(pn, s.lin1_w, s.lin1_b, s.norm1_w, s.norm1_b, F, D, &d.ff1, &d.ff1_c, &d.ff1_d));
    } else {
      TRY(pack_weight(pn, s.lin1_w, F, D, &d.ff1, pn->kind));
    }
    TRY(pack_weight(pn, s.lin2_w, D, F, &d.ff2, pn->kind));
    TRY(copy_vec(pn, s.in_proj_b, 3 * D, &d.qkv_b));
    TRY(copy_vec(pn, s.out_proj_b, D, &d.proj_b));
    TRY(copy_vec(pn, s.lin1_b, F, &d.ff1_b));
    TRY(copy_vec(pn, s.lin2_b, D, &d.ff2_b));
    TRY(copy_vec(pn, s.norm1_w, D, &d.n1_w));
    TRY(copy_vec(pn, s.norm1_b, D, &d.n1_b));
    TRY(copy_vec(pn, s.norm2_w, D, &d.n2_w));
    TRY(copy_vec(pn, s.norm2_b, D, &d.n2_b));
  }

  struct {
    float** p;
    int64_t n;
  } bufs[] = {{&pn->Ain_h, R * pn->Kin_p}, {&pn->Ain_l, R * pn->Kin_p}, {&pn->X, R * D},     {&pn->Xh, R * D},
              {&pn->Xl, R * D},           {&pn->Y, R * D},             {&pn->QKV, R * 3 * D}, {&pn->CTXh, R * D},
              {&pn->CTXl, R * D},         {&pn->Hh, R * F},            {&pn->Hl, R * F},      {&pn->condpe, R * D},
              {&pn->OUT, R * pn->Cout},
              {&pn->cond_traj, static_cast<int64_t>(max_batch) * (pn->traj > 0 ? pn->traj : 1) * max_frames}};
  for (auto& b : bufs) {
    *b.p = pn->pool.floats(b.n);
    if (*b.p == nullptr) {
      const int rc = fail(ctx, ROHM_ERR_CUDA, "workspace alloc failed: %s", cudaGetErrorString(pn->pool.last_error()));
      delete pn;
      return rc;
    }
  }

  // GEMM descriptors.  Input embedding: residual = cond embedding + positional rows (set per set_cond).
  TRY(setup_linear(pn, &pn->g_in, pn->Ain_h, pn->Ain_l, R, pn->C, pn->Kin_p, pn->w_in, pn->in_b));
  pn->g_in.residual = pn->condpe, pn->g_in.ldr = D;
  pn->g_in.out = pn->X, pn->g_in.ldo = D;
  pn->g_in.out_hi = pn->Xh, pn->g_in.out_lo = pn->Xl, pn->g_in.lds = D;
  // Condition embedding: residual = positional rows (held in condpe itself: written in place).
  TRY(setup_linear(pn, &pn->g_cond, pn->Ain_h, pn->Ain_l, R, pn->C, pn->Kin_p, pn->w_cond, pn->cond_b));
  pn->g_cond.residual = pn->condpe, pn->g_cond.ldr = D;
  pn->g_cond.out = pn->condpe, pn->g_cond.ldo = D;
  // Output head.
  TRY(setup_linear(pn, &pn->g_out, pn->Xh, pn->Xl, R, D, D, pn->w_out, pn->out_b));
  pn->g_out.out = pn->OUT, pn->g_out.ldo = pn->Cout;
  if (pn->fused_ln && pn->L > 0)
    pn->g_out.a_stats = pn->stats2, pn->g_out.a_corr = pn->out_c, pn->g_out.bias = pn->out_d, pn->g_out.ln_eps = 1e-5f;
  pn->g_qkv.resize(pn->L), pn->g_proj.resize(pn->L), pn->g_ff1.resize(pn->L), pn->g_ff2.resize(pn->L);
  for (int l = 0; l < pn->L; ++l) {
    PoseNetLayerDev& d = pn->layers[l];
    TRY(setup_linear(pn, &pn->g_qkv[l], pn->Xh, pn->Xl, R, D, D, d.qkv, d.qkv_b));
    if (pn->kind == kKindF16) {  // Q | K | V as fp16 hi/lo planes sharing the fp32 buffer's footprint
      pn->g_qkv[l].out_hi = pn->QKV;
      pn->g_qkv[l].out_lo = reinterpret_cast<__half*>(pn->QKV) + R * 3 * D;
      pn->g_qkv[l].lds = 3 * D;
    } else {
      pn->g_qkv[l].out = pn->QKV, pn->g_qkv[l].ldo = 3 * D;
    }
    // the residual adds (x + sa_block(x), x + ff_block(x)) happen in the LayerNorm kernel that follows, which leaves
    // the GEMM epilogues free of global reads
    TRY(setup_linear(pn, &pn->g_proj[l], pn->CTXh, pn->CTXl, R, D, D, d.proj, d.proj_b));
    pn->g_proj[l].out = pn->Y, pn->g_proj[l].ldo = D;
    // LayerNorm folding: producers write u in place over the residual pair + partial statistics; consumers correct
    auto producer = [&](GemmParams& g, float2* stats_out, const float2* res_stats, const float* res_gamma, const float* res_beta) {
      g.out = nullptr, g.ldo = 0;
      g.out_hi = pn->Xh, g.out_lo = pn->Xl, g.lds = D;
      g.stats_out = stats_out, g.res_stats = res_stats, g.res_gamma = res_gamma, g.res_beta = res_beta, g.ln_eps = 1e-5f;
    };
    auto consumer = [&](GemmParams& g, const float2* a_stats, const float* c, const float* dvec) {
      g.a_stats = a_stats, g.a_corr = c, g.bias = dvec, g.ln_eps = 1e-5f;
    };
    if (pn->fused_ln) {
      if (l > 0) consumer(pn->g_qkv[l], pn->stats2, d.qkv_c, d.qkv_d);
      // out-proj: u1 = LN2_prev(u2_prev) + attn   (layer 0: the embedded input, not normalised)
      producer(pn->g_proj[l], pn->stats1, l > 0 ? pn->stats2 : nullptr, l > 0 ? pn->layers[l - 1].n2_w : nullptr,
               l > 0 ? pn->layers[l - 1].n2_b : nullptr);
    }
    TRY(setup_linear(pn, &pn->g_ff1[l], pn->Xh, pn->Xl, R, D, D, d.ff1, d.ff1_b));
    pn->g_ff1[l].act = kActGelu;
    pn->g_ff1[l].out_hi = pn->Hh, pn->g_ff1[l].out_lo = pn->Hl, pn->g_ff1[l].lds = F;
    TRY(setup_linear(pn, &pn->g_ff2[l], pn->Hh, pn->Hl, R, F, F, d.ff2, d.ff2_b));
    pn->g_ff2[l].out = pn->Y, pn->g_ff2[l].ldo = D;
    if (pn->fused_ln) {
      consumer(pn->g_ff1[l], pn->stats1, d.ff1_c, d.ff1_d);
      producer(pn->g_ff2[l], pn->stats2, pn->stats1, d.n1_w, d.n1_b);  // u2 = LN1(u1) + ffn
    }
    for (GemmParams* g : {&pn->g_qkv[l], &pn->g_proj[l], &pn->g_ff1[l], &pn->g_ff2[l]}) {
      if (pn->use_tma_store && gemm_enable_tma_store(g, R, pn->kind) != 0) {
        const int rc__ = fail(ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (store map) failed");
        delete pn;
        return rc__;
      }
    }
  }
  if (pn->use_tma_store && gemm_enable_tma_store(&pn->g_out, R, pn->kind) != 0) {
    const int rc__ = fail(ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (store map) failed");
    delete pn;
    return rc__;
  }
#undef TRY

  {
    cudaError_t ea = gemm_init_attributes();
    auto set_mma = [&](auto kern, int nt) {
      if (ea == cudaSuccess)
        ea = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  static_cast<int>(attention_mma_smem_bytes(nt)));
    };
    set_mma(attention_mma_kernel<128, 4>, 4);
    set_mma(attention_mma_kernel<128, 8>, 8);
    set_mma(attention_mma_kernel<128, 12>, 12);
    set_mma(attention_mma_kernel<128, 16>, 16);
    set_mma(attention_mma_kernel<128, 20>, 20);
    set_mma(attention_mma_kernel<64, 8>, 8);
    set_mma(attention_mma_kernel<64, 20>, 20);
    auto set_f16 = [&](auto kern, size_t bytes) {
      if (ea == cudaSuccess) ea = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
    };
    set_f16(attention_f16_kernel<128, 2>, attention_f16_smem_bytes<128>(2));
    set_f16(attention_f16_kernel<128, 4>, attention_f16_smem_bytes<128>(4));
    set_f16(attention_f16_kernel<128, 6>, attention_f16_smem_bytes<128>(6));
    set_f16(attention_f16_kernel<128, 8>, attention_f16_smem_bytes<128>(8));
    set_f16(attention_f16_kernel<128, 10>, attention_f16_smem_bytes<128>(10));
    set_f16(attention_f16_kernel<64, 4>, attention_f16_smem_bytes<64>(4));
    set_f16(attention_f16_kernel<64, 10>, attention_f16_smem_bytes<64>(10));
    set_f16(attention_wgmma_kernel, kAwSmemBytes);
    if (pn->tc_attention) {
      __half* qkv_hi = reinterpret_cast<__half*>(pn->QKV);
      __half* qkv_lo = qkv_hi + R * 3 * D;
      int rcm = make_tile_tmap_f16_sw128(&pn->attn_wg.q_hi, qkv_hi, R, 3 * D, 3 * D, kAwQRows);
      rcm |= make_tile_tmap_f16_sw128(&pn->attn_wg.q_lo, qkv_lo, R, 3 * D, 3 * D, kAwQRows);
      rcm |= make_tile_tmap_f16_sw128(&pn->attn_wg.kv_hi, qkv_hi, R, 3 * D, 3 * D, kAwKeys);
      rcm |= make_tile_tmap_f16_sw128(&pn->attn_wg.kv_lo, qkv_lo, R, 3 * D, 3 * D, kAwKeys);
      if (rcm != 0) {
        delete pn;
        return fail(ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (attention tiles) failed (%d)", rcm);
      }
      pn->attn_wg.ctx_hi = reinterpret_cast<__half*>(pn->CTXh), pn->attn_wg.ctx_lo = reinterpret_cast<__half*>(pn->CTXl);
      pn->attn_wg.D = D, pn->attn_wg.H = pn->H;
      pn->attn_wg.scale = 1.0f / sqrtf(static_cast<float>(dh));
    }
    if (ea != cudaSuccess) {
      delete pn;
      return fail(ctx, ROHM_ERR_CUDA, "kernel attribute setup failed: %s", cudaGetErrorString(ea));
    }
  }
  // attention kernels need > 48 KB of dynamic shared memory
  const size_t smem_max = attention_smem_bytes(max_frames + 1, dh);
  if (smem_max > 227 * 1024) {
    delete pn;
    return fail(ctx, ROHM_ERR_INVALID, "clip too long for the attention kernel (%zu B smem)", smem_max);
  }
  cudaError_t e = dh == 128 ? cudaFuncSetAttribute(attention_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   static_cast<int>(smem_max))
                            : cudaFuncSetAttribute(attention_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                   static_cast<int>(smem_max));
  if (e != cudaSuccess) {
    delete pn;
    return fail(ctx, ROHM_ERR_CUDA, "cudaFuncSetAttribute(attention): %s", cudaGetErrorString(e));
  }
  e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    delete pn;
    return fail(ctx, ROHM_ERR_CUDA, "weight packing failed: %s", cudaGetErrorString(e));
  }
  *out = pn;
  return ROHM_OK;
}

extern "C" void rohm_posenet_destroy(rohm_posenet* pn) { delete pn; }

extern "C" int rohm_posenet_launches_per_forward(const rohm_posenet* pn) { return pn ? pn->launches : 0; }

extern "C" int rohm_posenet_set_cond(rohm_posenet* pn, const float* cond, int B, int T, void* stream) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (cond == nullptr || B <= 0 || T <= 0 || B > pn->max_batch || T > pn->max_frames)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_set_cond: B=%d T=%d outside the created capacity (%d, %d)", B, T,
                pn->max_batch, pn->max_frames);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int S = T + 1, D = pn->D;
  const int rows = B * S;
  // A_in <- tokens of cond (row (b,0) stays zero: the buffer was zero-initialised and is never written there)
  dim3 grid((T + 31) / 32, (pn->C + 31) / 32, B);
  pack_tokens_kernel<<<grid, dim3(32, 8), 0, st>>>(cond, pn->Ain_h, pn->Ain_l, pn->C, T, S, pn->Kin_p,
                                                   pn->kind == kKindF16 ? 1 : 0);
  ROHM_CUDA(ctx, cudaGetLastError());
  const int64_t total4 = static_cast<int64_t>(rows) * D / 4;
  pe_rows_kernel<<<static_cast<unsigned>((total4 + 255) / 256), 256, 0, st>>>(pn->pe, pn->condpe, S, D, total4);
  ROHM_CUDA(ctx, cudaGetLastError());
  // condpe <- cond_embed(cond) + cond_b + pe rows   (in place; rows (b,0) become cond_b + pe[0]: overwritten later
  // by the timestep token, so their value is irrelevant)
  const int saved = pn->launches;
  int rc = run_gemm(pn, pn->g_cond, pn->w_cond, rows, st);
  pn->launches = saved;
  if (rc != ROHM_OK) return rc;
  if (pn->traj > 0) {
    const size_t width = static_cast<size_t>(pn->traj) * T * sizeof(float);
    ROHM_CUDA(ctx, cudaMemcpy2DAsync(pn->cond_traj, width, cond, static_cast<size_t>(pn->C) * T * sizeof(float), width,
                                     B, cudaMemcpyDeviceToDevice, st));
  }
  pn->cond_B = B, pn->cond_T = T;
  return ROHM_OK;
}

// The raw launch sequence of one forward (what gets captured into the graph).
static int forward_launches(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B, int T,
                            cudaStream_t st) {
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const int S = T + 1, D = pn->D;
  const int rows = B * S;
  pn->launches = 0;
  int rc;

  dim3 grid((T + 31) / 32, (pn->C + 31) / 32, B);
  prof_begin(pn, kCatOther, st);
  const bool pdl = pn->use_pdl && !pn->profiling;
  ROHM_CUDA(ctx, launch_chain(pack_tokens_kernel, grid, dim3(32, 8), 0, st, pdl, x_t, pn->Ain_h, pn->Ain_l, pn->C, T, S, pn->Kin_p,
                              pn->kind == kKindF16 ? 1 : 0));
  prof_end(pn, st);
  ROHM_CUDA(ctx, cudaGetLastError());
  pn->launches++;
  if ((rc = run_gemm(pn, pn->g_in, pn->w_in, rows, st)) != ROHM_OK) return rc;
  prof_begin(pn, kCatOther, st);
  ROHM_CUDA(ctx, launch_chain(time_token_gather_kernel, dim3(B), dim3(128), 0, st, pdl, timesteps, pn->time_table, pn->pe_len,
                              pn->X, pn->Xh, pn->Xl, S, D, pn->kind == kKindF16 ? 1 : 0, nullptr, 0));
  prof_end(pn, st);
  ROHM_CUDA(ctx, cudaGetLastError());
  pn->launches++;

  for (int l = 0; l < pn->L; ++l) {
    PoseNetLayerDev& d = pn->layers[l];
    if ((rc = run_gemm(pn, pn->g_qkv[l], d.qkv, rows, st)) != ROHM_OK) return rc;
    if (pn->tc_attention && S <= kAwKeys) {
      if ((rc = run_attention_wgmma(pn, B, S, st)) != ROHM_OK) return rc;
    } else {
      if ((rc = run_attention(pn, B, S, st)) != ROHM_OK) return rc;
    }
    if ((rc = run_gemm(pn, pn->g_proj[l], d.proj, rows, st)) != ROHM_OK) return rc;
    if (!pn->fused_ln && (rc = run_ln(pn, pn->Y, pn->X, d.n1_w, d.n1_b, pn->X, pn->Xh, pn->Xl, rows, st)) != ROHM_OK) return rc;
    if ((rc = run_gemm(pn, pn->g_ff1[l], d.ff1, rows, st)) != ROHM_OK) return rc;
    if ((rc = run_gemm(pn, pn->g_ff2[l], d.ff2, rows, st)) != ROHM_OK) return rc;
    if (!pn->fused_ln && (rc = run_ln(pn, pn->Y, pn->X, d.n2_w, d.n2_b, pn->X, pn->Xh, pn->Xl, rows, st)) != ROHM_OK) return rc;
  }
  if ((rc = run_gemm(pn, pn->g_out, pn->w_out, rows, st)) != ROHM_OK) return rc;
  dim3 grid_o((T + 31) / 32, (pn->Cout + 31) / 32, B);
  prof_begin(pn, kCatOther, st);
  ROHM_CUDA(ctx, launch_chain(unpack_tokens_kernel, grid_o, dim3(32, 8), 0, st, pdl, pn->OUT, pn->cond_traj, out, pn->C, pn->Cout,
                              pn->traj, T, S, pn->Cout));
  prof_end(pn, st);
  ROHM_CUDA(ctx, cudaGetLastError());
  pn->launches++;
  return ROHM_OK;
}

extern "C" int rohm_posenet_forward(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B,
                                    int T, void* stream);

// One forward with CUDA events around every kernel launch (on `stream`, the launching stream); synchronises and
// returns the summed device time and launch count per category {GEMM, attention, LayerNorm, other}.
extern "C" int rohm_posenet_profile(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B,
                                    int T, void* stream, float* ms_by_category, int* launches_by_category) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  if (ms_by_category == nullptr || launches_by_category == nullptr)
    return fail(pn->ctx, ROHM_ERR_INVALID, "rohm_posenet_profile: null output");
  pn->profiling = true;
  pn->prof_events.clear();
  pn->prof_cat.clear();
  int rc = rohm_posenet_forward(pn, x_t, timesteps, out, B, T, stream);
  pn->profiling = false;
  cudaError_t e = cudaStreamSynchronize(static_cast<cudaStream_t>(stream));
  for (int c = 0; c < kNumCats; ++c) ms_by_category[c] = 0.0f, launches_by_category[c] = 0;
  for (size_t i = 0; i < pn->prof_cat.size(); ++i) {
    float ms = 0.0f;
    if (rc == ROHM_OK && e == cudaSuccess) cudaEventElapsedTime(&ms, pn->prof_events[2 * i], pn->prof_events[2 * i + 1]);
    ms_by_category[pn->prof_cat[i]] += ms;
    launches_by_category[pn->prof_cat[i]]++;
  }
  for (cudaEvent_t ev : pn->prof_events) cudaEventDestroy(ev);
  pn->prof_events.clear();
  pn->prof_cat.clear();
  if (rc != ROHM_OK) return rc;
  ROHM_CUDA(pn->ctx, e);
  return ROHM_OK;
}

struct StepArgs {  // the ancestral update appended to the forward (rohm_posenet_sample_step)
  float* x_next;
  const float* coef_row;
  unsigned long long seed, offset;
  int64_t G;
  int iters;
};

static int build_forward_graph(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B, int T,
                               cudaStream_t st, rohm_posenet::FwdGraph* fg, const StepArgs* step = nullptr) {
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  // Capture on a private stream: the caller's stream may be the legacy default stream, which cannot be captured.
  // Nothing executes during capture; the instantiated graph is then launched on the caller's stream.
  (void)st;
  if (pn->capture_stream == nullptr)
    ROHM_CUDA(ctx, cudaStreamCreateWithFlags(&pn->capture_stream, cudaStreamNonBlocking));
  cudaStream_t cs = pn->capture_stream;
  ROHM_CUDA(ctx, cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
  int rc = forward_launches(pn, x_t, timesteps, out, B, T, cs);
  if (rc == ROHM_OK && step != nullptr) {
    const int64_t clip_elems = static_cast<int64_t>(pn->C) * T;
    if (launch_ddpm_step_philox(out, x_t, step->x_next, clip_elems * B, clip_elems, step->coef_row, step->seed, step->offset,
                                step->G, step->iters, cs, pn->use_pdl) != cudaSuccess)
      rc = fail(ctx, ROHM_ERR_CUDA, "ddpm step launch failed during capture");
    pn->launches++;
  }
  cudaGraph_t graph = nullptr;
  cudaError_t e = cudaStreamEndCapture(cs, &graph);
  if (rc != ROHM_OK) {
    if (graph) cudaGraphDestroy(graph);
    return rc;
  }
  ROHM_CUDA(ctx, e);
  size_t n = 0;
  ROHM_CUDA(ctx, cudaGraphGetNodes(graph, nullptr, &n));
  std::vector<cudaGraphNode_t> nodes(n);
  ROHM_CUDA(ctx, cudaGraphGetNodes(graph, nodes.data(), &n));
  fg->B = B, fg->T = T, fg->graph = graph, fg->with_step = step != nullptr;
  for (cudaGraphNode_t node : nodes) {
    cudaGraphNodeType ty;
    ROHM_CUDA(ctx, cudaGraphNodeGetType(node, &ty));
    if (ty != cudaGraphNodeTypeKernel) continue;
    cudaKernelNodeParams kp{};
    ROHM_CUDA(ctx, cudaGraphKernelNodeGetParams(node, &kp));
    if (kp.func == reinterpret_cast<void*>(pack_tokens_kernel)) fg->n_pack = node, fg->p_pack = kp;
    else if (kp.func == reinterpret_cast<void*>(time_token_gather_kernel)) fg->n_time = node, fg->p_time = kp;
    else if (kp.func == reinterpret_cast<void*>(unpack_tokens_kernel)) fg->n_unpack = node, fg->p_unpack = kp;
    else if (kp.func == const_cast<void*>(ddpm_step_philox_kernel_address())) fg->n_step = node, fg->p_step = kp;
  }
  if (!fg->n_pack || !fg->n_time || !fg->n_unpack || (step != nullptr && !fg->n_step)) {
    cudaGraphDestroy(graph);
    fg->graph = nullptr;
    return fail(ctx, ROHM_ERR_CUDA, "forward graph: could not locate the boundary kernel nodes");
  }
  ROHM_CUDA(ctx, cudaGraphInstantiate(&fg->exec, graph, 0));
  return ROHM_OK;
}

static int forward_or_step(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B, int T,
                           void* stream, const StepArgs* step) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (x_t == nullptr || timesteps == nullptr || out == nullptr)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_forward: null pointer");
  if (B != pn->cond_B || T != pn->cond_T)
    return fail(ctx, ROHM_ERR_STATE, "rohm_posenet_forward: B=%d T=%d but set_cond was called with B=%d T=%d", B, T,
                pn->cond_B, pn->cond_T);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  ROHM_CUDA(ctx, cudaStreamIsCapturing(st, &cap));
  if (!pn->use_graph || pn->profiling || cap != cudaStreamCaptureStatusNone) {
    int rc = forward_launches(pn, x_t, timesteps, out, B, T, st);
    if (rc == ROHM_OK && step != nullptr) {
      const int64_t clip_elems = static_cast<int64_t>(pn->C) * T;
      ROHM_CUDA(ctx, launch_ddpm_step_philox(out, x_t, step->x_next, clip_elems * B, clip_elems, step->coef_row, step->seed,
                                             step->offset, step->G, step->iters, st, pn->use_pdl && !pn->profiling));
      pn->launches++;
    }
    return rc;
  }

  rohm_posenet::FwdGraph* fg = nullptr;
  for (auto& g : pn->graphs)
    if (g.B == B && g.T == T && g.with_step == (step != nullptr)) fg = &g;
  if (fg == nullptr) {
    rohm_posenet::FwdGraph ng;
    int rc = build_forward_graph(pn, x_t, timesteps, out, B, T, st, &ng, step);
    if (rc != ROHM_OK) return rc;
    if (pn->graphs.size() >= 8) {  // bounded cache
      if (pn->graphs.front().exec) cudaGraphExecDestroy(pn->graphs.front().exec);
      if (pn->graphs.front().graph) cudaGraphDestroy(pn->graphs.front().graph);
      pn->graphs.erase(pn->graphs.begin());
    }
    pn->graphs.push_back(ng);
    fg = &pn->graphs.back();
  }
  // patch the caller-memory pointers (argument 0 of pack / time-token, arguments 0.. of unpack: tok, cond, out)
  const void* a_x = x_t;
  const void* a_t = timesteps;
  void* a_o = out;
  {
    cudaKernelNodeParams kp = fg->p_pack;
    std::vector<void*> args(kp.kernelParams, kp.kernelParams + 8);
    args[0] = &a_x;
    kp.kernelParams = args.data();
    ROHM_CUDA(ctx, cudaGraphExecKernelNodeSetParams(fg->exec, fg->n_pack, &kp));
  }
  {
    cudaKernelNodeParams kp = fg->p_time;
    std::vector<void*> args(kp.kernelParams, kp.kernelParams + 11);
    args[0] = &a_t;
    kp.kernelParams = args.data();
    ROHM_CUDA(ctx, cudaGraphExecKernelNodeSetParams(fg->exec, fg->n_time, &kp));
  }
  {
    cudaKernelNodeParams kp = fg->p_unpack;
    std::vector<void*> args(kp.kernelParams, kp.kernelParams + 9);
    args[2] = &a_o;
    kp.kernelParams = args.data();
    ROHM_CUDA(ctx, cudaGraphExecKernelNodeSetParams(fg->exec, fg->n_unpack, &kp));
  }
  if (step != nullptr) {  // x0, x_t, out, coef row, Philox seed / offset of this step
    cudaKernelNodeParams kp = fg->p_step;
    std::vector<void*> args(kp.kernelParams, kp.kernelParams + 14);
    const void* a_x0 = out;
    void* a_next = step->x_next;
    const void* a_coef = step->coef_row;
    unsigned long long a_seed = step->seed, a_off = step->offset;
    args[0] = &a_x0, args[1] = &a_x, args[5] = &a_next, args[8] = &a_coef, args[10] = &a_seed, args[11] = &a_off;
    kp.kernelParams = args.data();
    ROHM_CUDA(ctx, cudaGraphExecKernelNodeSetParams(fg->exec, fg->n_step, &kp));
  }
  ROHM_CUDA(ctx, cudaGraphLaunch(fg->exec, st));
  return ROHM_OK;
}

extern "C" int rohm_posenet_forward(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B,
                                    int T, void* stream) {
  return forward_or_step(pn, x_t, timesteps, out, B, T, stream, nullptr);
}

extern "C" int rohm_posenet_sample_step(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* x0_out,
                                        float* x_next, const float* coef_row, uint64_t seed, uint64_t offset,
                                        uint64_t* offset_increment, int B, int T, void* stream) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  if (x_next == nullptr || coef_row == nullptr)
    return fail(pn->ctx, ROHM_ERR_INVALID, "rohm_posenet_sample_step: null pointer");
  StepArgs sa{x_next, coef_row, seed, offset, 0, 0};
  unsigned long long inc = 0;
  int rc = ddpm_step_philox_policy(pn->ctx, static_cast<int64_t>(pn->C) * T * B, &sa.G, &sa.iters, &inc);
  if (rc != ROHM_OK) return rc;
  if (offset_increment != nullptr) *offset_increment = inc;
  return forward_or_step(pn, x_t, timesteps, x0_out, B, T, stream, &sa);
}

extern "C" int rohm_posenet_set_option(rohm_posenet* pn, int option, int value) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  if (option == 0) {
    pn->use_graph = value != 0;
    return ROHM_OK;
  }
  if (option == 1) {  // programmatic dependent launch on the GEMMs (graphs are re-captured)
    pn->use_pdl = value != 0;
    for (auto& g : pn->graphs) {
      if (g.exec) cudaGraphExecDestroy(g.exec);
      if (g.graph) cudaGraphDestroy(g.graph);
    }
    pn->graphs.clear();
    return ROHM_OK;
  }
  return fail(pn->ctx, ROHM_ERR_INVALID, "rohm_posenet_set_option: unknown option %d", option);
}
