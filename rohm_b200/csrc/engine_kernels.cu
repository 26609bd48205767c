// The engines' small per-row kernels: PoseNet's LayerNorm and LayerNorm folding, TrajNet's time path and split-K sum; see
// engine_kernels.cuh.
#include "common.h"
#include "engine_kernels.cuh"
#include "groupnorm.cuh"
#include "ptx.cuh"

namespace rohm {
namespace {

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

template <int D>
cudaError_t launch_ln(const float* in, const float* res, const float* g, const float* b, float* out, float* oh, float* ol,
                      int rows, cudaStream_t st, int f16, bool pdl) {
  return launch_chain(layernorm_kernel<D>, dim3((rows + 7) / 8), dim3(256), 0, st, pdl, in, res, g, b, out, oh, ol, rows,
                      f16);
}

// LayerNorm folding of a consumer GEMM y = LN(u) W^T + b, LN(u) = (u - mean) rstd gamma + beta:
//   Wf[n,k] = gamma_k W[n,k],  c_n = sum_k Wf[n,k],  d_n = b_n + sum_k beta_k W[n,k]      (one CTA per output row n)
__global__ void fold_ln_kernel(const float* __restrict__ W, const float* __restrict__ gamma, const float* __restrict__ beta,
                               const float* __restrict__ bias, int K, float* __restrict__ Wf, float* __restrict__ c,
                               float* __restrict__ d) {
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

// Timestep path of TrajNet (trajnet.py:120-125, 189) and the per-block time projections (heads.py:34-38, 51-52):
//   temb = W3 mish(W1 sinusoid(t) + b1) + b3;  tp[b, :] = Wcat mish(temb) + bcat   (all blocks' Linear(32,out) stacked)
__device__ __forceinline__ void trajnet_time_compute(float t, int b, int time_dim, const float* __restrict__ w1,
                                                     const float* __restrict__ b1, const float* __restrict__ w3,
                                                     const float* __restrict__ b3, const float* __restrict__ wcat,
                                                     const float* __restrict__ bcat, int total_out, float* __restrict__ tp,
                                                     float* sm) {
  float* e = sm;                  // [time_dim]
  float* h = e + time_dim;        // [4 * time_dim]
  float* m = h + 4 * time_dim;    // [time_dim]  mish(temb)
  const int half = time_dim / 2;
  if (threadIdx.x < half) {
    const float f = expf(static_cast<float>(threadIdx.x) * -(logf(10000.0f) / static_cast<float>(half - 1)));
    const float a = t * f;
    e[threadIdx.x] = sinf(a);
    e[half + threadIdx.x] = cosf(a);
  }
  __syncthreads();
  for (int n = threadIdx.x; n < 4 * time_dim; n += blockDim.x) {
    float acc = b1[n];
    for (int k = 0; k < time_dim; ++k) acc = fmaf(w1[n * time_dim + k], e[k], acc);
    h[n] = mish_f(acc);
  }
  __syncthreads();
  for (int n = threadIdx.x; n < time_dim; n += blockDim.x) {
    float acc = b3[n];
    for (int k = 0; k < 4 * time_dim; ++k) acc = fmaf(w3[n * 4 * time_dim + k], h[k], acc);
    m[n] = mish_f(acc);
  }
  __syncthreads();
  // the stacked projections are split over blockIdx.y (each CTA recomputes the small time MLP above)
  for (int n = blockIdx.y * blockDim.x + threadIdx.x; n < total_out; n += blockDim.x * gridDim.y) {
    float acc = bcat[n];
    for (int k = 0; k < time_dim; ++k) acc = fmaf(wcat[n * time_dim + k], m[k], acc);
    tp[static_cast<int64_t>(b) * total_out + n] = acc;
  }
}

// Split-K convolution without a GroupNorm behind it (the stride-2 downsampling convolutions): out = bias + the partials (in
// split order) on real rows, 0 on pad rows.  4 channels per thread over the [B * Tp, C] output.  kPacked: row r is real iff
// row_mask[r] != 0.
template <bool kPacked>
__global__ void __launch_bounds__(256) sum_split_kernel(const float* __restrict__ part, int splits, int64_t split_stride,
                                                        const float* __restrict__ bias, float* __restrict__ out,
                                                        float* __restrict__ out_hi, float* __restrict__ out_lo, int C, int Tp,
                                                        int T, int64_t total4, int f16,
                                                        const unsigned char* __restrict__ row_mask) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int c4 = C / 4;
  const int64_t row = i / c4;
  const int c = static_cast<int>(i - row * c4) * 4;
  const bool real = kPacked ? row_mask[row] != 0 : static_cast<int>(row % Tp) < T;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (real) {
    float4 a[kMaxSplitsDev];
#pragma unroll
    for (int sp = 0; sp < kMaxSplitsDev; ++sp)
      if (sp < splits) a[sp] = __ldcg(reinterpret_cast<const float4*>(part + sp * split_stride) + i);
    v = *reinterpret_cast<const float4*>(bias + c);
#pragma unroll
    for (int sp = 0; sp < kMaxSplitsDev; ++sp)
      if (sp < splits) v.x += a[sp].x, v.y += a[sp].y, v.z += a[sp].z, v.w += a[sp].w;
  }
  store_act4(out, out_hi, out_lo, i, v, f16);
}

}  // namespace

cudaError_t launch_layernorm(int D, const float* in, const float* res, const float* gamma, const float* beta, float* out,
                             float* out_hi, float* out_lo, int rows, int f16, cudaStream_t st, bool pdl) {
  switch (D) {
    case 128: return launch_ln<128>(in, res, gamma, beta, out, out_hi, out_lo, rows, st, f16, pdl);
    case 256: return launch_ln<256>(in, res, gamma, beta, out, out_hi, out_lo, rows, st, f16, pdl);
    case 512: return launch_ln<512>(in, res, gamma, beta, out, out_hi, out_lo, rows, st, f16, pdl);
    case 1024: return launch_ln<1024>(in, res, gamma, beta, out, out_hi, out_lo, rows, st, f16, pdl);
    default: return cudaErrorInvalidValue;
  }
}

cudaError_t launch_fold_ln(const float* W, const float* gamma, const float* beta, const float* bias, int N, int K, float* Wf,
                           float* c, float* d) {
  fold_ln_kernel<<<N, 256>>>(W, gamma, beta, bias, K, Wf, c, d);
  return cudaGetLastError();
}

// Per step the embedding depends on the (integer) timestep only, so the whole path is tabulated at create time for
// t in [0, table_rows) (the direct evaluation is latency-bound) and the per-forward kernel is a row
// gather; timesteps outside the table are evaluated directly.  `table` == nullptr: always evaluate (used to build the table).
__global__ void __launch_bounds__(256) trajnet_time_kernel(const int64_t* __restrict__ time, int time_dim,
                                                           const float* __restrict__ w1, const float* __restrict__ b1,
                                                           const float* __restrict__ w3, const float* __restrict__ b3,
                                                           const float* __restrict__ wcat, const float* __restrict__ bcat,
                                                           int total_out, float* __restrict__ tp,
                                                           const float* __restrict__ table, int table_rows) {
  extern __shared__ float sm[];
  const int b = blockIdx.x;
  const int64_t ti = time[b];
  if (table != nullptr && ti >= 0 && ti < table_rows) {  // block-uniform
    const float4* src = reinterpret_cast<const float4*>(table + ti * total_out);
    float4* dst = reinterpret_cast<float4*>(tp + static_cast<int64_t>(b) * total_out);
    for (int n = blockIdx.y * blockDim.x + threadIdx.x; n < total_out / 4; n += blockDim.x * gridDim.y) dst[n] = src[n];
    return;
  }
  trajnet_time_compute(static_cast<float>(ti), b, time_dim, w1, b1, w3, b3, wcat, bcat, total_out, tp, sm);
}

cudaError_t launch_sum_split(const float* part, int splits, int64_t split_stride, const float* bias, float* out,
                             float* out_hi, float* out_lo, int C, int Tp, int T, int64_t rows, int f16,
                             const unsigned char* row_mask, cudaStream_t st, bool pdl) {
  const int64_t total4 = rows * C / 4;
  return launch_chain(row_mask != nullptr ? sum_split_kernel<true> : sum_split_kernel<false>,
                      dim3(static_cast<unsigned>((total4 + 255) / 256)), dim3(256), 0, st, pdl, part, splits, split_stride,
                      bias, out, out_hi, out_lo, C, Tp, T, total4, f16, row_mask);
}

}  // namespace rohm
