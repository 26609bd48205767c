// The small per-row kernels of the two denoiser engines (engine_kernels.cu): PoseNet's LayerNorm and LayerNorm folding
// (posenet.cu), TrajNet's time path and split-K sum (trajnet.cu).  Kept in a translation unit of their own, like the GroupNorm
// kernel (groupnorm.cuh), so that the kernel probe (tests/native) launches the same compiled code the engines run.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

namespace rohm {

// LayerNorm over the last dim D (eps 1e-5) of in + res (res = the residual stream, may be null), one warp per row and 8 rows
// per CTA; writes fp32 `out` and the hi/lo pair (fp16 when f16, else tf32) of every row.  `out` may alias `res` (each row is
// read completely before it is written).  D in {128, 256, 512, 1024}; any other D returns cudaErrorInvalidValue.
cudaError_t launch_layernorm(int D, const float* in, const float* res, const float* gamma, const float* beta, float* out,
                             float* out_hi, float* out_lo, int rows, int f16, cudaStream_t st, bool pdl);

// LayerNorm folding of a consumer GEMM y = LN(u) W^T + b, LN(u) = (u - mean) rstd gamma + beta (one CTA per output row n):
//   Wf[n,k] = gamma_k W[n,k],  c_n = sum_k Wf[n,k],  d_n = b_n + sum_k beta_k W[n,k]
// W, Wf: [N, K]; the sums are taken in double and rounded once.  Launched on the default stream.
cudaError_t launch_fold_ln(const float* W, const float* gamma, const float* beta, const float* bias, int N, int K, float* Wf,
                           float* c, float* d);

// TrajNet's timestep path (trajnet.py:120-125, 189) and the per-block time projections (heads.py:34-38, 51-52), one clip
// b = blockIdx.x per CTA row:
//   temb = W3 mish(W1 sinusoid(t) + b1) + b3;  tp[b, :] = Wcat mish(temb) + bcat   (all blocks' Linear(32,out) stacked)
// The stacked projections [total_out] are split over gridDim.y CTAs.  With a `table` ([table_rows, total_out], built by this
// kernel with table = nullptr), t in [0, table_rows) is a row gather and every other t is evaluated directly.  256 threads,
// 6 * time_dim floats of dynamic shared memory.
__global__ void __launch_bounds__(256) trajnet_time_kernel(const int64_t* __restrict__ time, int time_dim,
                                                           const float* __restrict__ w1, const float* __restrict__ b1,
                                                           const float* __restrict__ w3, const float* __restrict__ b3,
                                                           const float* __restrict__ wcat, const float* __restrict__ bcat,
                                                           int total_out, float* __restrict__ tp,
                                                           const float* __restrict__ table, int table_rows);
constexpr size_t kTrajnetTimeT = 0;  // the argument replaced on every replay of a cached forward graph

// Split-K convolution without a GroupNorm behind it (the stride-2 downsampling convolutions): out = bias + the `splits`
// partials (added in split order) on real rows, 0 on pad rows, as fp32 (out) and / or the operand pair of the next
// convolution (out_hi / out_lo: fp16 when f16, else tf32), over `rows` rows of C channels.  row_mask (device, one byte per
// row; packed clips): row r is real iff row_mask[r] != 0; nullptr: row r is real iff r % Tp < T.
cudaError_t launch_sum_split(const float* part, int splits, int64_t split_stride, const float* bias, float* out,
                             float* out_hi, float* out_lo, int C, int Tp, int T, int64_t rows, int f16,
                             const unsigned char* row_mask, cudaStream_t st, bool pdl);

}  // namespace rohm
