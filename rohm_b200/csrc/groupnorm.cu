// GroupNorm + Mish of TrajNet's GroupNorm'd convolutions as thread-block clusters; see groupnorm.cuh.
#include <cooperative_groups.h>

#include <algorithm>

#include "common.h"
#include "groupnorm.cuh"

namespace cg = cooperative_groups;

namespace rohm {
namespace {

// One cluster of n CTAs per (clip, group); CTA `rank` owns rows [rank * ceil(T / n), ...) of the group's T real rows (with
// clip_off: of the clip's own real rows, fewer than T for a short clip, in the slices sized for T).
// kCluster = false is the n = 1 instantiation (a plain launch): with n and rank compile-time constants it is the one-CTA
// kernel without any cluster code.  kPacked = false is the uniform-clip code (clip b at b * Tp, T real rows); kPacked = true
// reads clip b's first row and real-row count from clip_off.
// y = bias + the `splits` fp32 partials (added in split order: deterministic; an un-split convolution passes its output as the
// one partial) is formed once into shared memory while each CTA sums its slice in double; the CTAs' (s1, s2) are then added
// in rank order by every CTA through distributed shared memory, so all hold bit-identical statistics (n = 1: the CTA's own
// sums, nothing added).  Pad rows are written as zeros, spread over the cluster.
// kClipSlices (with kCluster and kPacked: the batch-invariant engines' instance): clip b's statistics are the reduction of
// v = gn_pick_cluster(Tc, C, groups, kGnClipBudget) slices, the cluster a clip of Tc real rows is launched with alone, whatever
// the launch's n >= v: CTA r < v sums virtual slice r exactly as rank r of a v-CTA cluster does, the slice sums are added in
// slice order, and CTAs r >= v hold no rows (they only write pad zeros).  With v = n it is the kPacked instance.
template <bool kCluster, bool kPacked, bool kClipSlices>
__device__ __forceinline__ void gn_mish_split(const float* __restrict__ part, int splits, int64_t split_stride,
                                              const float* __restrict__ bias, const float* __restrict__ gamma,
                                              const float* __restrict__ beta, const float* __restrict__ tp, int tp_stride,
                                              const float* __restrict__ r1, const float* __restrict__ r2,
                                              float* __restrict__ out, float* __restrict__ out_hi, float* __restrict__ out_lo,
                                              int C, int Tp, int T, int groups, int f16, const int* __restrict__ clip_off) {
  static_assert(!kClipSlices || (kCluster && kPacked), "virtual slices are a packed-cluster instance");
  extern __shared__ float4 gn_vals[];  // ceil(T / n) * (C / groups) / 4
  __shared__ double red[2][8];         // per-warp sums; then [0][0], [1][0]: this CTA's (s1, s2), read by the whole cluster
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  int n = 1, rank = 0;
  if constexpr (kCluster)
    n = static_cast<int>(cg::this_cluster().num_blocks()), rank = static_cast<int>(cg::this_cluster().block_rank());
  const unsigned bg = blockIdx.x / static_cast<unsigned>(n);  // unsigned, as blockIdx.x: n = 1 is the one-CTA code
  const int b = bg / groups, g = bg - b * groups;
  const int gs = C / groups, gs4 = gs / 4;
  // packed clips: clip b takes rows [clip_off[b], clip_off[b + 1]), the last Tp - T of them pad rows
  int Tc = T;
  int64_t clip0 = static_cast<int64_t>(b) * Tp;
  if constexpr (kPacked) clip0 = clip_off[b], Tc = clip_off[b + 1] - clip_off[b] - (Tp - T);
  int slices = n;  // the slices the statistics are reduced over
  if constexpr (kClipSlices) slices = gn_pick_cluster(Tc, C, groups, kGnClipBudget);
  const int rows = (Tc + slices - 1) / slices;
  const int t0 = rank * rows;                      // past Tc in trailing CTAs of a short group: their slice is empty
  const int n4 = (min(Tc, t0 + rows) - t0) * gs4;  // <= 0 for an empty slice
  const int c4 = C / 4;
  const int64_t row0 = clip0 + t0;
  double s1 = 0.0, s2 = 0.0;
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const int t = i / gs4;
    const int c = g * gs + (i - t * gs4) * 4;
    const int64_t idx = (row0 + t) * c4 + c / 4;
    // all partials of this float4 are requested before the first is used (one L2 round trip instead of `splits`); they are
    // still added in split order
    float4 a[kMaxSplitsDev];
#pragma unroll
    for (int sp = 0; sp < kMaxSplitsDev; ++sp)
      if (sp < splits) a[sp] = __ldcg(reinterpret_cast<const float4*>(part + sp * split_stride) + idx);
    float4 v = *reinterpret_cast<const float4*>(bias + c);
#pragma unroll
    for (int sp = 0; sp < kMaxSplitsDev; ++sp)
      if (sp < splits) v.x += a[sp].x, v.y += a[sp].y, v.z += a[sp].z, v.w += a[sp].w;
    gn_vals[i] = v;
    s1 += static_cast<double>(v.x) + static_cast<double>(v.y) + static_cast<double>(v.z) + static_cast<double>(v.w);
    s2 += static_cast<double>(v.x) * v.x + static_cast<double>(v.y) * v.y + static_cast<double>(v.z) * v.z +
          static_cast<double>(v.w) * v.w;
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s1 += __shfl_xor_sync(0xffffffffu, s1, off);
    s2 += __shfl_xor_sync(0xffffffffu, s2, off);
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) red[0][warp] = s1, red[1][warp] = s2;
  __syncthreads();
  s1 = 0.0, s2 = 0.0;
  for (int wv = 0; wv < static_cast<int>(blockDim.x >> 5); ++wv) s1 += red[0][wv], s2 += red[1][wv];
  if constexpr (kCluster) {
    cg::cluster_group cluster = cg::this_cluster();
    __syncthreads();  // every warp has read the per-warp sums
    if (threadIdx.x == 0) red[0][0] = s1, red[1][0] = s2;
    cluster.sync();   // every CTA's pair is written
    s1 = 0.0, s2 = 0.0;
    for (int r = 0; r < slices; ++r) {
      const double* peer = cluster.map_shared_rank(&red[0][0], r);
      s1 += peer[0], s2 += peer[8];
    }
    // this CTA is done reading its peers; its own pair must stay readable until every peer has arrived too (the wait is
    // at the end of the kernel)
    cluster.barrier_arrive();
  }
  const double cnt = static_cast<double>(gs) * static_cast<double>(Tc);
  const double mean = s1 / cnt;
  double var = s2 / cnt - mean * mean;
  var = var < 0.0 ? 0.0 : var;
  const float mu = static_cast<float>(mean);
  const float rstd = static_cast<float>(1.0 / sqrt(var + 1e-5));
  for (int i = threadIdx.x; i < n4; i += blockDim.x) {
    const int t = i / gs4;
    const int c = g * gs + (i - t * gs4) * 4;
    const int64_t idx = (row0 + t) * c4 + c / 4;
    const float4 x = gn_vals[i];
    const float4 ga = *reinterpret_cast<const float4*>(gamma + c);
    const float4 be = *reinterpret_cast<const float4*>(beta + c);
    float4 v;
    v.x = mish_f((x.x - mu) * rstd * ga.x + be.x);
    v.y = mish_f((x.y - mu) * rstd * ga.y + be.y);
    v.z = mish_f((x.z - mu) * rstd * ga.z + be.z);
    v.w = mish_f((x.w - mu) * rstd * ga.w + be.w);
    if (tp != nullptr) {
      const float4 a = *reinterpret_cast<const float4*>(tp + static_cast<int64_t>(b) * tp_stride + c);
      v.x += a.x, v.y += a.y, v.z += a.z, v.w += a.w;
    }
    if (r1 != nullptr) {
      const float4 a = reinterpret_cast<const float4*>(r1)[idx];
      v.x += a.x, v.y += a.y, v.z += a.z, v.w += a.w;
    }
    if (r2 != nullptr) {
      const float4 a = reinterpret_cast<const float4*>(r2)[idx];
      v.x += a.x, v.y += a.y, v.z += a.z, v.w += a.w;
    }
    store_act4(out, out_hi, out_lo, idx, v, f16);
  }
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  // pad rows: the next convolution's zero padding
  for (int i = rank * blockDim.x + threadIdx.x; i < (Tp - T) * gs4; i += n * blockDim.x) {
    const int t = Tc + i / gs4;
    const int c = g * gs + (i % gs4) * 4;
    store_act4(out, out_hi, out_lo, (clip0 + t) * c4 + c / 4, zero, f16);
  }
  if constexpr (kCluster) cg::this_cluster().barrier_wait();
}

template <bool kCluster, bool kPacked>
__global__ void __launch_bounds__(256) gn_mish_split_kernel(const float* __restrict__ part, int splits, int64_t split_stride,
                                                            const float* __restrict__ bias, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, const float* __restrict__ tp,
                                                            int tp_stride, const float* __restrict__ r1,
                                                            const float* __restrict__ r2, float* __restrict__ out,
                                                            float* __restrict__ out_hi, float* __restrict__ out_lo, int C, int Tp,
                                                            int T, int groups, int f16, const int* __restrict__ clip_off) {
  gn_mish_split<kCluster, kPacked, false>(part, splits, split_stride, bias, gamma, beta, tp, tp_stride, r1, r2, out, out_hi,
                                          out_lo, C, Tp, T, groups, f16, clip_off);
}

// The fifth instance: packed clips in clusters, each clip's statistics over the slices it has alone
__global__ void __launch_bounds__(256) gn_mish_split_clip_kernel(const float* __restrict__ part, int splits,
                                                                 int64_t split_stride, const float* __restrict__ bias,
                                                                 const float* __restrict__ gamma,
                                                                 const float* __restrict__ beta, const float* __restrict__ tp,
                                                                 int tp_stride, const float* __restrict__ r1,
                                                                 const float* __restrict__ r2, float* __restrict__ out,
                                                                 float* __restrict__ out_hi, float* __restrict__ out_lo, int C,
                                                                 int Tp, int T, int groups, int f16,
                                                                 const int* __restrict__ clip_off) {
  gn_mish_split<true, true, true>(part, splits, split_stride, bias, gamma, beta, tp, tp_stride, r1, r2, out, out_hi, out_lo, C,
                                  Tp, T, groups, f16, clip_off);
}

}  // namespace

cudaError_t gn_smem_budgets(size_t* default_budget, size_t* max_budget) {
  cudaFuncAttributes single{}, cluster{};
  cudaError_t e = cudaFuncGetAttributes(&single, gn_mish_split_kernel<false, false>);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&cluster, gn_mish_split_kernel<true, false>);
  if (e != cudaSuccess) return e;
  int dev = 0, optin = 0;
  if ((e = cudaGetDevice(&dev)) != cudaSuccess) return e;
  if ((e = cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev)) != cudaSuccess) return e;
  const size_t static_smem = std::max(single.sharedSizeBytes, cluster.sharedSizeBytes);
  *default_budget = 48 * 1024 - static_smem;
  *max_budget = static_cast<size_t>(optin) - static_smem;
  return cudaSuccess;
}

cudaError_t gn_reserve_smem(size_t bytes) {
  for (auto kern : {gn_mish_split_kernel<false, false>, gn_mish_split_kernel<true, false>, gn_mish_split_kernel<false, true>,
                    gn_mish_split_kernel<true, true>, gn_mish_split_clip_kernel}) {
    cudaFuncAttributes fa{};
    cudaError_t e = cudaFuncGetAttributes(&fa, kern);
    if (e == cudaSuccess && bytes > static_cast<size_t>(fa.maxDynamicSharedSizeBytes))
      e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(bytes));
    if (e != cudaSuccess) return e;
  }
  return cudaSuccess;
}

cudaError_t launch_gn_mish(const GnArgs& a, int B, int n, cudaStream_t st, bool pdl, const int* clip_off) {
  if (n < 1 || n > kGnMaxCluster || a.groups <= 0 || a.C % (4 * a.groups) != 0) return cudaErrorInvalidValue;
  auto kern = clip_off != nullptr ? (n == 1 ? gn_mish_split_kernel<false, true> : gn_mish_split_kernel<true, true>)
                                     : (n == 1 ? gn_mish_split_kernel<false, false> : gn_mish_split_kernel<true, false>);
  return launch_chain(kern, dim3(static_cast<unsigned>(B * a.groups * n)), dim3(256),
                      gn_slice_bytes(a.T, a.C, a.groups, n), st, ChainAttrs(pdl, static_cast<unsigned>(n)), a.part,
                      a.splits, a.split_stride, a.bias, a.gamma, a.beta, a.tp, a.tp_stride, a.r1, a.r2, a.out, a.out_hi,
                      a.out_lo, a.C, a.Tp, a.T, a.groups, a.f16, clip_off);
}

cudaError_t launch_gn_mish_clip_slices(const GnArgs& a, int B, int n, size_t smem_bytes, cudaStream_t st, bool pdl,
                                       const int* clip_off) {
  if (n < 2 || n > kGnMaxCluster || a.groups <= 0 || a.C % (4 * a.groups) != 0 || clip_off == nullptr)
    return cudaErrorInvalidValue;
  return launch_chain(gn_mish_split_clip_kernel, dim3(static_cast<unsigned>(B * a.groups * n)), dim3(256), smem_bytes, st,
                      ChainAttrs(pdl, static_cast<unsigned>(n)), a.part, a.splits, a.split_stride, a.bias, a.gamma, a.beta,
                      a.tp, a.tp_stride, a.r1, a.r2, a.out, a.out_hi, a.out_lo, a.C, a.Tp, a.T, a.groups, a.f16, clip_off);
}

}  // namespace rohm
