// GroupNorm + Mish behind TrajNet's GroupNorm'd convolutions (gn_mish_split_kernel, groupnorm.cu) and the per-element helpers
// it shares with the engine's other kernels (trajnet.cu).
//
// One thread-block cluster of n CTAs per (clip, group): each CTA holds a contiguous slice of the group's real rows in its own
// shared memory, and the group's statistics are reduced through distributed shared memory, so a group larger than one SM's
// shared memory still takes one pass over global memory.  n is chosen per convolution at engine creation
// (gn_pick_cluster): the smallest power of two whose slice fits the default 48 KB budget, so n = 1 wherever the group fits
// one CTA.  Batch-invariant engines (rohm_trajnet_create_batch_invariant) reduce each packed clip over the slices it would
// have alone (launch_gn_mish_clip_slices), so its statistics do not depend on the engine's T.
#pragma once
#include <cuda_runtime.h>

#include <cstddef>
#include <cstdint>

#include "ptx.cuh"

namespace rohm {

__device__ __forceinline__ float mish_f(float x) {
  const float sp = x > 20.0f ? x : log1pf(expf(x));
  return x * tanhf(sp);
}

constexpr int kMaxSplitsDev = 8;  // most K ranges a convolution is cut into (= kMaxSplits of the host-side choice)

// One float4 of an activation in its stored forms: fp32 and / or the hi/lo operand pair of the next convolution.
__device__ __forceinline__ void store_act4(float* out, float* out_hi, float* out_lo, int64_t idx, const float4& v, int f16) {
  if (out != nullptr) reinterpret_cast<float4*>(out)[idx] = v;
  if (out_hi != nullptr && f16) {
    uint2 h, l;
    ptx::split_f16x4(v, h, l);
    reinterpret_cast<uint2*>(out_hi)[idx] = h;
    reinterpret_cast<uint2*>(out_lo)[idx] = l;
  } else if (out_hi != nullptr) {
    float4 h, l;
    h.x = ptx::to_tf32(v.x), h.y = ptx::to_tf32(v.y), h.z = ptx::to_tf32(v.z), h.w = ptx::to_tf32(v.w);
    l.x = v.x - h.x, l.y = v.y - h.y, l.z = v.z - h.z, l.w = v.w - h.w;
    reinterpret_cast<float4*>(out_hi)[idx] = h;
    reinterpret_cast<float4*>(out_lo)[idx] = l;
  }
}

constexpr int kGnMaxCluster = 8;  // the portable cluster size limit

// One GroupNorm + Mish launch.  part: [splits][split_stride] floats, each a [B * Tp, C] matrix of the convolution without
// bias; out = Mish(GroupNorm(bias + partials)) [+ tp[b]] [+ r1] [+ r2] on the T real rows of each clip, 0 on its Tp - T pad
// rows, as fp32 (out) and / or the operand pair of the next convolution (out_hi / out_lo: fp16 when f16, else tf32).
// C / groups must be a multiple of 4.
struct GnArgs {
  const float* part;
  int splits;
  int64_t split_stride;
  const float* bias;
  const float* gamma;
  const float* beta;
  const float* tp;
  int tp_stride;
  const float* r1;
  const float* r2;
  float* out;
  float* out_hi;
  float* out_lo;
  int C, Tp, T, groups, f16;
};

// Dynamic shared memory of one CTA of an n-CTA cluster: ceil(T / n) rows of C / groups floats.
__host__ __device__ inline size_t gn_slice_bytes(int T, int C, int groups, int n) {
  return static_cast<size_t>((T + n - 1) / n) * static_cast<size_t>(C / groups) * sizeof(float);
}
// The kernel's dynamic shared-memory budget per CTA without raising its attribute (48 KB less its static shared memory),
// and the most it can be raised to on the current device.
cudaError_t gn_smem_budgets(size_t* default_budget, size_t* max_budget);
// Smallest power of two n <= kGnMaxCluster whose slice fits `budget`; kGnMaxCluster when none does.
__host__ __device__ inline int gn_pick_cluster(int T, int C, int groups, size_t budget) {
  for (int n = 1; n <= kGnMaxCluster; n *= 2)
    if (gn_slice_bytes(T, C, groups, n) <= budget) return n;
  return kGnMaxCluster;
}
// The slice budget of batch-invariant engines: a constant of the library, so a clip's slices follow from its own length
// alone (the default engines' budget, 48 KB less the kernel's static shared memory, is read from the device at creation).
// A little under 48 KB, so slices of fewer than 8 CTAs never need the raised shared-memory attribute.
constexpr size_t kGnClipBudget = 47 * 1024;
// Raises the kernel's dynamic shared-memory limit on the current device to at least `bytes` (never lowers it).
cudaError_t gn_reserve_smem(size_t bytes);
// Launches B x groups clusters of n CTAs (256 threads each), with programmatic dependent launch when pdl.  clip_off (device
// int[B + 1], or nullptr for clips at b * Tp): packed clips, clip b at rows [clip_off[b], clip_off[b + 1]) with its Tp - T
// pad rows last, so clip_off[b + 1] - clip_off[b] - (Tp - T) <= T real rows; statistics over those rows only.
cudaError_t launch_gn_mish(const GnArgs& a, int B, int n, cudaStream_t st, bool pdl, const int* clip_off = nullptr);
// The same launch of packed clips (clip_off required, n >= 2) in batch-invariant engines: clip b's statistics are reduced
// over v = gn_pick_cluster(its real rows, C, groups, kGnClipBudget) <= n slices, as a v-CTA cluster on that clip alone
// reduces them.  smem_bytes: the largest of those slices over the batch.
cudaError_t launch_gn_mish_clip_slices(const GnArgs& a, int B, int n, size_t smem_bytes, cudaStream_t st, bool pdl,
                                       const int* clip_off);

}  // namespace rohm
