// Sampler arithmetic: fused DDPM posterior step, q_sample, DDIM step.  HBM-bound elementwise kernels:
// 128-bit vectorised, grid sized as a multiple of the SM count, every product/sum individually rounded so the
// result is bit-identical to the reference's chain of separate elementwise ops
// (diffusion/gaussian_diffusion_posenet.py:212-234, 426-434, 461-479, 192-210, 696-715).
#include <curand_kernel.h>

#include <algorithm>
#include <cstdint>

#include "graph.cuh"

namespace rohm {
namespace {

constexpr int kThreads = 256;

__device__ __forceinline__ float ddpm_one(float x0, float xt, float nz, float g0, float g1, int n_grads, float c1,
                                          float c2, float sigma, float gs0, float gs1) {
  float mean = __fadd_rn(__fmul_rn(c1, x0), __fmul_rn(c2, xt));
  if (n_grads > 0) mean = __fadd_rn(mean, __fmul_rn(gs0, g0));
  if (n_grads > 1) mean = __fadd_rn(mean, __fmul_rn(gs1, g1));
  return __fadd_rn(mean, __fmul_rn(sigma, nz));
}

// grid = (chunks per clip, clips); each clip reads its own coefficient row.
template <bool kVec>
__global__ void __launch_bounds__(kThreads) ddpm_step_kernel(const float* __restrict__ x0, const float* x_t,
                                                             const float* __restrict__ noise,
                                                             const float* __restrict__ g0,
                                                             const float* __restrict__ g1, int n_grads, float* out,
                                                             int64_t clip_elems, const float* __restrict__ coef,
                                                             int64_t coef_stride) {
  const int64_t clip = blockIdx.y;
  const float* cf = coef + clip * coef_stride;
  const float c1 = cf[0], c2 = cf[1], sigma = cf[2], gs0 = cf[3], gs1 = cf[4];
  const int64_t base = clip * clip_elems;
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  const int64_t nthreads = static_cast<int64_t>(gridDim.x) * kThreads;
  if (kVec) {
    const int64_t n4 = clip_elems >> 2;  // host guarantees clip_elems % 4 == 0 and 16-byte aligned bases
    const float4* a4 = reinterpret_cast<const float4*>(x0 + base);
    const float4* b4 = reinterpret_cast<const float4*>(x_t + base);
    const float4* z4 = reinterpret_cast<const float4*>(noise + base);
    const float4* p4 = reinterpret_cast<const float4*>(n_grads > 0 ? g0 + base : x0 + base);
    const float4* q4 = reinterpret_cast<const float4*>(n_grads > 1 ? g1 + base : x0 + base);
    float4* o4 = reinterpret_cast<float4*>(out + base);
    for (int64_t i = tid; i < n4; i += nthreads) {
      const float4 a = a4[i], b = b4[i], z = z4[i];
      float4 p = make_float4(0.f, 0.f, 0.f, 0.f), q = p;
      if (n_grads > 0) p = p4[i];
      if (n_grads > 1) q = q4[i];
      float4 r;
      r.x = ddpm_one(a.x, b.x, z.x, p.x, q.x, n_grads, c1, c2, sigma, gs0, gs1);
      r.y = ddpm_one(a.y, b.y, z.y, p.y, q.y, n_grads, c1, c2, sigma, gs0, gs1);
      r.z = ddpm_one(a.z, b.z, z.z, p.z, q.z, n_grads, c1, c2, sigma, gs0, gs1);
      r.w = ddpm_one(a.w, b.w, z.w, p.w, q.w, n_grads, c1, c2, sigma, gs0, gs1);
      o4[i] = r;
    }
  } else {
    for (int64_t i = tid; i < clip_elems; i += nthreads) {
      const int64_t k = base + i;
      out[k] = ddpm_one(x0[k], x_t[k], noise[k], n_grads > 0 ? g0[k] : 0.f, n_grads > 1 ? g1[k] : 0.f, n_grads, c1, c2,
                        sigma, gs0, gs1);
    }
  }
}

__global__ void __launch_bounds__(kThreads) q_sample_kernel(const float* __restrict__ xs,
                                                            const float* __restrict__ noise, float* out, int64_t n,
                                                            float a, float b) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  const int64_t nthreads = static_cast<int64_t>(gridDim.x) * kThreads;
  for (int64_t i = tid; i < n; i += nthreads) out[i] = __fadd_rn(__fmul_rn(a, xs[i]), __fmul_rn(b, noise[i]));
}

__global__ void __launch_bounds__(kThreads) ddim_step_kernel(const float* __restrict__ x0, const float* x_t,
                                                             const float* __restrict__ noise, float* out, int64_t n,
                                                             float sr, float srm1, float sap, float dir, float sigma) {
  const int64_t tid = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  const int64_t nthreads = static_cast<int64_t>(gridDim.x) * kThreads;
  for (int64_t i = tid; i < n; i += nthreads) {
    const float eps = __fdiv_rn(__fsub_rn(__fmul_rn(sr, x_t[i]), x0[i]), srm1);
    const float mean = __fadd_rn(__fmul_rn(x0[i], sap), __fmul_rn(dir, eps));
    out[i] = __fadd_rn(mean, __fmul_rn(sigma, noise[i]));
  }
}

// The same update with the Gaussian noise drawn inside the kernel, bit-identical to what `torch.randn_like(x)` would have
// produced from the same generator state (ATen distribution_elementwise_grid_stride_kernel with curand_normal4, unroll 4):
// virtual thread `vidx` of torch's grid (G = grid * 256 threads) owns elements vidx + G * j; its j-th normal is component
// j % 4 of its (j / 4)-th curand_normal4 call on Philox4_32_10(seed, subsequence = vidx, offset).  One real thread per
// virtual thread, so the launch reads x0 / x_t and writes x_{t-1} once and the noise never touches memory.
__global__ void __launch_bounds__(kThreads) ddpm_step_philox_kernel(const float* __restrict__ x0, const float* x_t,
                                                                    const float* __restrict__ g0,
                                                                    const float* __restrict__ g1, int n_grads, float* out,
                                                                    int64_t numel, int64_t clip_elems,
                                                                    const float* __restrict__ coef, int64_t coef_stride,
                                                                    unsigned long long seed, unsigned long long offset,
                                                                    int64_t G, int iters) {
  // as the programmatic dependent of the denoiser's last kernel (posenet.cu): the Philox state is set up while that kernel
  // drains; x0 / x_t are read after it has completed.  A no-op for a plain launch.
  const int64_t vidx = static_cast<int64_t>(blockIdx.x) * kThreads + threadIdx.x;
  curandStatePhilox4_32_10_t state;
  if (vidx < G) curand_init(seed, static_cast<unsigned long long>(vidx), offset, &state);
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (vidx >= G) return;
  for (int k = 0; k < iters; ++k) {
    const float4 nz = curand_normal4(&state);
    const float z[4] = {nz.x, nz.y, nz.z, nz.w};
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const int64_t li = vidx + G * (4 * k + ii);
      if (li < numel) {
        const int64_t clip = li / clip_elems;
        const float* cf = coef + clip * coef_stride;
        out[li] = ddpm_one(x0[li], x_t[li], z[ii], n_grads > 0 ? g0[li] : 0.f, n_grads > 1 ? g1[li] : 0.f, n_grads, cf[0],
                           cf[1], cf[2], cf[3], cf[4]);
      }
    }
  }
}
// The arguments of ddpm_step_philox_kernel that change from step to step in a replayed graph (ddpm_step_patch)
constexpr size_t kStepX0 = 0, kStepXt = 1, kStepOut = 5, kStepCoef = 8, kStepSeed = 10, kStepOffset = 11;

// Per-clip noise streams (graph.cuh ClipPlan).  Block blockIdx.x belongs to the clip b with blk[b] <= blockIdx.x <
// blk[b + 1]; its threads are virtual threads vidx of torch's normal_ grid for that clip alone (G_b = 256 * its block count),
// so thread vidx draws curand_normal4 on Philox4_32_10(seed_b, subsequence = vidx, offset_b + draw * inc_b) and owns the
// clip-alone elements li = vidx + G_b * j, mapped to padded positions (c, t): li = c * n_b + t channel-major, li = t * C + c
// channels-last.  The same threads then write zeros to the clip's padded frames.  kUpdate: the value written is the DDPM
// update of ddpm_step_kernel with that noise (0-2 gradient terms, coefficient row shared or per clip); else the noise itself.
template <bool kUpdate>
__global__ void __launch_bounds__(kThreads) clip_noise_kernel(const float* __restrict__ x0, const float* x_t,
                                                              const float* __restrict__ g0, const float* __restrict__ g1,
                                                              int n_grads, float* out, const float* __restrict__ coef,
                                                              int64_t coef_stride,
                                                              const unsigned long long* __restrict__ streams,
                                                              unsigned long long draw, const __grid_constant__ ClipPlan plan) {
  const int bx = static_cast<int>(blockIdx.x);
  int b = 0, hi = plan.B;  // plan.blk[b] <= bx < plan.blk[hi]
  while (hi - b > 1) {
    const int mid = (b + hi) >> 1;
    if (plan.blk[mid] <= bx) b = mid;
    else hi = mid;
  }
  const int n = plan.n[b], C = plan.C, T = plan.T;
  const int64_t G = static_cast<int64_t>(plan.blk[b + 1] - plan.blk[b]) * kThreads;
  const int64_t vidx = static_cast<int64_t>(bx - plan.blk[b]) * kThreads + threadIdx.x;
  const int64_t numel = static_cast<int64_t>(C) * n;
  const int iters = static_cast<int>((numel - 1) / (G * 4) + 1);
  // as the programmatic dependent of the denoiser's last kernel: memory, the stream table included, is read after it completes
  asm volatile("griddepcontrol.wait;" ::: "memory");
  curandStatePhilox4_32_10_t state;
  curand_init(streams[2 * b], static_cast<unsigned long long>(vidx), streams[2 * b + 1] + draw * 4ull * iters, &state);
  float c1 = 0.f, c2 = 0.f, sigma = 0.f, gs0 = 0.f, gs1 = 0.f;
  if (kUpdate) {
    const float* cf = coef + b * coef_stride;
    c1 = cf[0], c2 = cf[1], sigma = cf[2], gs0 = cf[3], gs1 = cf[4];
  }
  const int64_t base = static_cast<int64_t>(b) * C * T;
  for (int k = 0; k < iters; ++k) {
    const float4 nz = curand_normal4(&state);
    const float z[4] = {nz.x, nz.y, nz.z, nz.w};
#pragma unroll
    for (int ii = 0; ii < 4; ++ii) {
      const int64_t li = vidx + G * (4 * k + ii);
      if (li < numel) {
        int64_t idx;
        if (plan.channels_last) {
          idx = base + li;  // t * C + c is also the offset inside the padded clip
        } else {
          const unsigned l = static_cast<unsigned>(li), c = l / static_cast<unsigned>(n);
          idx = base + static_cast<int64_t>(c) * T + (l - c * static_cast<unsigned>(n));
        }
        if (kUpdate)
          out[idx] = ddpm_one(x0[idx], x_t[idx], z[ii], n_grads > 0 ? g0[idx] : 0.f, n_grads > 1 ? g1[idx] : 0.f, n_grads, c1,
                              c2, sigma, gs0, gs1);
        else
          out[idx] = z[ii];
      }
    }
  }
  const int pad = T - n;
  const int64_t npad = static_cast<int64_t>(C) * pad;
  for (int64_t j = vidx; j < npad; j += G) {
    if (plan.channels_last) {
      out[base + static_cast<int64_t>(n) * C + j] = 0.f;
    } else {
      const int64_t c = j / pad;
      out[base + c * T + n + (j - c * pad)] = 0.f;
    }
  }
}
// The arguments of clip_noise_kernel<true> that change from step to step in a replayed graph (ddpm_clip_step_patch)
constexpr size_t kClipX0 = 0, kClipXt = 1, kClipOut = 5, kClipCoef = 6, kClipStreams = 8, kClipDraw = 9;

int grid_for(const rohm_ctx* ctx, int64_t work_items) {
  const int sms = ctx->sm_count > 0 ? ctx->sm_count : 132;
  int64_t blocks = (work_items + kThreads - 1) / kThreads;
  const int64_t cap = static_cast<int64_t>(sms) * 8;  // 8 resident CTAs of 256 threads per SM
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  return static_cast<int>(blocks);
}

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

}  // namespace
}  // namespace rohm

using namespace rohm;

extern "C" int rohm_ddpm_step(rohm_ctx* ctx, const float* x0, const float* x_t, const float* noise, const float* grad0,
                              const float* grad1, int n_grads, float* out, int64_t n_clips, int64_t clip_elems,
                              const float* coef, int64_t coef_clip_stride, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (n_clips < 0 || clip_elems < 0 || x0 == nullptr || x_t == nullptr || noise == nullptr || out == nullptr ||
      coef == nullptr || n_grads < 0 || n_grads > 2 || (n_grads > 0 && grad0 == nullptr) ||
      (n_grads > 1 && grad1 == nullptr) || n_clips > 65535)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_ddpm_step: bad arguments");
  if (n_clips == 0 || clip_elems == 0) return ROHM_OK;
  const bool vec = (clip_elems % 4 == 0) && aligned16(x0) && aligned16(x_t) && aligned16(noise) && aligned16(out) &&
                   (n_grads < 1 || aligned16(grad0)) && (n_grads < 2 || aligned16(grad1));
  const int sms = ctx->sm_count > 0 ? ctx->sm_count : 132;
  const int64_t items = vec ? clip_elems / 4 : clip_elems;
  int64_t bx = (items + kThreads - 1) / kThreads;
  const int64_t cap = (static_cast<int64_t>(sms) * 8 + n_clips - 1) / n_clips;  // ~8 resident CTAs per SM in total
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  dim3 grid(static_cast<unsigned>(bx), static_cast<unsigned>(n_clips));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (vec)
    ddpm_step_kernel<true><<<grid, kThreads, 0, st>>>(x0, x_t, noise, grad0, grad1, n_grads, out, clip_elems, coef,
                                                      coef_clip_stride);
  else
    ddpm_step_kernel<false><<<grid, kThreads, 0, st>>>(x0, x_t, noise, grad0, grad1, n_grads, out, clip_elems, coef,
                                                       coef_clip_stride);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

// Launch geometry of torch's normal_ kernel for `numel` fp32 elements on this device (ATen calc_execution_policy):
// G = virtual threads, iters = curand_normal4 calls per thread, *increment = what the generator's offset advances by.
static int torch_normal_policy(rohm_ctx* ctx, int64_t numel, int64_t* G, int* iters, unsigned long long* increment) {
  int threads_per_sm = 0;
  ROHM_CUDA(ctx, cudaDeviceGetAttribute(&threads_per_sm, cudaDevAttrMaxThreadsPerMultiProcessor, ctx->device));
  const int64_t blocks_per_sm = threads_per_sm / 256;
  int64_t grid = (numel + 255) / 256;
  const int64_t cap = static_cast<int64_t>(ctx->sm_count) * blocks_per_sm;
  if (grid > cap) grid = cap;
  *G = grid * 256;
  *iters = static_cast<int>((numel - 1) / (*G * 4) + 1);
  *increment = static_cast<unsigned long long>(*iters) * 4ull;
  return ROHM_OK;
}

extern "C" int rohm_ddpm_step_philox(rohm_ctx* ctx, const float* x0, const float* x_t, const float* grad0, const float* grad1,
                                     int n_grads, float* out, int64_t n_clips, int64_t clip_elems, const float* coef,
                                     int64_t coef_clip_stride, uint64_t seed, uint64_t offset, uint64_t* offset_increment,
                                     void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (n_clips < 0 || clip_elems < 0 || x0 == nullptr || x_t == nullptr || out == nullptr || coef == nullptr || n_grads < 0 ||
      n_grads > 2 || (n_grads > 0 && grad0 == nullptr) || (n_grads > 1 && grad1 == nullptr))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_ddpm_step_philox: bad arguments");
  const int64_t numel = n_clips * clip_elems;
  if (offset_increment != nullptr) *offset_increment = 0;
  if (numel == 0) return ROHM_OK;
  int64_t G = 0;
  int iters = 0;
  unsigned long long inc = 0;
  int rc = torch_normal_policy(ctx, numel, &G, &iters, &inc);
  if (rc != ROHM_OK) return rc;
  if (offset_increment != nullptr) *offset_increment = inc;
  ddpm_step_philox_kernel<<<static_cast<unsigned>(G / kThreads), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x0, x_t, grad0, grad1, n_grads, out, numel, clip_elems, coef, coef_clip_stride, seed, offset, G, iters);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

// The update the denoiser engines append to their forward (graph.cuh DdpmStep).
namespace rohm {
int ddpm_step_plan(rohm_ctx* ctx, DdpmStep* s, uint64_t* offset_increment) {
  unsigned long long inc = 0;
  const int rc = torch_normal_policy(ctx, s->numel, &s->G, &s->iters, &inc);
  if (rc != ROHM_OK) return rc;
  if (offset_increment != nullptr) *offset_increment = inc;
  return ROHM_OK;
}
int launch_ddpm_step(rohm_ctx* ctx, const DdpmStep& s, cudaStream_t st, bool pdl) {
  ROHM_CUDA(ctx, launch_chain(ddpm_step_philox_kernel, dim3(static_cast<unsigned>(s.G / kThreads)), dim3(kThreads), 0, st, pdl,
                              s.x0, s.x_t, nullptr, nullptr, 0, s.x_next, s.numel, s.clip_elems, s.coef_row, 0, s.seed,
                              s.offset, s.G, s.iters));
  return ROHM_OK;
}
KernelPatch ddpm_step_patch(const DdpmStep& s) {
  return {ddpm_step_philox_kernel, arg<kStepX0>(s.x0),         arg<kStepXt>(s.x_t),       arg<kStepOut>(s.x_next),
          arg<kStepCoef>(s.coef_row), arg<kStepSeed>(s.seed), arg<kStepOffset>(s.offset)};
}

int clip_plan(rohm_ctx* ctx, int B, int C, int T, bool channels_last, const int* lengths, ClipPlan* p, uint64_t* incs) {
  if (B < 1 || B > kMaxStreamClips || C < 1 || T < 1)
    return fail(ctx, ROHM_ERR_INVALID, "per-clip noise streams: B=%d (at most %d), C=%d, T=%d", B, kMaxStreamClips, C, T);
  // torch's normal_ grid (ATen calc_execution_policy, as torch_normal_policy): min(ceil(numel / 256), SMs * blocks per SM)
  int threads_per_sm = 0;
  ROHM_CUDA(ctx, cudaDeviceGetAttribute(&threads_per_sm, cudaDevAttrMaxThreadsPerMultiProcessor, ctx->device));
  const int64_t cap = static_cast<int64_t>(ctx->sm_count) * (threads_per_sm / 256);
  p->B = B, p->C = C, p->T = T, p->channels_last = channels_last ? 1 : 0;
  p->blk[0] = 0;
  for (int b = 0; b < B; ++b) {
    const int n = lengths != nullptr ? lengths[b] : T;
    if (n < 1 || n > T) return fail(ctx, ROHM_ERR_INVALID, "per-clip noise streams: lengths[%d] = %d outside [1, %d]", b, n, T);
    const int64_t numel = static_cast<int64_t>(C) * n;
    const int64_t grid = std::min((numel + kThreads - 1) / kThreads, cap);
    if (p->blk[b] + grid > INT32_MAX) return fail(ctx, ROHM_ERR_INVALID, "per-clip noise streams: grid too large");
    p->n[b] = n;
    p->blk[b + 1] = p->blk[b] + static_cast<int>(grid);
    if (incs != nullptr) incs[b] = 4ull * static_cast<uint64_t>((numel - 1) / (grid * kThreads * 4) + 1);
  }
  return ROHM_OK;
}
int launch_ddpm_clip_step(rohm_ctx* ctx, const DdpmClipStep& s, cudaStream_t st, bool pdl) {
  ROHM_CUDA(ctx, launch_chain(clip_noise_kernel<true>, dim3(static_cast<unsigned>(s.plan.blk[s.plan.B])), dim3(kThreads), 0,
                              st, pdl, s.x0, s.x_t, nullptr, nullptr, 0, s.x_next, s.coef_row, 0, s.streams, s.draw, s.plan));
  return ROHM_OK;
}
KernelPatch ddpm_clip_step_patch(const DdpmClipStep& s) {
  return {clip_noise_kernel<true>,      arg<kClipX0>(s.x0),           arg<kClipXt>(s.x_t),   arg<kClipOut>(s.x_next),
          arg<kClipCoef>(s.coef_row), arg<kClipStreams>(s.streams), arg<kClipDraw>(s.draw)};
}
}  // namespace rohm

extern "C" int rohm_randn_clips(rohm_ctx* ctx, float* out, int B, int C, int T, int channels_last, const int* lengths,
                                const uint64_t* streams, uint64_t draw, uint64_t* offset_increments, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (out == nullptr || streams == nullptr) return fail(ctx, ROHM_ERR_INVALID, "rohm_randn_clips: null pointer");
  ClipPlan plan;
  const int rc = clip_plan(ctx, B, C, T, channels_last != 0, lengths, &plan, offset_increments);
  if (rc != ROHM_OK) return rc;
  clip_noise_kernel<false><<<static_cast<unsigned>(plan.blk[B]), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      nullptr, nullptr, nullptr, nullptr, 0, out, nullptr, 0, reinterpret_cast<const unsigned long long*>(streams), draw, plan);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_ddpm_step_philox_clips(rohm_ctx* ctx, const float* x0, const float* x_t, const float* grad0,
                                           const float* grad1, int n_grads, float* out, int B, int C, int T,
                                           int channels_last, const int* lengths, const float* coef,
                                           int64_t coef_clip_stride, const uint64_t* streams, uint64_t draw,
                                           uint64_t* offset_increments, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (x0 == nullptr || x_t == nullptr || out == nullptr || coef == nullptr || streams == nullptr || n_grads < 0 ||
      n_grads > 2 || (n_grads > 0 && grad0 == nullptr) || (n_grads > 1 && grad1 == nullptr) || coef_clip_stride < 0)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_ddpm_step_philox_clips: bad arguments");
  ClipPlan plan;
  const int rc = clip_plan(ctx, B, C, T, channels_last != 0, lengths, &plan, offset_increments);
  if (rc != ROHM_OK) return rc;
  clip_noise_kernel<true><<<static_cast<unsigned>(plan.blk[B]), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x0, x_t, grad0, grad1, n_grads, out, coef, coef_clip_stride, reinterpret_cast<const unsigned long long*>(streams), draw,
      plan);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_q_sample(rohm_ctx* ctx, const float* x_start, const float* noise, float* out, int64_t n,
                             float sqrt_ac, float sqrt_one_minus_ac, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (n < 0 || x_start == nullptr || noise == nullptr || out == nullptr)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_q_sample: bad arguments");
  if (n == 0) return ROHM_OK;
  q_sample_kernel<<<grid_for(ctx, n), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(x_start, noise, out, n, sqrt_ac,
                                                                                       sqrt_one_minus_ac);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_ddim_step(rohm_ctx* ctx, const float* x0, const float* x_t, const float* noise, float* out,
                              int64_t n, float sqrt_recip_ac, float sqrt_recipm1_ac, float sqrt_ac_prev, float dir_coef,
                              float sigma, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (n < 0 || x0 == nullptr || x_t == nullptr || noise == nullptr || out == nullptr)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_ddim_step: bad arguments");
  if (n == 0) return ROHM_OK;
  ddim_step_kernel<<<grid_for(ctx, n), kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      x0, x_t, noise, out, n, sqrt_recip_ac, sqrt_recipm1_ac, sqrt_ac_prev, dir_coef, sigma);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}
