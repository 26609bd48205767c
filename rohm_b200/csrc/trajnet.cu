// TrajNet denoiser engine: RoHM's 1-D conv U-Net with the TrajControl side branch
// (reference model/trajnet.py:10-75 ControlNet.forward, :177-275 TrajNet.forward; blocks model/heads.py:20-106).
//
// Layout: every activation is a channels-last matrix [B * Tp_L, C] per pyramid level L (T_L = T / 2^L real frames
// per clip followed by Tp_L - T_L >= 2 all-zero rows, Tp_L = (T + 32) / 2^L).  In that layout
//   * Conv1d(k, pad k/2)        = k shifted reads of the same matrix: the zero rows between clips ARE the padding,
//   * channel concat [x, skip]  = two K-segments of one GEMM,
//   * Downsample (k3, stride 2) = the same with a row-stride-2 TMA descriptor,
//   * ConvTranspose (k4, s2)    = two GEMMs (even / odd output frames), 2 taps each, row-interleaved stores,
// so every convolution is one launch of the wgmma segmented-A GEMM (gemm.cu) and no im2col / concat / transpose
// buffer exists.  The convolutions of the deep pyramid levels are cut along K into 3-6 ranges (pick_split: 128-wide tiles x K
// ranges cover the SMs where 6-22 row tiles alone cannot); one kernel per GroupNorm'd convolution (gn_mish_split_kernel, a
// CTA per (clip, group)) adds bias + the fp32 partial(s) in split order, takes the group's statistics, applies GroupNorm + Mish
// (+ time projection, + residual, + TrajControl residual) and emits the hi/lo operand pair of the next convolution.  The
// step-invariant condition pyramid and control_zero_conv_0 run once per condition (set_cond).  rohm_trajnet_sample_step appends
// the in-kernel-noise sampler update to the forward graph.
#include <cmath>
#include <map>
#include <new>
#include <string>

#include "common.h"
#include "gemm.cuh"
#include "ptx.cuh"

namespace rohm {
namespace {

__device__ __forceinline__ float mish_f(float x) {
  const float sp = x > 20.0f ? x : log1pf(expf(x));
  return x * tanhf(sp);
}

// [B, T, C] channels-last API tensor -> padded-clip hi/lo rows (b * Tp + t), pitch ld.  Pad rows stay zero.
__global__ void pack_rows_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, int T,
                                 int Tp, int C, int ld, int64_t total, int f16) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % C);
  const int64_t bt = i / C;
  const int t = static_cast<int>(bt % T);
  const int64_t b = bt / T;
  const float v = x[i];
  const int64_t o = (b * Tp + t) * ld + c;
  if (f16) {
    ptx::split_f16(v, reinterpret_cast<__half*>(hi)[o], reinterpret_cast<__half*>(lo)[o]);
  } else {
    const float h = ptx::to_tf32(v);
    hi[o] = h;
    lo[o] = v - h;
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

// Split-K convolution without a GroupNorm behind it (the stride-2 downsampling convolutions): out = bias + the partials (in
// split order) on real rows, 0 on pad rows.  4 channels per thread over the [B * Tp, C] output.
__global__ void __launch_bounds__(256) sum_split_kernel(const float* __restrict__ part, int splits, int64_t split_stride,
                                                        const float* __restrict__ bias, float* __restrict__ out,
                                                        float* __restrict__ out_hi, float* __restrict__ out_lo, int C, int Tp,
                                                        int T, int64_t total4, int f16) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total4) return;
  const int c4 = C / 4;
  const int64_t row = i / c4;
  const int c = static_cast<int>(i - row * c4) * 4;
  const int t = static_cast<int>(row % Tp);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (t < T) {
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

// GroupNorm + Mish behind every GroupNorm'd convolution: one CTA per (clip, group).  y = bias + the `splits` fp32 partials
// (added in split order: deterministic; an un-split convolution passes its output as the one partial) of the group's
// T x (C / groups) real elements is formed once into shared memory, its mean / variance are reduced inside the CTA (the
// producing GEMM writes no statistics), then out = Mish(GroupNorm(y)) [+ tp] [+ r1] [+ r2]; pad rows are written as zeros.
// part: [splits][split_stride] floats, each a [B * Tp, C] matrix.  C / groups must be a multiple of 4 (float4 units).
__global__ void __launch_bounds__(256) gn_mish_split_kernel(const float* __restrict__ part, int splits, int64_t split_stride,
                                                            const float* __restrict__ bias, const float* __restrict__ gamma,
                                                            const float* __restrict__ beta, const float* __restrict__ tp,
                                                            int tp_stride, const float* __restrict__ r1,
                                                            const float* __restrict__ r2, float* __restrict__ out,
                                                            float* __restrict__ out_hi, float* __restrict__ out_lo, int C, int Tp,
                                                            int T, int groups, int f16) {
  extern __shared__ float4 gn_vals[];  // T * (C / groups) / 4
  __shared__ double red[2][8];
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  const int b = blockIdx.x / groups, g = blockIdx.x - b * groups;
  const int gs = C / groups, gs4 = gs / 4;
  const int n4 = T * gs4;
  const int c4 = C / 4;
  const int64_t row0 = static_cast<int64_t>(b) * Tp;
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
  const double n = static_cast<double>(gs) * static_cast<double>(T);
  const double mean = s1 / n;
  double var = s2 / n - mean * mean;
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
  for (int i = threadIdx.x; i < (Tp - T) * gs4; i += blockDim.x) {  // pad rows: the next convolution's zero padding
    const int t = T + i / gs4;
    const int c = g * gs + (i % gs4) * 4;
    store_act4(out, out_hi, out_lo, (row0 + t) * c4 + c / 4, zero, f16);
  }
}

// padded-clip rows [B * Tp, ld] -> compact [B, T, C]
__global__ void unpack_rows_kernel(const float* __restrict__ x, float* __restrict__ out, int T, int Tp, int C, int ld,
                                   int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % C);
  const int64_t bt = i / C;
  const int t = static_cast<int>(bt % T);
  const int64_t b = bt / T;
  out[i] = x[(b * Tp + t) * ld + c];
}

// One segment of a convolution weight -> columns [seg_off, seg_off + Cs) of the packed [Np, Ktot] hi/lo pair.
// conv:      w[co][src_off + c][tap]   (Conv1d weight [Cout, Cin, k])
// transposed: w[src_off + c][co][tap]  (ConvTranspose1d weight [Cin, Cout, k])
__global__ void pack_conv_segment_kernel(const float* __restrict__ w, float* __restrict__ hi, float* __restrict__ lo,
                                         int Cout, int Cin_total, int ks, int src_off, int Cs, int tap, int seg_off,
                                         int Ktot, int transposed, int f16, float scale) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(Cout) * Cs) return;
  const int co = static_cast<int>(i / Cs), c = static_cast<int>(i % Cs);
  const float v = transposed ? w[(static_cast<int64_t>(src_off + c) * Cout + co) * ks + tap]
                             : w[(static_cast<int64_t>(co) * Cin_total + src_off + c) * ks + tap];
  const int64_t o = static_cast<int64_t>(co) * Ktot + seg_off + c;
  if (f16) {
    ptx::split_f16(v * scale, reinterpret_cast<__half*>(hi)[o], reinterpret_cast<__half*>(lo)[o]);
  } else {
    const float h = ptx::to_tf32(v);
    hi[o] = h;
    lo[o] = v - h;
  }
}

constexpr int kLevels = 5;
constexpr int kTimeTableRows = 1024;  // timesteps whose time path is tabulated at create time (RoHM: 100 or 1000 steps)
constexpr int kGroups = 8;

struct Act {  // one activation tensor at pyramid level `level`
  float* f32 = nullptr;
  float* hi = nullptr;
  float* lo = nullptr;
  int C = 0, ld = 0, level = 0;
};

struct Conv {
  GemmParams g{};
  PackedWeight w;
  float* bias = nullptr;
  int level_out = 0;   // GEMM rows are the rows of this level (for transposed convs: the INPUT level)
  // GroupNorm'd convolutions store the GEMM result without bias in `partial`, and gn_mish_split_kernel adds bias, takes the
  // statistics and applies GroupNorm.  Split-K (deep pyramid levels): `splits` fp32 partial results of [split_rows, Cout]
  // each in the branch's partial scratch; otherwise the one partial is the convolution's own fp32 output.
  int splits = 1;
  float* partial = nullptr;
  int64_t split_rows = 0;
  bool sum_after = false;  // no GroupNorm behind it: sum_split_kernel writes `sum_out` right after the GEMM
  Act sum_out;
};

}  // namespace
}  // namespace rohm

using namespace rohm;

struct rohm_trajnet {
  rohm_ctx* ctx = nullptr;
  DevicePool pool;
  int time_dim = 32, cond_dim = 13, traj_dim = 13, mid = 512, control_dim = 272;
  bool control = false;
  int passes = 3;
  int kind = kKindTf32;  // operand element type of the convolution GEMMs (kKindF16 in ROHM_PRECISION_F16X2)
  int max_batch = 0, T = 0;
  int Tl[kLevels], Tp[kLevels];
  std::map<std::string, std::pair<const float*, int64_t>> sd;  // caller's tensors, valid during create only
  // time path
  float *w1 = nullptr, *b1 = nullptr, *w3 = nullptr, *b3 = nullptr, *wcat = nullptr, *bcat = nullptr, *tp = nullptr;
  float* time_table = nullptr;  // [kTimeTableRows, tp_total]: the stacked projections of every tabulated timestep
  int tp_total = 0;
  std::map<std::string, int> tp_off;  // block prefix -> offset in the stacked time projection
  // activations
  std::map<std::string, Act> acts;
  std::map<std::string, Conv> convs;
  std::map<std::string, std::pair<float*, float*>> norms;  // GroupNorm gamma/beta by conv-block prefix
  // RTB-internal scratch, one set per concurrently running branch (0: U-Net, 1: TrajControl)
  float *scratchY[2] = {nullptr, nullptr}, *scratchRes[2] = {nullptr, nullptr};
  Act scratchA[2];
  // Split-K partials of the GroupNorm'd convolutions (ROHM_B200_TRAJ_SPLITK=0 turns split-K off): kMaxSplits x the largest
  // 128-row-padded [rows, C] level matrix, per branch
  float* scratchSplit[2] = {nullptr, nullptr};
  bool use_splitk = true;
  // The forward is captured as a graph with parallel branches: the TrajControl branch next to the U-Net encoder, every
  // block's 1x1 residual convolution next to its conv1 -> GroupNorm -> conv2 chain.  None of these GEMMs fills the 132 SMs
  // (11 to 96 tiles), so running them side by side shortens the critical path at no cost.  ROHM_B200_TRAJ_PARALLEL=0: serial.
  bool parallel = true;
  cudaStream_t side[3] = {nullptr, nullptr, nullptr};  // 0: TrajControl branch, 1 / 2: residual convolutions of branch 0 / 1
  std::vector<cudaEvent_t> events;
  size_t ev_next = 0;
  cudaEvent_t time_ready = nullptr;     // recorded after the time kernel; each branch waits for it before its first GroupNorm
  bool time_pending[2] = {false, false};
  int cond_B = -1;
  int launches = 0;
  // CUDA graph of one forward per batch size
  struct FwdGraph {
    int B = 0;
    bool with_step = false;  // forward + Philox-fused ancestral update (rohm_trajnet_sample_step)
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t exec = nullptr;
    cudaGraphNode_t n_pack = nullptr, n_time = nullptr, n_unpack = nullptr, n_step = nullptr;
    cudaKernelNodeParams p_pack{}, p_time{}, p_unpack{}, p_step{};
  };
  std::vector<FwdGraph> graphs;
  bool use_graph = true;
  bool use_pdl = true;  // ROHM_B200_PDL / rohm_trajnet_set_option(1): programmatic dependent launch along the conv / GroupNorm chains
  cudaStream_t capture_stream = nullptr;
  void drop_graphs() {
    for (auto& g : graphs) {
      if (g.exec) cudaGraphExecDestroy(g.exec);
      if (g.graph) cudaGraphDestroy(g.graph);
    }
    graphs.clear();
  }
  ~rohm_trajnet() {
    if (capture_stream) cudaStreamDestroy(capture_stream);
    for (cudaStream_t q : side)
      if (q) cudaStreamDestroy(q);
    for (cudaEvent_t e : events) cudaEventDestroy(e);
    if (time_ready) cudaEventDestroy(time_ready);
    for (auto& g : graphs) {
      if (g.exec) cudaGraphExecDestroy(g.exec);
      if (g.graph) cudaGraphDestroy(g.graph);
    }
  }
};

namespace {

int64_t rows_of(const rohm_trajnet* tn, int level) { return static_cast<int64_t>(tn->max_batch) * tn->Tp[level]; }

const float* param(rohm_trajnet* tn, const std::string& key, int64_t expect_numel, int* rc) {
  auto it = tn->sd.find(key);
  if (it == tn->sd.end()) {
    *rc = fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: missing parameter '%s'", key.c_str());
    return nullptr;
  }
  if (expect_numel >= 0 && it->second.second != expect_numel) {
    *rc = fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: parameter '%s' has %lld elements, expected %lld",
               key.c_str(), static_cast<long long>(it->second.second), static_cast<long long>(expect_numel));
    return nullptr;
  }
  return it->second.first;
}

float* dev_copy(rohm_trajnet* tn, const float* src, int64_t n, int* rc) {
  float* d = tn->pool.floats(n);
  if (d == nullptr) {
    *rc = fail(tn->ctx, ROHM_ERR_CUDA, "alloc failed: %s", cudaGetErrorString(tn->pool.last_error()));
    return nullptr;
  }
  cudaError_t e = cudaMemcpy(d, src, static_cast<size_t>(n) * sizeof(float), cudaMemcpyDeviceToDevice);
  if (e != cudaSuccess) {
    *rc = fail(tn->ctx, ROHM_ERR_CUDA, "memcpy failed: %s", cudaGetErrorString(e));
    return nullptr;
  }
  return d;
}

// Allocates an activation (fp32 and/or hi/lo) at a level.
int make_act(rohm_trajnet* tn, const std::string& name, int C, int level, bool want_f32, bool want_split) {
  Act a;
  a.C = C, a.level = level, a.ld = static_cast<int>(round_up(C, tn->kind == kKindF16 ? 8 : 4));  // 16-byte row pitch
  const int64_t n = rows_of(tn, level) * a.ld;
  if (want_f32) a.f32 = tn->pool.floats(n);
  if (want_split) a.hi = tn->pool.floats(n), a.lo = tn->pool.floats(n);
  if ((want_f32 && !a.f32) || (want_split && (!a.hi || !a.lo)))
    return fail(tn->ctx, ROHM_ERR_CUDA, "activation alloc failed: %s", cudaGetErrorString(tn->pool.last_error()));
  tn->acts[name] = a;
  return ROHM_OK;
}

constexpr int kModelSms = 132;  // H100 SXM: the wave size of the tile-count models below

// Output-tile width of a convolution GEMM.  The deep pyramid levels have few 128-row tiles (11 at level 3 with 64 clips), so
// 128-wide tiles would leave most of the SMs idle; a narrower tile multiplies the tile count at a modest cost per tile
// (operand fill per 32 K-columns: 32 KB of A + BLOCK_N / 4 KB of B).  Choose the width that minimises waves x fill.
int pick_bn(int N, int64_t rows) {
  const int64_t m_tiles = (rows + kGemmBlockM - 1) / kGemmBlockM;
  int best = 0;
  double best_cost = 0.0;
  for (int bn : {128, 64, 32}) {
    if (bn > 32 && bn > N) continue;
    const int64_t tiles = m_tiles * ((N + bn - 1) / bn);
    const double cost = static_cast<double>((tiles + kModelSms - 1) / kModelSms) * (32.0 + bn / 4.0);
    if (best == 0 || cost < best_cost) best = bn, best_cost = cost;
  }
  return best;
}

// Split-K choice for a GroupNorm'd convolution (conv1 / conv2 of a ResidualTemporalBlock) with `stages` K blocks of `blk_cols`
// columns.  On the deep levels a tile's K loop (2560 to 5120 columns) is the whole launch: cutting it into S ranges lets
// 128-wide tiles (the cheapest per flop: the A stripe is read once per 128 columns) still cover the SMs.  Model, in us: one
// wave of work items costs (columns / S / 64) * t64(bn) + fixed launch / prologue / epilogue; the consumer reads S partials.
// The per-64-column times t64 and the fixed costs are estimates, not H100 measurements.
// Returns S (1 = keep the single-pass path and pick_bn's width); *bn_out is only written when S > 1.
constexpr int kMaxSplits = kMaxSplitsDev;
int pick_split(int N, int64_t rows, int stages, int blk_cols, int* bn_out, double extra_us = 0.0) {
  const double unit = blk_cols / 64.0;  // K blocks -> 64-column units of the model
  if (stages * unit < 16 || N % 32 != 0) return 1;
  const int64_t m_tiles = (rows + kGemmBlockM - 1) / kGemmBlockM;
  auto t64 = [](int bn) { return bn == 128 ? 0.60 : bn == 64 ? 0.42 : 0.41; };  // A-bound below 128 (estimate)
  const double t_fixed = 4.5, t_partial = 0.4;
  auto cost = [&](int bn, int S) {
    const int64_t items = m_tiles * ((N + bn - 1) / bn) * S;
    const int per = (stages + S - 1) / S;
    return static_cast<double>((items + kModelSms - 1) / kModelSms) * (per * unit * t64(bn) + t_fixed) + (S > 1 ? S * t_partial : 0.0);
  };
  const int bn1 = pick_bn(N, rows);
  const double base = cost(bn1, 1);
  int best_bn = bn1, best_S = 1;
  double best = base;
  for (int bn : {128, 64}) {
    if (bn > N || N % bn != 0) continue;
    for (int S = 2; S <= kMaxSplits; ++S) {
      const int per = (stages + S - 1) / S;
      if (per * unit < 4 || (S - 1) * per >= stages) continue;  // at least 256 columns per item, no empty range
      const double c = cost(bn, S);
      if (c < best) best = c, best_bn = bn, best_S = S;
    }
  }
  if (best_S == 1 || best + extra_us > 0.85 * base) return 1;  // not worth a second code path (extra_us: an added launch)
  *bn_out = best_bn;
  return best_S;
}

// Builds one convolution as a segmented GEMM.
//   kind 0: Conv1d(ks, stride, pad = ks/2 for stride 1, 1 for the stride-2 k3 downsample)
//   kind 1 / 2: even / odd output phase of ConvTranspose1d(k4, s2, p1) (GEMM rows = input level rows)
int make_conv(rohm_trajnet* tn, const std::string& name, const std::string& wkey, std::vector<const Act*> srcs, int Cout,
              int ks, int stride, int kind, const Act* out, bool with_stats) {
  int rc = ROHM_OK;
  int Cin = 0;
  for (auto* s : srcs) Cin += s->C;
  const float* w = param(tn, wkey + ".weight", static_cast<int64_t>(Cout) * Cin * ks, &rc);
  if (rc != ROHM_OK) return rc;
  const float* b = param(tn, wkey + ".bias", Cout, &rc);
  if (rc != ROHM_OK) return rc;
  Conv cv;
  // taps: (weight tap index, row shift)
  std::vector<std::pair<int, int>> taps;
  if (kind == 0) {
    const int pad = (stride == 2) ? 1 : ks / 2;
    for (int j = 0; j < ks; ++j) taps.push_back({j, j - pad});
  } else if (kind == 1) {  // out[2u] = W[1] x[u] + W[3] x[u-1]
    taps = {{1, 0}, {3, -1}};
  } else {  // out[2u+1] = W[0] x[u+1] + W[2] x[u]
    taps = {{0, 1}, {2, 0}};
  }
  const int nseg = static_cast<int>(taps.size() * srcs.size());
  if (nseg > kMaxSegs) return fail(tn->ctx, ROHM_ERR_INVALID, "conv '%s' needs %d segments", name.c_str(), nseg);
  const int kblk = gemm_block_k(tn->kind);  // every source's channels are padded to a whole K block (zero columns)
  int Ktot = 0;
  for (size_t i = 0; i < taps.size(); ++i)
    for (auto* s : srcs) Ktot += static_cast<int>(round_up(s->C, kblk));
  PackedWeight& pw = cv.w;
  pw.N = Cout, pw.K = Ktot, pw.Kp = Ktot;
  pw.block_n = pick_bn(Cout, rows_of(tn, (kind == 0) ? out->level : srcs[0]->level));
  const bool can_split = tn->use_splitk && kind == 0 && out->ld == Cout && Cout % 4 == 0;
  if (can_split && ((with_stats && stride == 1 && out->f32 != nullptr && out->hi == nullptr) || (!with_stats && ks > 1))) {
    int bn = pw.block_n;
    cv.splits = pick_split(Cout, rows_of(tn, out->level), Ktot / kblk, kblk, &bn, with_stats ? 0.0 : 4.0);
    if (cv.splits > 1) {
      pw.block_n = bn;
      if (!with_stats) cv.sum_after = true, cv.sum_out = *out;
    }
  }
  pw.Np = static_cast<int>(round_up(Cout, pw.block_n));
  pw.kind = tn->kind;
  pw.hi = static_cast<float*>(tn->pool.bytes(static_cast<int64_t>(pw.Np) * Ktot * gemm_elem_bytes(tn->kind)));
  pw.lo = static_cast<float*>(tn->pool.bytes(static_cast<int64_t>(pw.Np) * Ktot * gemm_elem_bytes(tn->kind)));
  if (!pw.hi || !pw.lo) return fail(tn->ctx, ROHM_ERR_CUDA, "weight alloc failed");
  if (tn->kind == kKindF16) ROHM_CUDA(tn->ctx, f16_weight_scale(w, static_cast<int64_t>(Cout) * Cin * ks, &pw.scale));
  cv.bias = dev_copy(tn, b, Cout, &rc);
  if (rc != ROHM_OK) return rc;

  GemmParams& g = cv.g;
  g = GemmParams{};
  int seg = 0, seg_off = 0;
  const int in_level = srcs[0]->level;
  for (auto& tap : taps) {
    int src_off = 0;
    for (auto* s : srcs) {
      if (s->level != in_level || s->hi == nullptr)
        return fail(tn->ctx, ROHM_ERR_INVALID, "conv '%s': bad source", name.c_str());
      const int Cs = s->C;
      const int64_t n = static_cast<int64_t>(Cout) * Cs;
      pack_conv_segment_kernel<<<static_cast<unsigned>((n + 255) / 256), 256>>>(w, pw.hi, pw.lo, Cout, Cin, ks, src_off,
                                                                              Cs, tap.first, seg_off, Ktot, kind != 0,
                                                                              tn->kind == kKindF16 ? 1 : 0, pw.scale);
      int e1 = make_tmap_2d(&g.a_hi[seg], s->hi, rows_of(tn, in_level), Cs, s->ld, kGemmBlockM, stride, tn->kind);
      int e2 = make_tmap_2d(&g.a_lo[seg], s->lo, rows_of(tn, in_level), Cs, s->ld, kGemmBlockM, stride, tn->kind);
      if (e1 || e2) return fail(tn->ctx, ROHM_ERR_CUDA, "tensor map failed for conv '%s' (%d, %d)", name.c_str(), e1, e2);
      g.seg_kblocks[seg] = static_cast<int>(round_up(Cs, kblk)) / kblk;
      g.seg_row_shift[seg] = tap.second;
      g.seg_row_mul[seg] = stride;
      seg_off += static_cast<int>(round_up(Cs, kblk));
      src_off += Cs;
      ++seg;
    }
  }
  ROHM_CUDA(tn->ctx, cudaGetLastError());
  g.num_segs = nseg;
  g.acc_scale = 1.0f / pw.scale;
  if (make_tmap_2d(&g.b_hi, pw.hi, pw.Np, Ktot, Ktot, pw.block_n, 1, tn->kind) ||
      make_tmap_2d(&g.b_lo, pw.lo, pw.Np, Ktot, Ktot, pw.block_n, 1, tn->kind))
    return fail(tn->ctx, ROHM_ERR_CUDA, "tensor map failed for weights of '%s'", name.c_str());
  g.bias = cv.bias;
  g.N = Cout;
  // GEMM rows: output level rows, except transposed convs whose rows are the input level's
  const int row_level = (kind == 0) ? out->level : in_level;
  cv.level_out = row_level;
  g.clip_rows = tn->Tp[row_level];
  g.clip_valid = tn->Tl[row_level];
  g.out_row_mul = (kind == 0) ? 1 : 2;
  g.out_row_add = (kind == 2) ? 1 : 0;
  if (out->f32) g.out = out->f32, g.ldo = out->ld;
  if (out->hi) g.out_hi = out->hi, g.out_lo = out->lo, g.lds = out->ld;
  if (cv.splits > 1) {
    // partial results instead of the block's fp32 scratch; bias / statistics / GroupNorm happen in gn_mish_split_kernel
    const int br = (name.rfind("controlnet.", 0) == 0 || name[0] == 'k') ? 1 : 0;  // TrajControl convolutions: "controlnet.*", "k*"
    cv.split_rows = static_cast<int64_t>(round_up(rows_of(tn, row_level), kGemmBlockM));
    cv.partial = tn->scratchSplit[br];
    g.out = cv.partial, g.ldo = Cout, g.out_hi = nullptr, g.out_lo = nullptr;
    g.bias = nullptr;
    g.k_splits = cv.splits;
    g.split_row_stride = static_cast<int>(cv.split_rows);
  } else if (with_stats) {
    // y = conv without bias; bias + statistics + GroupNorm in gn_mish_split_kernel (one "partial").  Every GroupNorm'd output
    // is an fp32-only [rows, Cout] scratch whose width is a multiple of 4 * kGroups (rohm_trajnet_create's mid_dim rule).
    cv.partial = out->f32;
    g.bias = nullptr;
  }
  // fp32-only or fp16-pair-only outputs with the identity row map leave through TMA bulk stores (the transposed-conv phases
  // and the few convolutions that write both forms keep the per-thread epilogue)
  if (gemm_enable_tma_store(&g, cv.splits > 1 ? cv.splits * cv.split_rows : rows_of(tn, row_level), tn->kind) != 0)
    return fail(tn->ctx, ROHM_ERR_CUDA, "store tensor map failed for conv '%s'", name.c_str());
  tn->convs[name] = cv;
  return ROHM_OK;
}

int load_norm(rohm_trajnet* tn, const std::string& block_prefix, int C) {
  int rc = ROHM_OK;
  const float* g = param(tn, block_prefix + "block.2.weight", C, &rc);
  if (rc != ROHM_OK) return rc;
  const float* b = param(tn, block_prefix + "block.2.bias", C, &rc);
  if (rc != ROHM_OK) return rc;
  float* dg = dev_copy(tn, g, C, &rc);
  if (rc != ROHM_OK) return rc;
  float* db = dev_copy(tn, b, C, &rc);
  if (rc != ROHM_OK) return rc;
  tn->norms[block_prefix] = {dg, db};
  return ROHM_OK;
}

// Declares the convolutions of a ResidualTemporalBlock named `p` (e.g. "diff_enc1.") reading `srcs`, writing `out`.
int make_rtb(rohm_trajnet* tn, const std::string& p, std::vector<const Act*> srcs, int Cout, int level) {
  int Cin = 0;
  for (auto* s : srcs) Cin += s->C;
  int rc;
  Act y;  // fp32 scratch view with this block's width
  const int br = p.rfind("controlnet.", 0) == 0 ? 1 : 0;
  y.f32 = tn->scratchY[br], y.C = Cout, y.ld = Cout, y.level = level;
  Act a1 = tn->scratchA[br];
  a1.C = Cout, a1.ld = Cout, a1.level = level;
  tn->acts[p + "#y"] = y;
  tn->acts[p + "#a1"] = a1;
  if ((rc = make_conv(tn, p + "c1", p + "blocks.0.block.0", srcs, Cout, 5, 1, 0, &tn->acts[p + "#y"], true)) != ROHM_OK) return rc;
  if ((rc = make_conv(tn, p + "c2", p + "blocks.1.block.0", {&tn->acts[p + "#a1"]}, Cout, 5, 1, 0, &tn->acts[p + "#y"], true)) != ROHM_OK) return rc;
  if ((rc = load_norm(tn, p + "blocks.0.", Cout)) != ROHM_OK) return rc;
  if ((rc = load_norm(tn, p + "blocks.1.", Cout)) != ROHM_OK) return rc;
  if (Cin != Cout) {
    Act r;
    r.f32 = tn->scratchRes[br], r.C = Cout, r.ld = Cout, r.level = level;
    tn->acts[p + "#res"] = r;
    if ((rc = make_conv(tn, p + "res", p + "residual_conv", srcs, Cout, 1, 1, 0, &tn->acts[p + "#res"], false)) != ROHM_OK) return rc;
  }
  return ROHM_OK;
}

int run_conv(rohm_trajnet* tn, const std::string& name, int B, cudaStream_t st) {
  auto it = tn->convs.find(name);
  if (it == tn->convs.end()) return fail(tn->ctx, ROHM_ERR_STATE, "unknown conv '%s'", name.c_str());
  Conv& cv = it->second;
  const int rows = B * tn->Tp[cv.level_out];
  cv.g.M = rows;
  // developer instrumentation: ROHM_B200_TRAJ_TS=<conv name>[,<conv name>...] prints CTA 0's %globaltimer stamps of that convolution's third
  // launch outside stream capture (use with ROHM_B200_GRAPH=0)
  unsigned long long* d_ts = nullptr;
  if (const char* want = getenv("ROHM_B200_TRAJ_TS")) {
    static std::map<std::string, int> ts_calls;
    cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(st, &cap);
    const bool listed = ("," + std::string(want) + ",").find("," + name + ",") != std::string::npos;  // comma-separated names
    if (listed && cap == cudaStreamCaptureStatusNone && ++ts_calls[name] == 3 &&
        cudaMalloc(&d_ts, 32 * sizeof(unsigned long long)) == cudaSuccess) {
      cudaMemset(d_ts, 0, 32 * sizeof(unsigned long long));
      cudaStreamSynchronize(st);
    }
  }
  GemmParams launch_params = cv.g;
  launch_params.debug_ts = d_ts;
  ROHM_CUDA(tn->ctx, launch_gemm(launch_params, rows, cv.w.N, cv.w.block_n, tn->passes, st, tn->use_pdl, tn->kind));
  tn->launches++;
  if (d_ts != nullptr) {
    unsigned long long h[32];
    cudaStreamSynchronize(st);
    cudaMemcpy(h, d_ts, sizeof h, cudaMemcpyDeviceToHost);
    cudaFree(d_ts);
    int iters = 0;
    for (int sgi = 0; sgi < cv.g.num_segs; ++sgi) iters += cv.g.seg_kblocks[sgi];
    fprintf(stderr, "conv %s (rows %d, N %d, block_n %d, %d K blocks, %d splits) CTA0 timeline (ns): setup %llu | first A tma %llu | "
            "first stage landed %llu | item0 mma issued %llu | item0 acc ready %llu | item0 epilogue done %llu | all mma issued %llu | "
            "last item drained %llu | stores done %llu | end %llu\n", name.c_str(), rows, cv.w.N, cv.w.block_n, iters, cv.splits,
            h[1] - h[0], h[2] - h[0], h[3] - h[0], h[4] - h[0], h[5] - h[0], h[6] - h[0], h[12] - h[0], h[13] - h[0], h[14] - h[0],
            h[7] - h[0]);
  }
  if (cv.sum_after) {
    const int C = cv.w.N;
    const int64_t total4 = static_cast<int64_t>(rows) * C / 4;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>((total4 + 255) / 256)), cfg.blockDim = dim3(256), cfg.stream = st;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr, cfg.numAttrs = tn->use_pdl ? 1 : 0;
    ROHM_CUDA(tn->ctx, cudaLaunchKernelEx(&cfg, sum_split_kernel, static_cast<const float*>(cv.partial), cv.splits,
                                          static_cast<int64_t>(cv.split_rows) * C, static_cast<const float*>(cv.bias),
                                          cv.sum_out.f32, cv.sum_out.hi, cv.sum_out.lo, C, tn->Tp[cv.level_out],
                                          tn->Tl[cv.level_out], total4, tn->kind == kKindF16 ? 1 : 0));
    tn->launches++;
  }
  return ROHM_OK;
}

// partial(s) + bias -> statistics -> GroupNorm / Mish of a GroupNorm'd convolution, one CTA per (clip, group)
int run_gn(rohm_trajnet* tn, const std::string& conv_name, const std::string& norm_prefix, int C, int level, int B,
           const float* tp, const float* r1, const float* r2, const Act* out, cudaStream_t st) {
  const Conv& cv = tn->convs[conv_name];
  auto nb = tn->norms[norm_prefix];
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(static_cast<unsigned>(B * kGroups)), cfg.blockDim = dim3(256), cfg.stream = st;
  cfg.dynamicSmemBytes = static_cast<size_t>(tn->Tl[level]) * (C / kGroups) * sizeof(float);
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr, cfg.numAttrs = tn->use_pdl ? 1 : 0;
  ROHM_CUDA(tn->ctx, cudaLaunchKernelEx(&cfg, gn_mish_split_kernel, static_cast<const float*>(cv.partial), cv.splits,
                                        static_cast<int64_t>(cv.split_rows) * C, static_cast<const float*>(cv.bias),
                                        static_cast<const float*>(nb.first), static_cast<const float*>(nb.second), tp,
                                        tn->tp_total, r1, r2, out->f32, out->hi, out->lo, C, tn->Tp[level], tn->Tl[level],
                                        kGroups, tn->kind == kKindF16 ? 1 : 0));
  tn->launches++;
  return ROHM_OK;
}

// Executes a ResidualTemporalBlock: out = Mish(GN(conv2(Mish(GN(conv1(x))) + time))) + res(x) [+ extra]
// fork: everything recorded on `from` so far happens-before what is launched on `to` afterwards (event record + wait; during
// stream capture this adds a graph edge)
int order_after(rohm_trajnet* tn, cudaStream_t from, cudaStream_t to) {
  if (from == to) return ROHM_OK;
  if (tn->ev_next == tn->events.size()) {
    cudaEvent_t e = nullptr;
    ROHM_CUDA(tn->ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    tn->events.push_back(e);
  }
  cudaEvent_t e = tn->events[tn->ev_next++];
  ROHM_CUDA(tn->ctx, cudaEventRecord(e, from));
  ROHM_CUDA(tn->ctx, cudaStreamWaitEvent(to, e, 0));
  return ROHM_OK;
}

int run_rtb(rohm_trajnet* tn, const std::string& p, const float* identity_res, const Act* out, const float* extra, int B,
            cudaStream_t st, cudaStream_t side = nullptr, int branch = 0) {
  int rc;
  const Act& y = tn->acts[p + "#y"];
  const Act& a1 = tn->acts[p + "#a1"];
  const int C = y.C, level = y.level;
  const bool has_res = tn->convs.count(p + "res") != 0;
  if (side == nullptr) side = st;
  if (has_res) {  // the 1x1 residual convolution only reads the block's input: run it next to the main chain
    if ((rc = order_after(tn, st, side)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, p + "res", B, side)) != ROHM_OK) return rc;
  }
  if ((rc = run_conv(tn, p + "c1", B, st)) != ROHM_OK) return rc;
  const float* tp = nullptr;
  auto t = tn->tp_off.find(p);
  if (t != tn->tp_off.end()) tp = tn->tp + t->second;
  if (tp != nullptr && tn->time_pending[branch]) {  // first use of the time projections on this branch
    ROHM_CUDA(tn->ctx, cudaStreamWaitEvent(st, tn->time_ready, 0));
    tn->time_pending[branch] = false;
  }
  if ((rc = run_gn(tn, p + "c1", p + "blocks.0.", C, level, B, tp, nullptr, nullptr, &a1, st)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, p + "c2", B, st)) != ROHM_OK) return rc;
  const float* res = identity_res;
  if (has_res) {
    if ((rc = order_after(tn, side, st)) != ROHM_OK) return rc;
    res = tn->acts[p + "#res"].f32;
  }
  return run_gn(tn, p + "c2", p + "blocks.1.", C, level, B, nullptr, res, extra, out, st);
}

}  // namespace

extern "C" int rohm_trajnet_create(rohm_ctx* ctx, int n_params, const char* const* names, const float* const* ptrs,
                                   const int64_t* numels, int time_dim, int cond_dim, int traj_feat_dim, int mid_dim,
                                   int trajcontrol, int control_cond_dim, int max_batch, int frames, int precision,
                                   rohm_trajnet** out) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (names == nullptr || ptrs == nullptr || numels == nullptr || out == nullptr || max_batch <= 0)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: bad arguments");
  if (frames <= 0 || frames % 16 != 0)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: frames (%d) must be a positive multiple of 16 (four "
                "stride-2 stages)", frames);
  // mid_dim: the narrowest GroupNorm'd convolution is mid_dim / 8 wide, and gn_mish_split_kernel needs each of its 8 groups
  // to be a whole number of float4s, i.e. a width that is a multiple of 32
  if (mid_dim <= 0 || mid_dim % 256 != 0 || time_dim % 2 != 0 || time_dim > 64)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: mid_dim (%d) must be a positive multiple of 256 (the GroupNorm "
                "groups of its mid_dim / 8-wide level need a multiple of 4 channels each), time_dim even and <= 64", mid_dim);
  if (precision != ROHM_PRECISION_TF32X3 && precision != ROHM_PRECISION_TF32 && precision != ROHM_PRECISION_F16X2)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: precision must be 3 (TF32x3), 2 (F16x2) or 1 (TF32)");
  ROHM_CUDA(ctx, gemm_init_attributes());
  rohm_trajnet* tn = new (std::nothrow) rohm_trajnet();
  if (tn == nullptr) return fail(ctx, ROHM_ERR_INVALID, "out of host memory");
  tn->ctx = ctx;
  tn->time_dim = time_dim, tn->cond_dim = cond_dim, tn->traj_dim = traj_feat_dim, tn->mid = mid_dim;
  tn->control = trajcontrol != 0, tn->control_dim = control_cond_dim, tn->passes = precision == ROHM_PRECISION_TF32 ? 1 : 3;
  tn->kind = precision == ROHM_PRECISION_F16X2 ? kKindF16 : kKindTf32;
  tn->max_batch = max_batch, tn->T = frames;
  for (int l = 0; l < kLevels; ++l) tn->Tl[l] = frames >> l, tn->Tp[l] = (frames + 32) >> l;
  for (int i = 0; i < n_params; ++i) tn->sd[names[i]] = {ptrs[i], numels[i]};
  const int m = mid_dim, td = time_dim;
  int rc = ROHM_OK;

#define TRY(expr)          \
  do {                     \
    rc = (expr);           \
    if (rc != ROHM_OK) {   \
      delete tn;           \
      return rc;           \
    }                      \
  } while (0)

  // ---- scratch ----
  int64_t max_elems = 0;
  {
    const int widths[kLevels] = {m / 8, m / 4, m / 2, m, 2 * m};
    for (int l = 0; l < kLevels; ++l) max_elems = std::max<int64_t>(max_elems, rows_of(tn, l) * widths[l]);
  }
  for (int br = 0; br < 2; ++br) {
    tn->scratchY[br] = tn->pool.floats(max_elems);
    tn->scratchRes[br] = tn->pool.floats(max_elems);
    tn->scratchA[br].hi = tn->pool.floats(max_elems);
    tn->scratchA[br].lo = tn->pool.floats(max_elems);
  }
  if (const char* env = getenv("ROHM_B200_TRAJ_PARALLEL")) tn->parallel = env[0] != '0';
  if (const char* env = getenv("ROHM_B200_TRAJ_SPLITK")) tn->use_splitk = env[0] != '0';
  if (tn->use_splitk) {
    int64_t max_padded = 0;
    const int widths[kLevels] = {m / 8, m / 4, m / 2, m, 2 * m};
    for (int l = 0; l < kLevels; ++l)
      max_padded = std::max<int64_t>(max_padded, static_cast<int64_t>(round_up(rows_of(tn, l), kGemmBlockM)) * widths[l]);
    for (int br = 0; br < 2; ++br) {
      tn->scratchSplit[br] = tn->pool.floats(kMaxSplits * max_padded);
      if (!tn->scratchSplit[br]) {
        delete tn;
        return fail(ctx, ROHM_ERR_CUDA, "split-K scratch alloc failed");
      }
    }
  }
  if (!tn->scratchY[1] || !tn->scratchRes[1] || !tn->scratchA[1].hi || !tn->scratchA[1].lo || !tn->scratchY[0] ||
      !tn->scratchRes[0] || !tn->scratchA[0].hi || !tn->scratchA[0].lo) {
    delete tn;
    return fail(ctx, ROHM_ERR_CUDA, "scratch alloc failed");
  }

  // ---- activations ----
  TRY(make_act(tn, "xin", traj_feat_dim, 0, false, true));
  TRY(make_act(tn, "cin", cond_dim, 0, false, true));
  const int enc_w[4] = {m / 8, m / 4, m / 2, m};
  for (int l = 0; l < 4; ++l) {
    const std::string L = std::to_string(l + 1);
    TRY(make_act(tn, "c" + L, enc_w[l], l, false, true));           // cond pyramid level (skip into the U-Net / control)
    if (l < 3) TRY(make_act(tn, "cd" + L, enc_w[l], l + 1, true, true));  // cond downsample (identity residual never needed, f32 for safety)
    TRY(make_act(tn, "d" + L, enc_w[l], l, false, true));           // U-Net encoder output (skip connection)
    TRY(make_act(tn, "e" + L, 2 * enc_w[l], l + 1, true, true));    // downsampled concat (identity residual of next RTB)
  }
  TRY(make_act(tn, "m1", m, 4, true, true));
  TRY(make_act(tn, "m2", m, 4, false, true));
  const int dec_w[4] = {32, m / 8, m / 4, m / 2};  // dec1..dec4 output widths
  for (int l = 3; l >= 0; --l) {
    const std::string L = std::to_string(l + 1);
    TRY(make_act(tn, "up" + L, (l == 3 ? m : dec_w[l + 1]), l, false, true));
    TRY(make_act(tn, "u" + L, dec_w[l], l, false, true));
  }
  TRY(make_act(tn, "f1", 32, 0, false, true));
  TRY(make_act(tn, "outp", traj_feat_dim, 0, true, false));
  if (tn->control) {
    TRY(make_act(tn, "kin", control_cond_dim, 0, false, true));
    TRY(make_act(tn, "k0", traj_feat_dim, 0, false, true));
    const int zw[4] = {32, m / 8, m / 4, m / 2};
    for (int l = 0; l < 4; ++l) {
      const std::string L = std::to_string(l + 1);
      TRY(make_act(tn, "k" + L, enc_w[l], l, false, true));
      TRY(make_act(tn, "z" + L, zw[l], l, true, false));
      TRY(make_act(tn, "ke" + L, 2 * enc_w[l], l + 1, true, true));
    }
    TRY(make_act(tn, "km1", m, 4, true, true));
    TRY(make_act(tn, "km2", m, 4, false, true));
    TRY(make_act(tn, "zm", m, 4, true, false));
  }
  auto A = [&](const std::string& n) { return &tn->acts[n]; };

  // ---- time path: stacked Linear(time_dim -> out) of every block with input_t ----
  {
    std::vector<std::pair<std::string, int>> blocks = {
        {"diff_enc1.", m / 8}, {"diff_enc2.", m / 4}, {"diff_enc3.", m / 2}, {"diff_enc4.", m},
        {"diff_mid_block1.", m}, {"diff_mid_block2.", m}, {"diff_dec4.", m / 2}, {"diff_dec3.", m / 4},
        {"diff_dec2.", m / 8}, {"diff_dec1.", 32}};
    if (tn->control) {
      blocks.insert(blocks.end(), {{"controlnet.control_enc1.", m / 8}, {"controlnet.control_enc2.", m / 4},
                                   {"controlnet.control_enc3.", m / 2}, {"controlnet.control_enc4.", m},
                                   {"controlnet.control_mid_block1.", m}, {"controlnet.control_mid_block2.", m}});
    }
    int total = 0;
    for (auto& b : blocks) tn->tp_off[b.first] = total, total += b.second;
    tn->tp_total = total;
    tn->wcat = tn->pool.floats(static_cast<int64_t>(total) * td);
    tn->bcat = tn->pool.floats(total);
    tn->tp = tn->pool.floats(static_cast<int64_t>(max_batch) * total);
    if (!tn->wcat || !tn->bcat || !tn->tp) {
      delete tn;
      return fail(ctx, ROHM_ERR_CUDA, "time projection alloc failed");
    }
    for (auto& b : blocks) {
      const float* w = param(tn, b.first + "time_mlp.1.weight", static_cast<int64_t>(b.second) * td, &rc);
      if (rc != ROHM_OK) { delete tn; return rc; }
      const float* bb = param(tn, b.first + "time_mlp.1.bias", b.second, &rc);
      if (rc != ROHM_OK) { delete tn; return rc; }
      const int off = tn->tp_off[b.first];
      cudaMemcpy(tn->wcat + static_cast<int64_t>(off) * td, w, sizeof(float) * b.second * td, cudaMemcpyDeviceToDevice);
      cudaMemcpy(tn->bcat + off, bb, sizeof(float) * b.second, cudaMemcpyDeviceToDevice);
    }
    const float* p1 = param(tn, "time_mlp.1.weight", static_cast<int64_t>(4) * td * td, &rc);
    if (rc != ROHM_OK) { delete tn; return rc; }
    tn->w1 = dev_copy(tn, p1, static_cast<int64_t>(4) * td * td, &rc);
    const float* p2 = param(tn, "time_mlp.1.bias", 4 * td, &rc);
    if (rc != ROHM_OK) { delete tn; return rc; }
    tn->b1 = dev_copy(tn, p2, 4 * td, &rc);
    const float* p3 = param(tn, "time_mlp.3.weight", static_cast<int64_t>(4) * td * td, &rc);
    if (rc != ROHM_OK) { delete tn; return rc; }
    tn->w3 = dev_copy(tn, p3, static_cast<int64_t>(4) * td * td, &rc);
    const float* p4 = param(tn, "time_mlp.3.bias", td, &rc);
    if (rc != ROHM_OK) { delete tn; return rc; }
    tn->b3 = dev_copy(tn, p4, td, &rc);
    if (rc != ROHM_OK) { delete tn; return rc; }
    // tabulate the whole time path for t = 0 .. kTimeTableRows-1 with the direct-evaluation branch of the kernel
    tn->time_table = tn->pool.floats(static_cast<int64_t>(kTimeTableRows) * total);
    std::vector<int64_t> ts(kTimeTableRows);
    for (int i = 0; i < kTimeTableRows; ++i) ts[i] = i;
    int64_t* d_ts = static_cast<int64_t*>(tn->pool.bytes(sizeof(int64_t) * kTimeTableRows));
    if (!tn->time_table || !d_ts) { delete tn; return fail(ctx, ROHM_ERR_CUDA, "time table alloc failed"); }
    cudaMemcpy(d_ts, ts.data(), sizeof(int64_t) * kTimeTableRows, cudaMemcpyHostToDevice);
    trajnet_time_kernel<<<dim3(kTimeTableRows, 8), 256, sizeof(float) * 6 * td>>>(d_ts, td, tn->w1, tn->b1, tn->w3, tn->b3, tn->wcat,
                                                                                tn->bcat, total, tn->time_table, nullptr, 0);
    if (cudaDeviceSynchronize() != cudaSuccess) { delete tn; return fail(ctx, ROHM_ERR_CUDA, "time table build failed"); }
  }

  // ---- convolutions ----
  // condition pyramid (trajnet.py:192-208): RTBs without time input
  TRY(make_rtb(tn, "cond_enc1.", {A("cin")}, m / 8, 0));
  TRY(make_conv(tn, "cond_down1", "cond_downsample1.conv", {A("c1")}, m / 8, 3, 2, 0, A("cd1"), false));
  TRY(make_rtb(tn, "cond_enc2.", {A("cd1")}, m / 4, 1));
  TRY(make_conv(tn, "cond_down2", "cond_downsample2.conv", {A("c2")}, m / 4, 3, 2, 0, A("cd2"), false));
  TRY(make_rtb(tn, "cond_enc3.", {A("cd2")}, m / 2, 2));
  TRY(make_conv(tn, "cond_down3", "cond_downsample3.conv", {A("c3")}, m / 2, 3, 2, 0, A("cd3"), false));
  TRY(make_rtb(tn, "cond_enc4.", {A("cd3")}, m, 3));
  // U-Net (trajnet.py:216-275)
  TRY(make_rtb(tn, "diff_enc1.", {A("xin")}, m / 8, 0));
  TRY(make_conv(tn, "diff_down1", "diff_downsample1.conv", {A("d1"), A("c1")}, m / 4, 3, 2, 0, A("e1"), false));
  TRY(make_rtb(tn, "diff_enc2.", {A("e1")}, m / 4, 1));
  TRY(make_conv(tn, "diff_down2", "diff_downsample2.conv", {A("d2"), A("c2")}, m / 2, 3, 2, 0, A("e2"), false));
  TRY(make_rtb(tn, "diff_enc3.", {A("e2")}, m / 2, 2));
  TRY(make_conv(tn, "diff_down3", "diff_downsample3.conv", {A("d3"), A("c3")}, m, 3, 2, 0, A("e3"), false));
  TRY(make_rtb(tn, "diff_enc4.", {A("e3")}, m, 3));
  TRY(make_conv(tn, "diff_down4", "diff_downsample4.conv", {A("d4"), A("c4")}, 2 * m, 3, 2, 0, A("e4"), false));
  TRY(make_rtb(tn, "diff_mid_block1.", {A("e4")}, m, 4));
  TRY(make_rtb(tn, "diff_mid_block2.", {A("m1")}, m, 4));
  TRY(make_conv(tn, "up4e", "diff_upsample4.conv", {A("m2")}, m, 4, 1, 1, A("up4"), false));
  TRY(make_conv(tn, "up4o", "diff_upsample4.conv", {A("m2")}, m, 4, 1, 2, A("up4"), false));
  TRY(make_rtb(tn, "diff_dec4.", {A("up4"), A("d4")}, m / 2, 3));
  TRY(make_conv(tn, "up3e", "diff_upsample3.conv", {A("u4")}, m / 2, 4, 1, 1, A("up3"), false));
  TRY(make_conv(tn, "up3o", "diff_upsample3.conv", {A("u4")}, m / 2, 4, 1, 2, A("up3"), false));
  TRY(make_rtb(tn, "diff_dec3.", {A("up3"), A("d3")}, m / 4, 2));
  TRY(make_conv(tn, "up2e", "diff_upsample2.conv", {A("u3")}, m / 4, 4, 1, 1, A("up2"), false));
  TRY(make_conv(tn, "up2o", "diff_upsample2.conv", {A("u3")}, m / 4, 4, 1, 2, A("up2"), false));
  TRY(make_rtb(tn, "diff_dec2.", {A("up2"), A("d2")}, m / 8, 1));
  TRY(make_conv(tn, "up1e", "diff_upsample1.conv", {A("u2")}, m / 8, 4, 1, 1, A("up1"), false));
  TRY(make_conv(tn, "up1o", "diff_upsample1.conv", {A("u2")}, m / 8, 4, 1, 2, A("up1"), false));
  TRY(make_rtb(tn, "diff_dec1.", {A("up1"), A("d1")}, 32, 0));
  {
    Act y;
    y.f32 = tn->scratchY[0], y.C = 32, y.ld = 32, y.level = 0;
    tn->acts["final#y"] = y;
    TRY(make_conv(tn, "final_c", "diff_final_conv.0.block.0", {A("u1")}, 32, 5, 1, 0, A("final#y"), true));
    TRY(load_norm(tn, "diff_final_conv.0.", 32));
    TRY(make_conv(tn, "final_o", "diff_final_conv.1", {A("f1")}, traj_feat_dim, 1, 1, 0, A("outp"), false));
  }
  if (tn->control) {  // trajnet.py:43-75
    const std::string c = "controlnet.";
    TRY(make_conv(tn, "kz0", c + "control_zero_conv_0", {A("kin")}, traj_feat_dim, 1, 1, 0, A("k0"), false));
    TRY(make_rtb(tn, c + "control_enc1.", {A("k0")}, m / 8, 0));
    TRY(make_conv(tn, "kz1", c + "control_zero_conv_1", {A("k1")}, 32, 1, 1, 0, A("z1"), false));
    TRY(make_conv(tn, "kd1", c + "control_downsample1.conv", {A("k1"), A("c1")}, m / 4, 3, 2, 0, A("ke1"), false));
    TRY(make_rtb(tn, c + "control_enc2.", {A("ke1")}, m / 4, 1));
    TRY(make_conv(tn, "kz2", c + "control_zero_conv_2", {A("k2")}, m / 8, 1, 1, 0, A("z2"), false));
    TRY(make_conv(tn, "kd2", c + "control_downsample2.conv", {A("k2"), A("c2")}, m / 2, 3, 2, 0, A("ke2"), false));
    TRY(make_rtb(tn, c + "control_enc3.", {A("ke2")}, m / 2, 2));
    TRY(make_conv(tn, "kz3", c + "control_zero_conv_3", {A("k3")}, m / 4, 1, 1, 0, A("z3"), false));
    TRY(make_conv(tn, "kd3", c + "control_downsample3.conv", {A("k3"), A("c3")}, m, 3, 2, 0, A("ke3"), false));
    TRY(make_rtb(tn, c + "control_enc4.", {A("ke3")}, m, 3));
    TRY(make_conv(tn, "kz4", c + "control_zero_conv_4", {A("k4")}, m / 2, 1, 1, 0, A("z4"), false));
    TRY(make_conv(tn, "kd4", c + "control_downsample4.conv", {A("k4"), A("c4")}, 2 * m, 3, 2, 0, A("ke4"), false));
    TRY(make_rtb(tn, c + "control_mid_block1.", {A("ke4")}, m, 4));
    TRY(make_rtb(tn, c + "control_mid_block2.", {A("km1")}, m, 4));
    TRY(make_conv(tn, "kzm", c + "control_zero_conv_mid", {A("km2")}, m, 1, 1, 0, A("zm"), false));
  }
#undef TRY
  cudaError_t e = cudaDeviceSynchronize();
  tn->sd.clear();
  if (e != cudaSuccess) {
    delete tn;
    return fail(ctx, ROHM_ERR_CUDA, "weight packing failed: %s", cudaGetErrorString(e));
  }
  *out = tn;
  return ROHM_OK;
}

extern "C" void rohm_trajnet_destroy(rohm_trajnet* tn) { delete tn; }

extern "C" int rohm_trajnet_launches_per_forward(const rohm_trajnet* tn) { return tn ? tn->launches : 0; }

static int trajnet_pack(rohm_trajnet* tn, const float* x, const Act& a, int B, cudaStream_t st) {
  const int64_t total = static_cast<int64_t>(B) * tn->T * a.C;
  pack_rows_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(x, a.hi, a.lo, tn->T, tn->Tp[0], a.C, a.ld,
                                                                             total, tn->kind == kKindF16 ? 1 : 0);
  ROHM_CUDA(tn->ctx, cudaGetLastError());
  tn->launches++;
  return ROHM_OK;
}

// Step-invariant part: the condition pyramid (and control_zero_conv_0).  cond: [B, T, cond_dim];
// control_cond: [B, T, control_cond_dim] or NULL for the vanilla network.
extern "C" int rohm_trajnet_set_cond(rohm_trajnet* tn, const float* cond, const float* control_cond, int B, void* stream) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = tn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (cond == nullptr || B <= 0 || B > tn->max_batch || (tn->control && control_cond == nullptr))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_set_cond: bad arguments (B=%d, capacity %d)", B, tn->max_batch);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  int rc;
  const int saved = tn->launches;
  if ((rc = trajnet_pack(tn, cond, tn->acts["cin"], B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "cond_enc1.", nullptr, &tn->acts["c1"], nullptr, B, st)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "cond_down1", B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "cond_enc2.", nullptr, &tn->acts["c2"], nullptr, B, st)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "cond_down2", B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "cond_enc3.", nullptr, &tn->acts["c3"], nullptr, B, st)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "cond_down3", B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "cond_enc4.", nullptr, &tn->acts["c4"], nullptr, B, st)) != ROHM_OK) return rc;
  if (tn->control) {
    if ((rc = trajnet_pack(tn, control_cond, tn->acts["kin"], B, st)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kz0", B, st)) != ROHM_OK) return rc;
  }
  tn->launches = saved;
  tn->cond_B = B;
  return ROHM_OK;
}

static int trajnet_forward_launches(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* out, int B,
                                    cudaStream_t st) {
  rohm_ctx* ctx = tn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  int rc;
  tn->launches = 0;
  auto A = [&](const char* n) { return &tn->acts[n]; };
  if ((rc = trajnet_pack(tn, x_t, *A("xin"), B, st)) != ROHM_OK) return rc;
  const int td = tn->time_dim;
  trajnet_time_kernel<<<dim3(B, 8), 256, sizeof(float) * 6 * td, st>>>(time, td, tn->w1, tn->b1, tn->w3, tn->b3, tn->wcat, tn->bcat,
                                                            tn->tp_total, tn->tp, tn->time_table, kTimeTableRows);
  ROHM_CUDA(ctx, cudaGetLastError());
  tn->launches++;

  // Parallel branches (see rohm_trajnet::parallel): sC carries the TrajControl branch, r0 / r1 the residual 1x1 convolutions
  // (and the odd phases of the transposed convolutions) of the U-Net / TrajControl blocks.
  tn->ev_next = 0;
  if (tn->parallel)
    for (cudaStream_t& q : tn->side)
      if (q == nullptr) ROHM_CUDA(ctx, cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));
  cudaStream_t sC = (tn->parallel && tn->control) ? tn->side[0] : st;
  cudaStream_t r0 = tn->parallel ? tn->side[1] : st;
  cudaStream_t r1 = tn->parallel ? tn->side[2] : sC;
  if (tn->control) {
    const std::string c = "controlnet.";
    if ((rc = order_after(tn, st, sC)) != ROHM_OK) return rc;  // fork after pack + time
    if ((rc = run_rtb(tn, c + "control_enc1.", nullptr, A("k1"), nullptr, B, sC, r1, 1)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kz1", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kd1", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_rtb(tn, c + "control_enc2.", A("ke1")->f32, A("k2"), nullptr, B, sC, r1, 1)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kz2", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kd2", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_rtb(tn, c + "control_enc3.", A("ke2")->f32, A("k3"), nullptr, B, sC, r1, 1)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kz3", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kd3", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_rtb(tn, c + "control_enc4.", A("ke3")->f32, A("k4"), nullptr, B, sC, r1, 1)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kz4", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kd4", B, sC)) != ROHM_OK) return rc;
    if ((rc = run_rtb(tn, c + "control_mid_block1.", nullptr, A("km1"), nullptr, B, sC, r1, 1)) != ROHM_OK) return rc;
    if ((rc = run_rtb(tn, c + "control_mid_block2.", A("km1")->f32, A("km2"), nullptr, B, sC, r1, 1)) != ROHM_OK) return rc;
    if ((rc = run_conv(tn, "kzm", B, sC)) != ROHM_OK) return rc;
  }
  const float* z1 = tn->control ? A("z1")->f32 : nullptr;
  const float* z2 = tn->control ? A("z2")->f32 : nullptr;
  const float* z3 = tn->control ? A("z3")->f32 : nullptr;
  const float* z4 = tn->control ? A("z4")->f32 : nullptr;
  const float* zm = tn->control ? A("zm")->f32 : nullptr;

  if ((rc = run_rtb(tn, "diff_enc1.", nullptr, A("d1"), nullptr, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "diff_down1", B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_enc2.", A("e1")->f32, A("d2"), nullptr, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "diff_down2", B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_enc3.", A("e2")->f32, A("d3"), nullptr, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "diff_down3", B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_enc4.", A("e3")->f32, A("d4"), nullptr, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "diff_down4", B, st)) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_mid_block1.", nullptr, A("m1"), nullptr, B, st, r0, 0)) != ROHM_OK) return rc;
  if (tn->control && (rc = order_after(tn, sC, st)) != ROHM_OK) return rc;  // join: the decoder adds the TrajControl residuals
  if ((rc = run_rtb(tn, "diff_mid_block2.", A("m1")->f32, A("m2"), zm, B, st, r0, 0)) != ROHM_OK) return rc;
  // ConvTranspose1d = two independent GEMMs (even / odd output frames) with row-interleaved stores
  auto upsample = [&](const char* even, const char* odd) -> int {
    int r;
    if ((r = order_after(tn, st, r0)) != ROHM_OK) return r;
    if ((r = run_conv(tn, odd, B, r0)) != ROHM_OK) return r;
    if ((r = run_conv(tn, even, B, st)) != ROHM_OK) return r;
    return order_after(tn, r0, st);
  };
  if ((rc = upsample("up4e", "up4o")) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_dec4.", nullptr, A("u4"), z4, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = upsample("up3e", "up3o")) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_dec3.", nullptr, A("u3"), z3, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = upsample("up2e", "up2o")) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_dec2.", nullptr, A("u2"), z2, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = upsample("up1e", "up1o")) != ROHM_OK) return rc;
  if ((rc = run_rtb(tn, "diff_dec1.", nullptr, A("u1"), z1, B, st, r0, 0)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "final_c", B, st)) != ROHM_OK) return rc;
  if ((rc = run_gn(tn, "final_c", "diff_final_conv.0.", 32, 0, B, nullptr, nullptr, nullptr, A("f1"), st)) != ROHM_OK) return rc;
  if ((rc = run_conv(tn, "final_o", B, st)) != ROHM_OK) return rc;
  const Act& o = *A("outp");
  const int64_t total = static_cast<int64_t>(B) * tn->T * o.C;
  unpack_rows_kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(o.f32, out, tn->T, tn->Tp[0], o.C, o.ld, total);
  ROHM_CUDA(ctx, cudaGetLastError());
  tn->launches++;
  return ROHM_OK;
}

struct TrajStepArgs {  // the ancestral update appended to the forward (rohm_trajnet_sample_step)
  float* x_next;
  const float* coef_row;
  unsigned long long seed, offset;
  int64_t G;
  int iters;
};

static int trajnet_forward_or_step(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* out, int B, void* stream,
                                   const TrajStepArgs* step) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = tn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (x_t == nullptr || time == nullptr || out == nullptr) return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_forward: null pointer");
  if (B != tn->cond_B)
    return fail(ctx, ROHM_ERR_STATE, "rohm_trajnet_forward: B=%d but set_cond was called with B=%d", B, tn->cond_B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  ROHM_CUDA(ctx, cudaStreamIsCapturing(st, &cap));
  const int64_t clip_elems = static_cast<int64_t>(tn->T) * tn->traj_dim;
  auto launch_step = [&](cudaStream_t s_) {
    return launch_ddpm_step_philox(out, x_t, step->x_next, clip_elems * B, clip_elems, step->coef_row, step->seed, step->offset,
                                   step->G, step->iters, s_, tn->use_pdl);
  };
  if (!tn->use_graph || cap != cudaStreamCaptureStatusNone) {
    int rc = trajnet_forward_launches(tn, x_t, time, out, B, st);
    if (rc == ROHM_OK && step != nullptr) {
      ROHM_CUDA(ctx, launch_step(st));
      tn->launches++;
    }
    return rc;
  }

  rohm_trajnet::FwdGraph* fg = nullptr;
  for (auto& g : tn->graphs)
    if (g.B == B && g.with_step == (step != nullptr)) fg = &g;
  if (fg == nullptr) {
    if (tn->capture_stream == nullptr) ROHM_CUDA(ctx, cudaStreamCreateWithFlags(&tn->capture_stream, cudaStreamNonBlocking));
    cudaStream_t cs = tn->capture_stream;
    ROHM_CUDA(ctx, cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal));
    int rc = trajnet_forward_launches(tn, x_t, time, out, B, cs);
    if (rc == ROHM_OK && step != nullptr) {
      if (launch_step(cs) != cudaSuccess) rc = fail(ctx, ROHM_ERR_CUDA, "ddpm step launch failed during capture");
      tn->launches++;
    }
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamEndCapture(cs, &graph);
    if (rc != ROHM_OK) {
      if (graph) cudaGraphDestroy(graph);
      return rc;
    }
    ROHM_CUDA(ctx, e);
    rohm_trajnet::FwdGraph ng;
    ng.B = B, ng.graph = graph, ng.with_step = step != nullptr;
    size_t n = 0;
    ROHM_CUDA(ctx, cudaGraphGetNodes(graph, nullptr, &n));
    std::vector<cudaGraphNode_t> nodes(n);
    ROHM_CUDA(ctx, cudaGraphGetNodes(graph, nodes.data(), &n));
    for (cudaGraphNode_t node : nodes) {
      cudaGraphNodeType ty;
      ROHM_CUDA(ctx, cudaGraphNodeGetType(node, &ty));
      if (ty != cudaGraphNodeTypeKernel) continue;
      cudaKernelNodeParams kp{};
      ROHM_CUDA(ctx, cudaGraphKernelNodeGetParams(node, &kp));
      if (kp.func == reinterpret_cast<void*>(pack_rows_kernel)) ng.n_pack = node, ng.p_pack = kp;
      else if (kp.func == reinterpret_cast<void*>(trajnet_time_kernel)) ng.n_time = node, ng.p_time = kp;
      else if (kp.func == reinterpret_cast<void*>(unpack_rows_kernel)) ng.n_unpack = node, ng.p_unpack = kp;
      else if (kp.func == const_cast<void*>(ddpm_step_philox_kernel_address())) ng.n_step = node, ng.p_step = kp;
    }
    if (!ng.n_pack || !ng.n_time || !ng.n_unpack || (step != nullptr && !ng.n_step)) {
      cudaGraphDestroy(graph);
      return fail(ctx, ROHM_ERR_CUDA, "trajnet graph: boundary nodes not found");
    }
    ROHM_CUDA(ctx, cudaGraphInstantiate(&ng.exec, graph, 0));
    if (tn->graphs.size() >= 8) {
      cudaGraphExecDestroy(tn->graphs.front().exec);
      cudaGraphDestroy(tn->graphs.front().graph);
      tn->graphs.erase(tn->graphs.begin());
    }
    tn->graphs.push_back(ng);
    fg = &tn->graphs.back();
  }
  const void* a_x = x_t;
  const void* a_t = time;
  void* a_o = out;
  {
    cudaKernelNodeParams kp = fg->p_pack;
    std::vector<void*> args(kp.kernelParams, kp.kernelParams + 9);
    args[0] = &a_x;
    kp.kernelParams = args.data();
    ROHM_CUDA(ctx, cudaGraphExecKernelNodeSetParams(fg->exec, fg->n_pack, &kp));
  }
  {
    cudaKernelNodeParams kp = fg->p_time;
    std::vector<void*> args(kp.kernelParams, kp.kernelParams + 12);
    args[0] = &a_t;
    kp.kernelParams = args.data();
    ROHM_CUDA(ctx, cudaGraphExecKernelNodeSetParams(fg->exec, fg->n_time, &kp));
  }
  {
    cudaKernelNodeParams kp = fg->p_unpack;
    std::vector<void*> args(kp.kernelParams, kp.kernelParams + 7);
    args[1] = &a_o;
    kp.kernelParams = args.data();
    ROHM_CUDA(ctx, cudaGraphExecKernelNodeSetParams(fg->exec, fg->n_unpack, &kp));
  }
  if (step != nullptr) {  // x0, x_t, out, coef row, Philox seed / offset of this step (ddpm_step_philox_kernel's argument list)
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

// TrajNet.forward (trajnet.py:177-275).  x_t: [B, T, traj_dim]; time: int64 [B]; out: [B, T, traj_dim].
extern "C" int rohm_trajnet_forward(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* out, int B,
                                    void* stream) {
  return trajnet_forward_or_step(tn, x_t, time, out, B, stream, nullptr);
}

// One whole ancestral step (gaussian_diffusion_trajnet.py p_sample without cond_fn): forward + in-kernel-noise update as one
// graph launch; see rohm_posenet_sample_step.
extern "C" int rohm_trajnet_sample_step(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* x0_out, float* x_next,
                                        const float* coef_row, uint64_t seed, uint64_t offset, uint64_t* offset_increment,
                                        int B, void* stream) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  if (x_next == nullptr || coef_row == nullptr)
    return fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_sample_step: null pointer");
  TrajStepArgs sa{x_next, coef_row, seed, offset, 0, 0};
  unsigned long long inc = 0;
  int rc = ddpm_step_philox_policy(tn->ctx, static_cast<int64_t>(tn->T) * tn->traj_dim * B, &sa.G, &sa.iters, &inc);
  if (rc != ROHM_OK) return rc;
  if (offset_increment != nullptr) *offset_increment = inc;
  return trajnet_forward_or_step(tn, x_t, time, x0_out, B, stream, &sa);
}

extern "C" int rohm_trajnet_set_option(rohm_trajnet* tn, int option, int value) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  if (option == 0) {
    tn->use_graph = value != 0;
    return ROHM_OK;
  }
  if (option == 1) {  // programmatic dependent launch along the convolution / GroupNorm chains (captured graphs are rebuilt)
    if (tn->use_pdl != (value != 0)) tn->drop_graphs();
    tn->use_pdl = value != 0;
    return ROHM_OK;
  }
  return fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_set_option: unknown option %d", option);
}
