// TrajNet denoiser engine: RoHM's 1-D conv U-Net with the TrajControl side branch
// (reference model/trajnet.py:10-75 ControlNet.forward, :177-275 TrajNet.forward; blocks model/heads.py:20-106).
//
// Layout: every activation is a channels-last matrix [B * Tp_L, C] per pyramid level L (T_L = T / 2^L real frames
// per clip followed by Tp_L - T_L >= 2 all-zero rows, Tp_L = (T + 32) / 2^L).  With per-clip lengths
// (rohm_trajnet_set_lengths) the clips are packed instead: clip b takes (lengths[b] + 32) / 2^L rows from
// off_L[b] = sum_{c<b} (lengths[c] + 32) / 2^L = off_0[b] / 2^L (exact: every lengths[c] + 32 is a multiple of 16), its
// lengths[b] / 2^L real frames first, and every GEMM runs over off_L[B] rows.  Stride-2 reads and the transposed
// convolution's interleaved stores still map clip b onto clip b, and every clip keeps >= 2 zero rows at every level.  In
// either layout
//   * Conv1d(k, pad k/2)        = k shifted reads of the same matrix: the zero rows between clips ARE the padding,
//   * channel concat [x, skip]  = two K-segments of one GEMM,
//   * Downsample (k3, stride 2) = the same with a row-stride-2 TMA descriptor,
//   * ConvTranspose (k4, s2)    = two GEMMs (even / odd output frames), 2 taps each, row-interleaved stores,
// so every convolution is one launch of the wgmma segmented-A GEMM (gemm.cu) and no im2col / concat / transpose
// buffer exists.  The convolutions of the deep pyramid levels are cut along K into 3-6 ranges (pick_split: 128-wide tiles x K
// ranges cover the SMs where 6-22 row tiles alone cannot); one kernel per GroupNorm'd convolution (gn_mish_split_kernel in
// groupnorm.cu, a cluster of CTAs per (clip, group)) adds bias + the fp32 partial(s) in split order, takes the group's
// statistics, applies GroupNorm + Mish
// (+ time projection, + residual, + TrajControl residual) and emits the hi/lo operand pair of the next convolution.  The
// step-invariant condition pyramid and control_zero_conv_0 run once per condition (set_cond).  rohm_trajnet_sample_step appends
// the in-kernel-noise sampler update to the forward graph.
// Batch-invariant engines (rohm_trajnet_create_batch_invariant) choose every convolution's tile width and K ranges at one
// canonical row count per level instead of the engine's capacity, and reduce each packed clip's GroupNorm statistics over the
// slices the clip has alone, so a clip's frames depend on that clip only, not on B, T or max_batch.
#include <cmath>
#include <memory>
#include <new>
#include <string>

#include "common.h"
#include "gemm.cuh"
#include "graph.cuh"
#include "groupnorm.cuh"
#include "ptx.cuh"

namespace rohm {
namespace {

// Real frames of packed clip b: its rows less the Tp - T pad rows every clip ends with.
__device__ __forceinline__ int packed_frames(const int* clip_off, int b, int T, int Tp) {
  return clip_off[b + 1] - clip_off[b] - (Tp - T);
}

// [B, T, C] channels-last API tensor -> padded-clip hi/lo rows (b * Tp + t), pitch ld.  Pad rows stay zero.
// kPacked (clip_off: level-0 offsets of packed clips): `total` covers B x Tp x C instead, and every row of clip b is
// written, its real frames from x and its pad rows as zeros; frames of x past the clip are never read.  Each of these
// boundary kernels has a uniform-clip instance of its own, which runs the code it ran before packed clips existed.
template <bool kPacked>
__global__ void pack_rows_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, int T,
                                 int Tp, int C, int ld, int64_t total, int f16, const int* __restrict__ clip_off) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % C);
  const int64_t bt = i / C;
  float v;
  int64_t o;
  if constexpr (!kPacked) {
    const int t = static_cast<int>(bt % T);
    const int64_t b = bt / T;
    v = x[i];
    o = (b * Tp + t) * ld + c;
  } else {
    const int t = static_cast<int>(bt % Tp);
    const int b = static_cast<int>(bt / Tp);
    if (t >= clip_off[b + 1] - clip_off[b]) return;
    v = t < packed_frames(clip_off, b, T, Tp) ? x[(static_cast<int64_t>(b) * T + t) * C + c] : 0.0f;
    o = (static_cast<int64_t>(clip_off[b]) + t) * ld + c;
  }
  if (f16) {
    ptx::split_f16(v, reinterpret_cast<__half*>(hi)[o], reinterpret_cast<__half*>(lo)[o]);
  } else {
    const float h = ptx::to_tf32(v);
    hi[o] = h;
    lo[o] = v - h;
  }
}
constexpr size_t kPackRowsX = 0;  // the argument replaced on every replay of a cached forward graph

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
constexpr size_t kTrajnetTimeT = 0;  // the argument replaced on every replay of a cached forward graph

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

// padded-clip rows [B * Tp, ld] -> compact [B, T, C]; kPacked (clip_off: packed clips): frames past a clip are zero
template <bool kPacked>
__global__ void unpack_rows_kernel(const float* __restrict__ x, float* __restrict__ out, int T, int Tp, int C, int ld,
                                   int64_t total, const int* __restrict__ clip_off) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = static_cast<int>(i % C);
  const int64_t bt = i / C;
  const int t = static_cast<int>(bt % T);
  const int64_t b = bt / T;
  if constexpr (!kPacked)
    out[i] = x[(b * Tp + t) * ld + c];
  else
    out[i] = t < packed_frames(clip_off, static_cast<int>(b), T, Tp) ? x[(static_cast<int64_t>(clip_off[b]) + t) * ld + c]
                                                                      : 0.0f;
}
constexpr size_t kUnpackRowsOut = 1;  // the argument replaced on every replay of a cached forward graph

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

// Scratch buffer `a` viewed as a [rows, C] matrix at `level` (row pitch C)
Act view(Act a, int C, int level) {
  a.C = C, a.ld = C, a.level = level;
  return a;
}

enum ConvKind : int {
  kConv,            // Conv1d(ks, stride, pad = ks/2 for stride 1, 1 for the stride-2 k3 downsample)
  kTransposedEven,  // even output phase of ConvTranspose1d(k4, s2, p1) (GEMM rows = input level rows)
  kTransposedOdd,   // odd output phase
};

struct Conv {
  std::string name;  // for error messages
  GemmParams g{};
  PackedWeight w;
  float* bias = nullptr;
  Act out;
  int level_out = 0;   // GEMM rows are the rows of this level (for transposed convs: the INPUT level)
  // GroupNorm'd convolutions store the GEMM result without bias in `partial`, and gn_mish_split_kernel adds bias, takes the
  // statistics and applies GroupNorm.  Split-K (deep pyramid levels): `splits` fp32 partial results of [split_rows, Cout]
  // each in the branch's partial scratch; otherwise the one partial is the convolution's own fp32 output.
  int splits = 1;
  float* partial = nullptr;
  int64_t split_rows = 0;
  bool sum_after = false;  // no GroupNorm behind it: sum_split_kernel writes `out` right after the GEMM
  int gn_cluster = 1;      // GroupNorm'd: CTAs per (clip, group) of its gn_mish_split_kernel launch (gn_pick_cluster)
};

struct GroupNorm {
  float* gamma = nullptr;
  float* beta = nullptr;
};

// ResidualTemporalBlock: out = Mish(GN(conv2(Mish(GN(conv1(x))) + time))) + residual [+ extra]
struct Rtb {
  std::string name;  // state-dict prefix, e.g. "diff_enc1."
  Conv c1, c2, res;
  bool has_res = false;  // the block changes the width: `res` is its 1x1 residual convolution
  GroupNorm gn[2];
  int tp_off = -1;  // offset of its rows in the stacked time projection; -1: no time input
  Act a1;           // Mish(GN(conv1(x))) + time: conv2's input
  const float* residual = nullptr;  // res's output, or the block's input
  const float* extra = nullptr;     // the TrajControl residual added by the U-Net's mid_block2 and decoder
  Act out;
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
  // caller's parameters by state-dict key, valid during create only
  int n_params = 0;
  const char* const* names = nullptr;
  const float* const* ptrs = nullptr;
  const int64_t* numels = nullptr;
  // time path
  float *w1 = nullptr, *b1 = nullptr, *w3 = nullptr, *b3 = nullptr, *wcat = nullptr, *bcat = nullptr, *tp = nullptr;
  float* time_table = nullptr;  // [kTimeTableRows, tp_total]: the stacked projections of every tabulated timestep
  int tp_total = 0;
  // the network (trajnet.py); U-Net decoder arrays are indexed by the level they write, like the encoder's
  Act xin, cin, kin;  // packed x_t, cond, control_cond
  Rtb cond_enc[4];    // condition pyramid
  Conv cond_down[3];
  Rtb enc[4], mid_block[2], dec[4];  // U-Net
  Conv down[4], up_even[4], up_odd[4];
  Conv final_c, final_o;
  GroupNorm final_gn;
  Act f1;  // final GroupNorm's output
  struct {
    Conv z0, zero[4], down[4], zero_mid;
    Rtb enc[4], mid_block[2];
  } ctl;  // TrajControl
  // RTB-internal scratch, one set per concurrently running branch (0: U-Net, 1: TrajControl)
  Act scratchY[2], scratchRes[2], scratchA[2];
  // Split-K partials of the GroupNorm'd convolutions (ROHM_B200_TRAJ_SPLITK=0 turns split-K off): kMaxSplits x the largest
  // 128-row-padded [rows, C] level matrix, per branch
  float* scratchSplit[2] = {nullptr, nullptr};
  bool use_splitk = true;
  // The forward is captured as a graph with parallel branches: the TrajControl branch next to the U-Net encoder, every
  // block's 1x1 residual convolution next to its conv1 -> GroupNorm -> conv2 chain.  None of these GEMMs fills the 132 SMs
  // (11 to 96 tiles), so running them side by side shortens the critical path at no cost.  ROHM_B200_TRAJ_PARALLEL=0: serial.
  bool parallel = true;
  cudaStream_t side[3] = {nullptr, nullptr, nullptr};  // 0: TrajControl branch, 1 / 2: residual convolutions of branch 0 / 1
  BranchEvents events;
  int cond_B = -1;
  int launches = 0;
  ForwardGraphs graphs;  // CUDA graph of one forward per batch size and lengths
  // Per-clip lengths (rohm_trajnet_set_lengths); empty: every clip has T frames at b * Tp[L].  Packed clips: clip_off[L]
  // (device int[max_batch + 1]) holds every clip's first row at level L, then the row count packed_rows[L]; row_mask[L]
  // (device, one byte per row) marks the real frames for the GEMM epilogue and sum_split_kernel.
  std::vector<int> lengths;
  std::vector<int> cond_lengths;  // the lengths set_cond embedded the condition with
  int* clip_off[kLevels] = {};
  unsigned char* row_mask[kLevels] = {};
  int packed_rows[kLevels] = {};
  bool use_pdl = true;  // ROHM_B200_PDL / rohm_trajnet_set_option(1): programmatic dependent launch along the conv / GroupNorm chains
  size_t gn_budget = 0;    // gn_mish_split_kernel's default dynamic shared-memory budget per CTA
  size_t gn_smem_max = 0;  // the largest slice of any of its launches
  // rohm_trajnet_create_batch_invariant: plans from kInvariantPlanRows, GroupNorm slices from kGnClipBudget and each clip's
  // own length (launch_gn_mish_clip_slices)
  bool batch_invariant = false;
  ~rohm_trajnet() {
    for (cudaStream_t q : side)
      if (q) cudaStreamDestroy(q);
  }
};

#define TRY(expr)                     \
  do {                                \
    const int rc__ = (expr);          \
    if (rc__ != ROHM_OK) return rc__; \
  } while (0)

namespace {

int64_t rows_of(const rohm_trajnet* tn, int level) { return static_cast<int64_t>(tn->max_batch) * tn->Tp[level]; }

// The rows a batch-invariant engine plans its convolutions for at level 0: the trajcontrol benchmark's 64 clips x (144 + 32)
// rows, so that shape runs the default engine's plan.  Level L plans for kInvariantPlanRows >> L rows.
constexpr int64_t kInvariantPlanRows = 64 * (144 + 32);

// The row count pick_bn / pick_split plan a convolution at `level` for: the engine's capacity, or in a batch-invariant
// engine a constant, so that the tile width and the K ranges (hence each output's summation order) depend on the layer alone.
int64_t plan_rows(const rohm_trajnet* tn, int level) {
  return tn->batch_invariant ? kInvariantPlanRows >> level : rows_of(tn, level);
}

int param(rohm_trajnet* tn, const std::string& key, int64_t expect_numel, const float** out) {
  for (int i = 0; i < tn->n_params; ++i) {
    if (key != tn->names[i]) continue;
    if (tn->numels[i] != expect_numel)
      return fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: parameter '%s' has %lld elements, expected %lld",
                  key.c_str(), static_cast<long long>(tn->numels[i]), static_cast<long long>(expect_numel));
    *out = tn->ptrs[i];
    return ROHM_OK;
  }
  return fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: missing parameter '%s'", key.c_str());
}

// The engine's own copy of parameter `key`
int dev_copy(rohm_trajnet* tn, const std::string& key, int64_t n, float** out) {
  const float* src = nullptr;
  TRY(param(tn, key, n, &src));
  *out = tn->pool.floats(n);
  if (*out == nullptr) return fail(tn->ctx, ROHM_ERR_CUDA, "alloc failed: %s", cudaGetErrorString(tn->pool.last_error()));
  ROHM_CUDA(tn->ctx, cudaMemcpy(*out, src, static_cast<size_t>(n) * sizeof(float), cudaMemcpyDeviceToDevice));
  return ROHM_OK;
}

// Allocates an activation (fp32 and/or hi/lo) at a level.
int make_act(rohm_trajnet* tn, Act& a, int C, int level, bool want_f32, bool want_split) {
  a.C = C, a.level = level, a.ld = static_cast<int>(round_up(C, tn->kind == kKindF16 ? 8 : 4));  // 16-byte row pitch
  const int64_t n = rows_of(tn, level) * a.ld;
  if (want_f32) a.f32 = tn->pool.floats(n);
  if (want_split) a.hi = tn->pool.floats(n), a.lo = tn->pool.floats(n);
  if ((want_f32 && !a.f32) || (want_split && (!a.hi || !a.lo)))
    return fail(tn->ctx, ROHM_ERR_CUDA, "activation alloc failed: %s", cudaGetErrorString(tn->pool.last_error()));
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

// Builds one convolution as a segmented GEMM writing `out` (Cout = out.C) from the channel concat of `srcs`.
// group_normed: gn_mish_split_kernel follows and adds the bias; branch: whose split-K partial scratch it uses.
int make_conv(rohm_trajnet* tn, Conv& cv, const std::string& name, const std::string& wkey, std::vector<const Act*> srcs,
              const Act& out, int ks, int stride, ConvKind kind, bool group_normed, int branch) {
  const int Cout = out.C;
  int Cin = 0;
  for (auto* s : srcs) Cin += s->C;
  const float* w = nullptr;
  TRY(param(tn, wkey + ".weight", static_cast<int64_t>(Cout) * Cin * ks, &w));
  cv.name = name;
  cv.out = out;
  // taps: (weight tap index, row shift)
  std::vector<std::pair<int, int>> taps;
  if (kind == kConv) {
    const int pad = (stride == 2) ? 1 : ks / 2;
    for (int j = 0; j < ks; ++j) taps.push_back({j, j - pad});
  } else if (kind == kTransposedEven) {  // out[2u] = W[1] x[u] + W[3] x[u-1]
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
  // GEMM rows: output level rows, except transposed convs whose rows are the input level's
  const int in_level = srcs[0]->level;
  const int row_level = (kind == kConv) ? out.level : in_level;
  PackedWeight& pw = cv.w;
  pw.N = Cout, pw.K = Ktot, pw.Kp = Ktot;
  pw.block_n = pick_bn(Cout, plan_rows(tn, row_level));
  const bool can_split = tn->use_splitk && kind == kConv && out.ld == Cout && Cout % 4 == 0;
  if (can_split && ((group_normed && stride == 1 && out.f32 != nullptr && out.hi == nullptr) || (!group_normed && ks > 1))) {
    int bn = pw.block_n;
    cv.splits = pick_split(Cout, plan_rows(tn, out.level), Ktot / kblk, kblk, &bn, group_normed ? 0.0 : 4.0);
    if (cv.splits > 1) {
      pw.block_n = bn;
      cv.sum_after = !group_normed;
    }
  }
  pw.Np = static_cast<int>(round_up(Cout, pw.block_n));
  pw.kind = tn->kind;
  pw.hi = static_cast<float*>(tn->pool.bytes(static_cast<int64_t>(pw.Np) * Ktot * gemm_elem_bytes(tn->kind)));
  pw.lo = static_cast<float*>(tn->pool.bytes(static_cast<int64_t>(pw.Np) * Ktot * gemm_elem_bytes(tn->kind)));
  if (!pw.hi || !pw.lo) return fail(tn->ctx, ROHM_ERR_CUDA, "weight alloc failed");
  if (tn->kind == kKindF16) ROHM_CUDA(tn->ctx, f16_weight_scale(w, static_cast<int64_t>(Cout) * Cin * ks, &pw.scale));
  TRY(dev_copy(tn, wkey + ".bias", Cout, &cv.bias));

  GemmParams& g = cv.g;
  int seg = 0, seg_off = 0;
  for (auto& tap : taps) {
    int src_off = 0;
    for (auto* s : srcs) {
      if (s->level != in_level || s->hi == nullptr)
        return fail(tn->ctx, ROHM_ERR_INVALID, "conv '%s': bad source", name.c_str());
      const int Cs = s->C;
      const int64_t n = static_cast<int64_t>(Cout) * Cs;
      pack_conv_segment_kernel<<<static_cast<unsigned>((n + 255) / 256), 256>>>(
          w, pw.hi, pw.lo, Cout, Cin, ks, src_off, Cs, tap.first, seg_off, Ktot, kind != kConv,
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
  cv.level_out = row_level;
  g.clip_rows = tn->Tp[row_level];
  g.clip_valid = tn->Tl[row_level];
  g.out_row_mul = (kind == kConv) ? 1 : 2;
  g.out_row_add = (kind == kTransposedOdd) ? 1 : 0;
  if (out.f32) g.out = out.f32, g.ldo = out.ld;
  if (out.hi) g.out_hi = out.hi, g.out_lo = out.lo, g.lds = out.ld;
  if (cv.splits > 1) {
    // partial results instead of the block's fp32 scratch; bias / statistics / GroupNorm happen in gn_mish_split_kernel
    cv.split_rows = static_cast<int64_t>(round_up(rows_of(tn, row_level), kGemmBlockM));
    cv.partial = tn->scratchSplit[branch];
    g.out = cv.partial, g.ldo = Cout, g.out_hi = nullptr, g.out_lo = nullptr;
    g.bias = nullptr;
    g.k_splits = cv.splits;
    g.split_row_stride = static_cast<int>(cv.split_rows);
  } else if (group_normed) {
    // y = conv without bias; bias + statistics + GroupNorm in gn_mish_split_kernel (one "partial").  Every GroupNorm'd output
    // is an fp32-only [rows, Cout] scratch whose width is a multiple of 4 * kGroups (rohm_trajnet_create's mid_dim rule).
    cv.partial = out.f32;
    g.bias = nullptr;
  }
  if (group_normed) {
    cv.gn_cluster = gn_pick_cluster(tn->Tl[row_level], Cout, kGroups, tn->batch_invariant ? kGnClipBudget : tn->gn_budget);
    tn->gn_smem_max = std::max(tn->gn_smem_max, gn_slice_bytes(tn->Tl[row_level], Cout, kGroups, cv.gn_cluster));
  }
  // fp32-only or fp16-pair-only outputs with the identity row map leave through TMA bulk stores (the transposed-conv phases
  // and the few convolutions that write both forms keep the per-thread epilogue)
  if (gemm_enable_tma_store(&g, cv.splits > 1 ? cv.splits * cv.split_rows : rows_of(tn, row_level), tn->kind) != 0)
    return fail(tn->ctx, ROHM_ERR_CUDA, "store tensor map failed for conv '%s'", name.c_str());
  return ROHM_OK;
}

int load_norm(rohm_trajnet* tn, GroupNorm& gn, const std::string& block_prefix, int C) {
  TRY(dev_copy(tn, block_prefix + "block.2.weight", C, &gn.gamma));
  return dev_copy(tn, block_prefix + "block.2.bias", C, &gn.beta);
}

// Declares the ResidualTemporalBlock `p` (its state-dict prefix, e.g. "diff_enc1.") reading `srcs` and writing `out`, with the
// RTB-internal scratch of `branch`.  timed: the block has a time input; it takes the next rows of the stacked time projection
// and is appended to *timed.
int make_rtb(rohm_trajnet* tn, Rtb& r, const std::string& p, std::vector<const Act*> srcs, const Act& out, int branch,
             std::vector<const Rtb*>* timed, const float* extra = nullptr) {
  int Cin = 0;
  for (auto* s : srcs) Cin += s->C;
  const int Cout = out.C, level = out.level;
  const Act y = view(tn->scratchY[branch], Cout, level);
  r.name = p;
  r.a1 = view(tn->scratchA[branch], Cout, level);
  r.extra = extra;
  r.out = out;
  TRY(make_conv(tn, r.c1, p + "c1", p + "blocks.0.block.0", srcs, y, 5, 1, kConv, true, branch));
  TRY(make_conv(tn, r.c2, p + "c2", p + "blocks.1.block.0", {&r.a1}, y, 5, 1, kConv, true, branch));
  TRY(load_norm(tn, r.gn[0], p + "blocks.0.", Cout));
  TRY(load_norm(tn, r.gn[1], p + "blocks.1.", Cout));
  r.has_res = Cin != Cout;
  if (r.has_res) {
    const Act res = view(tn->scratchRes[branch], Cout, level);
    TRY(make_conv(tn, r.res, p + "res", p + "residual_conv", srcs, res, 1, 1, kConv, false, branch));
    r.residual = res.f32;
  } else {
    if (srcs.size() != 1 || srcs[0]->f32 == nullptr)
      return fail(tn->ctx, ROHM_ERR_INVALID, "block '%s': the identity residual needs one fp32 input", p.c_str());
    r.residual = srcs[0]->f32;
  }
  if (timed != nullptr) {
    r.tp_off = tn->tp_total;
    tn->tp_total += Cout;
    timed->push_back(&r);
  }
  return ROHM_OK;
}

int run_conv(rohm_trajnet* tn, Conv& cv, int B, cudaStream_t st) {
  const bool packed = !tn->lengths.empty();
  const int rows = packed ? tn->packed_rows[cv.level_out] : B * tn->Tp[cv.level_out];
  const unsigned char* mask = packed ? tn->row_mask[cv.level_out] : nullptr;
  cv.g.M = rows;
  cv.g.row_mask = mask;
  ROHM_CUDA(tn->ctx, launch_gemm(cv.g, rows, cv.w.N, cv.w.block_n, tn->passes, st, tn->use_pdl, tn->kind));
  tn->launches++;
  if (cv.sum_after) {
    const int C = cv.w.N;
    const int64_t total4 = static_cast<int64_t>(rows) * C / 4;
    ROHM_CUDA(tn->ctx, launch_chain(packed ? sum_split_kernel<true> : sum_split_kernel<false>, dim3(static_cast<unsigned>((total4 + 255) / 256)), dim3(256), 0, st,
                                    tn->use_pdl, cv.partial, cv.splits, cv.split_rows * C, cv.bias, cv.out.f32, cv.out.hi,
                                    cv.out.lo, C, tn->Tp[cv.level_out], tn->Tl[cv.level_out], total4,
                                    tn->kind == kKindF16 ? 1 : 0, mask));
    tn->launches++;
  }
  return ROHM_OK;
}

// partial(s) + bias -> statistics -> GroupNorm / Mish of the GroupNorm'd convolution `cv`, one cluster of cv.gn_cluster
// CTAs per (clip, group)
int run_gn(rohm_trajnet* tn, const Conv& cv, const GroupNorm& gn, int B, const float* tp, const float* r1, const float* r2,
           const Act& out, cudaStream_t st) {
  const int C = cv.w.N, level = cv.level_out;
  const GnArgs a{cv.partial, cv.splits, cv.split_rows * C, cv.bias, gn.gamma, gn.beta, tp, tn->tp_total, r1, r2,
                 out.f32, out.hi, out.lo, C, tn->Tp[level], tn->Tl[level], kGroups, tn->kind == kKindF16 ? 1 : 0};
  if (tn->batch_invariant && !tn->lengths.empty() && cv.gn_cluster > 1) {
    // each packed clip over the slices it has alone (uniform clips have them already: v = n)
    size_t smem = 0;
    for (int len : tn->lengths) {
      const int Tc = len >> level;
      smem = std::max(smem, gn_slice_bytes(Tc, C, kGroups, gn_pick_cluster(Tc, C, kGroups, kGnClipBudget)));
    }
    ROHM_CUDA(tn->ctx, launch_gn_mish_clip_slices(a, B, cv.gn_cluster, smem, st, tn->use_pdl, tn->clip_off[level]));
  } else {
    ROHM_CUDA(tn->ctx, launch_gn_mish(a, B, cv.gn_cluster, st, tn->use_pdl,
                                      tn->lengths.empty() ? nullptr : tn->clip_off[level]));
  }
  tn->launches++;
  return ROHM_OK;
}

// Executes a ResidualTemporalBlock on `st`, its 1x1 residual convolution on `side`
int run_rtb(rohm_trajnet* tn, Rtb& r, int B, cudaStream_t st, cudaStream_t side) {
  if (r.has_res) {  // the 1x1 residual convolution only reads the block's input: run it next to the main chain
    TRY(tn->events.order_after(tn->ctx, st, side));
    TRY(run_conv(tn, r.res, B, side));
  }
  TRY(run_conv(tn, r.c1, B, st));
  const float* tp = r.tp_off >= 0 ? tn->tp + r.tp_off : nullptr;
  TRY(run_gn(tn, r.c1, r.gn[0], B, tp, nullptr, nullptr, r.a1, st));
  TRY(run_conv(tn, r.c2, B, st));
  if (r.has_res) TRY(tn->events.order_after(tn->ctx, side, st));
  return run_gn(tn, r.c2, r.gn[1], B, nullptr, r.residual, r.extra, r.out, st);
}

int trajnet_create(rohm_ctx* ctx, int n_params, const char* const* names, const float* const* ptrs, const int64_t* numels,
                   int time_dim, int cond_dim, int traj_feat_dim, int mid_dim, int trajcontrol, int control_cond_dim,
                   int max_batch, int frames, int precision, bool batch_invariant, rohm_trajnet** out) {
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
  // GroupNorm: a group of the widest levels (frames x mid_dim / 8 values at level 0, and the same count at levels 1-3) is
  // spread over a cluster of at most kGnMaxCluster CTAs, each of which holds its slice in shared memory
  size_t gn_budget = 0, gn_max = 0;
  ROHM_CUDA(ctx, gn_smem_budgets(&gn_budget, &gn_max));
  const int64_t gn_row_bytes = static_cast<int64_t>(mid_dim / 8 / kGroups) * sizeof(float);
  const int64_t max_frames = static_cast<int64_t>(gn_max) / gn_row_bytes * kGnMaxCluster / 16 * 16;
  if (frames > max_frames)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_create: frames (%d) exceeds %lld at mid_dim %d: a GroupNorm group of "
                "the widest levels holds frames x mid_dim / 64 values, spread over at most %d CTAs of %zu bytes of shared "
                "memory each (frames <= %d x floor(%zu / (mid_dim / 16)), a multiple of 16)", frames,
                static_cast<long long>(max_frames), mid_dim, kGnMaxCluster, gn_max, kGnMaxCluster, gn_max);
  ROHM_CUDA(ctx, gemm_init_attributes());
  std::unique_ptr<rohm_trajnet> owner(new (std::nothrow) rohm_trajnet());
  rohm_trajnet* tn = owner.get();
  if (tn == nullptr) return fail(ctx, ROHM_ERR_INVALID, "out of host memory");
  tn->ctx = ctx;
  tn->time_dim = time_dim, tn->cond_dim = cond_dim, tn->traj_dim = traj_feat_dim, tn->mid = mid_dim;
  tn->control = trajcontrol != 0, tn->control_dim = control_cond_dim, tn->passes = precision == ROHM_PRECISION_TF32 ? 1 : 3;
  tn->kind = precision == ROHM_PRECISION_F16X2 ? kKindF16 : kKindTf32;
  tn->max_batch = max_batch, tn->T = frames;
  tn->gn_budget = gn_budget;
  tn->batch_invariant = batch_invariant;
  for (int l = 0; l < kLevels; ++l) tn->Tl[l] = frames >> l, tn->Tp[l] = (frames + 32) >> l;
  tn->n_params = n_params, tn->names = names, tn->ptrs = ptrs, tn->numels = numels;
  const int m = mid_dim, td = time_dim;

  // ---- scratch ----
  int64_t max_elems = 0, max_padded = 0;  // the largest [rows, C] level matrix, unpadded and with 128-row-padded rows
  const int widths[kLevels] = {m / 8, m / 4, m / 2, m, 2 * m};
  for (int l = 0; l < kLevels; ++l) {
    max_elems = std::max<int64_t>(max_elems, rows_of(tn, l) * widths[l]);
    max_padded = std::max<int64_t>(max_padded, static_cast<int64_t>(round_up(rows_of(tn, l), kGemmBlockM)) * widths[l]);
  }
  for (int br = 0; br < 2; ++br) {
    tn->scratchY[br].f32 = tn->pool.floats(max_elems);
    tn->scratchRes[br].f32 = tn->pool.floats(max_elems);
    tn->scratchA[br].hi = tn->pool.floats(max_elems);
    tn->scratchA[br].lo = tn->pool.floats(max_elems);
    if (!tn->scratchY[br].f32 || !tn->scratchRes[br].f32 || !tn->scratchA[br].hi || !tn->scratchA[br].lo)
      return fail(ctx, ROHM_ERR_CUDA, "scratch alloc failed");
  }
  if (const char* env = getenv("ROHM_B200_TRAJ_PARALLEL")) tn->parallel = env[0] != '0';
  if (const char* env = getenv("ROHM_B200_TRAJ_SPLITK")) tn->use_splitk = env[0] != '0';
  for (int l = 0; l < kLevels; ++l) {
    tn->clip_off[l] = static_cast<int*>(tn->pool.bytes(static_cast<int64_t>(max_batch + 1) * sizeof(int)));
    tn->row_mask[l] = static_cast<unsigned char*>(tn->pool.bytes(rows_of(tn, l)));
    if (!tn->clip_off[l] || !tn->row_mask[l]) return fail(ctx, ROHM_ERR_CUDA, "clip table alloc failed");
  }
  if (tn->use_splitk) {
    for (int br = 0; br < 2; ++br) {
      tn->scratchSplit[br] = tn->pool.floats(kMaxSplits * max_padded);
      if (!tn->scratchSplit[br]) return fail(ctx, ROHM_ERR_CUDA, "split-K scratch alloc failed");
    }
  }

  // ---- activations ----
  // c: condition pyramid (skip into the U-Net / control), cd: its downsamplings, d: U-Net encoder outputs (skips),
  // e: downsampled concats, mb: mid blocks, up: upsamplings, u: decoder outputs; k, z, ke, kmb: the TrajControl counterparts
  Act c[4], cd[3], d[4], e[4], mb[2], up[4], u[4], outp, k0, k[4], z[4], ke[4], kmb[2], zm;
  TRY(make_act(tn, tn->xin, traj_feat_dim, 0, false, true));
  TRY(make_act(tn, tn->cin, cond_dim, 0, false, true));
  const int enc_w[4] = {m / 8, m / 4, m / 2, m};
  for (int l = 0; l < 4; ++l) {
    TRY(make_act(tn, c[l], enc_w[l], l, false, true));
    if (l < 3) TRY(make_act(tn, cd[l], enc_w[l], l + 1, true, true));  // identity residual never needed, f32 for safety
    TRY(make_act(tn, d[l], enc_w[l], l, false, true));
    TRY(make_act(tn, e[l], 2 * enc_w[l], l + 1, true, true));  // f32: identity residual of the next RTB
  }
  TRY(make_act(tn, mb[0], m, 4, true, true));
  TRY(make_act(tn, mb[1], m, 4, false, true));
  const int dec_w[4] = {32, m / 8, m / 4, m / 2};  // dec1..dec4 output widths
  for (int l = 3; l >= 0; --l) {
    TRY(make_act(tn, up[l], (l == 3 ? m : dec_w[l + 1]), l, false, true));
    TRY(make_act(tn, u[l], dec_w[l], l, false, true));
  }
  TRY(make_act(tn, tn->f1, 32, 0, false, true));
  TRY(make_act(tn, outp, traj_feat_dim, 0, true, false));
  if (tn->control) {
    TRY(make_act(tn, tn->kin, control_cond_dim, 0, false, true));
    TRY(make_act(tn, k0, traj_feat_dim, 0, false, true));
    const int zw[4] = {32, m / 8, m / 4, m / 2};
    for (int l = 0; l < 4; ++l) {
      TRY(make_act(tn, k[l], enc_w[l], l, false, true));
      TRY(make_act(tn, z[l], zw[l], l, true, false));
      TRY(make_act(tn, ke[l], 2 * enc_w[l], l + 1, true, true));
    }
    TRY(make_act(tn, kmb[0], m, 4, true, true));
    TRY(make_act(tn, kmb[1], m, 4, false, true));
    TRY(make_act(tn, zm, m, 4, true, false));
  }

  // ---- convolutions ----
  std::vector<const Rtb*> timed;  // blocks with a time input, in the order of the stacked time projection
  // condition pyramid (trajnet.py:192-208): RTBs without time input
  for (int l = 0; l < 4; ++l) {
    const std::string L = std::to_string(l + 1);
    TRY(make_rtb(tn, tn->cond_enc[l], "cond_enc" + L + ".", {l == 0 ? &tn->cin : &cd[l - 1]}, c[l], 0, nullptr));
    if (l < 3)
      TRY(make_conv(tn, tn->cond_down[l], "cond_down" + L, "cond_downsample" + L + ".conv", {&c[l]}, cd[l], 3, 2, kConv,
                    false, 0));
  }
  // U-Net (trajnet.py:216-275)
  for (int l = 0; l < 4; ++l) {
    const std::string L = std::to_string(l + 1);
    TRY(make_rtb(tn, tn->enc[l], "diff_enc" + L + ".", {l == 0 ? &tn->xin : &e[l - 1]}, d[l], 0, &timed));
    TRY(make_conv(tn, tn->down[l], "diff_down" + L, "diff_downsample" + L + ".conv", {&d[l], &c[l]}, e[l], 3, 2, kConv,
                  false, 0));
  }
  TRY(make_rtb(tn, tn->mid_block[0], "diff_mid_block1.", {&e[3]}, mb[0], 0, &timed));
  TRY(make_rtb(tn, tn->mid_block[1], "diff_mid_block2.", {&mb[0]}, mb[1], 0, &timed, zm.f32));
  for (int l = 3; l >= 0; --l) {
    const std::string L = std::to_string(l + 1);
    const Act* x = l == 3 ? &mb[1] : &u[l + 1];
    TRY(make_conv(tn, tn->up_even[l], "up" + L + "e", "diff_upsample" + L + ".conv", {x}, up[l], 4, 1,
                  kTransposedEven, false, 0));
    TRY(make_conv(tn, tn->up_odd[l], "up" + L + "o", "diff_upsample" + L + ".conv", {x}, up[l], 4, 1,
                  kTransposedOdd, false, 0));
    TRY(make_rtb(tn, tn->dec[l], "diff_dec" + L + ".", {&up[l], &d[l]}, u[l], 0, &timed, z[l].f32));
  }
  TRY(make_conv(tn, tn->final_c, "final_c", "diff_final_conv.0.block.0", {&u[0]}, view(tn->scratchY[0], 32, 0), 5, 1, kConv,
                true, 0));
  TRY(load_norm(tn, tn->final_gn, "diff_final_conv.0.", 32));
  TRY(make_conv(tn, tn->final_o, "final_o", "diff_final_conv.1", {&tn->f1}, outp, 1, 1, kConv, false, 0));
  if (tn->control) {  // trajnet.py:43-75
    const std::string cn = "controlnet.";
    auto& ctl = tn->ctl;
    TRY(make_conv(tn, ctl.z0, "kz0", cn + "control_zero_conv_0", {&tn->kin}, k0, 1, 1, kConv, false, 1));
    for (int l = 0; l < 4; ++l) {
      const std::string L = std::to_string(l + 1);
      TRY(make_rtb(tn, ctl.enc[l], cn + "control_enc" + L + ".", {l == 0 ? &k0 : &ke[l - 1]}, k[l], 1, &timed));
      TRY(make_conv(tn, ctl.zero[l], "kz" + L, cn + "control_zero_conv_" + L, {&k[l]}, z[l], 1, 1, kConv, false, 1));
      TRY(make_conv(tn, ctl.down[l], "kd" + L, cn + "control_downsample" + L + ".conv", {&k[l], &c[l]}, ke[l], 3, 2, kConv,
                    false, 1));
    }
    TRY(make_rtb(tn, ctl.mid_block[0], cn + "control_mid_block1.", {&ke[3]}, kmb[0], 1, &timed));
    TRY(make_rtb(tn, ctl.mid_block[1], cn + "control_mid_block2.", {&kmb[0]}, kmb[1], 1, &timed));
    TRY(make_conv(tn, ctl.zero_mid, "kzm", cn + "control_zero_conv_mid", {&kmb[1]}, zm, 1, 1, kConv, false, 1));
  }

  // one attribute for every GroupNorm launch of the engine; only needed when a slice exceeds the default budget (n = 8)
  if (tn->gn_smem_max > gn_budget) ROHM_CUDA(ctx, gn_reserve_smem(tn->gn_smem_max));

  // ---- time path: stacked Linear(time_dim -> out) of every block with input_t ----
  const int total = tn->tp_total;
  tn->wcat = tn->pool.floats(static_cast<int64_t>(total) * td);
  tn->bcat = tn->pool.floats(total);
  tn->tp = tn->pool.floats(static_cast<int64_t>(max_batch) * total);
  if (!tn->wcat || !tn->bcat || !tn->tp) return fail(ctx, ROHM_ERR_CUDA, "time projection alloc failed");
  for (const Rtb* r : timed) {
    const float *w = nullptr, *b = nullptr;
    TRY(param(tn, r->name + "time_mlp.1.weight", static_cast<int64_t>(r->out.C) * td, &w));
    TRY(param(tn, r->name + "time_mlp.1.bias", r->out.C, &b));
    ROHM_CUDA(ctx, cudaMemcpy(tn->wcat + static_cast<int64_t>(r->tp_off) * td, w, sizeof(float) * r->out.C * td,
                              cudaMemcpyDeviceToDevice));
    ROHM_CUDA(ctx, cudaMemcpy(tn->bcat + r->tp_off, b, sizeof(float) * r->out.C, cudaMemcpyDeviceToDevice));
  }
  TRY(dev_copy(tn, "time_mlp.1.weight", static_cast<int64_t>(4) * td * td, &tn->w1));
  TRY(dev_copy(tn, "time_mlp.1.bias", 4 * td, &tn->b1));
  TRY(dev_copy(tn, "time_mlp.3.weight", static_cast<int64_t>(4) * td * td, &tn->w3));
  TRY(dev_copy(tn, "time_mlp.3.bias", td, &tn->b3));
  // tabulate the whole time path for t = 0 .. kTimeTableRows-1 with the direct-evaluation branch of the kernel
  tn->time_table = tn->pool.floats(static_cast<int64_t>(kTimeTableRows) * total);
  std::vector<int64_t> ts(kTimeTableRows);
  for (int i = 0; i < kTimeTableRows; ++i) ts[i] = i;
  int64_t* d_ts = static_cast<int64_t*>(tn->pool.bytes(sizeof(int64_t) * kTimeTableRows));
  if (!tn->time_table || !d_ts) return fail(ctx, ROHM_ERR_CUDA, "time table alloc failed");
  ROHM_CUDA(ctx, cudaMemcpy(d_ts, ts.data(), sizeof(int64_t) * kTimeTableRows, cudaMemcpyHostToDevice));
  trajnet_time_kernel<<<dim3(kTimeTableRows, 8), 256, sizeof(float) * 6 * td>>>(d_ts, td, tn->w1, tn->b1, tn->w3, tn->b3, tn->wcat,
                                                                              tn->bcat, total, tn->time_table, nullptr, 0);
  ROHM_CUDA(ctx, cudaGetLastError());

  cudaError_t err = cudaDeviceSynchronize();
  tn->n_params = 0;
  if (err != cudaSuccess)
    return fail(ctx, ROHM_ERR_CUDA, "weight packing / time table build failed: %s", cudaGetErrorString(err));
  *out = owner.release();
  return ROHM_OK;
}

}  // namespace

extern "C" int rohm_trajnet_create(rohm_ctx* ctx, int n_params, const char* const* names, const float* const* ptrs,
                                   const int64_t* numels, int time_dim, int cond_dim, int traj_feat_dim, int mid_dim,
                                   int trajcontrol, int control_cond_dim, int max_batch, int frames, int precision,
                                   rohm_trajnet** out) {
  return trajnet_create(ctx, n_params, names, ptrs, numels, time_dim, cond_dim, traj_feat_dim, mid_dim, trajcontrol,
                        control_cond_dim, max_batch, frames, precision, false, out);
}

extern "C" int rohm_trajnet_create_batch_invariant(rohm_ctx* ctx, int n_params, const char* const* names,
                                                   const float* const* ptrs, const int64_t* numels, int time_dim,
                                                   int cond_dim, int traj_feat_dim, int mid_dim, int trajcontrol,
                                                   int control_cond_dim, int max_batch, int frames, int precision,
                                                   rohm_trajnet** out) {
  return trajnet_create(ctx, n_params, names, ptrs, numels, time_dim, cond_dim, traj_feat_dim, mid_dim, trajcontrol,
                        control_cond_dim, max_batch, frames, precision, true, out);
}

extern "C" void rohm_trajnet_destroy(rohm_trajnet* tn) { delete tn; }

extern "C" int rohm_trajnet_launches_per_forward(const rohm_trajnet* tn) { return tn ? tn->launches : 0; }

static int trajnet_pack(rohm_trajnet* tn, const float* x, const Act& a, int B, cudaStream_t st) {
  const bool packed = !tn->lengths.empty();
  const int64_t total = static_cast<int64_t>(B) * (packed ? tn->Tp[0] : tn->T) * a.C;
  (packed ? pack_rows_kernel<true> : pack_rows_kernel<false>)<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
      x, a.hi, a.lo, tn->T, tn->Tp[0], a.C, a.ld, total, tn->kind == kKindF16 ? 1 : 0, packed ? tn->clip_off[0] : nullptr);
  ROHM_CUDA(tn->ctx, cudaGetLastError());
  tn->launches++;
  return ROHM_OK;
}

// Step-invariant part: the condition pyramid (and control_zero_conv_0).  cond: [B, T, cond_dim];
// control_cond: [B, T, control_cond_dim] or NULL for the vanilla network.  Packed clips (rohm_trajnet_set_lengths) read only
// each clip's real frames.
extern "C" int rohm_trajnet_set_cond(rohm_trajnet* tn, const float* cond, const float* control_cond, int B, void* stream) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = tn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (cond == nullptr || B <= 0 || B > tn->max_batch || (tn->control && control_cond == nullptr))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_set_cond: bad arguments (B=%d, capacity %d)", B, tn->max_batch);
  if (!tn->lengths.empty() && static_cast<int>(tn->lengths.size()) != B)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_set_cond: lengths were set for %d clips, the call has B=%d",
                static_cast<int>(tn->lengths.size()), B);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int saved = tn->launches;
  TRY(trajnet_pack(tn, cond, tn->cin, B, st));
  for (int l = 0; l < 4; ++l) {
    TRY(run_rtb(tn, tn->cond_enc[l], B, st, st));
    if (l < 3) TRY(run_conv(tn, tn->cond_down[l], B, st));
  }
  if (tn->control) {
    TRY(trajnet_pack(tn, control_cond, tn->kin, B, st));
    TRY(run_conv(tn, tn->ctl.z0, B, st));
  }
  tn->launches = saved;
  tn->cond_B = B;
  tn->cond_lengths = tn->lengths;
  return ROHM_OK;
}

extern "C" int rohm_trajnet_set_lengths(rohm_trajnet* tn, const int* lengths, int B) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = tn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (lengths == nullptr) {
    if (tn->lengths.empty()) return ROHM_OK;
    // the uniform layout's pad rows of the packed inputs must be zero again (packing writes real frames there), and a
    // forward still in flight may be reading them
    ROHM_CUDA(ctx, cudaDeviceSynchronize());
    for (const Act* a : {&tn->xin, &tn->cin, &tn->kin}) {
      if (a->hi == nullptr) continue;
      const size_t n = static_cast<size_t>(rows_of(tn, 0)) * a->ld * sizeof(float);
      ROHM_CUDA(ctx, cudaMemset(a->hi, 0, n));
      ROHM_CUDA(ctx, cudaMemset(a->lo, 0, n));
    }
    tn->lengths.clear();
    return ROHM_OK;
  }
  if (B <= 0 || B > tn->max_batch)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_set_lengths: B=%d outside the created capacity %d", B, tn->max_batch);
  for (int b = 0; b < B; ++b)
    if (lengths[b] < 16 || lengths[b] > tn->T || lengths[b] % 16 != 0)
      return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_set_lengths: lengths[%d] = %d must be a multiple of 16 in [16, %d]",
                  b, lengths[b], tn->T);
  std::vector<int> v(lengths, lengths + B);
  if (v == tn->lengths) return ROHM_OK;
  std::vector<int> off[kLevels];
  std::vector<unsigned char> mask[kLevels];
  for (int l = 0; l < kLevels; ++l) {
    off[l].assign(B + 1, 0);
    for (int b = 0; b < B; ++b) {
      const int rows = (v[b] + 32) >> l, real = v[b] >> l;
      off[l][b + 1] = off[l][b] + rows;
      for (int t = 0; t < rows; ++t) mask[l].push_back(t < real ? 1 : 0);
    }
  }
  // a forward still in flight on any stream may be reading the tables being replaced
  ROHM_CUDA(ctx, cudaDeviceSynchronize());
  for (int l = 0; l < kLevels; ++l) {
    ROHM_CUDA(ctx, cudaMemcpy(tn->clip_off[l], off[l].data(), (B + 1) * sizeof(int), cudaMemcpyHostToDevice));
    ROHM_CUDA(ctx, cudaMemcpy(tn->row_mask[l], mask[l].data(), mask[l].size(), cudaMemcpyHostToDevice));
    tn->packed_rows[l] = off[l][B];
  }
  tn->lengths = std::move(v);
  return ROHM_OK;
}

static int trajnet_forward_launches(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* out, int B,
                                    cudaStream_t st) {
  rohm_ctx* ctx = tn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  tn->launches = 0;
  TRY(trajnet_pack(tn, x_t, tn->xin, B, st));
  const int td = tn->time_dim;
  trajnet_time_kernel<<<dim3(B, 8), 256, sizeof(float) * 6 * td, st>>>(time, td, tn->w1, tn->b1, tn->w3, tn->b3, tn->wcat, tn->bcat,
                                                            tn->tp_total, tn->tp, tn->time_table, kTimeTableRows);
  ROHM_CUDA(ctx, cudaGetLastError());
  tn->launches++;

  // Parallel branches (see rohm_trajnet::parallel): sC carries the TrajControl branch, r0 / r1 the residual 1x1 convolutions
  // (and the odd phases of the transposed convolutions) of the U-Net / TrajControl blocks.
  tn->events.rewind();
  if (tn->parallel)
    for (cudaStream_t& q : tn->side)
      if (q == nullptr) ROHM_CUDA(ctx, cudaStreamCreateWithFlags(&q, cudaStreamNonBlocking));
  cudaStream_t sC = (tn->parallel && tn->control) ? tn->side[0] : st;
  cudaStream_t r0 = tn->parallel ? tn->side[1] : st;
  cudaStream_t r1 = tn->parallel ? tn->side[2] : sC;
  if (tn->control) {
    auto& ctl = tn->ctl;
    TRY(tn->events.order_after(tn->ctx, st, sC));  // fork after pack + time
    for (int l = 0; l < 4; ++l) {
      TRY(run_rtb(tn, ctl.enc[l], B, sC, r1));
      TRY(run_conv(tn, ctl.zero[l], B, sC));
      TRY(run_conv(tn, ctl.down[l], B, sC));
    }
    for (Rtb& r : ctl.mid_block) TRY(run_rtb(tn, r, B, sC, r1));
    TRY(run_conv(tn, ctl.zero_mid, B, sC));
  }

  for (int l = 0; l < 4; ++l) {
    TRY(run_rtb(tn, tn->enc[l], B, st, r0));
    TRY(run_conv(tn, tn->down[l], B, st));
  }
  TRY(run_rtb(tn, tn->mid_block[0], B, st, r0));
  if (tn->control) TRY(tn->events.order_after(tn->ctx, sC, st));  // join: the decoder adds the TrajControl residuals
  TRY(run_rtb(tn, tn->mid_block[1], B, st, r0));
  for (int l = 3; l >= 0; --l) {
    // ConvTranspose1d = two independent GEMMs (even / odd output frames) with row-interleaved stores
    TRY(tn->events.order_after(tn->ctx, st, r0));
    TRY(run_conv(tn, tn->up_odd[l], B, r0));
    TRY(run_conv(tn, tn->up_even[l], B, st));
    TRY(tn->events.order_after(tn->ctx, r0, st));
    TRY(run_rtb(tn, tn->dec[l], B, st, r0));
  }
  TRY(run_conv(tn, tn->final_c, B, st));
  TRY(run_gn(tn, tn->final_c, tn->final_gn, B, nullptr, nullptr, nullptr, tn->f1, st));
  TRY(run_conv(tn, tn->final_o, B, st));
  const Act& o = tn->final_o.out;
  const int64_t total = static_cast<int64_t>(B) * tn->T * o.C;
  const bool packed = !tn->lengths.empty();
  (packed ? unpack_rows_kernel<true> : unpack_rows_kernel<false>)<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(
      o.f32, out, tn->T, tn->Tp[0], o.C, o.ld, total, packed ? tn->clip_off[0] : nullptr);
  ROHM_CUDA(ctx, cudaGetLastError());
  tn->launches++;
  return ROHM_OK;
}

// One forward, with the ancestral update appended when `step` (rohm_trajnet_sample_step) or `clip_step`
// (rohm_trajnet_sample_step_clips) is given.
static int trajnet_forward_or_step(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* out, int B, void* stream,
                                   const DdpmStep* step, const DdpmClipStep* clip_step = nullptr) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = tn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (x_t == nullptr || time == nullptr || out == nullptr) return fail(ctx, ROHM_ERR_INVALID, "rohm_trajnet_forward: null pointer");
  if (B != tn->cond_B)
    return fail(ctx, ROHM_ERR_STATE, "rohm_trajnet_forward: B=%d but set_cond was called with B=%d", B, tn->cond_B);
  if (tn->lengths != tn->cond_lengths)
    return fail(ctx, ROHM_ERR_STATE, "rohm_trajnet_forward: the clip lengths differ from those set_cond was called with");
  auto launches = [&](cudaStream_t st) {
    const int rc = trajnet_forward_launches(tn, x_t, time, out, B, st);
    if (rc != ROHM_OK || (step == nullptr && clip_step == nullptr)) return rc;
    tn->launches++;
    if (clip_step != nullptr) return launch_ddpm_clip_step(ctx, *clip_step, st, tn->use_pdl);
    return launch_ddpm_step(ctx, *step, st, tn->use_pdl);
  };
  const bool packed = !tn->lengths.empty();
  std::vector<KernelPatch> patches = {{packed ? pack_rows_kernel<true> : pack_rows_kernel<false>, arg<kPackRowsX>(x_t)},
                                      {trajnet_time_kernel, arg<kTrajnetTimeT>(time)},
                                      {packed ? unpack_rows_kernel<true> : unpack_rows_kernel<false>,
                                       arg<kUnpackRowsOut>(out)}};
  if (step != nullptr) patches.push_back(ddpm_step_patch(*step));
  if (clip_step != nullptr) patches.push_back(ddpm_clip_step_patch(*clip_step));
  const StepKind kind = clip_step != nullptr ? kStepPerClip : step != nullptr ? kStepSingleStream : kNoStep;
  return tn->graphs.run(ctx, B, tn->T, kind, false, static_cast<cudaStream_t>(stream), launches, patches, tn->lengths);
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
  const int64_t clip_elems = static_cast<int64_t>(tn->T) * tn->traj_dim;
  DdpmStep step{x0_out, x_t, x_next, clip_elems * B, clip_elems, coef_row, seed, offset};
  const int rc = ddpm_step_plan(tn->ctx, &step, offset_increment);
  if (rc != ROHM_OK) return rc;
  return trajnet_forward_or_step(tn, x_t, time, x0_out, B, stream, &step);
}

// The same step with per-clip noise streams (rohm_randn_clips); see rohm_posenet_sample_step_clips.
extern "C" int rohm_trajnet_sample_step_clips(rohm_trajnet* tn, const float* x_t, const int64_t* time, float* x0_out,
                                              float* x_next, const float* coef_row, const uint64_t* streams, uint64_t draw,
                                              uint64_t* offset_increments, int B, void* stream) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(tn->ctx);
  if (x_next == nullptr || coef_row == nullptr || streams == nullptr)
    return fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_sample_step_clips: null pointer");
  if (!tn->lengths.empty() && static_cast<int>(tn->lengths.size()) != B)
    return fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_sample_step_clips: lengths were set for %d clips, the call has B=%d",
                static_cast<int>(tn->lengths.size()), B);
  DdpmClipStep step{x0_out, x_t, x_next, coef_row, reinterpret_cast<const unsigned long long*>(streams), draw, {}};
  const int rc = clip_plan(tn->ctx, B, tn->traj_dim, tn->T, true, tn->lengths.empty() ? nullptr : tn->lengths.data(),
                           &step.plan, offset_increments);
  if (rc != ROHM_OK) return rc;
  return trajnet_forward_or_step(tn, x_t, time, x0_out, B, stream, nullptr, &step);
}

extern "C" int rohm_trajnet_set_option(rohm_trajnet* tn, int option, int value) {
  if (tn == nullptr) return ROHM_ERR_INVALID;
  if (option == 0) {
    tn->graphs.enabled = value != 0;
    return ROHM_OK;
  }
  if (option == 1) {  // programmatic dependent launch along the convolution / GroupNorm chains (captured graphs are rebuilt)
    if (tn->use_pdl != (value != 0)) tn->graphs.clear();
    tn->use_pdl = value != 0;
    return ROHM_OK;
  }
  return fail(tn->ctx, ROHM_ERR_INVALID, "rohm_trajnet_set_option: unknown option %d", option);
}
