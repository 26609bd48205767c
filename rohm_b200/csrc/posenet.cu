// PoseNet denoiser engine: the per-step transformer-encoder forward of RoHM's PoseNet
// (reference model/posenet.py:75-96, model/heads.py:112-176; torch nn.TransformerEncoderLayer post-norm, exact GELU).
//
// Token-major layout: every activation is a row-major [B*S, width] matrix, S = T + 1 tokens per clip (token 0 is the
// timestep embedding), clips contiguous.  With per-clip lengths (rohm_posenet_set_lengths) the clips are packed instead:
// clip b takes lengths[b] + 1 consecutive rows from clip_off[b], with no padding rows, so every GEMM runs over
// sum(lengths[b] + 1) rows.  Only attention crosses rows; everything else is per row and does not see the layout.  All linear layers run on the wgmma GEMM (gemm.cu); operands that feed a
// tensor-core product are kept as hi/lo pairs (fp16 halves by default, TF32 in the tf32 modes) written by the
// producing kernel's epilogue, so no separate conversion pass exists.
//
//   x_t [B,C,1,T] --pack--> A_in --GEMM(+bias+cond_embed+pe)--> X  (token 0 <- time-embedding table gather)
//   8 x { X --GEMM--> Q|K|V --attention (wgmma: S = QK^T, softmax on the fragments, O = PV)--> CTX --GEMM(+bias)--> Y
//         --LN(Y + X)--> X --GEMM(+bias,GELU)--> H --GEMM(+bias)--> Y --LN(Y + X)--> X }
//   X --GEMM--> OUT_tok --unpack(+copy cond[:, :traj])--> out [B,C,1,T]
// One forward = 45 launches, replayed as one CUDA graph with programmatic dependent launch along the chain.  With two or
// more uniform clips the layer chain runs as two clip groups on two streams (GroupPlan): pack, embedding and time token,
// then the two groups' 8 layers and output heads side by side, then unpack (+ the sampler update) for the whole batch.
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>

#include "attention.cuh"
#include "common.h"
#include "engine_kernels.cuh"
#include "gemm.cuh"
#include "graph.cuh"
#include "ptx.cuh"

namespace rohm {
namespace {

// ------------------------------------------------------------------------------------------------------------
// small kernels
// ------------------------------------------------------------------------------------------------------------

// First row and frame count of clip b: packed (clip_off[b], clip_off[b + 1] - clip_off[b] - 1) or uniform (b S, T).
__device__ __forceinline__ void clip_rows(const int* clip_off, int b, int S, int T, int64_t& row0, int& frames) {
  if (clip_off != nullptr) {
    row0 = clip_off[b];
    frames = clip_off[b + 1] - clip_off[b] - 1;
  } else {
    row0 = static_cast<int64_t>(b) * S;
    frames = T;
  }
}

// [B, C, T] (frames contiguous) -> token rows (row0(b) + 1 + t) of a [rows, ld] hi/lo pair, t < frames(b) (padded
// frames are never read).  32x32 smem transpose.
__global__ void pack_tokens_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo, int C,
                                   int T, int S, int ld, int f16, const int* __restrict__ clip_off) {
  __shared__ float tile[32][33];
  // programmatic dependent launch: the embedding GEMM behind this kernel may set itself up (barriers, weight tiles)
  // while it runs; as a dependent (a no-op for a plain launch) nothing is read before the previous kernel has completed
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;  // 32 x 8
  int64_t row0;
  int len;
  clip_rows(clip_off, b, S, T, row0, len);
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, t = t0 + tx;
    tile[j][tx] = (c < C && t < len) ? x[(static_cast<int64_t>(b) * C + c) * T + t] : 0.0f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int t = t0 + j, c = c0 + tx;
    if (t < len && c < C) {
      const float v = tile[tx][j];
      const int64_t o = (row0 + 1 + t) * ld + c;
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
constexpr size_t kPackTokensX = 0;  // the argument replaced on every replay of a cached forward graph

// Token rows -> [B, C, T]: channels [traj, traj+Cout) from tok[row0(b)+1+t][c - traj], channels [0, traj) from cond;
// frames at or past frames(b) are zero.
__global__ void unpack_tokens_kernel(const float* __restrict__ tok, const float* __restrict__ cond_traj,
                                     float* __restrict__ out, int C, int Cout, int traj, int T, int S, int ldt,
                                     const int* __restrict__ clip_off) {
  __shared__ float tile[32][33];
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();  // the output-head GEMM has completed
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;  // c0 indexes the Cout predicted channels
  const int tx = threadIdx.x, ty = threadIdx.y;
  int64_t row0;
  int len;
  clip_rows(clip_off, b, S, T, row0, len);
  for (int j = ty; j < 32; j += 8) {
    const int t = t0 + j, c = c0 + tx;
    tile[j][tx] = (t < len && c < Cout) ? tok[(row0 + 1 + t) * ldt + c] : 0.0f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, t = t0 + tx;
    if (c < Cout && t < T) out[(static_cast<int64_t>(b) * C + traj + c) * T + t] = tile[tx][j];
  }
  if (blockIdx.y == 0) {  // given trajectory channels are a verbatim copy of the condition (posenet.py:94-95)
    for (int c = ty; c < traj; c += 8) {
      const int t = t0 + tx;
      if (t < T) out[(static_cast<int64_t>(b) * C + c) * T + t] = t < len ? cond_traj[(static_cast<int64_t>(b) * traj + c) * T + t] : 0.0f;
    }
  }
}
constexpr size_t kUnpackTokensOut = 2;  // the argument replaced on every replay of a cached forward graph

// rows[row0(b) + s][:] = pe[s][:] for the frames(b) + 1 tokens of clip b = blockIdx.y (positional rows added to every
// token incl. the timestep token, posenet.py:90-91)
__global__ void pe_rows_kernel(const float* __restrict__ pe, float* __restrict__ rows, int T, int S, int D,
                               const int* __restrict__ clip_off) {
  int64_t row0;
  int len;
  clip_rows(clip_off, blockIdx.y, S, T, row0, len);
  const int d4 = D / 4;
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(len + 1) * d4) return;
  const int s = static_cast<int>(i / d4);
  const int c = static_cast<int>(i - static_cast<int64_t>(s) * d4);
  reinterpret_cast<float4*>(rows)[row0 * d4 + i] = reinterpret_cast<const float4*>(pe)[static_cast<int64_t>(s) * d4 + c];
}

// TimestepEmbedder (heads.py:132-146): e(t) = W2 silu(W0 pe[t] + b0) + b2 depends on the timestep only, so the whole
// table TE[t] = e(t) + pe[0] (the positional row of token 0) is computed once per weight set at create time (two GEMMs
// over all pe_len timesteps); per step the token row (b, 0) is a gather.
__global__ void time_token_gather_kernel(const int64_t* __restrict__ timesteps, const float* __restrict__ table,
                                         int table_rows, float* __restrict__ X, float* __restrict__ Xh,
                                         float* __restrict__ Xl, int S, int D, int f16, const int* __restrict__ clip_off) {
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();  // the embedding GEMM (which also writes row (b, 0)) has completed
  const int b = blockIdx.x;
  int64_t t = timesteps[b];
  // The reference indexes pe[timesteps] and raises on a bad index (heads.py:145).  A kernel cannot raise, so an
  // out-of-range timestep poisons the clip's timestep token with NaN (which attention spreads over the whole clip's
  // output) instead of being clamped to a plausible but wrong embedding.
  const bool bad = t < 0 || t >= table_rows;
  t = bad ? 0 : t;
  const float4* src = reinterpret_cast<const float4*>(table + t * D);
  const int64_t o = (clip_off != nullptr ? static_cast<int64_t>(clip_off[b]) : static_cast<int64_t>(b) * S) * D;
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
constexpr size_t kTimeTokenTimesteps = 0;  // the argument replaced on every replay of a cached forward graph

__global__ void add_vec_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ out, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i] + b[i];
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

// The launch parameters of the layer chain (L x {QKV, attention, out-proj, FFN1, FFN2} and the output head) over the
// workspace rows [row0, row0 + rows): the whole workspace, or one clip group of a split forward.  Every pointer starts at
// row0 and every tensor map's row extent ends at row0 + rows, so TMA loads past the end read zeros and TMA stores past it
// are clipped: the launches of one group never read or write another group's rows.
struct LayerChain {
  int64_t row0 = 0, rows = 0;
  std::vector<GemmParams> qkv, proj, ff1, ff2;
  GemmParams out{};
  AttnArgs attn{};  // Q|K|V planes and context pair (B and S set per launch)
  AttnWgmmaMaps attn_wg{};
};

// A forward of B uniform clips split into two clip groups, clips [0, split) and [split, B), whose layer chains run as two
// concurrent branches of the forward: the GEMMs of one group fill the SMs the other group's last wave leaves idle.
struct GroupPlan {
  int B = 0, T = 0, split = 0;
  LayerChain chain[2];
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
  // Per-clip lengths (rohm_posenet_set_lengths); empty: every clip has the call's T frames.  The clips are packed
  // (clip_off) and attention runs as up to two launches: the clips of at most 160 tokens on the 160-key wgmma kernel,
  // the longer ones on the streaming kernel, each clip on the kernel its own length picks when it runs alone.
  std::vector<int> lengths;
  std::vector<int> cond_lengths;  // the lengths set_cond embedded the condition with
  int* clip_off = nullptr;        // device [max_batch + 1]: first packed row of every clip, then the packed row count
  int* clip_ids = nullptr;        // device [max_batch]: the clips of at most 160 tokens, then the longer ones
  int packed_rows = 0, n_short = 0, short_tokens = 0, long_tokens = 0;
  int launches = 0;
  // CUDA graph of one forward per (B, T): 45 launches become one cudaGraphLaunch; the three nodes that touch caller
  // memory (pack: x_t, time-token gather: timesteps, unpack: out) get their pointers patched before every replay.
  ForwardGraphs graphs;
  bool use_pdl = true;
  // wgmma attention (F16X2, head dim 128): the maps serve both wgmma kernels; ROHM_B200_TC_ATTENTION=0 selects the
  // mma.sync kernel for clips of at most 160 tokens, longer clips always take the streaming wgmma kernel
  bool tc_attention = false;
  bool attn_maps = false;
  // LayerNorm folding (F16X2, d_model 512; ROHM_B200_FUSED_LN=0 keeps the separate layernorm_kernel): the residual stream
  // is stored un-normalised as an fp16 pair plus per-row partial statistics (stats1: after the attention sublayer, stats2:
  // after the feed-forward sublayer), LN(u) is never materialised: see GemmParams::stats_out / a_stats
  bool fused_ln = false;
  float2* stats1 = nullptr;
  float2* stats2 = nullptr;
  float *out_c = nullptr, *out_d = nullptr;  // output head: c_n, d_n of the folded last LayerNorm
  // optional per-kernel event timing (rohm_posenet_profile): category -> list of (start, stop) events
  bool profiling = false;
  std::vector<cudaEvent_t> prof_events;
  std::vector<int> prof_cat;
  // GEMM parameter blocks (tensor maps are built once; only the grid depends on B*S)
  GemmParams g_in{}, g_cond{};
  LayerChain whole;  // every workspace row: the serial chain (one clip group, packed clips, rohm_posenet_profile)
  // Two clip groups (GroupPlan) per (B, T), built on the first forward of the shape; the second group runs on `side`
  std::vector<std::unique_ptr<GroupPlan>> plans;
  cudaStream_t side = nullptr;
  BranchEvents forks;
  int num_sms = 0;
  int groups = 0;  // rohm_posenet_set_option(2): 0 = chosen from the input (use_groups), 1 = serial, 2 = two groups
  ~rohm_posenet() {
    if (side) cudaStreamDestroy(side);
  }
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
    if (launch_fold_ln(w, gamma, beta, bias, N, K, wf, *c, *d) != cudaSuccess)
      rc = fail(pn->ctx, ROHM_ERR_CUDA, "fold_ln_kernel launch failed");
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

static int run_ln(rohm_posenet* pn, const float* in, const float* res, const float* g, const float* b, float* out, float* oh,
           float* ol, int rows, cudaStream_t st) {
  prof_begin(pn, kCatLayerNorm, st);
  const int f16 = pn->kind == kKindF16 ? 1 : 0;
  const bool pdl = pn->use_pdl && !pn->profiling;
  if (launch_layernorm(pn->D, in, res, g, b, out, oh, ol, rows, f16, st, pdl) == cudaErrorInvalidValue)
    return fail(pn->ctx, ROHM_ERR_INVALID, "unsupported d_model %d for LayerNorm", pn->D);
  prof_end(pn, st);
  ROHM_CUDA(pn->ctx, cudaGetLastError());
  pn->launches++;
  return ROHM_OK;
}

// Attention of one layer (attention.cu): on fp16 pairs of head dim 128 the wgmma kernel up to 160 tokens (unless
// ROHM_B200_TC_ATTENTION=0) and the streaming wgmma kernel above; else the mma.sync kernel of the operand kind up to 160
// tokens and the SIMT kernel above.
static int run_attention(rohm_posenet* pn, const LayerChain& c, int B, int S, cudaStream_t st) {
  if (!pn->lengths.empty()) {  // packed clips: one launch per kernel that some clip's own length picks
    const int n_long = B - pn->n_short;
    for (int k = 0; k < 2; ++k) {
      AttnArgs a = c.attn;
      a.clip_off = pn->clip_off;
      a.clip_ids = pn->clip_ids + (k == 0 ? 0 : pn->n_short);
      a.B = k == 0 ? pn->n_short : n_long;
      a.S = k == 0 ? pn->short_tokens : pn->long_tokens;
      if (a.B == 0) continue;
      prof_begin(pn, kCatAttention, st);
      const cudaError_t e = launch_attention(a, k == 0 ? kAttnWgmma : kAttnWgmmaStream, &c.attn_wg, st,
                                             pn->use_pdl && !pn->profiling);
      prof_end(pn, st);
      ROHM_CUDA(pn->ctx, e);
      pn->launches++;
    }
    return ROHM_OK;
  }
  AttnArgs a = c.attn;
  a.B = B, a.S = S;
  const bool maps = pn->attn_maps && (pn->tc_attention || S > kAttnWgmmaMaxTokens);
  prof_begin(pn, kCatAttention, st);
  const cudaError_t e = launch_attention(a, kAttnAuto, maps ? &c.attn_wg : nullptr, st, pn->use_pdl && !pn->profiling);
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

// The launch parameters of the layer chain over workspace rows [row0, row0 + rows) (see LayerChain).
static int build_chain(rohm_posenet* pn, int64_t row0, int64_t rows, LayerChain* c) {
  const int D = pn->D, F = pn->F, eb = gemm_elem_bytes(pn->kind);
  const int64_t R = pn->max_rows;
  // row0 of a [*, ld] matrix of elements of `bytes` bytes
  auto at = [&](void* base, int64_t ld, int bytes) { return reinterpret_cast<float*>(static_cast<char*>(base) + row0 * ld * bytes); };
  float *Xh = at(pn->Xh, D, eb), *Xl = at(pn->Xl, D, eb), *CTXh = at(pn->CTXh, D, eb), *CTXl = at(pn->CTXl, D, eb);
  float *Hh = at(pn->Hh, F, eb), *Hl = at(pn->Hl, F, eb), *Y = at(pn->Y, D, 4), *OUT = at(pn->OUT, pn->Cout, 4);
  // Q | K | V: fp32 rows, or (fp16 kind) an fp16 hi plane followed by an fp16 lo plane in the fp32 buffer's footprint
  float* qkv_hi = at(pn->QKV, 3 * D, eb);
  float* qkv_lo = at(reinterpret_cast<__half*>(pn->QKV) + R * 3 * D, 3 * D, eb);
  float2* stats1 = pn->fused_ln ? pn->stats1 + row0 * 8 : nullptr;
  float2* stats2 = pn->fused_ln ? pn->stats2 + row0 * 8 : nullptr;
  c->row0 = row0, c->rows = rows;
  int rc;
  // Output head.
  if ((rc = setup_linear(pn, &c->out, Xh, Xl, rows, D, D, pn->w_out, pn->out_b)) != ROHM_OK) return rc;
  c->out.out = OUT, c->out.ldo = pn->Cout;
  if (pn->fused_ln && pn->L > 0)
    c->out.a_stats = stats2, c->out.a_corr = pn->out_c, c->out.bias = pn->out_d, c->out.ln_eps = 1e-5f;
  c->qkv.resize(pn->L), c->proj.resize(pn->L), c->ff1.resize(pn->L), c->ff2.resize(pn->L);
  for (int l = 0; l < pn->L; ++l) {
    PoseNetLayerDev& d = pn->layers[l];
    if ((rc = setup_linear(pn, &c->qkv[l], Xh, Xl, rows, D, D, d.qkv, d.qkv_b)) != ROHM_OK) return rc;
    if (pn->kind == kKindF16) {
      c->qkv[l].out_hi = qkv_hi, c->qkv[l].out_lo = qkv_lo, c->qkv[l].lds = 3 * D;
    } else {
      c->qkv[l].out = qkv_hi, c->qkv[l].ldo = 3 * D;
    }
    // the residual adds (x + sa_block(x), x + ff_block(x)) happen in the LayerNorm kernel that follows, which leaves
    // the GEMM epilogues free of global reads
    if ((rc = setup_linear(pn, &c->proj[l], CTXh, CTXl, rows, D, D, d.proj, d.proj_b)) != ROHM_OK) return rc;
    c->proj[l].out = Y, c->proj[l].ldo = D;
    // LayerNorm folding: producers write u in place over the residual pair + partial statistics; consumers correct
    auto producer = [&](GemmParams& g, float2* stats_out, const float2* res_stats, const float* res_gamma, const float* res_beta) {
      g.out = nullptr, g.ldo = 0;
      g.out_hi = Xh, g.out_lo = Xl, g.lds = D;
      g.stats_out = stats_out, g.res_stats = res_stats, g.res_gamma = res_gamma, g.res_beta = res_beta, g.ln_eps = 1e-5f;
    };
    auto consumer = [&](GemmParams& g, const float2* a_stats, const float* cv, const float* dvec) {
      g.a_stats = a_stats, g.a_corr = cv, g.bias = dvec, g.ln_eps = 1e-5f;
    };
    if (pn->fused_ln) {
      if (l > 0) consumer(c->qkv[l], stats2, d.qkv_c, d.qkv_d);
      // out-proj: u1 = LN2_prev(u2_prev) + attn   (layer 0: the embedded input, not normalised)
      producer(c->proj[l], stats1, l > 0 ? stats2 : nullptr, l > 0 ? pn->layers[l - 1].n2_w : nullptr,
               l > 0 ? pn->layers[l - 1].n2_b : nullptr);
    }
    if ((rc = setup_linear(pn, &c->ff1[l], Xh, Xl, rows, D, D, d.ff1, d.ff1_b)) != ROHM_OK) return rc;
    c->ff1[l].act = kActGelu;
    c->ff1[l].out_hi = Hh, c->ff1[l].out_lo = Hl, c->ff1[l].lds = F;
    if ((rc = setup_linear(pn, &c->ff2[l], Hh, Hl, rows, F, F, d.ff2, d.ff2_b)) != ROHM_OK) return rc;
    c->ff2[l].out = Y, c->ff2[l].ldo = D;
    if (pn->fused_ln) {
      consumer(c->ff1[l], stats1, d.ff1_c, d.ff1_d);
      producer(c->ff2[l], stats2, stats1, d.n1_w, d.n1_b);  // u2 = LN1(u1) + ffn
    }
    for (GemmParams* g : {&c->qkv[l], &c->proj[l], &c->ff1[l], &c->ff2[l]})
      if (gemm_enable_tma_store(g, rows, pn->kind) != 0) return fail(pn->ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (store map) failed");
  }
  if (gemm_enable_tma_store(&c->out, rows, pn->kind) != 0)
    return fail(pn->ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (store map) failed");
  AttnArgs& a = c->attn;
  a.qkv_hi = qkv_hi, a.qkv_lo = qkv_lo, a.rows = rows;
  a.ctx_hi = CTXh, a.ctx_lo = CTXl;
  a.D = D, a.H = pn->H;
  a.scale = 1.0f / sqrtf(static_cast<float>(D / pn->H));
  a.kind = pn->kind;
  if (pn->attn_maps && (rc = attention_wgmma_maps(&c->attn_wg, a)) != 0)
    return fail(pn->ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (attention tiles) failed (%d)", rc);
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
  if (max_frames + 1 > w->pe_len)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_create: %d frames need %d rows of the positional table, which has %d",
                max_frames, max_frames + 1, w->pe_len);
  // Clip length: fp16 pairs with head dim 128 stream K / V through the attention kernel and reach pe_len - 1 frames; the
  // TF32 precisions and head dim 64 run clips of more than 160 tokens on the SIMT kernel, whose K and V of the whole clip
  // must fit in shared memory (and at most 256 tokens).
  if (!(precision == ROHM_PRECISION_F16X2 && dh == 128)) {
    int simt_frames = kAttnSimtMaxTokens - 1;
    while (attention_smem_bytes(simt_frames + 1, dh) > kAttnSmemLimit) --simt_frames;
    if (max_frames > simt_frames)
      return fail(ctx, ROHM_ERR_INVALID,
                  "rohm_posenet_create: %d frames per clip: precision f16x2 with head dim 128 reaches pe_len - 1 = %d "
                  "frames; the tf32x3 / tf32 precisions and head dim 64 reach %d frames at head dim %d",
                  max_frames, w->pe_len - 1, simt_frames, dh);
  }

  rohm_posenet* pn = new (std::nothrow) rohm_posenet();
  if (pn == nullptr) return fail(ctx, ROHM_ERR_INVALID, "out of host memory");
  pn->ctx = ctx;
  pn->D = w->d_model, pn->F = w->ff_size, pn->L = w->num_layers, pn->H = w->num_heads;
  pn->C = w->in_feats, pn->Cout = w->out_feats, pn->traj = w->traj_feats, pn->pe_len = w->pe_len;
  pn->kind = precision == ROHM_PRECISION_F16X2 ? kKindF16 : kKindTf32;
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
    pn->fused_ln = pn->kind == kKindF16 && D == 512 && (env == nullptr || env[0] != '0');
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

  pn->clip_off = static_cast<int*>(pn->pool.bytes(static_cast<int64_t>(max_batch + 1) * sizeof(int)));
  pn->clip_ids = static_cast<int*>(pn->pool.bytes(static_cast<int64_t>(max_batch) * sizeof(int)));
  if (pn->clip_off == nullptr || pn->clip_ids == nullptr) {
    const int rc = fail(ctx, ROHM_ERR_CUDA, "clip table alloc failed: %s", cudaGetErrorString(pn->pool.last_error()));
    delete pn;
    return rc;
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
  // attention kernels need > 48 KB of dynamic shared memory
  {
    cudaError_t ea = gemm_init_attributes();
    if (ea == cudaSuccess) ea = attention_init_attributes(max_frames + 1, dh);
    if (ea != cudaSuccess) {
      delete pn;
      return fail(ctx, ROHM_ERR_CUDA, "kernel attribute setup failed: %s", cudaGetErrorString(ea));
    }
  }
  pn->attn_maps = pn->kind == kKindF16 && dh == 128;
  TRY(build_chain(pn, 0, R, &pn->whole));
#undef TRY
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&pn->num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaStreamCreateWithFlags(&pn->side, cudaStreamNonBlocking) != cudaSuccess) {
    delete pn;
    return fail(ctx, ROHM_ERR_CUDA, "stream creation failed");
  }
  const cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    delete pn;
    return fail(ctx, ROHM_ERR_CUDA, "weight packing failed: %s", cudaGetErrorString(e));
  }
  *out = pn;
  return ROHM_OK;
}

extern "C" void rohm_posenet_destroy(rohm_posenet* pn) { delete pn; }

extern "C" int rohm_posenet_launches_per_forward(const rohm_posenet* pn) { return pn ? pn->launches : 0; }

// The lengths set by rohm_posenet_set_lengths must describe the call's B clips of at most T frames.
static int check_lengths(rohm_posenet* pn, int B, int T, const char* fn) {
  if (pn->lengths.empty()) return ROHM_OK;
  if (static_cast<int>(pn->lengths.size()) != B)
    return fail(pn->ctx, ROHM_ERR_INVALID, "%s: lengths were set for %d clips, the call has B=%d", fn,
                static_cast<int>(pn->lengths.size()), B);
  for (int b = 0; b < B; ++b)
    if (pn->lengths[b] > T)
      return fail(pn->ctx, ROHM_ERR_INVALID, "%s: lengths[%d] = %d exceeds T=%d", fn, b, pn->lengths[b], T);
  return ROHM_OK;
}

extern "C" int rohm_posenet_set_cond(rohm_posenet* pn, const float* cond, int B, int T, void* stream) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (cond == nullptr || B <= 0 || T <= 0 || B > pn->max_batch || T > pn->max_frames)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_set_cond: B=%d T=%d outside the created capacity (%d, %d)", B, T,
                pn->max_batch, pn->max_frames);
  int rc = check_lengths(pn, B, T, "rohm_posenet_set_cond");
  if (rc != ROHM_OK) return rc;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int S = T + 1, D = pn->D;
  const bool packed = !pn->lengths.empty();
  const int* off = packed ? pn->clip_off : nullptr;
  const int rows = packed ? pn->packed_rows : B * S;
  // A_in <- tokens of cond (row (b,0) is never written: whatever it holds, the embedding GEMM's row (b,0) is overwritten
  // by the timestep token)
  dim3 grid((T + 31) / 32, (pn->C + 31) / 32, B);
  pack_tokens_kernel<<<grid, dim3(32, 8), 0, st>>>(cond, pn->Ain_h, pn->Ain_l, pn->C, T, S, pn->Kin_p,
                                                   pn->kind == kKindF16 ? 1 : 0, off);
  ROHM_CUDA(ctx, cudaGetLastError());
  const int64_t clip4 = static_cast<int64_t>(S) * D / 4;
  pe_rows_kernel<<<dim3(static_cast<unsigned>((clip4 + 255) / 256), B), 256, 0, st>>>(pn->pe, pn->condpe, T, S, D, off);
  ROHM_CUDA(ctx, cudaGetLastError());
  // condpe <- cond_embed(cond) + cond_b + pe rows   (in place; rows (b,0) become cond_b + pe[0]: overwritten later
  // by the timestep token, so their value is irrelevant)
  const int saved = pn->launches;
  rc = run_gemm(pn, pn->g_cond, pn->w_cond, rows, st);
  pn->launches = saved;
  if (rc != ROHM_OK) return rc;
  if (pn->traj > 0) {
    const size_t width = static_cast<size_t>(pn->traj) * T * sizeof(float);
    ROHM_CUDA(ctx, cudaMemcpy2DAsync(pn->cond_traj, width, cond, static_cast<size_t>(pn->C) * T * sizeof(float), width,
                                     B, cudaMemcpyDeviceToDevice, st));
  }
  pn->cond_B = B, pn->cond_T = T;
  pn->cond_lengths = pn->lengths;
  return ROHM_OK;
}

extern "C" int rohm_posenet_set_lengths(rohm_posenet* pn, const int* lengths, int B) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (lengths == nullptr) {
    pn->lengths.clear();
    return ROHM_OK;
  }
  if (!pn->attn_maps || !pn->tc_attention)
    return fail(ctx, ROHM_ERR_INVALID,
                "rohm_posenet_set_lengths: per-clip lengths run on the wgmma attention kernels: precision f16x2 with head "
                "dim 128 only (the tf32x3 / tf32 precisions, head dim 64 and ROHM_B200_TC_ATTENTION=0 are not supported)");
  if (B <= 0 || B > pn->max_batch)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_set_lengths: B=%d outside the created capacity %d", B, pn->max_batch);
  for (int b = 0; b < B; ++b)
    if (lengths[b] < 1 || lengths[b] > pn->max_frames)
      return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_set_lengths: lengths[%d] = %d outside [1, %d]", b, lengths[b],
                  pn->max_frames);
  std::vector<int> v(lengths, lengths + B);
  if (v == pn->lengths) return ROHM_OK;
  std::vector<int> off(B + 1), ids;
  int n_short = 0, short_tokens = 0, long_tokens = 0;
  off[0] = 0;
  for (int b = 0; b < B; ++b) off[b + 1] = off[b] + v[b] + 1;
  for (int pass = 0; pass < 2; ++pass)
    for (int b = 0; b < B; ++b) {
      const int S = v[b] + 1;
      const bool is_short = S <= kAttnWgmmaMaxTokens;
      if (is_short != (pass == 0)) continue;
      ids.push_back(b);
      if (is_short) ++n_short, short_tokens = S > short_tokens ? S : short_tokens;
      else long_tokens = S > long_tokens ? S : long_tokens;
    }
  // a forward still in flight on any stream may be reading the tables being replaced
  ROHM_CUDA(ctx, cudaDeviceSynchronize());
  ROHM_CUDA(ctx, cudaMemcpy(pn->clip_off, off.data(), (B + 1) * sizeof(int), cudaMemcpyHostToDevice));
  ROHM_CUDA(ctx, cudaMemcpy(pn->clip_ids, ids.data(), B * sizeof(int), cudaMemcpyHostToDevice));
  pn->lengths = std::move(v);
  pn->packed_rows = off[B];
  pn->n_short = n_short, pn->short_tokens = short_tokens, pn->long_tokens = long_tokens;
  return ROHM_OK;
}

// Layer l of a layer chain over `rows` rows (B clips of S tokens, or the packed clips).
static int run_layer(rohm_posenet* pn, LayerChain& c, int l, int B, int S, int rows, cudaStream_t st) {
  PoseNetLayerDev& d = pn->layers[l];
  int rc;
  if ((rc = run_gemm(pn, c.qkv[l], d.qkv, rows, st)) != ROHM_OK) return rc;
  if ((rc = run_attention(pn, c, B, S, st)) != ROHM_OK) return rc;
  if ((rc = run_gemm(pn, c.proj[l], d.proj, rows, st)) != ROHM_OK) return rc;
  const int64_t r0 = c.row0 * pn->D;
  const int eb = gemm_elem_bytes(pn->kind);
  float *X = pn->X + r0, *Y = pn->Y + r0;
  float* Xh = reinterpret_cast<float*>(reinterpret_cast<char*>(pn->Xh) + r0 * eb);
  float* Xl = reinterpret_cast<float*>(reinterpret_cast<char*>(pn->Xl) + r0 * eb);
  if (!pn->fused_ln && (rc = run_ln(pn, Y, X, d.n1_w, d.n1_b, X, Xh, Xl, rows, st)) != ROHM_OK) return rc;
  if ((rc = run_gemm(pn, c.ff1[l], d.ff1, rows, st)) != ROHM_OK) return rc;
  if ((rc = run_gemm(pn, c.ff2[l], d.ff2, rows, st)) != ROHM_OK) return rc;
  if (!pn->fused_ln && (rc = run_ln(pn, Y, X, d.n2_w, d.n2_b, X, Xh, Xl, rows, st)) != ROHM_OK) return rc;
  return ROHM_OK;
}

// Clip-aligned split of B clips of S tokens into two groups: the split with the fewest 128-row GEMM tiles over both
// groups, ties broken toward equal halves (32 x 145 tokens: 15 | 17 clips = 17 + 20 tiles, as many as the whole batch).
static int split_point(int B, int S) {
  int best = 1;
  int64_t best_tiles = -1;
  for (int k = 1; k < B; ++k) {
    const int64_t tiles = (static_cast<int64_t>(k) * S + kGemmBlockM - 1) / kGemmBlockM +
                          (static_cast<int64_t>(B - k) * S + kGemmBlockM - 1) / kGemmBlockM;
    if (best_tiles < 0 || tiles < best_tiles || (tiles == best_tiles && std::abs(2 * k - B) < std::abs(2 * best - B)))
      best = k, best_tiles = tiles;
  }
  return best;
}

// Whether a forward of B uniform clips of S tokens runs as two clip groups (see GroupPlan): when the whole batch's QKV
// GEMM, the widest of the layer, has more tiles than the GPU has SMs.  Below that every GEMM of the layer runs in one wave,
// no last wave leaves SMs idle for the other group to fill, and the second chain only adds launches (H100, T = 144: B = 8,
// 120 QKV tiles, runs 4 % slower split; B = 32 and 128 run 11 % and 7 % faster).
static bool use_groups(const rohm_posenet* pn, int B, int S) {
  const int64_t row_tiles = (static_cast<int64_t>(B) * S + kGemmBlockM - 1) / kGemmBlockM;
  const int64_t col_tiles = pn->L > 0 ? pn->layers[0].qkv.Np / pn->layers[0].qkv.block_n : 0;
  return row_tiles * col_tiles > pn->num_sms;
}

// The two-group plan of a forward of B clips of T frames, or nullptr for the serial chain: one clip, packed clips
// (per-clip lengths), rohm_posenet_profile (per-launch event timing needs one stream), or use_groups declines.
static int group_plan(rohm_posenet* pn, int B, int T, GroupPlan** plan) {
  *plan = nullptr;
  const int S = T + 1;
  const bool split = pn->groups == 2 || (pn->groups == 0 && use_groups(pn, B, S));
  if (B < 2 || !pn->lengths.empty() || pn->profiling || !split) return ROHM_OK;
  for (const auto& p : pn->plans)
    if (p->B == B && p->T == T) {
      *plan = p.get();
      return ROHM_OK;
    }
  std::unique_ptr<GroupPlan> p(new (std::nothrow) GroupPlan());
  if (p == nullptr) return fail(pn->ctx, ROHM_ERR_INVALID, "out of host memory");
  p->B = B, p->T = T, p->split = split_point(B, S);
  int rc = build_chain(pn, 0, static_cast<int64_t>(p->split) * S, &p->chain[0]);
  if (rc == ROHM_OK) rc = build_chain(pn, static_cast<int64_t>(p->split) * S, static_cast<int64_t>(B - p->split) * S, &p->chain[1]);
  if (rc != ROHM_OK) return rc;
  if (pn->plans.size() >= ForwardGraphs::kMaxGraphs) pn->plans.erase(pn->plans.begin());
  pn->plans.push_back(std::move(p));
  *plan = pn->plans.back().get();
  return ROHM_OK;
}

// The raw launch sequence of one forward (what gets captured into the graph).
static int forward_launches(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B, int T,
                            cudaStream_t st) {
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const int S = T + 1, D = pn->D;
  const bool packed = !pn->lengths.empty();
  const int* off = packed ? pn->clip_off : nullptr;
  const int rows = packed ? pn->packed_rows : B * S;
  pn->launches = 0;
  int rc;

  dim3 grid((T + 31) / 32, (pn->C + 31) / 32, B);
  prof_begin(pn, kCatOther, st);
  const bool pdl = pn->use_pdl && !pn->profiling;
  ROHM_CUDA(ctx, launch_chain(pack_tokens_kernel, grid, dim3(32, 8), 0, st, pdl, x_t, pn->Ain_h, pn->Ain_l, pn->C, T, S, pn->Kin_p,
                              pn->kind == kKindF16 ? 1 : 0, off));
  prof_end(pn, st);
  ROHM_CUDA(ctx, cudaGetLastError());
  pn->launches++;
  if ((rc = run_gemm(pn, pn->g_in, pn->w_in, rows, st)) != ROHM_OK) return rc;
  prof_begin(pn, kCatOther, st);
  ROHM_CUDA(ctx, launch_chain(time_token_gather_kernel, dim3(B), dim3(128), 0, st, pdl, timesteps, pn->time_table, pn->pe_len,
                              pn->X, pn->Xh, pn->Xl, S, D, pn->kind == kKindF16 ? 1 : 0, off));
  prof_end(pn, st);
  ROHM_CUDA(ctx, cudaGetLastError());
  pn->launches++;

  GroupPlan* plan = nullptr;
  if ((rc = group_plan(pn, B, T, &plan)) != ROHM_OK) return rc;
  if (plan == nullptr) {
    for (int l = 0; l < pn->L; ++l)
      if ((rc = run_layer(pn, pn->whole, l, B, S, rows, st)) != ROHM_OK) return rc;
    if ((rc = run_gemm(pn, pn->whole.out, pn->w_out, rows, st)) != ROHM_OK) return rc;
  } else {
    // fork after the time-token gather, join before unpack: group 0 runs on st, group 1 on the side stream
    const cudaStream_t gst[2] = {st, pn->side};
    const int clips[2] = {plan->split, B - plan->split};
    pn->forks.rewind();
    if ((rc = pn->forks.order_after(ctx, st, pn->side)) != ROHM_OK) return rc;
    for (int l = 0; l < pn->L; ++l)
      for (int g = 0; g < 2; ++g)
        if ((rc = run_layer(pn, plan->chain[g], l, clips[g], S, static_cast<int>(plan->chain[g].rows), gst[g])) != ROHM_OK)
          return rc;
    for (int g = 0; g < 2; ++g)
      if ((rc = run_gemm(pn, plan->chain[g].out, pn->w_out, static_cast<int>(plan->chain[g].rows), gst[g])) != ROHM_OK)
        return rc;
    if ((rc = pn->forks.order_after(ctx, pn->side, st)) != ROHM_OK) return rc;
  }
  dim3 grid_o((T + 31) / 32, (pn->Cout + 31) / 32, B);
  prof_begin(pn, kCatOther, st);
  ROHM_CUDA(ctx, launch_chain(unpack_tokens_kernel, grid_o, dim3(32, 8), 0, st, pdl, pn->OUT, pn->cond_traj, out, pn->C, pn->Cout,
                              pn->traj, T, S, pn->Cout, off));
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
  const int launches = pn->launches;  // launches_per_forward keeps describing the forward as it runs outside profiling
  int rc = rohm_posenet_forward(pn, x_t, timesteps, out, B, T, stream);
  pn->profiling = false;
  if (launches > 0) pn->launches = launches;
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

// One forward, with the ancestral update appended when `step` (rohm_posenet_sample_step) or `clip_step`
// (rohm_posenet_sample_step_clips) is given.
static int forward_or_step(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* out, int B, int T,
                           void* stream, const DdpmStep* step, const DdpmClipStep* clip_step = nullptr) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = pn->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (x_t == nullptr || timesteps == nullptr || out == nullptr)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_posenet_forward: null pointer");
  if (B != pn->cond_B || T != pn->cond_T)
    return fail(ctx, ROHM_ERR_STATE, "rohm_posenet_forward: B=%d T=%d but set_cond was called with B=%d T=%d", B, T,
                pn->cond_B, pn->cond_T);
  if (pn->lengths != pn->cond_lengths)
    return fail(ctx, ROHM_ERR_STATE, "rohm_posenet_forward: the clip lengths differ from those set_cond was called with");
  auto launches = [&](cudaStream_t st) {
    const int rc = forward_launches(pn, x_t, timesteps, out, B, T, st);
    if (rc != ROHM_OK || (step == nullptr && clip_step == nullptr)) return rc;
    pn->launches++;
    if (clip_step != nullptr) return launch_ddpm_clip_step(ctx, *clip_step, st, pn->use_pdl && !pn->profiling);
    return launch_ddpm_step(ctx, *step, st, pn->use_pdl && !pn->profiling);
  };
  std::vector<KernelPatch> patches = {{pack_tokens_kernel, arg<kPackTokensX>(x_t)},
                                      {time_token_gather_kernel, arg<kTimeTokenTimesteps>(timesteps)},
                                      {unpack_tokens_kernel, arg<kUnpackTokensOut>(out)}};
  if (step != nullptr) patches.push_back(ddpm_step_patch(*step));
  if (clip_step != nullptr) patches.push_back(ddpm_clip_step_patch(*clip_step));
  const StepKind kind = clip_step != nullptr ? kStepPerClip : step != nullptr ? kStepSingleStream : kNoStep;
  return pn->graphs.run(ctx, B, T, kind, pn->profiling, static_cast<cudaStream_t>(stream), launches, patches, pn->lengths);
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
  const int64_t clip_elems = static_cast<int64_t>(pn->C) * T;
  DdpmStep step{x0_out, x_t, x_next, clip_elems * B, clip_elems, coef_row, seed, offset};
  const int rc = ddpm_step_plan(pn->ctx, &step, offset_increment);
  if (rc != ROHM_OK) return rc;
  return forward_or_step(pn, x_t, timesteps, x0_out, B, T, stream, &step);
}

extern "C" int rohm_posenet_sample_step_clips(rohm_posenet* pn, const float* x_t, const int64_t* timesteps, float* x0_out,
                                              float* x_next, const float* coef_row, const uint64_t* streams, uint64_t draw,
                                              uint64_t* offset_increments, int B, int T, void* stream) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(pn->ctx);
  if (x_next == nullptr || coef_row == nullptr || streams == nullptr)
    return fail(pn->ctx, ROHM_ERR_INVALID, "rohm_posenet_sample_step_clips: null pointer");
  int rc = check_lengths(pn, B, T, "rohm_posenet_sample_step_clips");
  if (rc != ROHM_OK) return rc;
  DdpmClipStep step{x0_out, x_t, x_next, coef_row, reinterpret_cast<const unsigned long long*>(streams), draw, {}};
  rc = clip_plan(pn->ctx, B, pn->C, T, false, pn->lengths.empty() ? nullptr : pn->lengths.data(), &step.plan,
                 offset_increments);
  if (rc != ROHM_OK) return rc;
  return forward_or_step(pn, x_t, timesteps, x0_out, B, T, stream, nullptr, &step);
}

extern "C" int rohm_posenet_set_option(rohm_posenet* pn, int option, int value) {
  if (pn == nullptr) return ROHM_ERR_INVALID;
  if (option == 0) {
    pn->graphs.enabled = value != 0;
    return ROHM_OK;
  }
  if (option == 1) {  // programmatic dependent launch on the GEMMs (graphs are re-captured)
    if (pn->use_pdl != (value != 0)) pn->graphs.clear();
    pn->use_pdl = value != 0;
    return ROHM_OK;
  }
  if (option == 2) {  // clip groups: 0 = chosen from the input, 1 = the serial chain, 2 = two groups (graphs are re-captured)
    if (value < 0 || value > 2) return fail(pn->ctx, ROHM_ERR_INVALID, "rohm_posenet_set_option(2): value must be 0, 1 or 2");
    if (pn->groups != value) pn->graphs.clear();
    pn->groups = value;
    return ROHM_OK;
  }
  return fail(pn->ctx, ROHM_ERR_INVALID, "rohm_posenet_set_option: unknown option %d", option);
}
