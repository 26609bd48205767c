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

#include "attention.cuh"
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
  // wgmma attention (F16X2, head dim 128, <= 160 tokens per clip; ROHM_B200_TC_ATTENTION=0 selects the mma.sync kernel)
  bool tc_attention = false;
  AttnWgmmaMaps attn_wg{};
  AttnArgs attn{};  // Q|K|V planes and context pair of every layer (B and S set per forward)
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

// Attention of one layer (attention.cu): the wgmma kernel when the engine prepared its tensor maps and the clip fits,
// else the mma.sync kernel of the operand kind, else (more than 160 tokens) the SIMT kernel.
static int run_attention(rohm_posenet* pn, int B, int S, cudaStream_t st) {
  AttnArgs a = pn->attn;
  a.B = B, a.S = S;
  prof_begin(pn, kCatAttention, st);
  const cudaError_t e = launch_attention(a, kAttnAuto, pn->tc_attention ? &pn->attn_wg : nullptr, st, pn->use_pdl && !pn->profiling);
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
      if (gemm_enable_tma_store(g, R, pn->kind) != 0) {
        const int rc__ = fail(ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (store map) failed");
        delete pn;
        return rc__;
      }
    }
  }
  if (gemm_enable_tma_store(&pn->g_out, R, pn->kind) != 0) {
    const int rc__ = fail(ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (store map) failed");
    delete pn;
    return rc__;
  }
#undef TRY

  // attention kernels need > 48 KB of dynamic shared memory
  const size_t smem_max = attention_smem_bytes(max_frames + 1, dh);
  if (smem_max > 227 * 1024) {
    delete pn;
    return fail(ctx, ROHM_ERR_INVALID, "clip too long for the attention kernel (%zu B smem)", smem_max);
  }
  {
    cudaError_t ea = gemm_init_attributes();
    if (ea == cudaSuccess) ea = attention_init_attributes(max_frames + 1, dh);
    if (ea != cudaSuccess) {
      delete pn;
      return fail(ctx, ROHM_ERR_CUDA, "kernel attribute setup failed: %s", cudaGetErrorString(ea));
    }
  }
  // attention: Q|K|V in QKV (fp16 kind: hi plane, then lo plane, sharing the fp32 buffer's footprint), context in CTXh / CTXl
  pn->attn.qkv_hi = pn->QKV;
  pn->attn.qkv_lo = reinterpret_cast<const __half*>(pn->QKV) + R * 3 * D;
  pn->attn.rows = R;
  pn->attn.ctx_hi = pn->CTXh, pn->attn.ctx_lo = pn->CTXl;
  pn->attn.D = D, pn->attn.H = pn->H;
  pn->attn.scale = 1.0f / sqrtf(static_cast<float>(dh));
  pn->attn.kind = pn->kind;
  if (pn->tc_attention) {
    const int rcm = attention_wgmma_maps(&pn->attn_wg, pn->attn);
    if (rcm != 0) {
      delete pn;
      return fail(ctx, ROHM_ERR_CUDA, "cuTensorMapEncodeTiled (attention tiles) failed (%d)", rcm);
    }
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
    if ((rc = run_attention(pn, B, S, st)) != ROHM_OK) return rc;
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
