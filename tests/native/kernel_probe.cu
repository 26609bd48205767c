// Test-only entry points into the GEMM, attention, GroupNorm and engine kernels (rohm_b200/csrc/gemm.cu, attention.cu,
// groupnorm.cu, engine_kernels.cu), the operand-pair helpers of ptx.cuh and the rotation / trajectory helpers of kin.cuh and repr.cuh, driven from Python through ctypes by tests/kernel_probe.py and
// linked against the product's own objects of those sources.  Every function takes plain structs / device pointers, builds the tensor maps itself with the library's own
// helpers and returns 0, a cudaError_t (> 0) or -CUresult of a failed tensor-map encoding.  Every launch goes to the default
// stream; the probes that take `reps` run their launch that many times back to back, set-up done once, so that tools can
// time them.  The product
// library (librohm_b200.so, include/rohm_b200.h) exports none of this.
#include <cstdint>

#include <algorithm>

#include "../../rohm_b200/csrc/attention.cuh"
#include "../../rohm_b200/csrc/engine_kernels.cuh"
#include "../../rohm_b200/csrc/gemm.cuh"
#include "../../rohm_b200/csrc/groupnorm.cuh"
#include "../../rohm_b200/csrc/kin.cuh"
#include "../../rohm_b200/csrc/repr.cuh"

using namespace rohm;

namespace {

// `reps` calls of launch(), stopping at the first error
template <class F>
int repeat(int reps, F launch) {
  cudaError_t rc = cudaSuccess;
  for (int i = 0; i < reps && rc == cudaSuccess; ++i) rc = launch();
  return static_cast<int>(rc);
}

// Every operand-pair form of ptx.cuh applied to the same elements, four per thread: the scalar fp16 split, the packed fp16x2
// and fp16x4 splits (element 2k in the low half of word k) and the TF32 pair the kernels write (hi = to_tf32(x), lo = x - hi).
__global__ void pair_forms_kernel(const float4* __restrict__ x, int64_t n4, __half* __restrict__ s_hi,
                                  __half* __restrict__ s_lo, uint32_t* __restrict__ x2_hi, uint32_t* __restrict__ x2_lo,
                                  uint2* __restrict__ x4_hi, uint2* __restrict__ x4_lo, float4* __restrict__ t_hi,
                                  float4* __restrict__ t_lo) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n4;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float4 v = x[i];
    ptx::split_f16(v.x, s_hi[4 * i], s_lo[4 * i]);
    ptx::split_f16(v.y, s_hi[4 * i + 1], s_lo[4 * i + 1]);
    ptx::split_f16(v.z, s_hi[4 * i + 2], s_lo[4 * i + 2]);
    ptx::split_f16(v.w, s_hi[4 * i + 3], s_lo[4 * i + 3]);
    ptx::split_f16x2(v.x, v.y, x2_hi[2 * i], x2_lo[2 * i]);
    ptx::split_f16x2(v.z, v.w, x2_hi[2 * i + 1], x2_lo[2 * i + 1]);
    ptx::split_f16x4(v, x4_hi[i], x4_lo[i]);
    float4 h, l;
    h.x = ptx::to_tf32(v.x), h.y = ptx::to_tf32(v.y), h.z = ptx::to_tf32(v.z), h.w = ptx::to_tf32(v.w);
    l.x = v.x - h.x, l.y = v.y - h.y, l.z = v.z - h.z, l.w = v.w - h.w;
    t_hi[i] = h, t_lo[i] = l;
  }
}

// The kin.cuh / repr.cuh helpers, one element per iteration of a grid-stride loop.  Matrices are row-major [9].
using kin::M3;
using kin::V3;

__device__ __forceinline__ M3 load_m3(const float* m) {
  return {{m[0], m[3], m[6]}, {m[1], m[4], m[7]}, {m[2], m[5], m[8]}};
}
__device__ __forceinline__ void store_m3(const M3& R, float* o) {
  o[0] = R.c0.x, o[1] = R.c1.x, o[2] = R.c2.x, o[3] = R.c0.y, o[4] = R.c1.y, o[5] = R.c2.y;
  o[6] = R.c0.z, o[7] = R.c1.z, o[8] = R.c2.z;
}
__device__ __forceinline__ V3 load_v3(const float* v) { return {v[0], v[1], v[2]}; }
__device__ __forceinline__ void store_v3(V3 v, float* o) { o[0] = v.x, o[1] = v.y, o[2] = v.z; }

enum KinOp { kOpRot6d, kOpRot6dBackward, kOpMatToAa, kOpRodrigues, kOpRoundTrip, kOpRotvec, kOpHeading, kOpQrotZ,
             kOpTraj };

// a: inputs of element i at a + i * in_stride, b: second input (G of the backward, v of qrot_z) at b + i * 9 or i * 3,
// o: outputs at o + i * out_stride, o2: the (l1, l2, s) triple of rot6d_to_mat at o2 + i * 3.
__global__ void kin_kernel(int op, const float* __restrict__ a, const float* __restrict__ b, int64_t n,
                           float* __restrict__ o, float* __restrict__ o2) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    switch (op) {
      case kOpRot6d: {
        float x[6], l1, l2, s;
        for (int e = 0; e < 6; ++e) x[e] = a[i * 6 + e];
        store_m3(kin::rot6d_to_mat(x, &l1, &l2, &s), o + i * 9);
        o2[i * 3] = l1, o2[i * 3 + 1] = l2, o2[i * 3 + 2] = s;
        break;
      }
      case kOpRot6dBackward: {
        float x[6], gx[6];
        for (int e = 0; e < 6; ++e) x[e] = a[i * 6 + e];
        kin::rot6d_backward(x, load_m3(b + i * 9), gx);
        for (int e = 0; e < 6; ++e) o[i * 6 + e] = gx[e];
        break;
      }
      case kOpMatToAa: store_v3(kin::mat_to_aa(load_m3(a + i * 9)), o + i * 3); break;
      case kOpRodrigues: store_m3(kin::rodrigues(load_v3(a + i * 3)), o + i * 9); break;
      case kOpRoundTrip: {
        float x[6];
        for (int e = 0; e < 6; ++e) x[e] = a[i * 6 + e];
        store_m3(kin::rodrigues(kin::mat_to_aa(kin::rot6d_to_mat(x))), o + i * 9);
        break;
      }
      case kOpRotvec: store_m3(repr::rotvec_to_mat(load_v3(a + i * 3)), o + i * 9); break;
      case kOpHeading: {
        const float* j = a + i * 12;  // joints 1, 2, 17, 16
        repr::heading_quat(load_v3(j), load_v3(j + 3), load_v3(j + 6), load_v3(j + 9), o[i * 3], o[i * 3 + 1],
                           o[i * 3 + 2]);
        break;
      }
      case kOpQrotZ: store_v3(repr::qrot_z(a[i * 2], a[i * 2 + 1], load_v3(b + i * 3)), o + i * 3); break;
      case kOpTraj: {
        // w0, z0, w1, z1, root(0), root(1), rot(0), rot(1) (row-major), tr(0), tr(1)
        const float* t = a + i * 34;
        repr::traj_channels(
            o + i * repr::kTrajFull, t[0], t[1], t[2], t[3], [&](int k) { return load_v3(t + 4 + 3 * k); },
            [&](int k) { return load_m3(t + 10 + 9 * k); }, [&](int k, int c) { return t[28 + 3 * k + c]; });
        break;
      }
    }
  }
}

__global__ void clip_of_frame_kernel(const int* __restrict__ clip_off, int B, const int* __restrict__ f, int64_t n,
                                     int* __restrict__ out) {
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x)
    out[i] = kin::clip_of_frame(clip_off, B, f[i]);
}

unsigned grid_for(int64_t n) {
  const int64_t blocks = (n + 255) / 256;
  return static_cast<unsigned>(blocks < 4096 ? blocks : 4096);
}

}  // namespace

extern "C" {

// One kin.cuh / repr.cuh helper over n elements (KinOp, layouts at kin_kernel); n = 0 launches nothing.
int probe_kin(int op, const float* a, const float* b, int64_t n, float* out, float* out2) {
  if (n < 0 || op < kOpRot6d || op > kOpTraj) return static_cast<int>(cudaErrorInvalidValue);
  if (n == 0) return 0;
  kin_kernel<<<grid_for(n), 256>>>(op, a, b, n, out, out2);
  return static_cast<int>(cudaGetLastError());
}

// kin::clip_of_frame(clip_off, B, f[i]) for n packed frame indices.
int probe_clip_of_frame(const int* clip_off, int B, const int* f, int64_t n, int* out) {
  if (n < 0 || B < 1) return static_cast<int>(cudaErrorInvalidValue);
  if (n == 0) return 0;
  clip_of_frame_kernel<<<grid_for(n), 256>>>(clip_off, B, f, n, out);
  return static_cast<int>(cudaGetLastError());
}

// One A segment: rows of a row-major hi/lo matrix [rows, cols] with pitch ld (elements), read at row m * row_mul + row_shift.
struct ProbeSeg {
  const void* hi;
  const void* lo;
  int64_t rows;
  int cols;
  int ld;
  int row_shift;
  int row_mul;
  int kblocks;  // gemm_block_k(kind)-wide K blocks of this segment in the packed weight
};

struct ProbeGemm {
  int kind, passes, block_n;
  int m_rows, n_cols;  // extent of the tile grid
  int num_segs;
  ProbeSeg seg[kMaxSegs];
  const void* w_hi;  // [w_rows, w_cols] K-major packed weight pair
  const void* w_lo;
  int64_t w_rows;
  int w_cols;
  const float* bias;
  const float* residual;
  int ldr;
  float* out;
  int ldo;
  void* out_hi;
  void* out_lo;
  int lds;
  float acc_scale;
  int act;
  int M, N;
  int out_row_mul, out_row_add;
  int clip_rows, clip_valid;
  const float* a_stats;  // float2 [rows][8]
  const float* a_corr;
  const float* res_stats;  // float2 [rows][8]
  const float* res_gamma;
  const float* res_beta;
  float* stats_out;  // float2 [rows][8]
  float ln_eps;
  int k_splits, split_row_stride;
  int want_tma_store;   // ask gemm_enable_tma_store for the bulk-store epilogue over store_rows rows
  int64_t store_rows;
  int pdl;
  // set by probe_gemm: what the library decided
  int tma_store;
  const unsigned char* row_mask;  // packed clips: rows with row_mask[m] == 0 are stored as zeros (NULL: none)
};

int probe_gemm(ProbeGemm* g, int reps) {
  if (reps < 1) return static_cast<int>(cudaErrorInvalidValue);
  GemmParams p{};
  for (int s = 0; s < g->num_segs; ++s) {
    const ProbeSeg& sg = g->seg[s];
    int rc = make_tmap_2d(&p.a_hi[s], sg.hi, sg.rows, sg.cols, sg.ld, kGemmBlockM, sg.row_mul, g->kind);
    if (rc == 0) rc = make_tmap_2d(&p.a_lo[s], sg.lo, sg.rows, sg.cols, sg.ld, kGemmBlockM, sg.row_mul, g->kind);
    if (rc != 0) return -rc;
    p.seg_kblocks[s] = sg.kblocks;
    p.seg_row_shift[s] = sg.row_shift;
    p.seg_row_mul[s] = sg.row_mul;
  }
  int rc = make_tmap_2d(&p.b_hi, g->w_hi, g->w_rows, g->w_cols, g->w_cols, g->block_n, 1, g->kind);
  if (rc == 0) rc = make_tmap_2d(&p.b_lo, g->w_lo, g->w_rows, g->w_cols, g->w_cols, g->block_n, 1, g->kind);
  if (rc != 0) return -rc;
  p.num_segs = g->num_segs;
  p.bias = g->bias;
  p.residual = g->residual, p.ldr = g->ldr;
  p.out = g->out, p.ldo = g->ldo;
  p.out_hi = g->out_hi, p.out_lo = g->out_lo, p.lds = g->lds;
  p.acc_scale = g->acc_scale;
  p.act = g->act;
  p.M = g->M, p.N = g->N;
  p.out_row_mul = g->out_row_mul, p.out_row_add = g->out_row_add;
  p.clip_rows = g->clip_rows, p.clip_valid = g->clip_valid, p.row_mask = g->row_mask;
  p.a_stats = reinterpret_cast<const float2*>(g->a_stats), p.a_corr = g->a_corr;
  p.res_stats = reinterpret_cast<const float2*>(g->res_stats), p.res_gamma = g->res_gamma, p.res_beta = g->res_beta;
  p.stats_out = reinterpret_cast<float2*>(g->stats_out), p.ln_eps = g->ln_eps;
  p.k_splits = g->k_splits, p.split_row_stride = g->split_row_stride;
  if (g->want_tma_store && (rc = gemm_enable_tma_store(&p, g->store_rows, g->kind)) != 0) return -rc;
  g->tma_store = p.tma_store;
  return repeat(reps, [&] { return launch_gemm(p, g->m_rows, g->n_cols, g->block_n, g->passes, nullptr, g->pdl != 0, g->kind); });
}

// The library's operand splits: fp32 -> TF32 pair (kind 0) or fp16 pair of x * scale (kind 1).
int probe_split(int kind, const float* x, void* hi, void* lo, int64_t n, float scale) {
  if (kind == kKindF16) return static_cast<int>(launch_split_f16(x, hi, lo, n, scale, nullptr));
  return static_cast<int>(launch_split_tf32(x, static_cast<float*>(hi), static_cast<float*>(lo), n, nullptr));
}

// The operand-pair helpers of ptx.cuh on n fp32 values (n a multiple of 4, 16-byte aligned buffers): f16_hi / f16_lo
// [3][n] halves from split_f16, split_f16x2 and split_f16x4 in that order, tf32_hi / tf32_lo [n] the TF32 pair.
int probe_pair_forms(const float* x, int64_t n, void* f16_hi, void* f16_lo, float* tf32_hi, float* tf32_lo) {
  if (n <= 0 || n % 4 != 0) return static_cast<int>(cudaErrorInvalidValue);
  __half* h = static_cast<__half*>(f16_hi);
  __half* l = static_cast<__half*>(f16_lo);
  const int64_t n4 = n / 4;
  const int threads = 256;
  const int64_t blocks = (n4 + threads - 1) / threads < 4096 ? (n4 + threads - 1) / threads : 4096;
  pair_forms_kernel<<<static_cast<unsigned>(blocks), threads>>>(
      reinterpret_cast<const float4*>(x), n4, h, l, reinterpret_cast<uint32_t*>(h + n), reinterpret_cast<uint32_t*>(l + n),
      reinterpret_cast<uint2*>(h + 2 * n), reinterpret_cast<uint2*>(l + 2 * n), reinterpret_cast<float4*>(tf32_hi),
      reinterpret_cast<float4*>(tf32_lo));
  return static_cast<int>(cudaGetLastError());
}

// The engines' weight scale for fp16 pairs (synchronous).
int probe_f16_weight_scale(const float* w, int64_t n, float* scale) {
  return static_cast<int>(f16_weight_scale(w, n, scale));
}

struct ProbeAttn {
  const void* qkv_hi;
  const void* qkv_lo;
  int64_t rows;
  void* ctx_hi;
  void* ctx_lo;
  int B, S, D, H;
  float scale;
  int kind;
  int which;  // AttnKernel
  int pdl;
  // Packed clips (NULL: B uniform clips of S tokens): clip c holds rows [clip_off[c], clip_off[c + 1]) and the launch runs
  // the B clips listed in clip_ids, S being the most tokens among them.  fp16 pairs of head dim 128, wgmma kernels only.
  const int* clip_off;
  const int* clip_ids;
};

// Clips of any length: the shared-memory limits of every attention kernel are raised for S tokens (the SIMT kernel's is
// capped at what it can serve), and the wgmma tensor maps are built for both wgmma kernels; whatever launch_attention
// cannot run, it refuses.
int probe_attention(const ProbeAttn* q, int reps) {
  AttnArgs a{};
  a.qkv_hi = q->qkv_hi, a.qkv_lo = q->qkv_lo, a.rows = q->rows;
  a.ctx_hi = q->ctx_hi, a.ctx_lo = q->ctx_lo;
  a.B = q->B, a.S = q->S, a.D = q->D, a.H = q->H;
  a.scale = q->scale, a.kind = q->kind;
  a.clip_off = q->clip_off, a.clip_ids = q->clip_ids;
  const bool packed = q->clip_off != nullptr;
  if (q->H <= 0 || q->D % q->H != 0 || reps < 1 || (packed && (q->kind != kKindF16 || q->D / q->H != 128)))
    return static_cast<int>(cudaErrorInvalidValue);
  const int dh = q->D / q->H;
  const cudaError_t e = attention_init_attributes(q->S, dh);
  if (e != cudaSuccess) return static_cast<int>(e);
  AttnWgmmaMaps maps;
  const AttnWgmmaMaps* wg = nullptr;
  if (packed || (q->kind == kKindF16 && dh == 128 &&
                 (q->which == kAttnWgmma || q->which == kAttnWgmmaStream || q->which == kAttnAuto))) {
    const int rc = attention_wgmma_maps(&maps, a);
    if (rc != 0) return -rc;
    wg = &maps;
  }
  return repeat(reps, [&] { return launch_attention(a, q->which, wg, nullptr, q->pdl != 0); });
}

// GroupNorm + Mish over B clips with clusters of n CTAs per (clip, group), the kernel's shared-memory limit raised to the
// slice first (so n = 1 also runs groups above the default 48 KB).  clip_off (device int[B + 1], NULL: clips at b * Tp):
// packed clips, as launch_gn_mish takes them.
int probe_group_norm(const GnArgs* a, int B, int n, int reps, const int* clip_off) {
  if (reps < 1 || B < 1) return static_cast<int>(cudaErrorInvalidValue);
  const cudaError_t e = gn_reserve_smem(gn_slice_bytes(a->T, a->C, a->groups, n));
  if (e != cudaSuccess) return static_cast<int>(e);
  return repeat(reps, [&] { return launch_gn_mish(*a, B, n, nullptr, false, clip_off); });
}

// The batch-invariant engines' GroupNorm + Mish of packed clips (launch_gn_mish_clip_slices), n >= 2 CTAs per (clip, group),
// with the dynamic shared memory run_gn (trajnet.cu) gives it: the largest slice of any clip's own cluster.  real_rows (host
// int[B]): clip b's real rows, clip_off[b + 1] - clip_off[b] - (Tp - T).
int probe_group_norm_clip_slices(const GnArgs* a, int B, int n, const int* real_rows, const int* clip_off, int reps) {
  if (reps < 1 || B < 1) return static_cast<int>(cudaErrorInvalidValue);
  size_t smem = 0;
  for (int b = 0; b < B; ++b) {
    const int Tc = real_rows[b];
    smem = std::max(smem, gn_slice_bytes(Tc, a->C, a->groups, gn_pick_cluster(Tc, a->C, a->groups, kGnClipBudget)));
  }
  return repeat(reps, [&] { return launch_gn_mish_clip_slices(*a, B, n, smem, nullptr, false, clip_off); });
}

// The cluster size rohm_trajnet_create chooses for a (clip, group) of T rows of C / groups channels; 0 on error.
int probe_group_norm_cluster(int T, int C, int groups) {
  size_t budget = 0, max_budget = 0;
  if (gn_smem_budgets(&budget, &max_budget) != cudaSuccess) return 0;
  return gn_pick_cluster(T, C, groups, budget);
}

// PoseNet's LayerNorm (layernorm_kernel<D>) of in + res over `rows` rows of D floats: fp32 out and the hi/lo pair (fp16
// when f16, else tf32 in fp32 containers).  res may be NULL or alias out.
int probe_layernorm(int D, const float* in, const float* res, const float* gamma, const float* beta, float* out, void* out_hi,
                    void* out_lo, int rows, int f16) {
  if (rows < 1) return static_cast<int>(cudaErrorInvalidValue);
  return static_cast<int>(launch_layernorm(D, in, res, gamma, beta, out, static_cast<float*>(out_hi),
                                           static_cast<float*>(out_lo), rows, f16, nullptr, false));
}

// LayerNorm folding (fold_ln_kernel) of a [N, K] weight: Wf [N, K], c [N], d [N].
int probe_fold_ln(const float* W, const float* gamma, const float* beta, const float* bias, int N, int K, float* Wf, float* c,
                  float* d) {
  if (N < 1 || K < 1) return static_cast<int>(cudaErrorInvalidValue);
  return static_cast<int>(launch_fold_ln(W, gamma, beta, bias, N, K, Wf, c, d));
}

// TrajNet's time path (trajnet_time_kernel) for the B timesteps time[0 .. B), ctas_per_clip CTAs per clip as gridDim.y, into
// tp [B, total_out]; table (NULL: every timestep evaluated directly) [table_rows, total_out].
int probe_trajnet_time(const int64_t* time, int B, int ctas_per_clip, int time_dim, const float* w1, const float* b1,
                       const float* w3, const float* b3, const float* wcat, const float* bcat, int total_out, float* tp,
                       const float* table, int table_rows) {
  if (B < 1 || ctas_per_clip < 1) return static_cast<int>(cudaErrorInvalidValue);
  trajnet_time_kernel<<<dim3(B, ctas_per_clip), 256, sizeof(float) * 6 * time_dim>>>(time, time_dim, w1, b1, w3, b3, wcat,
                                                                                      bcat, total_out, tp, table, table_rows);
  return static_cast<int>(cudaGetLastError());
}

// The split-K sum (sum_split_kernel) over `rows` rows of C channels; row_mask NULL: uniform clips of Tp rows, T real.
int probe_sum_split(const float* part, int splits, int64_t split_stride, const float* bias, float* out, void* out_hi,
                    void* out_lo, int C, int Tp, int T, int64_t rows, int f16, const unsigned char* row_mask) {
  if (rows < 1 || splits < 1 || splits > kMaxSplitsDev || C % 4 != 0) return static_cast<int>(cudaErrorInvalidValue);
  return static_cast<int>(launch_sum_split(part, splits, split_stride, bias, out, static_cast<float*>(out_hi),
                                           static_cast<float*>(out_lo), C, Tp, T, rows, f16, row_mask, nullptr, false));
}

}  // extern "C"
