// Test-only entry points into the GEMM and attention kernels (rohm_b200/csrc/gemm.cu, attention.cu), driven from Python
// through ctypes by tests/kernel_probe.py.  Every function takes plain structs / device pointers, builds the tensor maps
// itself with the library's own helpers and returns 0, a cudaError_t (> 0) or -CUresult of a failed tensor-map encoding.
// The product library (librohm_b200.so, include/rohm_b200.h) exports none of this.
#include <cstdint>

#include "../../rohm_b200/csrc/attention.cuh"
#include "../../rohm_b200/csrc/gemm.cuh"

using namespace rohm;

extern "C" {

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
  double* gn_stats;
  int gn_groups, gn_group_size;
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
  int want_multicast;   // ask gemm_enable_multicast (segment 0 is the A operand)
  int pdl;
  // set by probe_gemm: what the library decided
  int tma_store;
  int multicast;
};

int probe_gemm(ProbeGemm* g) {
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
  p.clip_rows = g->clip_rows, p.clip_valid = g->clip_valid;
  p.gn_stats = g->gn_stats, p.gn_groups = g->gn_groups, p.gn_group_size = g->gn_group_size;
  p.a_stats = reinterpret_cast<const float2*>(g->a_stats), p.a_corr = g->a_corr;
  p.res_stats = reinterpret_cast<const float2*>(g->res_stats), p.res_gamma = g->res_gamma, p.res_beta = g->res_beta;
  p.stats_out = reinterpret_cast<float2*>(g->stats_out), p.ln_eps = g->ln_eps;
  p.k_splits = g->k_splits, p.split_row_stride = g->split_row_stride;
  if (g->want_tma_store && (rc = gemm_enable_tma_store(&p, g->store_rows, g->kind)) != 0) return -rc;
  if (g->want_multicast) {
    const ProbeSeg& s0 = g->seg[0];
    rc = gemm_enable_multicast(&p, s0.hi, s0.lo, s0.rows, s0.cols, s0.ld, g->n_cols, g->block_n, g->kind);
    if (rc != 0) return -rc;
  }
  g->tma_store = p.tma_store;
  g->multicast = p.multicast_a;
  return static_cast<int>(launch_gemm(p, g->m_rows, g->n_cols, g->block_n, g->passes, nullptr, g->pdl != 0, g->kind));
}

// The library's operand splits: fp32 -> TF32 pair (kind 0) or fp16 pair of x * scale (kind 1).
int probe_split(int kind, const float* x, void* hi, void* lo, int64_t n, float scale) {
  if (kind == kKindF16) return static_cast<int>(launch_split_f16(x, hi, lo, n, scale, nullptr));
  return static_cast<int>(launch_split_tf32(x, static_cast<float*>(hi), static_cast<float*>(lo), n, nullptr));
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
};

int probe_attention(const ProbeAttn* q) {
  AttnArgs a{};
  a.qkv_hi = q->qkv_hi, a.qkv_lo = q->qkv_lo, a.rows = q->rows;
  a.ctx_hi = q->ctx_hi, a.ctx_lo = q->ctx_lo;
  a.B = q->B, a.S = q->S, a.D = q->D, a.H = q->H;
  a.scale = q->scale, a.kind = q->kind;
  if (q->H <= 0 || q->D % q->H != 0) return static_cast<int>(cudaErrorInvalidValue);
  const int dh = q->D / q->H;
  // the SIMT kernel's shared memory grows with the clip; anything it cannot hold is refused by launch_attention
  if (attention_smem_bytes(q->S, dh) <= 227 * 1024) {
    const cudaError_t e = attention_init_attributes(q->S, dh);
    if (e != cudaSuccess) return static_cast<int>(e);
  }
  AttnWgmmaMaps maps;
  const AttnWgmmaMaps* wg = nullptr;
  if (q->kind == kKindF16 && dh == 128 && (q->which == kAttnWgmma || q->which == kAttnAuto)) {
    const int rc = attention_wgmma_maps(&maps, a);
    if (rc != 0) return -rc;
    wg = &maps;
  }
  return static_cast<int>(launch_attention(a, q->which, wg, nullptr, q->pdl != 0));
}

}  // extern "C"
