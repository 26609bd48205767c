// Test-only entry points into the packed-clip paths of TrajNet's kernels: the GEMM epilogue with a per-row mask
// (GemmParams::row_mask, gemm.cu) and GroupNorm + Mish with a per-clip offset table (launch_gn_mish, groupnorm.cu).
// Driven from Python through ctypes by tests/trajnet_packed_probe.py and linked against the product's own objects.  Every
// function returns 0, a cudaError_t (> 0) or -CUresult of a failed tensor-map encoding; `reps` >= 1 launches run back to
// back on the default stream.
#include <cstdint>

#include "../../rohm_b200/csrc/gemm.cuh"
#include "../../rohm_b200/csrc/groupnorm.cuh"

using namespace rohm;

extern "C" {

// One-segment GEMM (a 1x1 convolution) through the masked epilogue: A [a_rows, a_cols] hi/lo with pitch a_ld, the packed
// weight pair [w_rows, w_cols], bias, activation and fp32 output; rows with row_mask[m] == 0 are stored as zeros.
struct ProbeMaskedGemm {
  int kind, passes, block_n;
  const void* a_hi;
  const void* a_lo;
  int64_t a_rows;
  int a_cols, a_ld, kblocks;
  const void* w_hi;
  const void* w_lo;
  int64_t w_rows;
  int w_cols;
  const float* bias;
  float* out;
  int ldo;
  float acc_scale;
  int act;
  int M, N;
  int clip_rows, clip_valid;  // the padded-clip rule; must be set (it selects the masked variant)
  const unsigned char* row_mask;
  int want_tma_store;  // ask gemm_enable_tma_store for the bulk-store epilogue over store_rows rows
  int64_t store_rows;
  int tma_store;  // set by the probe: what the library decided
};

int probe_gemm_row_mask(ProbeMaskedGemm* g, int reps) {
  if (reps < 1) return static_cast<int>(cudaErrorInvalidValue);
  GemmParams p{};
  int rc = make_tmap_2d(&p.a_hi[0], g->a_hi, g->a_rows, g->a_cols, g->a_ld, kGemmBlockM, 1, g->kind);
  if (rc == 0) rc = make_tmap_2d(&p.a_lo[0], g->a_lo, g->a_rows, g->a_cols, g->a_ld, kGemmBlockM, 1, g->kind);
  if (rc == 0) rc = make_tmap_2d(&p.b_hi, g->w_hi, g->w_rows, g->w_cols, g->w_cols, g->block_n, 1, g->kind);
  if (rc == 0) rc = make_tmap_2d(&p.b_lo, g->w_lo, g->w_rows, g->w_cols, g->w_cols, g->block_n, 1, g->kind);
  if (rc != 0) return -rc;
  p.num_segs = 1;
  p.seg_kblocks[0] = g->kblocks, p.seg_row_shift[0] = 0, p.seg_row_mul[0] = 1;
  p.bias = g->bias;
  p.out = g->out, p.ldo = g->ldo;
  p.acc_scale = g->acc_scale;
  p.act = g->act;
  p.M = g->M, p.N = g->N;
  p.out_row_mul = 1;
  p.clip_rows = g->clip_rows, p.clip_valid = g->clip_valid, p.row_mask = g->row_mask;
  if (g->want_tma_store && (rc = gemm_enable_tma_store(&p, g->store_rows, g->kind)) != 0) return -rc;
  g->tma_store = p.tma_store;
  cudaError_t e = cudaSuccess;
  for (int i = 0; i < reps && e == cudaSuccess; ++i) e = launch_gemm(p, g->M, g->N, g->block_n, g->passes, nullptr, false, g->kind);
  return static_cast<int>(e);
}

// GroupNorm + Mish over B packed clips (clip_off: device int[B + 1]) with clusters of n CTAs per (clip, group), the kernel's
// shared-memory limit raised to the slice first.
int probe_group_norm_packed(const GnArgs* a, const int* clip_off, int B, int n, int reps) {
  if (reps < 1 || B < 1 || clip_off == nullptr) return static_cast<int>(cudaErrorInvalidValue);
  cudaError_t e = gn_reserve_smem(gn_slice_bytes(a->T, a->C, a->groups, n));
  for (int i = 0; i < reps && e == cudaSuccess; ++i) e = launch_gn_mish(*a, B, n, nullptr, false, clip_off);
  return static_cast<int>(e);
}

}  // extern "C"
