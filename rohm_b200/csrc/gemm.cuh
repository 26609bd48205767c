// Segmented-A GEMM on Hopper wgmma tensor cores with error-compensated hi/lo operand pairs for fp32-grade results.
//
//   C[m, n] = epilogue( sum_s sum_k A_s[m * row_mul_s + row_shift_s, k] * W[n, koff_s + k] )
//
// * A is a list of up to kMaxSegs "segments": each is a row-major matrix (given as a hi/lo pair: fp16 halves or TF32
//   values in fp32 containers, see GemmKind) read through its own TMA descriptor with a row shift.  One segment = a plain
//   linear layer (PoseNet, reference model/posenet.py:59-72).  Several segments = the taps of a Conv1d / the halves of a
//   channel concat (TrajNet, reference model/heads.py:90-106, model/trajnet.py:222-271): a k-tap convolution over
//   channels-last activations is k shifted copies of the same matrix, so no im2col buffer ever exists.  Out-of-range
//   rows/columns are zero-filled by TMA, which is exactly Conv1d's zero padding.
// * W is [N, K_total] K-major (torch Linear layout), also a hi/lo pair.  The roles are symmetric: the weight may just as
//   well be the A operand (transposed products, bias_per_row).
// * PASSES == 3: D += A_lo*W_hi + A_hi*W_lo + A_hi*W_hi  (drops only the lo*lo term, ~2^-22 relative).
//   PASSES == 1: D += A_hi*W_hi (plain TF32, ~2^-11 relative) -- the documented fast mode.
//
// * Split-K (GemmParams::k_splits, masked variant): a work item is a (tile, K range) pair; partial tiles are plain
//   fp32 stores at a per-split row offset and the consumer kernel adds them in split order (TrajNet's deep pyramid levels, where
//   6-22 row tiles with 40-80 K blocks each would otherwise leave most SMs idle or force 32-wide tiles).
//
// Kernel shape: persistent, grid = min(#work items, #SMs), 128 x BLOCK_N output tiles:
//   warpgroup 0   : TMA producer (one lane)             smem ring of (A + B) stages: full[]/empty[] mbarriers
//   warpgroups 1-2: wgmma, 64 rows each, accumulators in registers (two per thread with PASSES == 3); the finished tile
//                   goes to a shared-memory accumulator tile (acc_s), read back one row per thread by the epilogue: scale /
//                   bias / activation / row mask -> swizzled smem tile -> TMA bulk store, or per-thread stores with a
//                   residual.
//   Lean variants (no masks: every PoseNet launch), 512 threads: warpgroup 3 runs the epilogue while warpgroups 1-2 run
//   the next tile's MMAs (acc_full / acc_empty mbarriers around acc_s).  Masked (TrajNet) and skinning variants, 384
//   threads: warpgroups 1-2 run the epilogue after their MMAs.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace rohm {

constexpr int kSkinTileBones = 16;  // most distinct bones a 32-vertex column tile may touch (fused skinning epilogue)
constexpr int kGemmBlockM = 128;
// K extent of one pipeline stage in fp32 elements: 16 = 64-byte rows (SWIZZLE_64B).  Next to the shared-memory accumulator
// tile (66 KB at BLOCK_N = 128) and the epilogue staging tiles, the 227 KB of an H100 block hold three 32 KB stages of a
// 128-wide PASSES == 3 tile, where 128-byte rows (64 KB stages) would leave a single one.
constexpr int kGemmBlockK = 16;
constexpr int kMaxSegs = 10;

// Operand element type of a GEMM.  kKindTf32: fp32 containers holding TF32 hi/lo pairs (wgmma .tf32, 8 K-columns
// per instruction).  kKindF16: fp16 hi/lo pairs (wgmma .f16, 16 K-columns per instruction): the same 2 x 11 significant
// bits per value in half the bytes, so one 128-byte swizzle row -- one pipeline stage -- covers twice the K extent at the
// same tensor-pipe and shared-memory-fill cost.  Weights are pre-scaled by a power of two into the middle of the fp16
// range (GemmParams::acc_scale undoes it exactly in the epilogue); activations must stay below 1.3e5 in magnitude.
enum GemmKind : int { kKindTf32 = 0, kKindF16 = 1 };
// K extent of one pipeline stage in elements
__host__ __device__ constexpr int gemm_block_k(int kind) { return kind == kKindF16 ? 2 * kGemmBlockK : kGemmBlockK; }
__host__ __device__ constexpr int gemm_elem_bytes(int kind) { return kind == kKindF16 ? 2 : 4; }

enum GemmAct : int { kActNone = 0, kActGelu = 1, kActSilu = 2, kActMish = 3 };

struct alignas(64) GemmParams {
  CUtensorMap a_hi[kMaxSegs];
  CUtensorMap a_lo[kMaxSegs];
  // B must be constant for the lifetime of the launch chain (a packed weight matrix): the kernel requests its first B tiles
  // BEFORE griddepcontrol.wait, i.e. while the previous kernel of the stream may still be running
  CUtensorMap b_hi;
  CUtensorMap b_lo;
  int seg_kblocks[kMaxSegs];    // number of gemm_block_k(kind)-wide K blocks of this segment
  int seg_row_shift[kMaxSegs];  // A row coordinate = m0 * seg_row_mul + seg_row_shift
  int seg_row_mul[kMaxSegs];
  int num_segs;
  // ---- epilogue ----
  const float* bias;      // [N] (per output column) or, with bias_per_row, [M] (per output row); nullptr = none
  int bias_per_row;       // transposed products (C^T = W A^T): the bias follows the rows
  const float* residual;  // fp32 [*, ldr] added after the activation, or nullptr
  int ldr;
  float* out;  // fp32 [*, ldo] or nullptr
  int ldo;
  void* out_hi;  // hi/lo split of the result for a following GEMM (fp32 TF32 pairs or fp16 pairs, as the kind), or nullptr
  void* out_lo;
  int lds;        // pitch of out_hi / out_lo in elements
  float acc_scale;  // the accumulator is multiplied by this before the bias (0 = 1.0); kKindF16: 2^-s of the weight scale
  int act;
  int M;  // rows to store (rows >= M are never written)
  int N;  // columns to store
  int out_row_mul;  // output row = m * out_row_mul + out_row_add (transposed-conv phase interleave)
  int out_row_add;
  // Padded-clip layouts (TrajNet): rows are grouped in clips of clip_rows rows of which the first clip_valid
  // are real frames; the others are written as zeros so that they act as conv padding for the next layer.
  int clip_rows;  // 0 = disabled
  int clip_valid;
  // TMA-store epilogue (gemm_enable_tma_store): 32 x 32 output chunks go registers -> swizzled shared-memory tile ->
  // cp.async.bulk.tensor store.  Eligible launches: no residual, identity output row map (not the transposed-conv
  // phases), and either only `out` (fp32) or only an fp16 out_hi/out_lo pair.  Chunks on a ragged M or N edge still take
  // the per-thread path.
  CUtensorMap st_out;
  CUtensorMap st_hi;
  CUtensorMap st_lo;
  int tma_store;
  // ---- LayerNorm folding (PoseNet post-norm encoder layers; kKindF16, d_model = 512 = 8 x 64 columns) ----
  // The residual stream is kept UN-normalised: u = LN_prev(u_prev) + sublayer(.) is stored as an fp16 pair together with
  // per-row partial statistics, and x = LN(u) is never materialised:
  //  * the PRODUCER of u (out-proj / FFN2, `stats_out` != nullptr, BLOCK_N = 128, N = 512, output pair written in place
  //    over the residual pair through st_hi / st_lo) adds the residual tile -- optionally passed through the previous
  //    LayerNorm on the fly: (r - mean) rstd gamma + beta with `res_stats`, `res_gamma`, `res_beta` -- and writes, per thread,
  //    the (mean, M2) of its 64 columns of the row to stats_out[row][tile_n * 2 + half];
  //  * every CONSUMER GEMM of x = LN(u) (QKV, FFN1, output head; `a_stats` != nullptr) runs on the raw pair u with the
  //    LayerNorm scale folded into its weight, W'[n,k] = gamma_k W[n,k], and corrects in the epilogue:
  //      out[m,n] = rstd_m (acc[m,n] - mean_m c_n) + d_n,   c_n = sum_k W'[n,k] (`a_corr`),  d_n = b_n + sum_k beta_k W[n,k]
  //    (passed as `bias`).  (mean_m, rstd_m) come from Chan's combination of the row's 8 partials.
  // Statistics cross kernels through global memory; nothing waits inside a kernel.
  const float2* a_stats;    // [rows][8] partial (mean, M2) of the A rows, or nullptr
  const float* a_corr;      // [N]
  const float2* res_stats;  // [rows][8] partials of the residual rows, or nullptr: residual added as is
  const float* res_gamma;   // [N]
  const float* res_beta;    // [N]
  float2* stats_out;        // [rows][8], or nullptr: plain epilogue
  float ln_eps;
  // Linear-blend skinning in the epilogue (`skin_A` != nullptr; BLOCK_N = 96 = 32 vertices x 3, fp16 pairs): the
  // accumulator row of frame m is v_posed[m][32 vertices]; the epilogue applies  verts[m][v] = sum_b w[v][b] (R[m][b] v_posed +
  // t[m][b])  with the bone transforms skin_A [55][12][skin_lda frames] (row-major 3 x 4 per bone, translation folded in; frames contiguous:
  // one frame per lane = coalesced loads) and the per-tile tables
  // built by the host: skin_nb[tile] bones touched by the tile's 32 vertices, their indices skin_bone[tile][16] and the dense
  // weights skin_w[tile][16][32].  `out` (ldo = N = 3 V) receives the vertices; v_posed never exists in memory.
  const float* skin_A;
  int64_t skin_lda;  // frames per (bone, element) row of skin_A
  const int* skin_nb;
  const int* skin_bone;
  const float* skin_w;
  // Split-K (TrajNet convolutions on the deep pyramid levels; masked epilogue variant only): the K iterations of
  // every output tile are cut into `k_splits` contiguous ranges, one work item each, so that a level with 6 to 22 row tiles
  // still fills the SMs with 128-wide tiles.  Split s stores its fp32 partial tile (no bias) at output row
  // m + s * split_row_stride of `out`; the consumer (gn_mish_split_kernel) adds the partials in a fixed order, so the result is
  // deterministic.  0 / 1 = off.  Every range must be non-empty: (k_splits - 1) * ceil(iters / k_splits) < iters.
  int k_splits;
  int split_row_stride;
  // filled in by launch_gemm: extent of the tile grid
  int grid_m_rows;
  int grid_n_cols;
};

// Host side ------------------------------------------------------------------------------------
// Fills a 2-D fp32 tensor map: inner dim `cols` (contiguous), outer dim `rows`, row pitch `ld` elements,
// box = {gemm_block_k(kind), box_rows}, SWIZZLE_64B, zero OOB fill, optional row traversal stride.
// Returns 0 on success, a CUresult otherwise.
int make_tmap_2d(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows,
                 int row_elem_stride = 1, int kind = kKindTf32);

// Builds the store tensor maps of p for its current out / out_hi / out_lo pointers (rows_total = row capacity of those
// buffers) and sets p.tma_store when the launch is eligible (see GemmParams); otherwise clears it.  Returns 0 or a
// CUresult.
int gemm_enable_tma_store(GemmParams* p, int64_t rows_total, int kind);

// Tensor map for box_rows x 32-element TMA store boxes over a row-major [rows, cols] matrix with pitch ld: fp32 with
// SWIZZLE_128B (128-byte box rows) or fp16 with SWIZZLE_64B (64-byte box rows).  Returns 0 or a CUresult.
int make_store_tmap(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, bool half, int box_rows = 32);

// Tensor map for box_rows x 64-element fp16 load boxes (128-byte rows, SWIZZLE_128B) over a row-major [rows, cols] matrix
// with pitch ld: wgmma operand tiles of the attention kernel.  Returns 0 or a CUresult.
int make_tile_tmap_f16_sw128(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows);

// Launches the tile kernel.  block_n in {32, 64, 96, 128}; passes in {1, 3} (kKindF16: 3 only).
// grid = ceil(M_tiles) x ceil(N_tiles) where M_tiles covers `m_rows` GEMM rows.
cudaError_t launch_gemm(const GemmParams& p, int m_rows, int n_cols, int block_n, int passes, cudaStream_t stream,
                        bool pdl = false, int kind = kKindTf32);

// Raises the dynamic shared-memory limit of every kernel instantiation (call once per process, outside any stream
// capture).
cudaError_t gemm_init_attributes();

// fp32 -> (hi, lo) TF32 split, elementwise; n elements.
cudaError_t launch_split_tf32(const float* x, float* hi, float* lo, int64_t n, cudaStream_t stream);
// Power-of-two scale 2^s for storing a weight tensor as fp16 hi/lo pairs: max |w| 2^s lies in [2^13, 2^14), so every
// weight within 2^-13 of the largest keeps a normal-range lo half and nothing overflows (1.0 for an all-zero tensor).
// Synchronous (reads the maximum back); call at engine creation only.
cudaError_t f16_weight_scale(const float* w_dev, int64_t n, float* scale_out);

// fp32 -> (hi, lo) fp16 split of x * scale, elementwise; n elements.
cudaError_t launch_split_f16(const float* x, void* hi, void* lo, int64_t n, float scale, cudaStream_t stream);

}  // namespace rohm
