// wgmma / TMA implementation of the segmented-A hi/lo-pair GEMM declared in gemm.cuh.
#include "gemm.cuh"
#include "ptx.cuh"

#include <cudaTypedefs.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>

namespace rohm {

namespace {

// Warp roles.  Warpgroup 0: TMA producer (one lane).  Warpgroups 1, 2 (warps 4-11): wgmma, 64 tile rows each.
// EPI 0, 1, 3 (the lean variants the PoseNet forward runs): warpgroup 3 (warps 12-15) is a dedicated epilogue, one tile row
// per thread, so the MMA warpgroups go straight on to the next tile's K loop while it runs (512 threads).
// EPI 2 / 5 (TrajNet: split-K, activations, padded or packed clips) and EPI 4 (skinning, ~168 registers per epilogue thread): the MMA
// warpgroups run the epilogue themselves, after the tile's MMAs (384 threads) -- these epilogues do not fit the register
// budget of an epilogue warpgroup next to two MMA warpgroups.
constexpr int kFirstMmaWarp = 4;
constexpr int kMmaWarps = 8;
constexpr int kFirstEpiWarp = kFirstMmaWarp + kMmaWarps;  // the dedicated epilogue warpgroup
__host__ __device__ constexpr bool epi_role(int epi) { return epi == 0 || epi == 1 || epi == 3; }
__host__ __device__ constexpr int kernel_threads(int epi) { return 32 * (kFirstEpiWarp + (epi_role(epi) ? 4 : 0)); }
// setmaxnreg budgets of the 512-thread variants: producer + epilogue + 2 x MMA <= 65536 / 128 registers per thread
// (a launch starts every thread at 65536 / 512 = 128: the producer gives registers back, the other roles take them)
constexpr int kProducerRegs = 40, kEpiRoleRegs = 152, kMmaRegs = 160;
static_assert(kProducerRegs + kEpiRoleRegs + 2 * kMmaRegs <= 512, "register file of one SM");
static_assert(kProducerRegs <= 128 && kEpiRoleRegs >= 128 && kMmaRegs >= 128, "setmaxnreg.dec / .inc direction");
constexpr int kSmemLimit = 227 * 1024;  // H100: dynamic + static shared memory of one block
constexpr int kStaticSmemReserve = 8 * 1024;  // barriers, per-column vectors, skinning tables
constexpr int kEpiTileFloats = 32 * 32;   // per-epilogue-warp staging tile (32 x 32, XOR-swizzled columns): coalesced stores
// fused skinning epilogue (EPI 4): one 128 x 96 fp32 staging tile for the whole CTA.  Pitch 100 floats: the 16-byte
// row-per-thread writes (8 lanes per wavefront hit 8 distinct 16-byte bank groups: 25 r mod 8) and the 4-byte row-contiguous
// reads are both conflict-free
constexpr int kSkinPitch = 100;
constexpr int kSkinStageBytes = kGemmBlockM * kSkinPitch * 4;

template <int BLOCK_N, int PASSES, bool EPI_ROLE>
struct TileCfg {
  static constexpr int kEpiWarps = EPI_ROLE ? 4 : 8;  // warps that run the epilogue, 32 tile rows each
  static constexpr int kABytes = kGemmBlockM * kGemmBlockK * 4;
  static constexpr int kBBytes = BLOCK_N * kGemmBlockK * 4;
  static constexpr int kSplit = (PASSES == 3) ? 2 : 1;
  static constexpr int kStageBytes = kSplit * (kABytes + kBBytes);
  // The finished accumulator tile goes registers -> shared memory (fp32, 128 x BLOCK_N, pitch BLOCK_N + 4: the fragment
  // writes and the row-per-thread 16-byte reads of the epilogue are at most 2-way conflicted) -> one row per thread.
  static constexpr int kAccPitch = BLOCK_N + 4;
  static constexpr int kAccBytes = kGemmBlockM * kAccPitch * 4;
  // the epilogue staging area: per-warp 32 x 32 tiles, or (BLOCK_N = 96, 384-thread variants) the skinning epilogue's
  // CTA-wide tile.  The four epilogue-warpgroup tiles leave room for 4 stages at BLOCK_N = 128 (3 with eight tiles).
  static constexpr int kEpiBytes = !EPI_ROLE && BLOCK_N == 96 && kSkinStageBytes > kEpiWarps * kEpiTileFloats * 4
                                       ? kSkinStageBytes
                                       : kEpiWarps * kEpiTileFloats * 4;
  static constexpr int kStagesRaw = (kSmemLimit - kStaticSmemReserve - 1024 - kAccBytes - kEpiBytes) / kStageBytes;
  static constexpr int kStages = kStagesRaw > 10 ? 10 : kStagesRaw;
  static constexpr int kSmemBytes = kStages * kStageBytes + 1024 + kAccBytes + kEpiWarps * kEpiTileFloats * 4;
  // PASSES == 3 keeps two register accumulators: one takes the leading hi*hi products, the other the two small cross
  // terms.  The tensor core truncates when it adds into the accumulator, so keeping the ~2^-11-sized terms out of the big
  // sum cuts the rounding count of the main accumulator by 3x.  They are added once, when the tile leaves the registers.
  static constexpr int kAccRegs = BLOCK_N / 2;  // per thread and accumulator: m64 x BLOCK_N over a warpgroup
  static_assert(kStages >= 2, "need at least a double buffer");
  static_assert(BLOCK_N % 32 == 0 && BLOCK_N >= 32 && BLOCK_N <= 128, "wgmma N and the epilogue's 32-column chunks");
};

// One wgmma step of the operand kind on an m64 x BLOCK_N accumulator.
template <int KIND, int R>
__device__ __forceinline__ void mma_step(float (&d)[R], uint64_t a, uint64_t b) {
  if constexpr (KIND == kKindF16) ptx::wgmma_f16(d, a, b);
  else ptx::wgmma_tf32(d, a, b);
}

// N consecutive accumulator columns of one row out of the shared-memory accumulator tile
template <int PITCH, int N>
__device__ __forceinline__ void acc_load(const float* acc, int row, int col, float (&v)[N]) {
  const float4* src = reinterpret_cast<const float4*>(acc + row * PITCH + col);
#pragma unroll
  for (int j = 0; j < N / 4; ++j) {
    const float4 t = src[j];
    v[4 * j] = t.x, v[4 * j + 1] = t.y, v[4 * j + 2] = t.z, v[4 * j + 3] = t.w;
  }
}

__device__ __forceinline__ float apply_act(float x, int act) {
  if (act == kActGelu) {
    return 0.5f * x * (1.0f + erff(x * 0.70710678118654752440f));  // exact (erf) GELU, nn.GELU default
  } else if (act == kActSilu) {
    return x / (1.0f + expf(-x));
  } else if (act == kActMish) {
    // x * tanh(softplus(x)); softplus with torch's threshold=20
    float sp = x > 20.0f ? x : log1pf(expf(x));
    return x * tanhf(sp);
  }
  return x;
}

// Exact (erf) GELU, nn.GELU's default, as x Phi(x) = max(x, 0) - |x| Phi(-|x|) with Phi(-u) = 2^Q(u): one degree-8
// polynomial in u = min(|x|, 6.5), one MUFU.EX2, no erf branches -- 12 instructions per element (the two-branch erf form
// it replaces took 28, and the FFN1 epilogue is bound by the FP32 pipe).  Only the absolute error of |x| Phi(-|x|) matters,
// so Q is a least-squares fit of log2 Phi(-u) weighted by u Phi(-u) (tools/fit_gelu_erf.py); max |error| of the whole GELU
// against float64: 2.5e-7, i.e. the rounding of the result (the fp32 erff formulation: 4.5e-7).  Below x = -6.5 the clamp
// takes the tail |x| Phi(-|x|) as |x| 2^Q(6.5) = 3.5e-11 |x|, which adds up to that much: the 2.5e-7 holds for |x| up to
// about 7000, beyond it the error stays below 3.6e-11 |x|, far under one ulp of x (tests/test_gpu_operand_pairs.py).
__device__ __forceinline__ float gelu_erf(float x) {
  const float u = fminf(fabsf(x), 6.5f);
  float q = -1.657032612e-06f;
  q = fmaf(q, u, 2.461445729e-05f);
  q = fmaf(q, u, -1.118122309e-04f);
  q = fmaf(q, u, -3.311361652e-04f);
  q = fmaf(q, u, 7.346248254e-03f);
  q = fmaf(q, u, -5.272617936e-02f);
  q = fmaf(q, u, -4.591094553e-01f);
  q = fmaf(q, u, -1.151124716e+00f);
  q = fmaf(q, u, -9.999987483e-01f);
  float p;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(p) : "f"(q));
  return fmaf(-fabsf(x), p, fmaxf(x, 0.0f));
}

// fused skinning epilogue: the 3 x 4 transform of one bone for this thread's frame, from the [bone][12][frames] table
__device__ __forceinline__ void load_bone_transform(const float* frame_col, int64_t lda, int bone, float4& r0, float4& r1,
                                                    float4& r2) {
  const float* a = frame_col + static_cast<int64_t>(bone) * 12 * lda;
  r0 = make_float4(__ldg(a), __ldg(a + lda), __ldg(a + 2 * lda), __ldg(a + 3 * lda));
  r1 = make_float4(__ldg(a + 4 * lda), __ldg(a + 5 * lda), __ldg(a + 6 * lda), __ldg(a + 7 * lda));
  r2 = make_float4(__ldg(a + 8 * lda), __ldg(a + 9 * lda), __ldg(a + 10 * lda), __ldg(a + 11 * lda));
}

struct EpiParams {
  const float* bias;
  const float* residual;
  const float2* a_stats;
  const float* a_corr;
  const float2* res_stats;
  const float* res_gamma;
  const float* res_beta;
  float2* stats_out;
  float ln_eps;
  float* out;
  void* out_hi;
  void* out_lo;
  float acc_scale;
  int tma_store;
  int bias_per_row;
  int ldr, ldo, lds, act, M, N, out_row_mul, out_row_add, clip_rows, clip_valid;
};

// (mean, rstd) of a 512-wide row from its 8 partial (mean_i, M2_i) over 64 columns each (Chan et al. pairwise combination);
// row8: 64 contiguous bytes in global memory, written by the previous kernel.
__device__ __forceinline__ float2 combine_row_stats(const float2* row8, float eps) {
  const float4* q4 = reinterpret_cast<const float4*>(row8);
  float4 t[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) t[i] = __ldcg(q4 + i);
  const float mean = ((t[0].x + t[0].z) + (t[1].x + t[1].z) + (t[2].x + t[2].z) + (t[3].x + t[3].z)) * 0.125f;
  float m2 = 0.0f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float d0 = t[i].x - mean, d1 = t[i].z - mean;
    m2 += fmaf(64.0f * d0, d0, t[i].y) + fmaf(64.0f * d1, d1, t[i].w);
  }
  return make_float2(mean, rsqrtf(m2 * (1.0f / 512.0f) + eps));
}

// One 32 x 32 chunk (row per lane) as an fp16 hi/lo pair: registers -> two SWIZZLE_64B planes of the warp's staging tile
// (hi at +0, lo at +2048; chunk c of row r at slot c ^ ((r >> 1) & 3)) -> two TMA bulk stores.
__device__ __forceinline__ void stage_pair_chunk(const float (&v)[32], uint8_t* tb, int lane, const CUtensorMap* st_hi,
                                                 const CUtensorMap* st_lo, int col0, int row0) {
  if (lane == 0) ptx::bulk_wait_read_all();  // an earlier bulk store may still be reading the tile
  __syncwarp();
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    uint2 h0, l0, h1, l1;
    ptx::split_f16x4(make_float4(v[8 * c], v[8 * c + 1], v[8 * c + 2], v[8 * c + 3]), h0, l0);
    ptx::split_f16x4(make_float4(v[8 * c + 4], v[8 * c + 5], v[8 * c + 6], v[8 * c + 7]), h1, l1);
    const int off = lane * 64 + ((c ^ ((lane >> 1) & 3)) << 4);
    *reinterpret_cast<uint4*>(tb + off) = make_uint4(h0.x, h0.y, h1.x, h1.y);
    *reinterpret_cast<uint4*>(tb + 2048 + off) = make_uint4(l0.x, l0.y, l1.x, l1.y);
  }
  ptx::fence_proxy_async();
  __syncwarp();
  if (lane == 0) {
    ptx::tma_store_2d(st_hi, tb, col0, row0);
    ptx::tma_store_2d(st_lo, tb + 2048, col0, row0);
    ptx::bulk_commit();
  }
}

// Persistent, warp-specialised: grid = min(#tiles, #SMs); every CTA walks tiles blockIdx.x, +gridDim.x, ...
// (N-tile index fastest, so CTAs running concurrently share the same A rows in L2).
// Epilogue variants: 0 = bias + residual + fp32 / hi-lo stores (the PoseNet linears), 1 = the same + exact GELU (FFN1),
// 2 = everything (other activations, padded-clip row masks, split-K partials: TrajNet), 3 = bias + residual pair +
// LayerNorm with the row statistics exchanged between the four column-tile CTAs of a row stripe (PoseNet out-proj / FFN2,
// see GemmParams::ln_gamma).  Separate instantiations keep the hot variants' code small (the full
// epilogue is ~7000 SASS instructions, most of them predicated-off activation code when unused).
//
// EPI 0 / 1 / 3 hand the finished accumulator tile over through acc_s and two mbarriers: the MMA warpgroups wait on
// acc_empty (the epilogue has read the previous tile) before they write acc_s, then arrive on acc_full and start the next
// work item's K loop; the epilogue warpgroup stages the next tile's per-column vectors, row statistics and (EPI 3) residual
// while those MMAs run, waits on acc_full, and arrives on acc_empty once it has read the tile.
template <int BLOCK_N, int PASSES, int EPI, int KIND>
__global__ void __launch_bounds__(kernel_threads(EPI), 1) gemm_tile_kernel(const __grid_constant__ GemmParams p) {
  // EPI: 0 bias / stores, 1 + exact GELU, 2 everything (TrajNet), 3 LayerNorm-folding producer, 4 skinning, 5 = 2 with the
  // pad rows given by GemmParams::row_mask (TrajNet on packed clips; a separate instance keeps 2's code as it is)
  constexpr bool LEAN = EPI != 2 && EPI != 5;
  constexpr bool EPI_ROLE = epi_role(EPI);  // a dedicated epilogue warpgroup (see kFirstMmaWarp)
  constexpr int kElemK = gemm_block_k(KIND);  // K elements per pipeline stage (TMA coordinates are in elements)
  using Cfg = TileCfg<BLOCK_N, PASSES, EPI_ROLE>;
  constexpr int kEpiWarps = Cfg::kEpiWarps;
  extern __shared__ uint8_t smem_raw[];
  __shared__ uint64_t full_bar[Cfg::kStages];
  __shared__ uint64_t empty_bar[Cfg::kStages];
  // Epilogue parameters are copied from the (3 KB, tensor-map dominated) kernel parameter block into shared memory
  // once: reading them late from the constant bank is slow on first touch.
  __shared__ EpiParams epi_s;
  // per-column vectors of the current tile (single-buffered, see the staging block of the epilogue): bias; LayerNorm
  // folding: c_n of a consumer GEMM, or (EPI 3) gamma | beta of the residual's LayerNorm
  __shared__ __align__(16) float bias_s[BLOCK_N];
  __shared__ __align__(16) float corr_s[BLOCK_N];
  __shared__ __align__(16) float beta_s[EPI == 3 ? BLOCK_N : 4];
  __shared__ uint64_t res_bar[EPI == 3 ? kEpiWarps : 1];  // EPI 3: one transaction barrier per epilogue warp (residual tile loads)
  __shared__ uint64_t acc_full, acc_empty;  // EPI_ROLE: the acc_s hand-over between the MMA and the epilogue warpgroups
  // EPI 4 (skinning): the current column tile's bone list and dense [bone][vertex] weights
  __shared__ __align__(16) float skin_w_s[EPI == 4 ? 2 : 1][EPI == 4 ? kSkinTileBones * 32 : 4];  // double-buffered across tiles
  __shared__ int skin_bone_s[EPI == 4 ? 2 : 1][EPI == 4 ? kSkinTileBones : 1];
  __shared__ int skin_nb_s[2];

  // 128B-swizzled tiles need 1024-byte alignment.
  const uint32_t raw_addr = ptx::smem_u32(smem_raw);
  uint8_t* smem = smem_raw + ((1024u - (raw_addr & 1023u)) & 1023u);
  float* const acc_s = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes);
  uint8_t* const epi_smem = smem + Cfg::kStages * Cfg::kStageBytes + Cfg::kAccBytes;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int tiles_n = (p.grid_n_cols + BLOCK_N - 1) / BLOCK_N;
  const int tiles_m = (p.grid_m_rows + kGemmBlockM - 1) / kGemmBlockM;
  const int num_tiles = tiles_m * tiles_n;

  int total_iters = 0;
  for (int s = 0; s < p.num_segs; ++s) total_iters += p.seg_kblocks[s];
  // Split-K (GemmParams::k_splits, masked variant only): work item w = tile * S + split; split s runs the K
  // iterations [s * per_split, min(total_iters, (s + 1) * per_split)).  S == 1 everywhere else: one item per tile.
  const int S = (!LEAN && p.k_splits > 1) ? p.k_splits : 1;
  const int per_split = (total_iters + S - 1) / S;
  const int num_work = num_tiles * S;

  if (warp_idx == 0 && lane == 0) {
    ptx::prefetch_tmap(&p.b_hi);  // needed first: the weight tiles are requested right below
    if (PASSES == 3) ptx::prefetch_tmap(&p.b_lo);
    for (int s = 0; s < p.num_segs; ++s) {
      ptx::prefetch_tmap(&p.a_hi[s]);
      if (PASSES == 3) ptx::prefetch_tmap(&p.a_lo[s]);
    }
    for (int i = 0; i < Cfg::kStages; ++i) {
      ptx::mbar_init(&full_bar[i], 1);
      ptx::mbar_init(&empty_bar[i], 2);  // one arrival per MMA warpgroup
    }
    if (EPI == 3)
      for (int i = 0; i < kEpiWarps; ++i) ptx::mbar_init(&res_bar[i], 1);
    if (EPI_ROLE) {
      ptx::mbar_init(&acc_full, kMmaWarps);  // one arrival per warp
      ptx::mbar_init(&acc_empty, kEpiWarps);
    }
    ptx::fence_barrier_init();
  }
  // The B operand is a weight matrix that no kernel of the chain writes: the producer thread puts the B tiles of the first
  // pipeline stages in flight right after it has initialised the barriers -- BEFORE the CTA-wide setup barrier and before
  // it waits for the previous grid -- so the pipeline fill overlaps both the setup and that grid's tail.
  int prefetched = 0;
  if (warp_idx == 0 && lane == 0 && static_cast<int>(blockIdx.x) < num_work) {
    const int tile0 = static_cast<int>(blockIdx.x) / S;
    const int it_b = (static_cast<int>(blockIdx.x) - tile0 * S) * per_split;
    const int cnt = (total_iters < it_b + per_split ? total_iters : it_b + per_split) - it_b;
    const int n0 = (tile0 % tiles_n) * BLOCK_N;
    prefetched = cnt < Cfg::kStages ? cnt : Cfg::kStages;
    for (int i = 0; i < prefetched; ++i) {
      uint8_t* st = smem + i * Cfg::kStageBytes;
      ptx::mbar_expect_tx(&full_bar[i], Cfg::kStageBytes);
      ptx::tma_load_2d(st + Cfg::kSplit * Cfg::kABytes, &p.b_hi, &full_bar[i], (it_b + i) * kElemK, n0);
      if (PASSES == 3)
        ptx::tma_load_2d(st + 2 * Cfg::kABytes + Cfg::kBBytes, &p.b_lo, &full_bar[i], (it_b + i) * kElemK, n0);
    }
  }
  if (warp_idx == kFirstMmaWarp && lane == 0) {
    epi_s.bias = p.bias, epi_s.residual = p.residual, epi_s.ldr = p.ldr, epi_s.out = p.out, epi_s.ldo = p.ldo;
    epi_s.out_hi = p.out_hi, epi_s.out_lo = p.out_lo, epi_s.lds = p.lds, epi_s.act = p.act, epi_s.M = p.M, epi_s.N = p.N;
    epi_s.out_row_mul = p.out_row_mul, epi_s.out_row_add = p.out_row_add, epi_s.clip_rows = p.clip_rows;
    epi_s.clip_valid = p.clip_valid;
    epi_s.acc_scale = p.acc_scale == 0.0f ? 1.0f : p.acc_scale;
    epi_s.tma_store = p.tma_store;
    epi_s.bias_per_row = p.bias_per_row;
    epi_s.a_stats = p.a_stats, epi_s.a_corr = p.a_corr, epi_s.res_stats = p.res_stats, epi_s.res_gamma = p.res_gamma;
    epi_s.res_beta = p.res_beta, epi_s.stats_out = p.stats_out, epi_s.ln_eps = p.ln_eps;
    if (p.tma_store) {
      ptx::prefetch_tmap(&p.st_out);
      ptx::prefetch_tmap(&p.st_hi);
      ptx::prefetch_tmap(&p.st_lo);
    }
  }
  __syncthreads();

  // Programmatic dependent launch: let the next kernel of the chain become resident as soon as SMs free up (its
  // prologue then overlaps this kernel's tail; it blocks in its own griddepcontrol.wait until this grid has completed
  // and flushed), then order everything below after the previous kernel.
  ptx::pdl_launch_dependents();
  ptx::pdl_wait_prior_grid();

  if (warp_idx < kFirstMmaWarp) {
    // ===================== TMA producer (warpgroup 0, one lane) =====================
    ptx::setmaxnreg_dec<kProducerRegs>();
    if (warp_idx == 0 && lane == 0) {
      int it = 0, stage = 0;
      uint32_t phase = 0;
      for (int w = blockIdx.x; w < num_work; w += gridDim.x) {
        const int tile = w / S;
        const int m0 = (tile / tiles_n) * kGemmBlockM;
        const int n0 = (tile % tiles_n) * BLOCK_N;
        const int it_b = (w - tile * S) * per_split;
        const int it_e = total_iters < it_b + per_split ? total_iters : it_b + per_split;
        // (segment, K block) of the item's first iteration; the packed weight column advances by one K block per iteration
        int s = 0, kb = it_b;
        while (s + 1 < p.num_segs && kb >= p.seg_kblocks[s]) kb -= p.seg_kblocks[s], ++s;
        int kcol = it_b * kElemK;
        for (int i = it_b; i < it_e; ++i, ++it, kcol += kElemK) {
          {
            const int row = m0 * p.seg_row_mul[s] + p.seg_row_shift[s];
            uint8_t* st = smem + stage * Cfg::kStageBytes;
            if (it < prefetched) {  // B of this stage is already in flight (see above): only A is missing
              ptx::tma_load_2d(st, &p.a_hi[s], &full_bar[stage], kb * kElemK, row);
              if (PASSES == 3) ptx::tma_load_2d(st + Cfg::kABytes, &p.a_lo[s], &full_bar[stage], kb * kElemK, row);
              if (++stage == Cfg::kStages) stage = 0, phase ^= 1;
              if (++kb == p.seg_kblocks[s]) kb = 0, ++s;
              continue;
            }
            ptx::mbar_wait(&empty_bar[stage], phase ^ 1);
            ptx::mbar_expect_tx(&full_bar[stage], Cfg::kStageBytes);
            ptx::tma_load_2d(st, &p.a_hi[s], &full_bar[stage], kb * kElemK, row);
            ptx::tma_load_2d(st + Cfg::kSplit * Cfg::kABytes, &p.b_hi, &full_bar[stage], kcol, n0);
            if (PASSES == 3) {
              ptx::tma_load_2d(st + Cfg::kABytes, &p.a_lo[s], &full_bar[stage], kb * kElemK, row);
              ptx::tma_load_2d(st + 2 * Cfg::kABytes + Cfg::kBBytes, &p.b_lo, &full_bar[stage], kcol, n0);
            }
            if (++stage == Cfg::kStages) stage = 0, phase ^= 1;
            if (++kb == p.seg_kblocks[s]) kb = 0, ++s;
          }
        }
      }
    }
  } else {
    // ===================== MMA (warpgroups 1, 2) and epilogue (warpgroup 3, or 1 and 2) =====================
    const bool mma_warp = warp_idx < kFirstEpiWarp;
    // (EPI_ROLE: each role sets its budget inside its own branch below -- ptxas allocates code reached from both
    // branches within the smaller budget)
    if constexpr (!EPI_ROLE) ptx::setmaxnreg_inc<232>();
    // MMA: warpgroup mhalf computes rows [64 mhalf, 64 mhalf + 64) of the tile, warp mq of it rows 16 mq + [0, 16).
    const int mq = (warp_idx - kFirstMmaWarp) & 3;
    const int mhalf = (warp_idx - kFirstMmaWarp) >> 2;
    // Epilogue: warp ew owns rows [32 q, 32 q + 32), one per lane, and the 32-column chunks half * 32 + 64 j (384 threads)
    // or all of them (EPI_ROLE: half = 0, chunks 32 j).
    const int ew = warp_idx - (EPI_ROLE ? kFirstEpiWarp : kFirstMmaWarp);  // epilogue warp 0..kEpiWarps-1
    const int q = ew & 3;
    const int half = EPI_ROLE ? 0 : ew >> 2;
    constexpr int kChunkStep = EPI_ROLE ? 32 : 64;
    int mma_stage = 0;
    uint32_t mma_phase = 0;
    // Runs the K loop of work item w (the CTA's item number tc) into registers, then publishes the finished tile in acc_s.
    // EPI_ROLE: waits on acc_empty before it writes acc_s and arrives on acc_full afterwards.  Otherwise a barrier over the
    // two warpgroups publishes it (afterwards every epilogue thread may read any row), and the caller guarantees that no
    // thread still reads acc_s for the previous tile.
    auto mma_tile = [&](int w, int tc) {
      float dm[Cfg::kAccRegs];
      float dc[PASSES == 3 ? Cfg::kAccRegs : 1];
#pragma unroll
      for (int i = 0; i < Cfg::kAccRegs; ++i) dm[i] = 0.0f;
#pragma unroll
      for (int i = 0; i < (PASSES == 3 ? Cfg::kAccRegs : 1); ++i) dc[i] = 0.0f;
      const int it_b = (w % S) * per_split;
      const int n_it = (total_iters < it_b + per_split ? total_iters : it_b + per_split) - it_b;
      const bool signaller = (threadIdx.x & 127) == 0;
      auto release = [&](int stg) {
        if (signaller) ptx::mbar_arrive(&empty_bar[stg]);
      };
      int prev = -1;
      for (int ki = 0; ki < n_it; ++ki) {
        ptx::mbar_wait(&full_bar[mma_stage], mma_phase);
        const uint32_t st = ptx::smem_u32(smem + mma_stage * Cfg::kStageBytes);
        const uint32_t a_off = static_cast<uint32_t>(mhalf * (Cfg::kABytes / 2));  // this warpgroup's 64 rows
        const uint64_t a_hi = ptx::make_desc_kmajor<kGemmBlockK * 4>(st + a_off);
        const uint64_t b_hi = ptx::make_desc_kmajor<kGemmBlockK * 4>(st + Cfg::kSplit * Cfg::kABytes);
        const uint64_t a_lo = ptx::make_desc_kmajor<kGemmBlockK * 4>(st + Cfg::kABytes + a_off);
        const uint64_t b_lo = ptx::make_desc_kmajor<kGemmBlockK * 4>(st + 2 * Cfg::kABytes + Cfg::kBBytes);
        ptx::wgmma_fence_regs(dm);
        if (PASSES == 3) ptx::wgmma_fence_regs(dc);
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < kGemmBlockK / 8; ++k) {
          // advancing K by one instruction (8 fp32 / 16 fp16 = 32 bytes) inside the swizzle span: +2 in the (>>4) address field
          const uint64_t koff = static_cast<uint64_t>(k * 2);
          mma_step<KIND>(dm, a_hi + koff, b_hi + koff);
          if constexpr (PASSES == 3) {
            mma_step<KIND>(dc, a_lo + koff, b_hi + koff);
            mma_step<KIND>(dc, a_hi + koff, b_lo + koff);
          }
        }
        ptx::wgmma_commit();
        ptx::wgmma_fence_regs(dm);
        if (PASSES == 3) ptx::wgmma_fence_regs(dc);
        // keep this stage's MMAs in flight; the previous stage's have completed, so its slot goes back to the producer
        ptx::wgmma_wait<1>();
        if (prev >= 0) release(prev);
        prev = mma_stage;
        if (++mma_stage == Cfg::kStages) mma_stage = 0, mma_phase ^= 1;
      }
      ptx::wgmma_wait<0>();
      ptx::wgmma_fence_regs(dm);
      if (PASSES == 3) ptx::wgmma_fence_regs(dc);
      if (prev >= 0) release(prev);
      if constexpr (EPI_ROLE) ptx::mbar_wait(&acc_empty, static_cast<uint32_t>((tc & 1) ^ 1));
      // fragment -> acc_s (the two accumulators of PASSES == 3 are added here)
      const int r0 = mhalf * 64 + mq * 16 + (lane >> 2);
      const int cc = 2 * (lane & 3);
#pragma unroll
      for (int j = 0; j < BLOCK_N / 8; ++j) {
        float v0 = dm[4 * j], v1 = dm[4 * j + 1], v2 = dm[4 * j + 2], v3 = dm[4 * j + 3];
        if (PASSES == 3) v0 += dc[4 * j], v1 += dc[4 * j + 1], v2 += dc[4 * j + 2], v3 += dc[4 * j + 3];
        *reinterpret_cast<float2*>(acc_s + r0 * Cfg::kAccPitch + 8 * j + cc) = make_float2(v0, v1);
        *reinterpret_cast<float2*>(acc_s + (r0 + 8) * Cfg::kAccPitch + 8 * j + cc) = make_float2(v2, v3);
      }
      if constexpr (EPI_ROLE) {
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&acc_full);
      } else {
        asm volatile("bar.sync 3, %0;" ::"n"(kMmaWarps * 32));
      }
    };
    const bool epi_warp = !EPI_ROLE || !mma_warp;
    if (!epi_warp) {
      // MMA warpgroups of the EPI_ROLE variants: nothing but K loops and the hand-over
      ptx::setmaxnreg_inc<kMmaRegs>();
      int tc = 0;
      for (int wi = blockIdx.x; wi < num_work; wi += gridDim.x, ++tc) mma_tile(wi, tc);
    } else if constexpr (EPI_ROLE) {
      ptx::setmaxnreg_inc<kEpiRoleRegs>();
    }
    // the 384-thread variants keep the epilogue parameters in registers; the epilogue warpgroup reads them from shared
    // memory (its register budget goes to the row's values)
    EpiParams e_regs;
    if constexpr (!EPI_ROLE) e_regs = epi_s;
    const EpiParams& e = EPI_ROLE ? epi_s : e_regs;
    const bool vec_ok = ((e.N & 3) == 0);
    float* tile = reinterpret_cast<float*>(epi_smem) + ew * kEpiTileFloats;
    const int tr = lane >> 3, tc = (lane & 7) * 4;  // transposed mapping: rows tr, tr+4, ..., columns tc..tc+3
    int tcount = 0;
    uint32_t res_phase = 0;  // EPI 3: parity of this warp's next residual load on res_bar[ew]
    if constexpr (EPI == 4) {
      // ===== linear-blend skinning epilogue: thread = frame m, 16 of the tile's 32 vertices (warp half) =====
      // Software pipeline over the CTA's tiles: the next tile's tables (bones, dense weights) are fetched into registers at the
      // top of a tile and published to the other shared-memory buffer after the compute phase; the next tile's bone transforms
      // of this thread's frame (up to kSkinRegBones x 12 registers, coalesced loads from the [bone][12][frames] table) are
      // requested right after that, so their L2 latency hides behind this tile's staging and stores.
      static_assert(BLOCK_N == 96 && PASSES == 3 && KIND == kKindF16, "skinning epilogue: 32 vertices x 3 per tile, fp16 pairs");
      constexpr int kSkinRegBones = 4;
      const int i = ew * 32 + lane;
      float4 sk[kSkinRegBones][3];
      float* const stg = reinterpret_cast<float*>(epi_smem);
      auto fetch_tables = [&](int tile_n, float& w0, float& w1, int& bone, int& nbv) {
        const float* wsrc = p.skin_w + static_cast<int64_t>(tile_n) * (kSkinTileBones * 32);
        w0 = __ldg(wsrc + i), w1 = __ldg(wsrc + i + 256);
        bone = i < kSkinTileBones ? __ldg(p.skin_bone + tile_n * kSkinTileBones + i) : 0;
        nbv = i == 0 ? __ldg(p.skin_nb + tile_n) : 0;
      };
      auto publish_tables = [&](int buf, float w0, float w1, int bone, int nbv) {
        skin_w_s[buf][i] = w0, skin_w_s[buf][i + 256] = w1;
        if (i < kSkinTileBones) skin_bone_s[buf][i] = bone;
        if (i == 0) skin_nb_s[buf] = nbv;
      };
      auto request_transforms = [&](int buf, int m_first) {
        const int mm = m_first + q * 32 + lane;
        const float* col = p.skin_A + (mm < e.M ? mm : 0);
        const int nbv = skin_nb_s[buf];
#pragma unroll
        for (int b = 0; b < kSkinRegBones; ++b)
          if (b < nbv) load_bone_transform(col, p.skin_lda, skin_bone_s[buf][b], sk[b][0], sk[b][1], sk[b][2]);
      };
      int buf = 0;
      if (static_cast<int>(blockIdx.x) < num_tiles) {
        float w0, w1;
        int bone, nbv;
        fetch_tables(static_cast<int>(blockIdx.x) % tiles_n, w0, w1, bone, nbv);
        publish_tables(0, w0, w1, bone, nbv);
        asm volatile("bar.sync 1, %0;" ::"n"(kEpiWarps * 32));
        request_transforms(0, (static_cast<int>(blockIdx.x) / tiles_n) * kGemmBlockM);
      }
      for (int tile_idx = blockIdx.x; tile_idx < num_tiles; tile_idx += gridDim.x, ++tcount, buf ^= 1) {
        const int m0 = (tile_idx / tiles_n) * kGemmBlockM;
        const int n0 = (tile_idx % tiles_n) * BLOCK_N;
        const int m = m0 + q * 32 + lane;
        const int next = tile_idx + static_cast<int>(gridDim.x);
        const bool has_next = next < num_tiles;
        float nw0 = 0.f, nw1 = 0.f;
        int nbone = 0, nnb = 0;
        if (has_next) fetch_tables(next % tiles_n, nw0, nw1, nbone, nnb);  // in flight during the accumulator wait and the compute

        mma_tile(tile_idx, tcount);  // the previous tile's reads of acc_s are behind the bar.sync 1 of its compute phase
        // verts = sum_b w[v][b] (R_b v_posed + t_b).  Within a 32-vertex tile nearly every (vertex, bone) pair carries weight
        // (vertices are indexed by body part), so every vertex is updated per bone: no branches, 12 FMAs per (vertex, bone).
        // Two rounds of 8 vertices keep the live registers (transforms 48 + v_posed 24 + results 48) under the 168 available.
        float o[48];
#pragma unroll
        for (int j = 0; j < 48; ++j) o[j] = 0.0f;
        const int nb = skin_nb_s[buf];
        const float* col = p.skin_A + (m < e.M ? m : 0);
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          float vp[24];
          {
            acc_load<Cfg::kAccPitch>(acc_s, q * 32 + lane, 48 * half + 24 * h2, vp);
#pragma unroll
            for (int j = 0; j < 24; ++j) vp[j] *= e.acc_scale;
          }
          auto apply_bone = [&](const float4& r0, const float4& r1, const float4& r2, const float* wrow) {
#pragma unroll
            for (int g = 0; g < 2; ++g) {
              const float4 w4 = *reinterpret_cast<const float4*>(wrow + 8 * h2 + 4 * g);
              const float wv[4] = {w4.x, w4.y, w4.z, w4.w};
#pragma unroll
              for (int u = 0; u < 4; ++u) {
                const int j = 4 * g + u;  // vertex inside this round
                const float x = vp[3 * j], y = vp[3 * j + 1], z = vp[3 * j + 2];
                float& ox = o[24 * h2 + 3 * j];
                float& oy = o[24 * h2 + 3 * j + 1];
                float& oz = o[24 * h2 + 3 * j + 2];
                ox = fmaf(wv[u], fmaf(r0.x, x, fmaf(r0.y, y, fmaf(r0.z, z, r0.w))), ox);
                oy = fmaf(wv[u], fmaf(r1.x, x, fmaf(r1.y, y, fmaf(r1.z, z, r1.w))), oy);
                oz = fmaf(wv[u], fmaf(r2.x, x, fmaf(r2.y, y, fmaf(r2.z, z, r2.w))), oz);
              }
            }
          };
#pragma unroll
          for (int b = 0; b < kSkinRegBones; ++b)
            if (b < nb) apply_bone(sk[b][0], sk[b][1], sk[b][2], &skin_w_s[buf][b * 32 + 16 * half]);
          if (nb > kSkinRegBones) {  // the rarer tiles that touch more bones: straight from L2, one bone ahead
            float4 c0, c1, c2;
            load_bone_transform(col, p.skin_lda, skin_bone_s[buf][kSkinRegBones], c0, c1, c2);
            for (int b = kSkinRegBones; b < nb; ++b) {
              const float4 r0 = c0, r1 = c1, r2 = c2;
              if (b + 1 < nb) load_bone_transform(col, p.skin_lda, skin_bone_s[buf][b + 1], c0, c1, c2);
              apply_bone(r0, r1, r2, &skin_w_s[buf][b * 32 + 16 * half]);
            }
          }
        }
        if (has_next) publish_tables(buf ^ 1, nw0, nw1, nbone, nnb);
        // TMA-store variant: the previous tile's bulk stores (issued by this thread) have finished reading the staging tile
        if (e.tma_store && ew == 0 && lane == 0) ptx::bulk_wait_read_all();
        // one barrier: the next tile's tables are visible, and every warp has finished storing the previous tile's rows out of
        // the staging tile that is overwritten below
        asm volatile("bar.sync 1, %0;" ::"n"(kEpiWarps * 32));
        if (has_next) request_transforms(buf ^ 1, (next / tiles_n) * kGemmBlockM);
        if (e.tma_store) {
          // Output rows with a 16-byte-multiple pitch (rohm_body_set_vertex_pitch): the tile leaves through TMA.  Staging = three
          // 128-row x 128-byte SWIZZLE_128B boxes (32 columns each; 16-byte chunk c of row r at slot c ^ (r & 7): the row-per-thread
          // 16-byte writes are conflict-free); one thread issues the three bulk tensor stores, which clip the ragged last row /
          // column tile themselves.  The 96 epilogue-issued 4-byte loads / stores per thread of the path below disappear.
          uint8_t* const sb = reinterpret_cast<uint8_t*>(stg);
          const int r = q * 32 + lane;
#pragma unroll
          for (int j = 0; j < 12; ++j) {
            const int cc = 12 * half + j;  // 16-byte chunk of the 96-column row
            *reinterpret_cast<float4*>(sb + (cc >> 3) * (kGemmBlockM * 128) + r * 128 + (((cc & 7) ^ (r & 7)) << 4)) =
                make_float4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
          }
          ptx::fence_proxy_async();
          asm volatile("bar.sync 2, %0;" ::"n"(kEpiWarps * 32));
          if (ew == 0 && lane == 0) {
#pragma unroll
            for (int j = 0; j < 3; ++j)
              if (n0 + 32 * j < e.N) ptx::tma_store_2d(&p.st_out, sb + j * (kGemmBlockM * 128), n0 + 32 * j, m0);
            ptx::bulk_commit();
          }
          continue;
        }
        // transpose through the CTA-wide staging tile: the output row pitch (3 V floats) is not a multiple of 16 bytes, so
        // neither TMA nor vector stores apply; lanes along the columns give fully coalesced 4-byte stores
        {
          float4* srow = reinterpret_cast<float4*>(stg + (q * 32 + lane) * kSkinPitch + 48 * half);
#pragma unroll
          for (int j = 0; j < 12; ++j) srow[j] = make_float4(o[4 * j], o[4 * j + 1], o[4 * j + 2], o[4 * j + 3]);
        }
        asm volatile("bar.sync 2, %0;" ::"n"(kEpiWarps * 32));
        {
          const int w8 = ew;
#pragma unroll 4
          for (int rr = 0; rr < kGemmBlockM / kEpiWarps; ++rr) {
            const int r = w8 * (kGemmBlockM / kEpiWarps) + rr;
            const int mr = m0 + r;
            if (mr >= e.M) break;
            float* dst = e.out + static_cast<int64_t>(mr) * e.ldo + n0;
            const float* src = stg + r * kSkinPitch;
#pragma unroll
            for (int c = 0; c < 3; ++c) {
              const int col = lane + 32 * c;
              if (n0 + col < e.N) __stcs(dst + col, src[col]);
            }
          }
        }
      }
    }
    for (int wi = blockIdx.x; EPI != 4 && epi_warp && wi < num_work; wi += gridDim.x, ++tcount) {
      const int tile_idx = wi / S;
      // split-K: the partial tile of split s goes to output rows m + s * split_row_stride
      const int split_rows = (wi - tile_idx * S) * (!LEAN ? p.split_row_stride : 0);
      const int m0 = (tile_idx / tiles_n) * kGemmBlockM;
      const int n0 = (tile_idx % tiles_n) * BLOCK_N;
      const int m = m0 + q * 32 + lane;
      const bool row_ok = m < e.M;
      bool row_real = true;
      if constexpr (EPI == 5) row_real = row_ok && __ldg(p.row_mask + m) != 0;
      else if (!LEAN && e.clip_rows > 0) row_real = (m % e.clip_rows) < e.clip_valid;
      const int64_t orow = static_cast<int64_t>(m) * e.out_row_mul + e.out_row_add + split_rows;
      const float bias_row = (e.bias != nullptr && e.bias_per_row && row_ok) ? __ldg(e.bias + m) : 0.0f;

      // stage this tile's per-column vectors before its accumulator is ready (EPI_ROLE: while its MMAs run; otherwise
      // before its main loop).  Single-buffered: the first barrier keeps the writers off the vectors until every epilogue
      // thread has finished the previous tile.
      {
        const int i = ew * 32 + lane;
        asm volatile("bar.sync 1, %0;" ::"n"(kEpiWarps * 32));
        if (i < BLOCK_N) {
          const bool col_ok = n0 + i < e.N;
          bias_s[i] = (e.bias != nullptr && !e.bias_per_row && col_ok) ? __ldg(e.bias + n0 + i) : 0.0f;
          if (EPI == 3) {
            corr_s[i] = e.res_stats != nullptr ? __ldg(e.res_gamma + n0 + i) : 1.0f;
            beta_s[i] = e.res_stats != nullptr ? __ldg(e.res_beta + n0 + i) : 0.0f;
          } else {
            corr_s[i] = (e.a_stats != nullptr && col_ok) ? __ldg(e.a_corr + n0 + i) : 0.0f;
          }
        }
        if (e.residual != nullptr && row_ok) {
          const float* r = e.residual + orow * e.ldr + n0 + half * 32;
#pragma unroll
          for (int c = 0; c < (EPI_ROLE ? BLOCK_N : (BLOCK_N > 64 ? 128 : 64)); c += kChunkStep)
            asm volatile("prefetch.global.L2 [%0];" ::"l"(r + c));
        }
        asm volatile("bar.sync 1, %0;" ::"n"(kEpiWarps * 32));
      }
      // LayerNorm folding, consumer side: (mean, rstd) of this thread's A row, fetched while the accumulator is still filling
      float a_mean = 0.0f, a_rstd = 1.0f;
      if (EPI != 3 && LEAN && e.a_stats != nullptr && row_ok) {
        const float2 mr = combine_row_stats(e.a_stats + static_cast<int64_t>(m) * 8, e.ln_eps);
        a_mean = mr.x, a_rstd = mr.y;
      }
      // LayerNorm folding, producer side: the residual tile (this thread: one row; the 2 x 32 columns of one 64-column
      // statistics group at a time, columns g * 32 + 64 h2) arrives through TMA into the warp's staging tile -- nearly all
      // of the shared memory is in use, so there is little L1 for per-thread loads -- and is passed through the previous
      // LayerNorm on the fly.  Group 0 is loaded before the accumulator is ready, group 1 after group 0 has been stored.
      float lnv[EPI == 3 ? 2 : 1][EPI == 3 ? 32 : 1];
      float r_mean = 0.0f, r_rstd = 1.0f;
      auto load_residual = [&](int g) {
        uint8_t* tb = reinterpret_cast<uint8_t*>(tile);
        uint64_t* rb = &res_bar[ew];
#pragma unroll
        for (int h2 = 0; h2 < 2; ++h2) {
          const int c0 = g * 32 + 64 * h2;
          if (lane == 0) {
            ptx::bulk_wait_read_all();  // this warp's stores have finished reading the staging tile
            ptx::mbar_expect_tx(rb, 4096);
            ptx::tma_load_2d(tb, &p.st_hi, rb, n0 + c0, m0 + q * 32);
            ptx::tma_load_2d(tb + 2048, &p.st_lo, rb, n0 + c0, m0 + q * 32);
          }
          ptx::mbar_wait(rb, res_phase);
          res_phase ^= 1;
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int off = lane * 64 + ((c ^ ((lane >> 1) & 3)) << 4);
            const uint4 hq = *reinterpret_cast<const uint4*>(tb + off);
            const uint4 lq = *reinterpret_cast<const uint4*>(tb + 2048 + off);
            const uint32_t hw[4] = {hq.x, hq.y, hq.z, hq.w};
            const uint32_t lw[4] = {lq.x, lq.y, lq.z, lq.w};
#pragma unroll
            for (int k = 0; k < 4; ++k) {
              const float2 fh = __half22float2(*reinterpret_cast<const __half2*>(&hw[k]));
              const float2 fl = __half22float2(*reinterpret_cast<const __half2*>(&lw[k]));
              const int j = 8 * c + 2 * k;
              lnv[h2][j] = fmaf(((fh.x + fl.x) - r_mean) * r_rstd, corr_s[c0 + j], beta_s[c0 + j]);
              lnv[h2][j + 1] = fmaf(((fh.y + fl.y) - r_mean) * r_rstd, corr_s[c0 + j + 1], beta_s[c0 + j + 1]);
            }
          }
          ptx::fence_proxy_async();  // generic-proxy reads above, async-proxy writes (next load / the stores) below
          __syncwarp();
        }
      };
      if constexpr (EPI == 3) {
        if (e.res_stats != nullptr && row_ok) {
          const float2 mr = combine_row_stats(e.res_stats + static_cast<int64_t>(m) * 8, e.ln_eps);
          r_mean = mr.x, r_rstd = mr.y;
        }
        load_residual(0);
      }
      if constexpr (EPI_ROLE) {
        ptx::mbar_wait(&acc_full, static_cast<uint32_t>(tcount & 1));
      } else {
        // the start-of-tile bar.sync 1 above keeps this tile's accumulator off acc_s until every thread has read the last one
        mma_tile(wi, tcount);
      }

      if constexpr (EPI == 3) {
        // ===== u = LN_prev(residual) + acc * 2^-s + bias, written in place as an fp16 pair + per-row partial statistics =====
        static_assert(BLOCK_N == 128 && PASSES == 3 && KIND == kKindF16, "LayerNorm-folding producer: fp16 pairs, 128-wide tiles");
        static_assert(EPI_ROLE, "one thread per row: both 64-column statistics groups");
        const int tile_n = tile_idx % tiles_n;
        float (&v)[2][32] = lnv;
        uint8_t* tb = reinterpret_cast<uint8_t*>(tile);
        const bool group_full = (m0 + q * 32 + 32 <= e.M);
#pragma unroll 1
        for (int g = 0; g < 2; ++g) {
          if (g == 1) load_residual(1);
#pragma unroll
          for (int h2 = 0; h2 < 2; ++h2) {
            const int c0 = g * 32 + 64 * h2;
            float raw[32];
            acc_load<Cfg::kAccPitch>(acc_s, q * 32 + lane, c0, raw);
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 b4 = *reinterpret_cast<const float4*>(&bias_s[c0 + j]);
              v[h2][j] += fmaf(raw[j], e.acc_scale, b4.x);
              v[h2][j + 1] += fmaf(raw[j + 1], e.acc_scale, b4.y);
              v[h2][j + 2] += fmaf(raw[j + 2], e.acc_scale, b4.z);
              v[h2][j + 3] += fmaf(raw[j + 3], e.acc_scale, b4.w);
            }
          }
          if (g == 1) {  // the last read of acc_s: the MMA warpgroups may write the next tile
            __syncwarp();
            if (lane == 0) ptx::mbar_arrive(&acc_empty);
          }
          auto store_chunk = [&](int h2) {
            const int nb = n0 + g * 32 + 64 * h2;
            if (group_full) {
              stage_pair_chunk(v[h2], tb, lane, &p.st_hi, &p.st_lo, nb, m0 + q * 32);
            } else if (row_ok) {  // ragged last row group: per-thread stores
              __half* oh = static_cast<__half*>(e.out_hi) + static_cast<int64_t>(m) * e.lds + nb;
              __half* ol = static_cast<__half*>(e.out_lo) + static_cast<int64_t>(m) * e.lds + nb;
#pragma unroll
              for (int j = 0; j < 32; ++j) ptx::split_f16(v[h2][j], oh[j], ol[j]);
            }
          };
          store_chunk(0);
          // partial row statistics over the group's 64 columns for the consumers of LN(u) -- computed while the TMA engine
          // reads the first chunk out of the staging tile (the second chunk has to wait for that anyway)
          float s1 = 0.0f;
#pragma unroll
          for (int j = 0; j < 32; ++j) s1 += v[0][j] + v[1][j];
          const float mean_i = s1 * (1.0f / 64.0f);
          float m2_i = 0.0f;
#pragma unroll
          for (int j = 0; j < 32; ++j) {
            const float d0 = v[0][j] - mean_i, d1 = v[1][j] - mean_i;
            m2_i = fmaf(d0, d0, fmaf(d1, d1, m2_i));
          }
          if (row_ok) e.stats_out[static_cast<int64_t>(m) * 8 + tile_n * 2 + g] = make_float2(mean_i, m2_i);
          store_chunk(1);
        }
        continue;
      }

#pragma unroll 1
      for (int c0 = half * 32; c0 < BLOCK_N; c0 += kChunkStep) {
        const int nb = n0 + c0;
        const bool full = vec_ok && (nb + 32 <= e.N);
        if (e.tma_store && full && (m0 + q * 32 + 32 <= e.M)) {
          // ---- TMA-store path: row-per-thread registers -> swizzled staging tile -> bulk tensor store ----
          float v[32];
          acc_load<Cfg::kAccPitch>(acc_s, q * 32 + lane, c0, v);
          if (KIND == kKindF16) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] *= e.acc_scale;
          }
          if (LEAN && e.a_stats != nullptr) {  // LayerNorm folding: out = rstd (acc - mean c_n) + d_n
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 c4 = *reinterpret_cast<const float4*>(&corr_s[c0 + j]);
              v[j] = a_rstd * fmaf(-a_mean, c4.x, v[j]), v[j + 1] = a_rstd * fmaf(-a_mean, c4.y, v[j + 1]);
              v[j + 2] = a_rstd * fmaf(-a_mean, c4.z, v[j + 2]), v[j + 3] = a_rstd * fmaf(-a_mean, c4.w, v[j + 3]);
            }
          }
          if (e.bias != nullptr) {
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
              const float4 b4 = *reinterpret_cast<const float4*>(&bias_s[c0 + j]);
              v[j] += b4.x, v[j + 1] += b4.y, v[j + 2] += b4.z, v[j + 3] += b4.w;
            }
            if (e.bias_per_row) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] += bias_row;
            }
          }
          if (EPI == 1) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
          }
          if (!LEAN) {  // TrajNet: other activations, zeroed pad rows
            if (e.act == kActGelu) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
            } else if (e.act == kActSilu) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = v[j] / (1.0f + expf(-v[j]));
            } else if (e.act == kActMish) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = apply_act(v[j], kActMish);
            }
            if (!row_real) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] = 0.0f;
            }
          }
          // the previous chunk's bulk store must have finished reading the staging tile
          if (lane == 0) ptx::bulk_wait_read_all();
          __syncwarp();
          uint8_t* tb = reinterpret_cast<uint8_t*>(tile);
          if (e.out != nullptr) {
            // 32 rows x 128 B, SWIZZLE_128B: 16-byte chunk c of row r lives at slot c ^ (r & 7)
#pragma unroll
            for (int c = 0; c < 8; ++c)
              *reinterpret_cast<float4*>(tb + lane * 128 + ((c ^ (lane & 7)) << 4)) =
                  make_float4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
          } else {
            // two planes of 32 rows x 64 B (hi at +0, lo at +2048), SWIZZLE_64B: chunk c of row r at slot c ^ ((r >> 1) & 3)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              uint2 h0, l0, h1, l1;
              ptx::split_f16x4(make_float4(v[8 * c], v[8 * c + 1], v[8 * c + 2], v[8 * c + 3]), h0, l0);
              ptx::split_f16x4(make_float4(v[8 * c + 4], v[8 * c + 5], v[8 * c + 6], v[8 * c + 7]), h1, l1);
              const int off = lane * 64 + ((c ^ ((lane >> 1) & 3)) << 4);
              *reinterpret_cast<uint4*>(tb + off) = make_uint4(h0.x, h0.y, h1.x, h1.y);
              *reinterpret_cast<uint4*>(tb + 2048 + off) = make_uint4(l0.x, l0.y, l1.x, l1.y);
            }
          }
          ptx::fence_proxy_async();
          __syncwarp();
          if (lane == 0) {
            if (e.out != nullptr) {
              ptx::tma_store_2d(&p.st_out, tb, nb, m0 + q * 32 + split_rows);
            } else {
              ptx::tma_store_2d(&p.st_hi, tb, nb, m0 + q * 32 + split_rows);
              ptx::tma_store_2d(&p.st_lo, tb + 2048, nb, m0 + q * 32 + split_rows);
            }
            ptx::bulk_commit();
          }
          continue;
        }
        // residual in the transposed (coalesced) layout
        float4 res[8];
        const bool use_res = e.residual != nullptr && full;
        if (use_res) {
#pragma unroll
          for (int rr = 0; rr < 8; ++rr) {
            const int mr = m0 + q * 32 + rr * 4 + tr;
            res[rr] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (mr < e.M)
              res[rr] = *reinterpret_cast<const float4*>(
                  e.residual + (static_cast<int64_t>(mr) * e.out_row_mul + e.out_row_add) * e.ldr + nb + tc);
          }
        }
        float v[32];
        acc_load<Cfg::kAccPitch>(acc_s, q * 32 + lane, c0, v);
        if (KIND == kKindF16) {  // undo the power-of-two weight scale (exact)
#pragma unroll
          for (int j = 0; j < 32; ++j) v[j] *= e.acc_scale;
        }
        if (nb >= e.N) continue;  // warp-uniform

        if (row_ok) {
          if (LEAN && e.a_stats != nullptr) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = a_rstd * fmaf(-a_mean, corr_s[c0 + j], v[j]);
          }
          if (e.bias != nullptr) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] += bias_s[c0 + j];  // smem broadcast; zero beyond N
            if (e.bias_per_row) {
#pragma unroll
              for (int j = 0; j < 32; ++j) v[j] += bias_row;
            }
          }
          // one warp-uniform branch per activation: a per-element switch compiles to ~3000 predicated-off
          // instructions per chunk that are still issued when act == none
          if (EPI == 0) {
          } else if (EPI == 1 || e.act == kActGelu) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = gelu_erf(v[j]);
          } else if (e.act == kActSilu) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = v[j] / (1.0f + expf(-v[j]));
          } else if (e.act == kActMish) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = apply_act(v[j], kActMish);
          }
          if (e.residual != nullptr && !full) {  // ragged N tail: row-per-thread scalar path
            const float* r = e.residual + orow * e.ldr + nb;
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (nb + j < e.N) v[j] += r[j];
          }
          if (!LEAN && !row_real) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = 0.0f;
          }
        }

        if (full) {
          // ---- coalesced path through the staging tile ----
          if (e.tma_store) {  // an earlier chunk's bulk store may still be reading the tile
            if (lane == 0) ptx::bulk_wait_read_all();
            __syncwarp();
          }
#pragma unroll
          for (int j = 0; j < 32; ++j) tile[lane * 32 + (j ^ lane)] = v[j];  // column ^ row: conflict-free both ways
          __syncwarp();
#pragma unroll
          for (int rr = 0; rr < 8; ++rr) {
            const int r = rr * 4 + tr;
            const int mr = m0 + q * 32 + r;
            float4 w;
            w.x = tile[r * 32 + (tc ^ r)], w.y = tile[r * 32 + ((tc + 1) ^ r)];
            w.z = tile[r * 32 + ((tc + 2) ^ r)], w.w = tile[r * 32 + ((tc + 3) ^ r)];
            if (mr < e.M) {
              if (use_res) {
                bool real = true;
                if constexpr (EPI == 5) real = __ldg(p.row_mask + mr) != 0;
                else if (!LEAN && e.clip_rows > 0) real = (mr % e.clip_rows) < e.clip_valid;
                if (real) w.x += res[rr].x, w.y += res[rr].y, w.z += res[rr].z, w.w += res[rr].w;
              }
              const int64_t orr = static_cast<int64_t>(mr) * e.out_row_mul + e.out_row_add + split_rows;
              if (e.out != nullptr) *reinterpret_cast<float4*>(e.out + orr * e.ldo + nb + tc) = w;
              if (e.out_hi != nullptr) {
                if (KIND == kKindF16) {
                  uint2 h, l;
                  ptx::split_f16x4(w, h, l);
                  *reinterpret_cast<uint2*>(static_cast<__half*>(e.out_hi) + orr * e.lds + nb + tc) = h;
                  *reinterpret_cast<uint2*>(static_cast<__half*>(e.out_lo) + orr * e.lds + nb + tc) = l;
                } else {
                  float4 h, l;
                  h.x = ptx::to_tf32(w.x), h.y = ptx::to_tf32(w.y), h.z = ptx::to_tf32(w.z), h.w = ptx::to_tf32(w.w);
                  l.x = w.x - h.x, l.y = w.y - h.y, l.z = w.z - h.z, l.w = w.w - h.w;
                  *reinterpret_cast<float4*>(static_cast<float*>(e.out_hi) + orr * e.lds + nb + tc) = h;
                  *reinterpret_cast<float4*>(static_cast<float*>(e.out_lo) + orr * e.lds + nb + tc) = l;
                }
              }
            }
          }
          __syncwarp();
        } else if (row_ok) {
          // ---- ragged N tail: scalar row-per-thread stores ----
          if (e.out != nullptr) {
            float* o = e.out + orow * e.ldo + nb;
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (nb + j < e.N) o[j] = v[j];
          }
          if (e.out_hi != nullptr && KIND == kKindF16) {
            __half* oh = static_cast<__half*>(e.out_hi) + orow * e.lds + nb;
            __half* ol = static_cast<__half*>(e.out_lo) + orow * e.lds + nb;
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (nb + j < e.N) ptx::split_f16(v[j], oh[j], ol[j]);
          } else if (e.out_hi != nullptr) {
            float* oh = static_cast<float*>(e.out_hi) + orow * e.lds + nb;
            float* ol = static_cast<float*>(e.out_lo) + orow * e.lds + nb;
#pragma unroll
            for (int j = 0; j < 32; ++j)
              if (nb + j < e.N) {
                const float h = ptx::to_tf32(v[j]);
                oh[j] = h;
                ol[j] = v[j] - h;
              }
          }
        }
      }
      if constexpr (EPI_ROLE) {  // every chunk has been read out of acc_s
        __syncwarp();
        if (lane == 0) ptx::mbar_arrive(&acc_empty);
      }
    }
    // outstanding TMA stores of this warp must have finished reading the staging tile before the CTA's shared memory is
    // released; their global writes are ordered before the grid's completion like any other store
    if (lane == 0) ptx::bulk_wait_read_all();
  }

  __syncthreads();
}

__global__ void split_tf32_kernel(const float* __restrict__ x, float* __restrict__ hi, float* __restrict__ lo,
                                  int64_t n) {
  int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) {
    const float v = x[i];
    const float h = ptx::to_tf32(v);
    hi[i] = h;
    lo[i] = v - h;
  }
}

__global__ void split_f16_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, int64_t n,
                                 float scale) {
  int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t stride = static_cast<int64_t>(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) ptx::split_f16(x[i] * scale, hi[i], lo[i]);
}

// max |w| over n elements (the bit pattern of a non-negative float is monotonic in its value)
__global__ void absmax_kernel(const float* __restrict__ w, int64_t n, unsigned int* __restrict__ out) {
  float m = 0.0f;
  for (int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += static_cast<int64_t>(gridDim.x) * blockDim.x) {
    const float a = fabsf(w[i]);
    m = (a <= 3.0e38f && a > m) ? a : m;  // ignores NaN / inf
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, off));
  if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));
}

PFN_cuTensorMapEncodeTiled_v12000 get_encode_fn() {
  static PFN_cuTensorMapEncodeTiled_v12000 fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled_v12000>(ptr);
  });
  return fn;
}

template <int BLOCK_N, int PASSES, int KIND>
static cudaError_t set_attr() {
  constexpr int kRoleSmem = TileCfg<BLOCK_N, PASSES, true>::kSmemBytes;
  cudaError_t e = cudaFuncSetAttribute(gemm_tile_kernel<BLOCK_N, PASSES, 0, KIND>,
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, kRoleSmem);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(gemm_tile_kernel<BLOCK_N, PASSES, 1, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRoleSmem);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(gemm_tile_kernel<BLOCK_N, PASSES, 2, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           TileCfg<BLOCK_N, PASSES, false>::kSmemBytes);
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(gemm_tile_kernel<BLOCK_N, PASSES, 5, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           TileCfg<BLOCK_N, PASSES, false>::kSmemBytes);
  if (e != cudaSuccess) return e;
  if constexpr (BLOCK_N == 128 && PASSES == 3 && KIND == kKindF16)
    e = cudaFuncSetAttribute(gemm_tile_kernel<BLOCK_N, PASSES, 3, KIND>, cudaFuncAttributeMaxDynamicSharedMemorySize, kRoleSmem);
  return e;
}

template <int BLOCK_N, int PASSES, int KIND>
cudaError_t launch_cfg(const GemmParams& p, int m_rows, int n_cols, cudaStream_t stream, bool pdl) {
  using Cfg = TileCfg<BLOCK_N, PASSES, false>;  // the 384-thread variants (EPI 2, 4)
  const bool plain = p.clip_rows == 0;
  const int epi = (plain && p.act == kActNone) ? 0 : (plain && p.act == kActGelu) ? 1 : p.row_mask != nullptr ? 5 : 2;
  auto kern = epi == 0   ? gemm_tile_kernel<BLOCK_N, PASSES, 0, KIND>
              : epi == 1 ? gemm_tile_kernel<BLOCK_N, PASSES, 1, KIND>
              : epi == 2 ? gemm_tile_kernel<BLOCK_N, PASSES, 2, KIND>
                         : gemm_tile_kernel<BLOCK_N, PASSES, 5, KIND>;
  int threads = kernel_threads(epi);
  int smem_bytes = epi_role(epi) ? TileCfg<BLOCK_N, PASSES, true>::kSmemBytes : Cfg::kSmemBytes;
  if (p.a_stats != nullptr && (!plain || p.a_corr == nullptr)) return cudaErrorInvalidValue;
  if (p.row_mask != nullptr && plain) return cudaErrorInvalidValue;  // the mask is read by the masked variant only
  if (p.stats_out != nullptr) {
    // LayerNorm-folding producer: the output pair overwrites the residual pair tile by tile (st_hi / st_lo both ways), rows are
    // four 128-column tiles wide, and the column tile of a CTA must not change between its tiles (per-column vectors)
    if constexpr (BLOCK_N == 128 && PASSES == 3 && KIND == kKindF16) {
      if (!plain || p.act != kActNone || n_cols != 4 * BLOCK_N || p.N != n_cols || !p.tma_store || p.out != nullptr ||
          p.out_hi == nullptr || p.a_stats != nullptr || (p.res_stats != nullptr && (p.res_gamma == nullptr || p.res_beta == nullptr)))
        return cudaErrorInvalidValue;
      kern = gemm_tile_kernel<BLOCK_N, PASSES, 3, KIND>;
      threads = kernel_threads(3);
      smem_bytes = TileCfg<BLOCK_N, PASSES, true>::kSmemBytes;
    } else {
      return cudaErrorInvalidValue;
    }
  }
  if (p.skin_A != nullptr) {
    if constexpr (BLOCK_N == 96 && PASSES == 3 && KIND == kKindF16) {
      if (!plain || p.act != kActNone || p.out == nullptr || p.skin_nb == nullptr || p.skin_bone == nullptr || p.skin_w == nullptr ||
          p.bias != nullptr || p.residual != nullptr || p.a_stats != nullptr || p.stats_out != nullptr)
        return cudaErrorInvalidValue;
      kern = gemm_tile_kernel<BLOCK_N, PASSES, 4, KIND>;
      threads = kernel_threads(4);
      smem_bytes = Cfg::kStages * Cfg::kStageBytes + 1024 + Cfg::kAccBytes + kSkinStageBytes;
      static bool skin_attr_set = false;
      if (!skin_attr_set) {
        cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes);
        if (e != cudaSuccess) return e;
        skin_attr_set = true;
      }
    } else {
      return cudaErrorInvalidValue;
    }
  }
  static bool attr_set = false;
  if (!attr_set) {  // normally done up front by gemm_init_attributes(); kept for stand-alone users of launch_gemm
    cudaError_t e = set_attr<BLOCK_N, PASSES, KIND>();
    if (e != cudaSuccess) return e;
    attr_set = true;
  }
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || num_sms <= 0) num_sms = 132;
  }
  GemmParams q = p;
  q.grid_m_rows = m_rows;
  q.grid_n_cols = n_cols;
  int tiles = ((n_cols + BLOCK_N - 1) / BLOCK_N) * ((m_rows + kGemmBlockM - 1) / kGemmBlockM);
  if (q.k_splits > 1) {  // split-K: masked variant, fp32 partials only, every K range non-empty
    int iters = 0;
    for (int s = 0; s < q.num_segs; ++s) iters += q.seg_kblocks[s];
    const int per = (iters + q.k_splits - 1) / q.k_splits;
    if (plain || q.out == nullptr || q.out_hi != nullptr || q.bias != nullptr || q.residual != nullptr ||
        q.act != kActNone || q.out_row_mul != 1 || q.out_row_add != 0 || (q.k_splits - 1) * per >= iters ||
        q.split_row_stride < m_rows)
      return cudaErrorInvalidValue;
    tiles *= q.k_splits;
  }
  cudaLaunchConfig_t cfg{};
  int grid = tiles < num_sms ? tiles : num_sms;
  if (p.stats_out != nullptr) grid -= grid % 4;  // a CTA keeps its column tile: tile % 4 == blockIdx % 4 on every round
  cfg.gridDim = dim3(grid, 1, 1);
  cfg.blockDim = dim3(threads, 1, 1);
  cfg.dynamicSmemBytes = smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, q);
}

}  // namespace

int make_tmap_2d(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows,
                 int row_elem_stride, int kind) {
  auto fn = get_encode_fn();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * gemm_elem_bytes(kind)};
  // With a traversal stride s the box spans box_rows * s tensor rows and TMA delivers every s-th of them
  // (ceil(boxDim / elementStride) elements), so smem still receives exactly box_rows rows.
  cuuint32_t box[2] = {static_cast<cuuint32_t>(gemm_block_k(kind)), static_cast<cuuint32_t>(box_rows * row_elem_stride)};
  cuuint32_t estride[2] = {1u, static_cast<cuuint32_t>(row_elem_stride)};
  CUresult r = fn(map, kind == kKindF16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                  const_cast<void*>(base), gdim, gstride, box, estride,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                  CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return static_cast<int>(r);
}

static int encode_store_map(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, bool half,
                            int box_rows = 32) {
  auto fn = get_encode_fn();
  if (fn == nullptr) return -1;
  const int eb = half ? 2 : 4;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * eb};
  cuuint32_t box[2] = {32u, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estride[2] = {1u, 1u};
  return static_cast<int>(fn(map, half ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2,
                             const_cast<void*>(base), gdim, gstride, box, estride, CU_TENSOR_MAP_INTERLEAVE_NONE,
                             half ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
}

int make_store_tmap(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, bool half, int box_rows) {
  return encode_store_map(map, base, rows, cols, ld, half, box_rows);
}

int make_tile_tmap_f16_sw128(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, int64_t ld, int box_rows) {
  auto fn = get_encode_fn();
  if (fn == nullptr) return -1;
  cuuint64_t gdim[2] = {static_cast<cuuint64_t>(cols), static_cast<cuuint64_t>(rows)};
  cuuint64_t gstride[1] = {static_cast<cuuint64_t>(ld) * 2};
  cuuint32_t box[2] = {64u, static_cast<cuuint32_t>(box_rows)};
  cuuint32_t estride[2] = {1u, 1u};
  return static_cast<int>(fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estride,
                             CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                             CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE));
}

int gemm_enable_tma_store(GemmParams* p, int64_t rows_total, int kind) {
  p->tma_store = 0;
  const bool plain = p->residual == nullptr && p->out_row_mul == 1 && p->out_row_add == 0;
  const bool only_out = p->out != nullptr && p->out_hi == nullptr;
  const bool only_pair = p->out == nullptr && p->out_hi != nullptr && kind == kKindF16;
  if (!plain || !(only_out || only_pair)) return 0;
  int rc = 0;
  if (only_out) {
    if ((p->ldo * 4) % 16 != 0 || (reinterpret_cast<uintptr_t>(p->out) & 15) != 0) return 0;
    rc = encode_store_map(&p->st_out, p->out, rows_total, p->N, p->ldo, false);
    p->st_hi = p->st_out, p->st_lo = p->st_out;
  } else {
    if ((p->lds * 2) % 16 != 0 || (reinterpret_cast<uintptr_t>(p->out_hi) & 15) != 0 ||
        (reinterpret_cast<uintptr_t>(p->out_lo) & 15) != 0)
      return 0;
    rc = encode_store_map(&p->st_hi, p->out_hi, rows_total, p->N, p->lds, true);
    if (rc == 0) rc = encode_store_map(&p->st_lo, p->out_lo, rows_total, p->N, p->lds, true);
    p->st_out = p->st_hi;
  }
  if (rc != 0) return rc;
  p->tma_store = 1;
  return 0;
}

cudaError_t launch_gemm(const GemmParams& p, int m_rows, int n_cols, int block_n, int passes, cudaStream_t stream,
                        bool pdl, int kind) {
  if (kind == kKindF16 && passes != 3) return cudaErrorInvalidValue;
#define ROHM_GEMM_CASE(BN)                                                                       \
  case BN:                                                                                       \
    if (kind == kKindF16) return launch_cfg<BN, 3, kKindF16>(p, m_rows, n_cols, stream, pdl);    \
    return passes == 3 ? launch_cfg<BN, 3, kKindTf32>(p, m_rows, n_cols, stream, pdl)            \
                       : launch_cfg<BN, 1, kKindTf32>(p, m_rows, n_cols, stream, pdl);
  switch (block_n) {
    ROHM_GEMM_CASE(32)
    ROHM_GEMM_CASE(64)
    ROHM_GEMM_CASE(96)
    ROHM_GEMM_CASE(128)
    default:
      return cudaErrorInvalidValue;
  }
#undef ROHM_GEMM_CASE
}

cudaError_t gemm_init_attributes() {
  cudaError_t e;
  if ((e = set_attr<32, 1, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<32, 3, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<64, 1, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<64, 3, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<96, 1, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<96, 3, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<128, 1, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<128, 3, kKindTf32>()) != cudaSuccess) return e;
  if ((e = set_attr<32, 3, kKindF16>()) != cudaSuccess) return e;
  if ((e = set_attr<64, 3, kKindF16>()) != cudaSuccess) return e;
  if ((e = set_attr<96, 3, kKindF16>()) != cudaSuccess) return e;
  if ((e = set_attr<128, 3, kKindF16>()) != cudaSuccess) return e;
  return cudaSuccess;
}

cudaError_t f16_weight_scale(const float* w_dev, int64_t n, float* scale_out) {
  *scale_out = 1.0f;
  if (n <= 0) return cudaSuccess;
  unsigned int* d_max = nullptr;
  cudaError_t e = cudaMalloc(&d_max, sizeof(unsigned int));
  if (e != cudaSuccess) return e;
  unsigned int bits = 0;
  e = cudaMemset(d_max, 0, sizeof(unsigned int));
  if (e == cudaSuccess) {
    absmax_kernel<<<132, 256>>>(w_dev, n, d_max);
    e = cudaGetLastError();
  }
  if (e == cudaSuccess) e = cudaMemcpy(&bits, d_max, sizeof bits, cudaMemcpyDeviceToHost);
  cudaFree(d_max);
  if (e != cudaSuccess) return e;
  float wmax;
  memcpy(&wmax, &bits, sizeof wmax);
  if (wmax > 0.0f) {
    int e2 = 0;
    frexpf(wmax, &e2);  // wmax = f * 2^e2, f in [0.5, 1)
    int sh = 14 - e2;
    sh = sh > 100 ? 100 : (sh < -100 ? -100 : sh);
    *scale_out = ldexpf(1.0f, sh);
  }
  return cudaSuccess;
}

cudaError_t launch_split_f16(const float* x, void* hi, void* lo, int64_t n, float scale, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const int threads = 256;
  int64_t blocks = (n + threads - 1) / threads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  split_f16_kernel<<<static_cast<unsigned>(blocks), threads, 0, stream>>>(x, static_cast<__half*>(hi), static_cast<__half*>(lo),
                                                                          n, scale);
  return cudaGetLastError();
}

cudaError_t launch_split_tf32(const float* x, float* hi, float* lo, int64_t n, cudaStream_t stream) {
  if (n <= 0) return cudaSuccess;
  const int threads = 256;
  int64_t blocks = (n + threads - 1) / threads;
  if (blocks > 132 * 16) blocks = 132 * 16;
  split_tf32_kernel<<<static_cast<unsigned>(blocks), threads, 0, stream>>>(x, hi, lo, n);
  return cudaGetLastError();
}

}  // namespace rohm
