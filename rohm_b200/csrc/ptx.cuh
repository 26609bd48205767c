// Thin inline-PTX wrappers for the sm_90a features the kernels use:
// mbarrier, TMA (cp.async.bulk.tensor), wgmma, clusters, fences.
// Everything here is device-only and header-only.
#pragma once
#include <cstdint>
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace rohm {
namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ bool elect_one() {
  uint32_t pred = 0;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(pred));
  return pred != 0;
}

// ----------------------------------------------------------------------------------------------
// mbarrier
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred P;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, P;\n\t"
      "}\n"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}

// ----------------------------------------------------------------------------------------------
// TMA
// ----------------------------------------------------------------------------------------------
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
// 2-D tiled load: coordinates are (c0 = innermost, c1 = row).  Out-of-bounds elements are zero-filled
// and still counted in the transaction bytes.
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                            int32_t c1, int32_t c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], "
      "[%2];" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}

// The same load delivered to the same shared-memory offset (and signalling the mbarrier at the same offset) of every CTA
// of the cluster whose bit is set in cta_mask: one L2 read feeds several SMs.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int32_t c0,
                                                      int32_t c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, "
      "%4}], [%2], %5;" ::"r"(smem_u32(smem_dst)),
      "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// 2-D tiled store shared -> global (bulk async group of the issuing thread); out-of-bounds parts of the box are clipped.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* m, const void* smem_src, int32_t c0, int32_t c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(m)),
               "r"(smem_u32(smem_src)), "r"(c0), "r"(c1)
               : "memory");
}
// 1-D bulk copy global -> shared (16-byte aligned addresses, size a multiple of 16), completion on an mbarrier
__device__ __forceinline__ void bulk_load_1d(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// all bulk groups of this thread have finished READING their shared-memory source
__device__ __forceinline__ void bulk_wait_read_all() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// all bulk groups of this thread are complete (writes performed)
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------
// wgmma: warpgroup MMA, operands in shared memory, FP32 accumulators in registers
// ----------------------------------------------------------------------------------------------
// Register layout of an m64nN accumulator d[N / 2] in warp w (0..3) of the warpgroup, lane l: element i sits at row
// 16 w + l / 4 + 8 ((i / 2) % 2), column 8 (i / 4) + 2 (l % 4) + (i % 2).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
// Keeps the compiler from touching accumulator registers across an asynchronous wgmma (they are written behind its back).
template <int R>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// Register budget of a warpgroup (all four warps execute it): producers give registers back, MMA warpgroups take them.
template <int R>
__device__ __forceinline__ void setmaxnreg_dec() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R));
}
template <int R>
__device__ __forceinline__ void setmaxnreg_inc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R));
}
// Arrive on the mbarrier at the same shared-memory offset in CTA `cta` of the cluster.
__device__ __forceinline__ void mbar_arrive_cluster(uint64_t* bar, uint32_t cta) {
  asm volatile(
      "{\n\t"
      ".reg .b32 remote;\n\t"
      "mapa.shared::cluster.u32 remote, %0, %1;\n\t"
      "mbarrier.arrive.release.cluster.shared::cluster.b64 _, [remote];\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(cta)
      : "memory");
}

// Shared-memory matrix descriptor of a K-major tile whose rows are exactly one swizzle span of kRowBytes (128 ->
// 128B swizzle, 64 -> 64B swizzle), as TMA writes it: 8-row core groups are 8 * kRowBytes apart.  sm_90 layout:
// start_address[0,14) (>>4), LBO[16,30) (unused for swizzled K-major, 1), SBO[32,46) (>>4), layout[62,64): 1 = 128B,
// 2 = 64B.  Advancing K by 32 bytes inside the span is +2 on the descriptor.
template <int kRowBytes>
__device__ __forceinline__ uint64_t make_desc_kmajor(uint32_t smem_addr) {
  static_assert(kRowBytes == 128 || kRowBytes == 64, "row = one swizzle span");
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>(1) << 16;
  d |= static_cast<uint64_t>((8 * kRowBytes) >> 4) << 32;
  d |= static_cast<uint64_t>(kRowBytes == 128 ? 1 : 2) << 62;
  return d;
}

// MN-major operand (the MN extent is contiguous) in 128B-swizzle atoms of 8 K-rows x 128 bytes: LBO = byte distance between
// atoms along MN (the next 64 16-bit elements), SBO = byte distance between atoms along K (the next 8 rows).
__device__ __forceinline__ uint64_t make_desc_mnmajor_sw128(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= static_cast<uint64_t>(1) << 62;
  return d;
}

// Operand lists of the wgmma wrappers below: accumulator registers %0.. in blocks of 16, "+f" constraints in blocks of 16.
#define ROHM_R16_0 "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15"
#define ROHM_R16_1 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31"
#define ROHM_R16_2 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47"
#define ROHM_R16_3 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63"
#define ROHM_R16_4 "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79"
#define ROHM_F4(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3])
#define ROHM_F16(i) ROHM_F4(i), ROHM_F4(i + 4), ROHM_F4(i + 8), ROHM_F4(i + 12)
#define ROHM_PRED(n) "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #n ", 0;\n\t"

// D (+)= A * B for one m64nNk16 (fp16) / m64nNk8 (tf32) step, both operands K-major in shared memory.
#define ROHM_WGMMA_SS(KIND, INSTR, R, REGS, A, B, P, IMM, ...)                                                       \
  __device__ __forceinline__ void wgmma_##KIND(float (&d)[R], uint64_t desc_a, uint64_t desc_b) {                 \
    asm volatile(ROHM_PRED(P) INSTR " {" REGS "}, %" #A ", %" #B ", p" IMM ";\n\t}\n"                           \
                 : __VA_ARGS__                                                                                    \
                 : "l"(desc_a), "l"(desc_b), "r"(1));                                                             \
  }
ROHM_WGMMA_SS(f16, "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16", 16, ROHM_R16_0, 16, 17, 18, ", 1, 1, 0, 0",
              ROHM_F16(0))
ROHM_WGMMA_SS(f16, "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16", 32, ROHM_R16_0 ", " ROHM_R16_1, 32, 33, 34,
              ", 1, 1, 0, 0", ROHM_F16(0), ROHM_F16(16))
ROHM_WGMMA_SS(f16, "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16", 48,
              ROHM_R16_0 ", " ROHM_R16_1 ", " ROHM_R16_2, 48, 49, 50, ", 1, 1, 0, 0", ROHM_F16(0), ROHM_F16(16), ROHM_F16(32))
ROHM_WGMMA_SS(f16, "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16", 64,
              ROHM_R16_0 ", " ROHM_R16_1 ", " ROHM_R16_2 ", " ROHM_R16_3, 64, 65, 66, ", 1, 1, 0, 0", ROHM_F16(0),
              ROHM_F16(16), ROHM_F16(32), ROHM_F16(48))
// m64n160k16: the S = Q K^T product of the attention kernel
ROHM_WGMMA_SS(f16, "wgmma.mma_async.sync.aligned.m64n160k16.f32.f16.f16", 80,
              ROHM_R16_0 ", " ROHM_R16_1 ", " ROHM_R16_2 ", " ROHM_R16_3 ", " ROHM_R16_4, 80, 81, 82, ", 1, 1, 0, 0",
              ROHM_F16(0), ROHM_F16(16), ROHM_F16(32), ROHM_F16(48), ROHM_F16(64))
ROHM_WGMMA_SS(tf32, "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32", 16, ROHM_R16_0, 16, 17, 18, ", 1, 1", ROHM_F16(0))
ROHM_WGMMA_SS(tf32, "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32", 32, ROHM_R16_0 ", " ROHM_R16_1, 32, 33, 34,
              ", 1, 1", ROHM_F16(0), ROHM_F16(16))
ROHM_WGMMA_SS(tf32, "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32", 48, ROHM_R16_0 ", " ROHM_R16_1 ", " ROHM_R16_2,
              48, 49, 50, ", 1, 1", ROHM_F16(0), ROHM_F16(16), ROHM_F16(32))
ROHM_WGMMA_SS(tf32, "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32", 64,
              ROHM_R16_0 ", " ROHM_R16_1 ", " ROHM_R16_2 ", " ROHM_R16_3, 64, 65, 66, ", 1, 1", ROHM_F16(0), ROHM_F16(16),
              ROHM_F16(32), ROHM_F16(48))

// m64n128k16 with A from registers (per warp the m16n8k16 A-fragment layout) and an MN-major B in shared memory: the
// O = P V product of the attention kernel
__device__ __forceinline__ void wgmma_f16_rs_tb(float (&d)[64], const uint32_t (&a)[4], uint64_t desc_b) {
  asm volatile(ROHM_PRED(69) "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {" ROHM_R16_0 ", " ROHM_R16_1 ", " ROHM_R16_2
               ", " ROHM_R16_3 "}, {%64, %65, %66, %67}, %68, p, 1, 1, 1;\n\t}\n"
               : ROHM_F16(0), ROHM_F16(16), ROHM_F16(32), ROHM_F16(48)
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(1));
}

// Round-to-nearest TF32 (10-bit mantissa), result kept in an fp32 container.
__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}

// Two-term fp16 split x ~= hi + lo (2 x 11 significant bits, the same 22 bits a TF32 hi/lo pair carries).  hi is
// clamped to the fp16 range so values up to 2 x 65504 still split into finite halves; below 2^-14 the halves go
// subnormal and the split degrades gracefully to an absolute error of 2^-25 per element.
__device__ __forceinline__ void split_f16(float x, __half& hi, __half& lo) {
  const float c = fminf(fmaxf(x, -65504.0f), 65504.0f);
  hi = __float2half_rn(c);
  lo = __float2half_rn(x - __half2float(hi));
}
// Packed form: (x, y) -> half2 words {x in the low half}.  cvt.rn.satfinite.f16x2.f32 rounds to nearest and saturates at
// +-65504, which is the clamp split_f16 applies; bit-identical to two split_f16 calls in 6 instructions.
__device__ __forceinline__ void split_f16x2(float x, float y, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(y), "f"(x));
  const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hi));
  const float lx = x - hf.x, ly = y - hf.y;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(ly), "f"(lx));
}
// (x, y, z, w) -> four hi halves and four lo halves packed for 8-byte stores
__device__ __forceinline__ void split_f16x4(const float4& v, uint2& hi, uint2& lo) {
  split_f16x2(v.x, v.y, hi.x, lo.x);
  split_f16x2(v.z, v.w, hi.y, lo.y);
}

// Programmatic dependent launch hooks (no-ops unless the launch carries the PDL attribute).
__device__ __forceinline__ void pdl_wait_prior_grid() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

}  // namespace ptx
}  // namespace rohm
