// Test-only entry point into the wgmma attention kernels on packed clips (rohm_b200/csrc/attention.cu), driven from Python
// through ctypes by tests/packed_attention_probe.py and linked against the product's own attention and GEMM objects.
// Returns 0, a cudaError_t (> 0) or -CUresult of a failed tensor-map encoding; runs its launch `reps` >= 1 times back to
// back on the default stream, set-up done once, so that tools can time it.  The product library exports none of this.
#include <cstdint>

#include "../../rohm_b200/csrc/attention.cuh"
#include "../../rohm_b200/csrc/gemm.cuh"

using namespace rohm;

extern "C" {

struct ProbePackedAttn {
  const void* qkv_hi;  // [rows, 3D] fp16 planes
  const void* qkv_lo;
  int64_t rows;
  void* ctx_hi;  // [rows, D] fp16 pair
  void* ctx_lo;
  const int* clip_off;  // device: clip c holds rows [clip_off[c], clip_off[c + 1])
  const int* clip_ids;  // device: the n clips this launch runs
  int n, S, D, H;       // S: the most tokens among the listed clips
  float scale;
  int which;  // AttnKernel: kAttnWgmma or kAttnWgmmaStream
  int pdl;
};

int probe_attention_packed(const ProbePackedAttn* q, int reps) {
  if (q->H <= 0 || q->D % q->H != 0 || q->D / q->H != 128 || reps < 1) return static_cast<int>(cudaErrorInvalidValue);
  AttnArgs a{};
  a.qkv_hi = q->qkv_hi, a.qkv_lo = q->qkv_lo, a.rows = q->rows;
  a.ctx_hi = q->ctx_hi, a.ctx_lo = q->ctx_lo;
  a.B = q->n, a.S = q->S, a.D = q->D, a.H = q->H;
  a.scale = q->scale, a.kind = kKindF16;
  a.clip_off = q->clip_off, a.clip_ids = q->clip_ids;
  const cudaError_t e = attention_init_attributes(q->S, 128);
  if (e != cudaSuccess) return static_cast<int>(e);
  AttnWgmmaMaps maps;
  const int rc = attention_wgmma_maps(&maps, a);
  if (rc != 0) return -rc;
  cudaError_t r = cudaSuccess;
  for (int i = 0; i < reps && r == cudaSuccess; ++i) r = launch_attention(a, q->which, &maps, nullptr, q->pdl != 0);
  return static_cast<int>(r);
}

}  // extern "C"
