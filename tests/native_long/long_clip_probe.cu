// Test-only entry point into the attention kernels (rohm_b200/csrc/attention.cu) for clips of any length, driven from
// Python through ctypes by tests/long_clip_probe.py.  Unlike probe_attention (tests/native/kernel_probe.cu) it raises the
// shared-memory limits of every attention kernel for every clip length and builds the wgmma tensor maps for the streaming
// kernel too, and it can repeat the launch for timing.  Returns 0, a cudaError_t (> 0) or -CUresult of a failed
// tensor-map encoding.
#include <cstdint>

#include "../../rohm_b200/csrc/attention.cuh"
#include "../../rohm_b200/csrc/gemm.cuh"

using namespace rohm;

extern "C" {

struct LongProbeAttn {  // the layout of ProbeAttn (tests/native/kernel_probe.cu)
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

// `reps` back-to-back launch_attention calls on the default stream (tensor maps and attributes set up once).
int long_probe_attention(const LongProbeAttn* q, int reps) {
  AttnArgs a{};
  a.qkv_hi = q->qkv_hi, a.qkv_lo = q->qkv_lo, a.rows = q->rows;
  a.ctx_hi = q->ctx_hi, a.ctx_lo = q->ctx_lo;
  a.B = q->B, a.S = q->S, a.D = q->D, a.H = q->H;
  a.scale = q->scale, a.kind = q->kind;
  if (q->H <= 0 || q->D % q->H != 0 || reps < 1) return static_cast<int>(cudaErrorInvalidValue);
  const int dh = q->D / q->H;
  // the SIMT kernel's limit is capped at what it can serve; a clip it cannot hold is refused by launch_attention
  const cudaError_t e = attention_init_attributes(q->S, dh);
  if (e != cudaSuccess) return static_cast<int>(e);
  AttnWgmmaMaps maps;
  const AttnWgmmaMaps* wg = nullptr;
  if (q->kind == kKindF16 && dh == 128 &&
      (q->which == kAttnWgmma || q->which == kAttnWgmmaStream || q->which == kAttnAuto)) {
    const int rc = attention_wgmma_maps(&maps, a);
    if (rc != 0) return -rc;
    wg = &maps;
  }
  cudaError_t rc = cudaSuccess;
  for (int i = 0; i < reps && rc == cudaSuccess; ++i) rc = launch_attention(a, q->which, wg, nullptr, q->pdl != 0);
  return static_cast<int>(rc);
}

}  // extern "C"
