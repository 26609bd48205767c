// Multi-head self-attention of the PoseNet encoder: softmax(scale Q K^T) V per (clip, head), no mask
// (reference model/posenet.py:63-69).  Five kernels, all reading the QKV GEMM's output rows [B*S, 3D] (Q | K | V, head h
// at columns h*dh) and writing context rows [B*S, D] as a hi/lo pair:
//   * kAttnWgmma:       wgmma on fp16 pairs, head dim 128, clips of at most 160 tokens (the default of ROHM_PRECISION_F16X2);
//   * kAttnWgmmaStream: wgmma on fp16 pairs, head dim 128, clips of any length: K and V stream through a two-stage TMA
//                       ring in blocks of 64 keys with an online (running max / running sum) softmax, so its shared
//                       memory does not grow with the clip (the default of ROHM_PRECISION_F16X2 above 160 tokens);
//   * kAttnMmaF16:      mma.sync m16n8k16 on fp16 pairs, head dim 64 or 128, at most 160 tokens;
//   * kAttnMmaTf32:     mma.sync m16n8k8 on fp32 Q|K|V split into TF32 pairs in registers, head dim 64 or 128, at most 160
//                       tokens; writes TF32 pairs;
//   * kAttnSimt:        fp32 on CUDA cores, either kind, any clip up to 256 tokens whose K and V fit in shared memory.
// Every kernel reads only the rows of its own clip: keys past the clip are masked and never multiply a value row of the
// next clip.
#pragma once
#include <cstddef>
#include <cstdint>
#include <cuda.h>
#include <cuda_runtime.h>

namespace rohm {

enum AttnKernel : int { kAttnAuto = 0, kAttnWgmma = 1, kAttnMmaF16 = 2, kAttnMmaTf32 = 3, kAttnSimt = 4, kAttnWgmmaStream = 5 };

constexpr int kAttnWgmmaMaxTokens = 160;    // padded key count of the wgmma kernel's S product
constexpr int kAttnSimtMaxTokens = 256;     // register budget of the SIMT kernel's logits (8 per lane)
constexpr size_t kAttnSmemLimit = 227 * 1024;  // dynamic shared memory of one CTA on sm_90

// Tensor maps of the wgmma kernels over the Q|K|V planes (built once per buffer: the encoding is a host-side cost).
struct AttnWgmmaMaps {
  CUtensorMap q_hi, q_lo;    // boxes of 64 columns x 64 rows (also the K / V blocks of the streaming kernel)
  CUtensorMap kv_hi, kv_lo;  // boxes of 64 columns x 160 rows
};

struct AttnArgs {
  const void* qkv_hi;  // [rows, 3D]: fp16 hi plane (kKindF16) or fp32 values (kKindTf32)
  const void* qkv_lo;  // [rows, 3D] fp16 lo plane (kKindF16); unused for kKindTf32
  int64_t rows;        // row capacity of the planes (>= B * S)
  void* ctx_hi;        // [B * S, D]: fp16 pair (kKindF16) or TF32 pair in fp32 containers (kKindTf32)
  void* ctx_lo;
  int B, S, D, H;
  float scale;  // usually 1 / sqrt(D / H)
  int kind;     // GemmKind of the planes
  // Packed clips (optional, device arrays, wgmma kernels only): clip c holds rows [clip_off[c], clip_off[c + 1]) of the
  // planes, and the launch runs the B clips listed in clip_ids, S being the most tokens among them.  Null: clip b holds
  // rows [b S, b S + S).
  const int* clip_off = nullptr;
  const int* clip_ids = nullptr;
};

// Encodes the wgmma kernels' tensor maps over the planes of a.  Returns 0 or a CUresult.
int attention_wgmma_maps(AttnWgmmaMaps* maps, const AttnArgs& a);

// Launches one attention.  kAttnAuto picks the kernel the PoseNet engine uses: with `wg` given on fp16 pairs of head
// dim 128, the wgmma kernel up to 160 tokens and the streaming wgmma kernel above; otherwise the mma.sync kernel of the
// kind up to 160 tokens, else the SIMT kernel.  A forced kernel that cannot run the launch (kind, head dim, token count,
// missing maps) is refused with cudaErrorInvalidValue before anything is launched.  Packed clips need a forced wgmma kernel:
// each clip runs with the block decomposition it would get alone, on the kernel the caller chose for the listed clips.
cudaError_t launch_attention(const AttnArgs& a, int which, const AttnWgmmaMaps* wg, cudaStream_t stream, bool pdl);

// Raises the dynamic shared-memory limit of every attention kernel; the SIMT kernel's for clips of up to max_tokens
// tokens of head dim dh, capped at the longest clip it can serve.  Call once per process, outside any stream capture.
cudaError_t attention_init_attributes(int max_tokens, int dh);

// Dynamic shared memory of the SIMT kernel for S tokens of head dim dh.
size_t attention_smem_bytes(int S, int DH);

}  // namespace rohm
