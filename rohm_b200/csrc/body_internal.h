// Internal layout of a rohm_body handle, shared by the translation units that run kernels against the body model
// (body.cu: FK / LBS / skating guidance; glue.cu: inter-round glue, 2-D reprojection guidance, representation recovery).
#pragma once
#include "common.h"
#include "gemm.cuh"

struct rohm_body {
  rohm_ctx* ctx = nullptr;
  rohm::DevicePool pool;
  int V = 0, sd_comps = 0, passes = 3;
  int kind = rohm::kKindTf32;  // operand element type of the blend GEMM (kKindF16 in ROHM_PRECISION_F16X2)
  int64_t max_frames = 0;
  float *Jt = nullptr, *Jd = nullptr;
  const float* lbs_w = nullptr;  // dense weights copy
  float* lbs_w_copy = nullptr;
  int* bone_idx = nullptr;
  float* bone_w = nullptr;
  bool sparse_ok = true;
  rohm::PackedWeight blend;  // [V*3 (padded), kBlendK]
  // per-frame workspace
  float *go = nullptr, *bp = nullptr, *betas = nullptr, *transl = nullptr, *A = nullptr, *feat_h = nullptr,
        *feat_l = nullptr, *vposed = nullptr;
  float *foot = nullptr, *gdir = nullptr, *sums = nullptr;
  float* clip_sums = nullptr;      // [max_frames][4] per-clip skating sums (per-clip normalisers; at most one clip per frame)
  int* parents_dev = nullptr;      // [55] kinematic tree on the device (glue.cu kernels; body.cu keeps a __constant__ copy)
  float* jwork = nullptr;          // [max_frames, 22, 3] scratch joints (glue)
  float* gwork = nullptr;          // [max_frames, 22, 3] scratch joint gradients (2-D guidance)
  rohm::GemmParams g_blend{};
  // fused LBS (blend GEMM with the skinning epilogue, gemm.cuh: GemmParams::skin_A): one launch, v_posed never leaves the SM.
  // Needs fp16 pairs and at most kSkinTileBones distinct bones per 32 consecutive vertices; ROHM_B200_FUSED_LBS=0 keeps the
  // two-kernel path (blend GEMM -> v_posed -> skin_kernel), which is also the fallback.
  rohm::GemmParams g_skin{};
  bool fused_lbs = false;
  int64_t vertex_pitch = 0;  // floats between the vertex rows of two frames in the caller's buffer; 0 = dense (3 V)
  int64_t a_frame_stride = 0;  // fused path: A is [55][12][a_frame_stride] (frames contiguous); two-kernel path: [frames][55][12]
  int* skin_nb = nullptr;
  int* skin_bone = nullptr;
  float* skin_w = nullptr;
  // full LBS pipeline: v_posed double buffer (one chunk each), second stream for the skinning kernels
  int64_t vposed_stride = 0;
  // frames per two-kernel chunk (ROHM_B200_LBS_CHUNK, a multiple of 128)
  int64_t chunk = 4608;
  CUtensorMap st_out_b{};
  cudaStream_t skin_stream = nullptr;
  cudaEvent_t gemm_done[2] = {nullptr, nullptr}, skin_done[2] = {nullptr, nullptr};
  ~rohm_body() {
    if (skin_stream) cudaStreamDestroy(skin_stream);
    for (int i = 0; i < 2; ++i) {
      if (gemm_done[i]) cudaEventDestroy(gemm_done[i]);
      if (skin_done[i]) cudaEventDestroy(skin_done[i]);
    }
  }
};
