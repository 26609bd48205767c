// SMPL-X body model kernels: joints-only forward kinematics, the foot-skating guidance gradient (analytic VJP, no
// autograd), and full linear-blend skinning.
//
// Algorithm provenance: the body model arithmetic is third-party smplx==0.1.28 (lbs.py: blend_shapes,
// vertices2joints, batch_rodrigues, batch_rigid_transform, lbs; body_models.py: SMPLX.forward) -- NOT part of the
// reference tree (reference environment.yml:198; call sites model/posenet.py:57-58,
// data_loaders/motion_representation.py:373-398).  The code around it restates the reference:
//   rot6d_to_rotmat                 data_loaders/common/quaternion.py:482-501
//   rotation_matrix_to_angle_axis   utils/konia_transform.py:317-340, 350-444, 561-631
//   recover_from_repr_smpl          data_loaders/motion_representation.py:285-398
//   guide_skating_with_smpl         model/posenet.py:196-257
//
// Guidance design.  The reference differentiates  x0 -> denorm -> {abs-traj joints, 6D -> R -> quat -> aa ->
// Rodrigues -> FK joints} -> foot velocity -> masked mean  with autograd and then zeroes channels [0, traj) and the
// 4 contact channels.  Only feet (joints 7, 10, 8, 11) enter the loss, so only the two leg chains
// 0-1-4-7-10 / 0-2-5-8-11 are evaluated; only local_positions of the 4 foot joints, the 6-D rotations of body joints
// {1,2,4,5,7,8} and betas receive a non-zero gradient.  R -> axis-angle -> Rodrigues is the identity on SO(3), and the
// Gram-Schmidt output only moves inside SO(3), so its Jacobian contribution is the identity: the VJP goes straight
// from the joint rotation matrices to the 6-D inputs (differences to the reference's autograd: its eps clamps below
// ~2e-3 rad and fp32 round-off of the round trip).
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <new>
#include <vector>

#include "common.h"
#include "gemm.cuh"
#include "kin.cuh"
#include "ptx.cuh"

namespace rohm {
namespace {

using namespace kin;

constexpr int kJ = 55;        // SMPL-X joints
constexpr int kBodyJ = 22;    // global + 21 body joints
constexpr int kBetas = 10;
constexpr int kPoseFeat = 189;  // (22 - 1) * 9 non-zero pose-corrective features (hands / jaw / eyes are identity)
constexpr int kBlendK = 256;    // 189 pose features + 10 betas + 1 (template), zero-padded to whole K blocks (64 fp16 / 32 TF32)
constexpr int kMaxBones = 8;    // compressed skinning weights per vertex

__constant__ int c_parents[kJ];

// ---------------------------------------------------------------------------------------------------------------
// model preparation
// ---------------------------------------------------------------------------------------------------------------
// Jt[j][k] = sum_v Jreg[j][v] * v_template[v][k];  Jd[j][k][l] = sum_v Jreg[j][v] * shapedirs[v][k][l]  (l < 10)
__global__ void joint_regress_kernel(const float* __restrict__ Jreg, const float* __restrict__ vt,
                                     const float* __restrict__ sdirs, int V, int sd_comps, float* __restrict__ Jt,
                                     float* __restrict__ Jd) {
  const int j = blockIdx.x;       // joint
  const int q = blockIdx.y;       // 0..2: template xyz; 3..32: dirs (k*10 + l)
  float acc = 0.0f;
  for (int v = threadIdx.x; v < V; v += blockDim.x) {
    const float w = Jreg[static_cast<int64_t>(j) * V + v];
    if (w != 0.0f) {
      const float val = q < 3 ? vt[static_cast<int64_t>(v) * 3 + q]
                              : sdirs[(static_cast<int64_t>(v) * 3 + (q - 3) / kBetas) * sd_comps + (q - 3) % kBetas];
      acc = fmaf(w, val, acc);
    }
  }
  __shared__ float red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    if (q < 3) Jt[j * 3 + q] = red[0];
    else Jd[j * 30 + (q - 3)] = red[0];
  }
}

// Blend matrix for the GEMM: Wb[n = v*3 + k][col]: cols [0,189) posedirs[col][n], [189,199) shapedirs[v][k][l],
// col 199 = v_template[v][k], rest 0; stored as TF32 hi/lo, or (f16) as fp16 hi/lo of the value times `scale`.
__global__ void build_blend_kernel(const float* __restrict__ posedirs, const float* __restrict__ sdirs,
                                   const float* __restrict__ vt, int V, int sd_comps, float* __restrict__ hi,
                                   float* __restrict__ lo, int64_t total, int f16, float scale) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int col = static_cast<int>(i % kBlendK);
  const int64_t n = i / kBlendK;
  float v = 0.0f;
  if (n < static_cast<int64_t>(V) * 3) {
    if (col < kPoseFeat) v = posedirs[static_cast<int64_t>(col) * V * 3 + n];
    else if (col < kPoseFeat + kBetas) v = sdirs[n * sd_comps + (col - kPoseFeat)];
    else if (col == kPoseFeat + kBetas) v = vt[n];
  }
  if (f16) {
    ptx::split_f16(v * scale, reinterpret_cast<__half*>(hi)[i], reinterpret_cast<__half*>(lo)[i]);
  } else {
    const float h = ptx::to_tf32(v);
    hi[i] = h;
    lo[i] = v - h;
  }
}

// one element of a GEMM operand pair: TF32 hi/lo in fp32 containers, or fp16 hi/lo
__device__ __forceinline__ void store_pair(float* hi, float* lo, int64_t i, float v, int f16) {
  if (f16) {
    ptx::split_f16(v, reinterpret_cast<__half*>(hi)[i], reinterpret_cast<__half*>(lo)[i]);
  } else {
    const float h = ptx::to_tf32(v);
    hi[i] = h;
    lo[i] = v - h;
  }
}

// up to kMaxBones (index, weight) pairs per vertex; overflow flag if a vertex has more non-zeros
__global__ void compress_weights_kernel(const float* __restrict__ W, int V, int* __restrict__ idx, float* __restrict__ wt,
                                        int* __restrict__ overflow) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  int n = 0;
  for (int j = 0; j < kJ; ++j) {
    const float w = W[static_cast<int64_t>(v) * kJ + j];
    if (w != 0.0f) {
      if (n < kMaxBones) idx[v * kMaxBones + n] = j, wt[v * kMaxBones + n] = w;
      ++n;
    }
  }
  for (int k = n; k < kMaxBones; ++k) idx[v * kMaxBones + k] = 0, wt[v * kMaxBones + k] = 0.0f;
  if (n > kMaxBones) atomicExch(overflow, 1);
}

// ---------------------------------------------------------------------------------------------------------------
// forward kinematics of all 55 joints + pose features + skinning transforms, one thread per frame
// ---------------------------------------------------------------------------------------------------------------
// go [N,3], bp [N,63] axis-angle, betas [N,10], transl [N,3].  Outputs (each optional):
//   joints [N, nj, 3] (posed joints + transl, nj <= 55), A [N, 55, 12] (rows of the 3x4 skinning transform),
//   feat hi/lo [N, kBlendK] (pose_feature | betas | 1 | 0...) for the blend GEMM.
// One WARP per frame: lane j (and j + 32) owns joint j; rest joints and local rotations are computed in parallel, the
// kinematic tree is then walked level by level (a joint is composed once its parent's world transform is in shared
// memory; SMPL-X depth is 12).  The thread-per-frame version kept 55 world transforms in local memory and ran at 36 CTAs.
constexpr int kFkWarps = 8;
__global__ void __launch_bounds__(32 * kFkWarps) fk_full_kernel(const float* __restrict__ go, const float* __restrict__ bp,
                                                                const float* __restrict__ betas,
                                                                const float* __restrict__ transl,
                                                                const float* __restrict__ Jt, const float* __restrict__ Jd,
                                                                int N, float* __restrict__ joints, int nj,
                                                                float* __restrict__ A, int64_t a_frame_stride,
                                                                float* __restrict__ feat_hi, float* __restrict__ feat_lo,
                                                                int f16) {
  __shared__ float sW[kFkWarps][kJ][12];   // world transforms [R | t] row-major 3x4
  __shared__ float sJ[kFkWarps][kJ][3];    // rest joints
  __shared__ int sDone[kFkWarps][kJ];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n = blockIdx.x * kFkWarps + warp;
  if (n >= N) return;  // whole warp
  float be[kBetas];
#pragma unroll
  for (int l = 0; l < kBetas; ++l) be[l] = betas[static_cast<int64_t>(n) * kBetas + l];
  const V3 tr = {transl[n * 3], transl[n * 3 + 1], transl[n * 3 + 2]};
  M3 Rl[2];
  for (int h = 0; h < 2; ++h) {
    const int j = lane + 32 * h;
    if (j >= kJ) break;
    V3 J = {Jt[j * 3], Jt[j * 3 + 1], Jt[j * 3 + 2]};
#pragma unroll
    for (int l = 0; l < kBetas; ++l) {
      J.x = fmaf(Jd[j * 30 + l], be[l], J.x);
      J.y = fmaf(Jd[j * 30 + 10 + l], be[l], J.y);
      J.z = fmaf(Jd[j * 30 + 20 + l], be[l], J.z);
    }
    sJ[warp][j][0] = J.x, sJ[warp][j][1] = J.y, sJ[warp][j][2] = J.z;
    M3 R = {{1.f, 0.f, 0.f}, {0.f, 1.f, 0.f}, {0.f, 0.f, 1.f}};
    if (j < kBodyJ) {
      const float* r = (j == 0) ? go + static_cast<int64_t>(n) * 3 : bp + static_cast<int64_t>(n) * 63 + (j - 1) * 3;
      R = rodrigues({r[0], r[1], r[2]});
      if (j > 0 && feat_hi != nullptr) {
        const float pf[9] = {R.c0.x - 1.f, R.c1.x, R.c2.x, R.c0.y, R.c1.y - 1.f, R.c2.y, R.c0.z, R.c1.z, R.c2.z - 1.f};
#pragma unroll
        for (int e = 0; e < 9; ++e) store_pair(feat_hi, feat_lo, static_cast<int64_t>(n) * kBlendK + (j - 1) * 9 + e, pf[e], f16);
      }
    }
    Rl[h] = R;
    sDone[warp][j] = 0;
  }
  if (feat_hi != nullptr) {
    for (int c = kPoseFeat + lane; c < kBlendK; c += 32) {  // betas | 1 | zero padding
      const int k = c - kPoseFeat;
      const float v = k < kBetas ? be[k < kBetas ? k : 0] : (k == kBetas ? 1.0f : 0.0f);
      store_pair(feat_hi, feat_lo, static_cast<int64_t>(n) * kBlendK + c, v, f16);
    }
  }
  __syncwarp();
  // level-synchronous walk of the kinematic tree (parents precede children in index order)
  bool mine_done[2] = {false, false};
  for (int level = 0; level < kJ; ++level) {
    bool progressed = false;
    for (int h = 0; h < 2; ++h) {
      const int j = lane + 32 * h;
      if (j >= kJ || mine_done[h]) continue;
      const int p = c_parents[j];
      if (p >= 0 && sDone[warp][p] == 0) continue;
      const V3 J = {sJ[warp][j][0], sJ[warp][j][1], sJ[warp][j][2]};
      M3 Wr;
      V3 Wt;
      if (p < 0) {
        Wr = Rl[h], Wt = J;
      } else {
        const float* w = sW[warp][p];
        const M3 Pr = {{w[0], w[4], w[8]}, {w[1], w[5], w[9]}, {w[2], w[6], w[10]}};
        const V3 Pt = {w[3], w[7], w[11]};
        const V3 Jp = {sJ[warp][p][0], sJ[warp][p][1], sJ[warp][p][2]};
        Wr = mul(Pr, Rl[h]);
        Wt = Pt + mul(Pr, J - Jp);
      }
      float* w = sW[warp][j];
      w[0] = Wr.c0.x, w[1] = Wr.c1.x, w[2] = Wr.c2.x, w[3] = Wt.x;
      w[4] = Wr.c0.y, w[5] = Wr.c1.y, w[6] = Wr.c2.y, w[7] = Wt.y;
      w[8] = Wr.c0.z, w[9] = Wr.c1.z, w[10] = Wr.c2.z, w[11] = Wt.z;
      mine_done[h] = true;
      progressed = true;
      if (joints != nullptr && j < nj) {
        float* o = joints + (static_cast<int64_t>(n) * nj + j) * 3;
        o[0] = Wt.x + tr.x, o[1] = Wt.y + tr.y, o[2] = Wt.z + tr.z;
      }
      if (A != nullptr) {  // A_j = [W_r | W_t - W_r J_rest + transl]
        const V3 t = Wt - mul(Wr, J) + tr;
        const float a12[12] = {Wr.c0.x, Wr.c1.x, Wr.c2.x, t.x, Wr.c0.y, Wr.c1.y, Wr.c2.y, t.y, Wr.c0.z, Wr.c1.z, Wr.c2.z, t.z};
        if (a_frame_stride == 0) {  // [frame][joint][12]: skin_kernel stages whole frames
          float* o = A + (static_cast<int64_t>(n) * kJ + j) * 12;
#pragma unroll
          for (int e = 0; e < 12; ++e) o[e] = a12[e];
        } else {  // [joint][12][frame]: the fused skinning epilogue reads one frame per lane, coalesced
          float* o = A + static_cast<int64_t>(j) * 12 * a_frame_stride + n;
#pragma unroll
          for (int e = 0; e < 12; ++e) o[e * a_frame_stride] = a12[e];
        }
      }
    }
    __syncwarp();
    for (int h = 0; h < 2; ++h) {
      const int j = lane + 32 * h;
      if (j < kJ && mine_done[h]) sDone[warp][j] = 1;
    }
    __syncwarp();
    if (!__any_sync(0xffffffffu, progressed)) break;
  }
}

// verts[n][v] = sum_k w_k A[n][j_k] [v_posed[n][v]; 1]   (translation already folded into A)
// One CTA = 256 vertices x kSkinFrames frames: the 8 (bone, weight) pairs of a vertex are read once and kept in
// registers for all frames (re-reading them per frame was 5x the algorithmic traffic), the frames' 55 x 12 transform
// tables are staged in shared memory.  HBM-bound: 12 B in + 12 B out per vertex and frame.
constexpr int kSkinFrames = 16;
// grid = (vertex blocks, Y): CTA (vb, y) keeps the (bone, weight) pairs of its 256 vertices in registers and walks the frame
// blocks y, y + Y, ... of the chunk; Y is chosen by the host so that the grid is one full wave (5 CTAs of 42 KB per SM), which
// removes the partial-wave tail that a (vertex blocks x frame blocks) grid has for most frame counts.
__global__ void __launch_bounds__(256, 4) skin_kernel(const float* __restrict__ vposed, int64_t vp_pitch,
                                                      const float* __restrict__ A, const int* __restrict__ idx,
                                                   const float* __restrict__ wt, int V, int64_t N,
                                                   float* __restrict__ verts) {
  __shared__ __align__(16) float sA[kSkinFrames][kJ * 12];
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  int bi[kMaxBones];
  float bw[kMaxBones];
  if (v < V) {
    const int4 i0 = *reinterpret_cast<const int4*>(idx + v * kMaxBones);
    const int4 i1 = *reinterpret_cast<const int4*>(idx + v * kMaxBones + 4);
    const float4 w0 = *reinterpret_cast<const float4*>(wt + v * kMaxBones);
    const float4 w1 = *reinterpret_cast<const float4*>(wt + v * kMaxBones + 4);
    bi[0] = i0.x, bi[1] = i0.y, bi[2] = i0.z, bi[3] = i0.w, bi[4] = i1.x, bi[5] = i1.y, bi[6] = i1.z, bi[7] = i1.w;
    bw[0] = w0.x, bw[1] = w0.y, bw[2] = w0.z, bw[3] = w0.w, bw[4] = w1.x, bw[5] = w1.y, bw[6] = w1.z, bw[7] = w1.w;
  }
  const int64_t frame_blocks = (N + kSkinFrames - 1) / kSkinFrames;
  for (int64_t fb = blockIdx.y; fb < frame_blocks; fb += gridDim.y) {
    const int64_t n0 = fb * kSkinFrames;
    const int nf = static_cast<int>(min(static_cast<int64_t>(kSkinFrames), N - n0));
    __syncthreads();  // the previous frame block's transforms are no longer read
    {
      const float4* src = reinterpret_cast<const float4*>(A + n0 * kJ * 12);
      float4* dst = reinterpret_cast<float4*>(&sA[0][0]);
      for (int i = threadIdx.x; i < nf * kJ * 3; i += blockDim.x) dst[i] = src[i];
    }
    __syncthreads();
    if (v >= V) continue;
    // Four frames per iteration: all streaming loads are issued before the first dependent use (the loop is bound by load
    // latency: ncu showed 12.6 stall cycles on long scoreboard per issued instruction with one frame in flight).
    constexpr int kFramesInFlight = 4;
    for (int f0 = 0; f0 < nf; f0 += kFramesInFlight) {
      float px[kFramesInFlight], py[kFramesInFlight], pz[kFramesInFlight];
#pragma unroll
      for (int u = 0; u < kFramesInFlight; ++u) {
        const int f = min(f0 + u, nf - 1);
        const float* p = vposed + (n0 + f) * vp_pitch + static_cast<int64_t>(v) * 3;
        px[u] = __ldcs(p), py[u] = __ldcs(p + 1), pz[u] = __ldcs(p + 2);  // read once: evict-first
      }
#pragma unroll
      for (int u = 0; u < kFramesInFlight; ++u) {
        const int f = f0 + u;
        if (f >= nf) break;
        float T[12];
#pragma unroll
        for (int e = 0; e < 12; ++e) T[e] = 0.0f;
#pragma unroll
        for (int k = 0; k < kMaxBones; ++k) {
          if (bw[k] != 0.0f) {
            const float4* a = reinterpret_cast<const float4*>(sA[f] + bi[k] * 12);  // 3 x 128-bit smem loads per bone
            const float4 r0 = a[0], r1 = a[1], r2 = a[2];
            const float w = bw[k];
            T[0] = fmaf(w, r0.x, T[0]), T[1] = fmaf(w, r0.y, T[1]), T[2] = fmaf(w, r0.z, T[2]), T[3] = fmaf(w, r0.w, T[3]);
            T[4] = fmaf(w, r1.x, T[4]), T[5] = fmaf(w, r1.y, T[5]), T[6] = fmaf(w, r1.z, T[6]), T[7] = fmaf(w, r1.w, T[7]);
            T[8] = fmaf(w, r2.x, T[8]), T[9] = fmaf(w, r2.y, T[9]), T[10] = fmaf(w, r2.z, T[10]), T[11] = fmaf(w, r2.w, T[11]);
          }
        }
        float* o = verts + ((n0 + f) * V + v) * 3;
        __stcs(o, T[0] * px[u] + T[1] * py[u] + T[2] * pz[u] + T[3]);  // written once, never re-read by this library
        __stcs(o + 1, T[4] * px[u] + T[5] * py[u] + T[6] * pz[u] + T[7]);
        __stcs(o + 2, T[8] * px[u] + T[9] * py[u] + T[10] * pz[u] + T[11]);
      }
    }
  }
}

// dense fallback when a vertex has more than kMaxBones non-zero weights
__global__ void __launch_bounds__(256) skin_dense_kernel(const float* __restrict__ vposed, int64_t vp_pitch,
                                                         const float* __restrict__ A, const float* __restrict__ W, int V,
                                                         float* __restrict__ verts) {
  __shared__ float sA[kJ * 12];
  const int n = blockIdx.y;
  for (int i = threadIdx.x; i < kJ * 12; i += blockDim.x) sA[i] = A[static_cast<int64_t>(n) * kJ * 12 + i];
  __syncthreads();
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= V) return;
  const float* p = vposed + static_cast<int64_t>(n) * vp_pitch + static_cast<int64_t>(v) * 3;
  const float x = p[0], y = p[1], z = p[2];
  float T[12];
#pragma unroll
  for (int e = 0; e < 12; ++e) T[e] = 0.0f;
  for (int j = 0; j < kJ; ++j) {
    const float w = W[static_cast<int64_t>(v) * kJ + j];
#pragma unroll
    for (int e = 0; e < 12; ++e) T[e] = fmaf(w, sA[j * 12 + e], T[e]);
  }
  float* o = verts + (static_cast<int64_t>(n) * V + v) * 3;
  o[0] = T[0] * x + T[1] * y + T[2] * z + T[3];
  o[1] = T[4] * x + T[5] * y + T[6] * z + T[7];
  o[2] = T[8] * x + T[9] * y + T[10] * z + T[11];
}

// ---------------------------------------------------------------------------------------------------------------
// motion representation [B, 294, 1, T] -> SMPL-X parameters (rot6d -> R -> axis-angle), one thread per (frame, joint)
// ---------------------------------------------------------------------------------------------------------------
constexpr int kC = 294;
constexpr int kChAngle = 0, kChRootPos = 2, kChHeight = 6, kChRot6d = 7, kChTrans = 16, kChLocalPos = 22,
              kChBodyPose = 154, kChBetas = 280, kChContact = 290;

// element (b, c, t) of x lives at x[b * sb + c * sc + t * st]: channel-major [B,294,1,T] (sb = 294 T, sc = T, st = 1,
// PoseNet tensors) or channels-last [B,T,294] (sb = 294 T, sc = 1, st = 294: TrajNet-side / driver tensors).
// kLengths: clip b has clip_off[b + 1] - clip_off[b] <= T frames; only those are gathered, packed: frame t of clip b
// becomes row f = clip_off[b] + t of go / bp / betas / transl (`total` rows), and frames past a clip are never read.
template <bool kLengths>
__global__ void repr_to_smplx_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int64_t st,
                                     const float* __restrict__ mean,
                                     const float* __restrict__ stdv, int B, int T, float* __restrict__ go,
                                     float* __restrict__ bp, float* __restrict__ betas, float* __restrict__ transl,
                                     const int* __restrict__ clip_off, int64_t total) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t frames = kLengths ? total : static_cast<int64_t>(B) * T;
  if (i >= frames * kBodyJ) return;
  const int j = static_cast<int>(i % kBodyJ);
  const int64_t f = i / kBodyJ;
  const int b = kLengths ? clip_of_frame(clip_off, B, static_cast<int>(f)) : static_cast<int>(f / T);
  const int t = kLengths ? static_cast<int>(f) - clip_off[b] : static_cast<int>(f % T);
  if (kLengths && (t >= clip_off[b + 1] - clip_off[b] || t >= T)) return;
  auto ch = [&](int c) { return x[b * sb + c * sc + t * st] * stdv[c] + mean[c]; };
  const int c0 = (j == 0) ? kChRot6d : kChBodyPose + (j - 1) * 6;
  float r6[6];
#pragma unroll
  for (int e = 0; e < 6; ++e) r6[e] = ch(c0 + e);
  const V3 aa = mat_to_aa(rot6d_to_mat(r6));
  float* o = (j == 0) ? go + f * 3 : bp + f * 63 + (j - 1) * 3;
  o[0] = aa.x, o[1] = aa.y, o[2] = aa.z;
  if (j == 0) {
#pragma unroll
    for (int l = 0; l < kBetas; ++l) betas[f * kBetas + l] = ch(kChBetas + l);
#pragma unroll
    for (int k = 0; k < 3; ++k) transl[f * 3 + k] = ch(kChTrans + k);
  }
}

// ---------------------------------------------------------------------------------------------------------------
// skating guidance (posenet.py:196-257), one thread per frame
// ---------------------------------------------------------------------------------------------------------------
// leg chains: joints 0-1-4-7-10 (left) and 0-2-5-8-11 (right); foot joints in the reference's order [7, 10, 8, 11]
struct LegFK {
  M3 W[4];  // world rotations of joints (0, hip, knee, ankle)
  V3 p[5];  // world positions of (0, hip, knee, ankle, toe)
  V3 d[5];  // rest offsets J_j - J_parent (d[0] = J_0)
};

__device__ __forceinline__ void leg_forward(const M3& R0, const M3* R, const V3* d, LegFK& L) {
  L.W[0] = R0;
  L.p[0] = d[0];
  for (int k = 1; k <= 4; ++k) {
    L.p[k] = L.p[k - 1] + mul(L.W[k - 1], d[k]);
    if (k <= 3) L.W[k] = mul(L.W[k - 1], R[k - 1]);
  }
}

struct GuideWs {
  float* foot;   // [2 paths][B*T][4][3] foot joint positions (path 0: abs traj, 1: SMPL-X)
  float* gdir;   // [2][B*T][4][3] dL/dposition before the 1/count normalisation
  float* sums;   // [4]: sum_abs, cnt_abs, sum_smpl, cnt_smpl; per-clip normalisers: [B][4], the same four per clip
};

__device__ __forceinline__ float ld_ch(const float* x, const float* mean, const float* stdv, int b, int t, int T, int c) {
  return x[(static_cast<int64_t>(b) * kC + c) * T + t] * stdv[c] + mean[c];
}

// pass 1: foot joint positions of both recovery paths
__global__ void __launch_bounds__(128) guide_forward_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                                            const float* __restrict__ stdv, const float* __restrict__ Jt,
                                                            const float* __restrict__ Jd, int B, int T, GuideWs ws) {
  const int64_t f = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t frames = static_cast<int64_t>(B) * T;
  if (f >= frames) return;
  const int b = static_cast<int>(f / T), t = static_cast<int>(f % T);
  auto ch = [&](int c) { return ld_ch(x, mean, stdv, b, t, T, c); };
  // ---- abs-traj path: p = Rz(-2a) lp + (rx, ry, 0)  (qrot(qinv(q)), q = (cos a, 0, 0, sin a)) ----
  {
    const float a = ch(kChAngle), rx = ch(kChRootPos), ry = ch(kChRootPos + 1);
    float sn, cs;
    sincosf(a, &sn, &cs);
    const int feet[4] = {7, 10, 8, 11};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const V3 v = {ch(kChLocalPos + feet[k] * 3), ch(kChLocalPos + feet[k] * 3 + 1), ch(kChLocalPos + feet[k] * 3 + 2)};
      // v + 2 (w (qv x v) + qv x (qv x v)), qv = (0, 0, -sin a), w = cos a
      const V3 qv = {0.0f, 0.0f, -sn};
      const V3 uv = cross(qv, v);
      const V3 uuv = cross(qv, uv);
      const V3 p = {v.x + 2.0f * (cs * uv.x + uuv.x) + rx, v.y + 2.0f * (cs * uv.y + uuv.y) + ry,
                    v.z + 2.0f * (cs * uv.z + uuv.z)};
      float* o = ws.foot + (f * 4 + k) * 3;
      o[0] = p.x, o[1] = p.y, o[2] = p.z;
    }
  }
  // ---- SMPL-X path ----
  {
    float be[kBetas];
#pragma unroll
    for (int l = 0; l < kBetas; ++l) be[l] = ch(kChBetas + l);
    auto restJ = [&](int j) {
      V3 J = {Jt[j * 3], Jt[j * 3 + 1], Jt[j * 3 + 2]};
#pragma unroll
      for (int l = 0; l < kBetas; ++l) {
        J.x = fmaf(Jd[j * 30 + l], be[l], J.x);
        J.y = fmaf(Jd[j * 30 + 10 + l], be[l], J.y);
        J.z = fmaf(Jd[j * 30 + 20 + l], be[l], J.z);
      }
      return J;
    };
    auto rotJ = [&](int j) {
      float r6[6];
      const int c0 = (j == 0) ? kChRot6d : kChBodyPose + (j - 1) * 6;
#pragma unroll
      for (int e = 0; e < 6; ++e) r6[e] = ch(c0 + e);
      return rodrigues(mat_to_aa(rot6d_to_mat(r6)));  // the reference's 6D -> R -> axis-angle -> R round trip
    };
    const V3 tr = {ch(kChTrans), ch(kChTrans + 1), ch(kChTrans + 2)};
    const M3 R0 = rotJ(0);
    const V3 J0 = restJ(0);
    const int chain[2][4] = {{1, 4, 7, 10}, {2, 5, 8, 11}};
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      M3 R[3];
      V3 d[5];
      d[0] = J0;
      V3 prev = J0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const V3 J = restJ(chain[s][k]);
        d[k + 1] = J - prev;
        prev = J;
        if (k < 3) R[k] = rotJ(chain[s][k]);
      }
      LegFK L;
      leg_forward(R0, R, d, L);
      float* o = ws.foot + ((frames + f) * 4 + s * 2) * 3;  // [ankle, toe] of this side: order 7,10 | 8,11
      o[0] = L.p[3].x + tr.x, o[1] = L.p[3].y + tr.y, o[2] = L.p[3].z + tr.z;
      o[3] = L.p[4].x + tr.x, o[4] = L.p[4].y + tr.y, o[5] = L.p[4].z + tr.z;
    }
  }
}

// pass 2: foot speeds, masks, loss sums, and dL/dposition directions.  kMasked: clip b has lengths[b] real frames (device
// int[B]); a velocity pair counts only inside them, so later frames add nothing and get no direction.  kPerClip: the sums
// go to clip b's row of ws.sums [B][4].  The counts are integer-valued floats below 2^24, so they come out exact whatever
// order the atomics land in; the speed sums do depend on that order.
template <bool kMasked, bool kPerClip>
__global__ void __launch_bounds__(128) guide_loss_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                                         const float* __restrict__ stdv, int B, int T, GuideWs ws,
                                                         const int* __restrict__ lengths) {
  const int64_t f = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t frames = static_cast<int64_t>(B) * T;
  float lsum[2] = {0.f, 0.f}, lcnt[2] = {0.f, 0.f};
  if (f < frames) {
    const int b = static_cast<int>(f / T), t = static_cast<int>(f % T);
    const int len = kMasked ? lengths[b] : T;
#pragma unroll
    for (int path = 0; path < 2; ++path) {
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        // gradient on p(t) = +m(t-1) vhat(t-1) - m(t) vhat(t), each scaled by fps (d|v|/dp)
        V3 g = {0.f, 0.f, 0.f};
        const float* p0 = ws.foot + ((path * frames + f) * 4 + k) * 3;
        if (t + 1 < len) {
          const float* p1 = p0 + 12;
          const V3 v = {(p1[0] - p0[0]) * 30.0f, (p1[1] - p0[1]) * 30.0f, (p1[2] - p0[2]) * 30.0f};
          const float sp = sqrtf(dot(v, v));
          const float contact = ld_ch(x, mean, stdv, b, t, T, kChContact + k) > 0.5f ? 1.0f : 0.0f;
          if (sp - 0.1f > 0.0f && contact > 0.0f) {
            lsum[path] += sp, lcnt[path] += 1.0f;
            g = g - (30.0f / sp) * v;
          }
        }
        if (t > 0 && (!kMasked || t < len)) {
          const float* pm = p0 - 12;
          const V3 v = {(p0[0] - pm[0]) * 30.0f, (p0[1] - pm[1]) * 30.0f, (p0[2] - pm[2]) * 30.0f};
          const float sp = sqrtf(dot(v, v));
          const float contact = ld_ch(x, mean, stdv, b, t - 1, T, kChContact + k) > 0.5f ? 1.0f : 0.0f;
          if (sp - 0.1f > 0.0f && contact > 0.0f) g = g + (30.0f / sp) * v;
        }
        float* o = ws.gdir + ((path * frames + f) * 4 + k) * 3;
        o[0] = g.x, o[1] = g.y, o[2] = g.z;
      }
    }
  }
  if constexpr (kPerClip) {
    // a warp whose frames all lie in one clip adds its warp totals; a warp that straddles clips adds per thread
    const unsigned lane = threadIdx.x & 31u;
    const int b = f < frames ? static_cast<int>(f / T) : -1;
    const int b0 = __shfl_sync(0xffffffffu, b, 0);
    float v[4] = {lsum[0], lcnt[0], lsum[1], lcnt[1]};
    if (__all_sync(0xffffffffu, b == b0 || b < 0)) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v[q] += __shfl_xor_sync(0xffffffffu, v[q], o);
      if (lane == 0 && b0 >= 0)
#pragma unroll
        for (int q = 0; q < 4; ++q)
          if (v[q] != 0.0f) atomicAdd(ws.sums + static_cast<int64_t>(b0) * 4 + q, v[q]);
    } else if (b >= 0) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (v[q] != 0.0f) atomicAdd(ws.sums + static_cast<int64_t>(b) * 4 + q, v[q]);
    }
    return;
  }
  // block reduction of the four scalars, then one atomic each
  __shared__ float red[4][128];
  red[0][threadIdx.x] = lsum[0], red[1][threadIdx.x] = lcnt[0], red[2][threadIdx.x] = lsum[1], red[3][threadIdx.x] = lcnt[1];
  __syncthreads();
  for (int s = blockDim.x / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s)
      for (int q = 0; q < 4; ++q) red[q][threadIdx.x] += red[q][threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x < 4 && red[threadIdx.x][0] != 0.0f) atomicAdd(ws.sums + threadIdx.x, red[threadIdx.x][0]);
}

// pass 3: VJP to the normalised representation; grad = d(-(loss_smpl + loss_abs))/dx0, channels [0,traj) and the
// contact channels are zero (the output buffer was cleared; only the channels with a non-zero gradient are written).
// kPerClip: clip b is scaled by its own counts, row b of ws.sums [B][4].
template <bool kPerClip>
__global__ void __launch_bounds__(128) guide_backward_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                                             const float* __restrict__ stdv, const float* __restrict__ Jt,
                                                             const float* __restrict__ Jd, int B, int T, GuideWs ws,
                                                             float* __restrict__ grad, const int* __restrict__ lengths) {
  const int64_t f = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t frames = static_cast<int64_t>(B) * T;
  if (f >= frames) return;
  const int b = static_cast<int>(f / T), t = static_cast<int>(f % T);
  if (lengths != nullptr && t >= lengths[b]) return;  // past the clip: the cleared zero gradient
  auto ch = [&](int c) { return ld_ch(x, mean, stdv, b, t, T, c); };
  auto put = [&](int c, float g) { grad[(static_cast<int64_t>(b) * kC + c) * T + t] = g * stdv[c]; };
  const float* sums = kPerClip ? ws.sums + static_cast<int64_t>(b) * 4 : ws.sums;
  const float cnt_abs = sums[1], cnt_smpl = sums[3];
  const float sc_abs = cnt_abs != 0.0f ? -1.0f / cnt_abs : 0.0f;   // loss enters as -(loss)
  const float sc_smpl = cnt_smpl != 0.0f ? -1.0f / cnt_smpl : 0.0f;
  // ---- abs path: p = Rz(-2a) lp + ...;  dL/dlp = Rz(-2a)^T g ----
  {
    const float a = ch(kChAngle);
    float sn, cs;
    sincosf(2.0f * a, &sn, &cs);  // Rz(-2a) = [[c, s, 0], [-s, c, 0], [0, 0, 1]]
    const int feet[4] = {7, 10, 8, 11};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float* g = ws.gdir + (f * 4 + k) * 3;
      const float gx = sc_abs * g[0], gy = sc_abs * g[1], gz = sc_abs * g[2];
      put(kChLocalPos + feet[k] * 3, cs * gx - sn * gy);
      put(kChLocalPos + feet[k] * 3 + 1, sn * gx + cs * gy);
      put(kChLocalPos + feet[k] * 3 + 2, gz);
    }
  }
  // ---- SMPL-X path ----
  {
    float be[kBetas], gbe[kBetas];
#pragma unroll
    for (int l = 0; l < kBetas; ++l) be[l] = ch(kChBetas + l), gbe[l] = 0.0f;
    auto restJ = [&](int j) {
      V3 J = {Jt[j * 3], Jt[j * 3 + 1], Jt[j * 3 + 2]};
#pragma unroll
      for (int l = 0; l < kBetas; ++l) {
        J.x = fmaf(Jd[j * 30 + l], be[l], J.x);
        J.y = fmaf(Jd[j * 30 + 10 + l], be[l], J.y);
        J.z = fmaf(Jd[j * 30 + 20 + l], be[l], J.z);
      }
      return J;
    };
    // dL/dbeta += (dJ_j/dbeta)^T g  for a gradient g on the rest position of joint j (sign: +1 for J_j, -1 for parent)
    auto acc_beta = [&](int j, V3 g, float sign) {
#pragma unroll
      for (int l = 0; l < kBetas; ++l)
        gbe[l] += sign * (Jd[j * 30 + l] * g.x + Jd[j * 30 + 10 + l] * g.y + Jd[j * 30 + 20 + l] * g.z);
    };
    float r6[7][6];  // joints 0, then (1,4,7), (2,5,8)
    const int rot_joint[7] = {0, 1, 4, 7, 2, 5, 8};
#pragma unroll
    for (int q = 0; q < 7; ++q) {
      const int c0 = (rot_joint[q] == 0) ? kChRot6d : kChBodyPose + (rot_joint[q] - 1) * 6;
#pragma unroll
      for (int e = 0; e < 6; ++e) r6[q][e] = ch(c0 + e);
    }
    const M3 R0 = rot6d_to_mat(r6[0]);
    const V3 J0 = restJ(0);
    const int chain[2][4] = {{1, 4, 7, 10}, {2, 5, 8, 11}};
    V3 a0 = {0.f, 0.f, 0.f};  // gradient reaching the root position (-> betas through J_0)
#pragma unroll
    for (int s = 0; s < 2; ++s) {
      M3 R[3];
      V3 d[5];
      d[0] = J0;
      V3 prev = J0;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const V3 J = restJ(chain[s][k]);
        d[k + 1] = J - prev;
        prev = J;
        if (k < 3) R[k] = rot6d_to_mat(r6[1 + s * 3 + k]);
      }
      LegFK L;
      leg_forward(R0, R, d, L);
      const float* g = ws.gdir + ((frames + f) * 4 + s * 2) * 3;
      const V3 g_ankle = {sc_smpl * g[0], sc_smpl * g[1], sc_smpl * g[2]};
      const V3 g_toe = {sc_smpl * g[3], sc_smpl * g[4], sc_smpl * g[5]};
      // a[k]: gradient w.r.t. the world position of chain node k (0 root, 1 hip, 2 knee, 3 ankle, 4 toe)
      const V3 a4 = g_toe, a3 = g_ankle + g_toe;
      const V3 a2 = a3, a1 = a3;
      a0 = a0 + a1;
      const V3 a[5] = {a1, a1, a2, a3, a4};
      // rest offsets: p_k = p_{k-1} + W_{k-1} d_k  ->  dL/dd_k = W_{k-1}^T a_k
#pragma unroll
      for (int k = 1; k <= 4; ++k) {
        const V3 gd = mulT(L.W[k - 1], a[k]);
        acc_beta(chain[s][k - 1], gd, 1.0f);
        acc_beta(k == 1 ? 0 : chain[s][k - 2], gd, -1.0f);
      }
      // world-rotation gradients, leaf to root: GW_k = a_{k+1} d_{k+1}^T + GW_{k+1} R_{k+1}^T ; dL/dR_k = W_{k-1}^T GW_k
      // (outer product u v^T stored by columns: column c = v_c * u)
      M3 GW = {d[4].x * a[4], d[4].y * a[4], d[4].z * a[4]};  // node 3 (ankle joint rotation)
#pragma unroll
      for (int k = 3; k >= 1; --k) {
        // gradient of the local rotation of chain node k (joint chain[s][k-1])
        const M3 GR = {mulT(L.W[k - 1], GW.c0), mulT(L.W[k - 1], GW.c1), mulT(L.W[k - 1], GW.c2)};
        float gx[6];
        rot6d_backward(r6[1 + s * 3 + (k - 1)], GR, gx);
        const int c0 = kChBodyPose + (chain[s][k - 1] - 1) * 6;
#pragma unroll
        for (int e = 0; e < 6; ++e) put(c0 + e, gx[e]);
        if (k > 1) {
          // GW_{k-1} = a_k d_k^T + GW_k R_k^T ; (GW R^T) column c = sum_m R[c][m] GW.col(m) = GW * (row c of R)
          const M3& Rk = R[k - 1];
          const M3 GWR = {Rk.c0.x * GW.c0 + Rk.c1.x * GW.c1 + Rk.c2.x * GW.c2,
                          Rk.c0.y * GW.c0 + Rk.c1.y * GW.c1 + Rk.c2.y * GW.c2,
                          Rk.c0.z * GW.c0 + Rk.c1.z * GW.c1 + Rk.c2.z * GW.c2};
          GW = {d[k].x * a[k] + GWR.c0, d[k].y * a[k] + GWR.c1, d[k].z * a[k] + GWR.c2};
        }
      }
    }
    acc_beta(0, a0, 1.0f);
#pragma unroll
    for (int l = 0; l < kBetas; ++l) put(kChBetas + l, gbe[l]);
  }
}

}  // namespace
}  // namespace rohm

using namespace rohm;

#include "body_internal.h"

extern "C" int rohm_body_create(rohm_ctx* ctx, const float* v_template, const float* shapedirs, int shape_comps,
                                const float* posedirs, const float* J_regressor, const float* lbs_weights,
                                const int* parents_host, int num_verts, int64_t max_frames, int with_vertices,
                                int precision, rohm_body** out) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!v_template || !shapedirs || !J_regressor || !parents_host || !out || num_verts <= 0 || max_frames <= 0 ||
      shape_comps < kBetas || (with_vertices && (!posedirs || !lbs_weights)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_body_create: bad arguments");
  for (int j = 0; j < kJ; ++j)
    if (parents_host[j] >= j) return fail(ctx, ROHM_ERR_INVALID, "rohm_body_create: parents must precede children");
  rohm_body* bd = new (std::nothrow) rohm_body();
  if (!bd) return fail(ctx, ROHM_ERR_INVALID, "out of host memory");
  bd->ctx = ctx, bd->V = num_verts, bd->sd_comps = shape_comps, bd->max_frames = max_frames, bd->passes = precision == ROHM_PRECISION_TF32 ? 1 : 3;
  bd->kind = precision == ROHM_PRECISION_F16X2 ? kKindF16 : kKindTf32;
  ROHM_CUDA(ctx, cudaMemcpyToSymbol(c_parents, parents_host, sizeof(int) * kJ));
  const int V = num_verts;
  const int64_t F = max_frames;
  bd->Jt = bd->pool.floats(kJ * 3);
  bd->Jd = bd->pool.floats(kJ * 30);
  bd->foot = bd->pool.floats(2 * F * 12);
  bd->gdir = bd->pool.floats(2 * F * 12);
  bd->sums = bd->pool.floats(16);
  bd->clip_sums = bd->pool.floats(F * 4);
  bd->go =bd->pool.floats(F * 3), bd->bp = bd->pool.floats(F * 63), bd->betas = bd->pool.floats(F * kBetas);
  bd->transl = bd->pool.floats(F * 3);
  bd->jwork = bd->pool.floats(F * kBodyJ * 3), bd->gwork = bd->pool.floats(F * kBodyJ * 3);
  bd->parents_dev = static_cast<int*>(bd->pool.bytes(sizeof(int) * kJ));
  bool ok = bd->Jt && bd->Jd && bd->foot && bd->gdir && bd->sums && bd->clip_sums && bd->go && bd->bp && bd->betas && bd->transl &&
            bd->jwork && bd->gwork && bd->parents_dev;
  if (ok) ok = cudaMemcpy(bd->parents_dev, parents_host, sizeof(int) * kJ, cudaMemcpyHostToDevice) == cudaSuccess;
  if (ok && with_vertices) {
    bd->a_frame_stride = round_up(F, 128);  // whole 128-frame row tiles: the epilogue's bulk copies never leave a row
    bd->A = bd->pool.floats(bd->a_frame_stride * kJ * 12);
    bd->feat_h = bd->pool.floats(F * kBlendK), bd->feat_l = bd->pool.floats(F * kBlendK);
    // two-kernel path: v_posed lives for one chunk of bd->chunk frames at a time (the blend GEMM writes it, the skinning
    // kernel reads it back), in two buffers so that the next chunk's GEMM can run beside this chunk's skinning.  The default
    // chunk of 4608 frames is 4608 x 31 488 x 4 B = 580 MB per buffer; a chunk small enough for the 50 MB L2 (384 frames:
    // 48 MB) would keep the round trip out of HBM at the price of more, smaller launches
    if (const char* env = getenv("ROHM_B200_LBS_CHUNK")) {  // developer switch: frames per chunk (multiple of 128)
      const long v = atol(env);
      if (v >= 128 && v % 128 == 0) bd->chunk = v;
    }
    bd->vposed_stride = std::min<int64_t>(F, bd->chunk) * round_up(V * 3, 384);
    bd->vposed = bd->pool.floats(2 * bd->vposed_stride);
    bd->bone_idx = static_cast<int*>(bd->pool.bytes(static_cast<int64_t>(V) * kMaxBones * sizeof(int)));
    bd->bone_w = bd->pool.floats(static_cast<int64_t>(V) * kMaxBones);
    bd->lbs_w_copy = bd->pool.floats(static_cast<int64_t>(V) * kJ);
    bd->blend.N = V * 3, bd->blend.K = kBlendK, bd->blend.Kp = kBlendK, bd->blend.block_n = 128;
    bd->blend.Np = static_cast<int>(round_up(V * 3, 384));  // whole 128-column (two-kernel path) and 96-column (fused path) tiles
    bd->blend.hi = bd->pool.floats(static_cast<int64_t>(bd->blend.Np) * kBlendK);
    bd->blend.lo = bd->pool.floats(static_cast<int64_t>(bd->blend.Np) * kBlendK);
    ok = bd->A && bd->feat_h && bd->feat_l && bd->vposed && bd->bone_idx && bd->bone_w && bd->lbs_w_copy && bd->blend.hi &&
         bd->blend.lo;
  }
  if (!ok) {
    const int rc = fail(ctx, ROHM_ERR_CUDA, "rohm_body_create: alloc failed: %s", cudaGetErrorString(bd->pool.last_error()));
    delete bd;
    return rc;
  }
  joint_regress_kernel<<<dim3(kJ, 33), 256>>>(J_regressor, v_template, shapedirs, V, shape_comps, bd->Jt, bd->Jd);
  if (with_vertices) {
    int* overflow = static_cast<int*>(bd->pool.bytes(sizeof(int)));
    cudaMemcpy(bd->lbs_w_copy, lbs_weights, sizeof(float) * V * kJ, cudaMemcpyDeviceToDevice);
    compress_weights_kernel<<<(V + 255) / 256, 256>>>(lbs_weights, V, bd->bone_idx, bd->bone_w, overflow);
    const int64_t total = static_cast<int64_t>(bd->blend.Np) * kBlendK;
    bd->blend.kind = bd->kind;
    if (bd->kind == kKindF16) {  // one power-of-two scale for the whole matrix: the smallest of its three sources' scales
      float s1 = 1.0f, s2 = 1.0f, s3 = 1.0f;
      cudaError_t es = f16_weight_scale(posedirs, static_cast<int64_t>(kPoseFeat) * V * 3, &s1);
      if (es == cudaSuccess) es = f16_weight_scale(shapedirs, static_cast<int64_t>(V) * 3 * shape_comps, &s2);
      if (es == cudaSuccess) es = f16_weight_scale(v_template, static_cast<int64_t>(V) * 3, &s3);
      if (es != cudaSuccess) {
        delete bd;
        return fail(ctx, ROHM_ERR_CUDA, "rohm_body_create: %s", cudaGetErrorString(es));
      }
      bd->blend.scale = fminf(s1, fminf(s2, s3));
    }
    build_blend_kernel<<<static_cast<unsigned>((total + 255) / 256), 256>>>(posedirs, shapedirs, v_template, V,
                                                                            shape_comps, bd->blend.hi, bd->blend.lo, total,
                                                                            bd->kind == kKindF16 ? 1 : 0, bd->blend.scale);
    int h_over = 0;
    cudaError_t e = cudaMemcpy(&h_over, overflow, sizeof(int), cudaMemcpyDeviceToHost);
    if (e != cudaSuccess) {
      delete bd;
      return fail(ctx, ROHM_ERR_CUDA, "rohm_body_create: %s", cudaGetErrorString(e));
    }
    bd->sparse_ok = (h_over == 0);
    // developer / test switch: run the dense skinning kernel (the fallback for models with > 8 bones per vertex)
    if (const char* env = getenv("ROHM_B200_DENSE_SKIN")) bd->sparse_ok = bd->sparse_ok && env[0] == '0';
    cudaError_t ea = gemm_init_attributes();
    GemmParams& g = bd->g_blend;
    g = GemmParams{};
    int rc = make_tmap_2d(&g.a_hi[0], bd->feat_h, F, kBlendK, kBlendK, kGemmBlockM, 1, bd->kind);
    rc |= make_tmap_2d(&g.a_lo[0], bd->feat_l, F, kBlendK, kBlendK, kGemmBlockM, 1, bd->kind);
    rc |= make_tmap_2d(&g.b_hi, bd->blend.hi, bd->blend.Np, kBlendK, kBlendK, 128, 1, bd->kind);
    rc |= make_tmap_2d(&g.b_lo, bd->blend.lo, bd->blend.Np, kBlendK, kBlendK, 128, 1, bd->kind);
    if (rc != 0 || ea != cudaSuccess) {
      delete bd;
      return fail(ctx, ROHM_ERR_CUDA, "rohm_body_create: GEMM setup failed (%d)", rc);
    }
    g.num_segs = 1, g.seg_kblocks[0] = kBlendK / gemm_block_k(bd->kind), g.seg_row_mul[0] = 1;
    g.acc_scale = 1.0f / bd->blend.scale;
    g.out = bd->vposed, g.ldo = bd->blend.Np, g.N = bd->blend.Np, g.out_row_mul = 1;  // padded columns are exact zeros
    if (gemm_enable_tma_store(&g, std::min<int64_t>(F, bd->chunk), bd->kind) != 0 ||  // 32 x 32 fp32 chunks leave through TMA bulk stores
        make_store_tmap(&bd->st_out_b, bd->vposed + bd->vposed_stride, std::min<int64_t>(F, bd->chunk), bd->blend.Np, bd->blend.Np,
                        false) != 0) {
      delete bd;
      return fail(ctx, ROHM_ERR_CUDA, "rohm_body_create: store tensor map failed");
    }
    // ---- fused LBS tables: per 32-vertex column tile the bones it touches and the dense [bone][vertex] weights ----
    {
      const char* env = getenv("ROHM_B200_FUSED_LBS");
      bool want = bd->kind == kKindF16 && !(env != nullptr && env[0] == '0');
      const int tiles = bd->blend.Np / 96;  // column tiles of the fused launch (those past the last vertex touch no bone)
      std::vector<float> hw;
      std::vector<int> h_nb(tiles, 0), h_bone(static_cast<size_t>(tiles) * kSkinTileBones, 0);
      std::vector<float> h_w(static_cast<size_t>(tiles) * kSkinTileBones * 32, 0.0f);
      if (want) {
        hw.resize(static_cast<size_t>(V) * kJ);
        want = cudaMemcpy(hw.data(), lbs_weights, sizeof(float) * hw.size(), cudaMemcpyDeviceToHost) == cudaSuccess;
      }
      for (int t = 0; t < tiles && want; ++t) {
        int slot_of[kJ];
        for (int j = 0; j < kJ; ++j) slot_of[j] = -1;
        for (int vl = 0; vl < 32 && want; ++vl) {
          const int v = t * 32 + vl;
          if (v >= V) break;
          for (int j = 0; j < kJ; ++j) {
            const float w = hw[static_cast<size_t>(v) * kJ + j];
            if (w == 0.0f) continue;
            if (slot_of[j] < 0) {
              if (h_nb[t] == kSkinTileBones) {
                want = false;  // more distinct bones than the epilogue's table holds: keep the two-kernel path
                break;
              }
              slot_of[j] = h_nb[t];
              h_bone[static_cast<size_t>(t) * kSkinTileBones + h_nb[t]++] = j;
            }
            h_w[(static_cast<size_t>(t) * kSkinTileBones + slot_of[j]) * 32 + vl] = w;
          }
        }
      }
      if (want) {
        bd->skin_nb = static_cast<int*>(bd->pool.bytes(sizeof(int) * h_nb.size()));
        bd->skin_bone = static_cast<int*>(bd->pool.bytes(sizeof(int) * h_bone.size()));
        bd->skin_w = bd->pool.floats(static_cast<int64_t>(h_w.size()));
        want = bd->skin_nb && bd->skin_bone && bd->skin_w &&
               cudaMemcpy(bd->skin_nb, h_nb.data(), sizeof(int) * h_nb.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
               cudaMemcpy(bd->skin_bone, h_bone.data(), sizeof(int) * h_bone.size(), cudaMemcpyHostToDevice) == cudaSuccess &&
               cudaMemcpy(bd->skin_w, h_w.data(), sizeof(float) * h_w.size(), cudaMemcpyHostToDevice) == cudaSuccess;
      }
      if (want) {
        GemmParams& k = bd->g_skin;
        k = GemmParams{};
        // The tensor maps end at the last live K column (200 -> 208: the rest of the fourth K block is zero-filled by TMA without
        // being read: 19 % less L2 -> SM operand traffic).
        constexpr int kLiveK = (kPoseFeat + kBetas + 1 + 15) / 16 * 16;
        int rs = make_tmap_2d(&k.a_hi[0], bd->feat_h, F, kLiveK, kBlendK, kGemmBlockM, 1, bd->kind);
        rs |= make_tmap_2d(&k.a_lo[0], bd->feat_l, F, kLiveK, kBlendK, kGemmBlockM, 1, bd->kind);
        rs |= make_tmap_2d(&k.b_hi, bd->blend.hi, bd->blend.Np, kLiveK, kBlendK, 96, 1, bd->kind);
        rs |= make_tmap_2d(&k.b_lo, bd->blend.lo, bd->blend.Np, kLiveK, kBlendK, 96, 1, bd->kind);
        k.num_segs = 1, k.seg_kblocks[0] = kBlendK / gemm_block_k(bd->kind), k.seg_row_mul[0] = 1;
        k.acc_scale = 1.0f / bd->blend.scale;
        k.ldo = V * 3, k.N = V * 3, k.out_row_mul = 1;
        k.skin_A = bd->A, k.skin_lda = bd->a_frame_stride, k.skin_nb = bd->skin_nb, k.skin_bone = bd->skin_bone, k.skin_w = bd->skin_w;
        want = rs == 0 && bd->blend.Np % 96 == 0;
      }
      bd->fused_lbs = want;
    }
    bool ev_ok = cudaStreamCreateWithFlags(&bd->skin_stream, cudaStreamNonBlocking) == cudaSuccess;
    for (int i = 0; i < 2 && ev_ok; ++i)
      ev_ok = cudaEventCreateWithFlags(&bd->gemm_done[i], cudaEventDisableTiming) == cudaSuccess &&
              cudaEventCreateWithFlags(&bd->skin_done[i], cudaEventDisableTiming) == cudaSuccess;
    if (!ev_ok) {
      delete bd;
      return fail(ctx, ROHM_ERR_CUDA, "rohm_body_create: stream / event creation failed");
    }
    if (const char* env = getenv("ROHM_B200_LBS_OVERLAP"))
      if (env[0] == '0') cudaStreamDestroy(bd->skin_stream), bd->skin_stream = nullptr;
  }
  cudaError_t e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    delete bd;
    return fail(ctx, ROHM_ERR_CUDA, "rohm_body_create: %s", cudaGetErrorString(e));
  }
  *out = bd;
  return ROHM_OK;
}

extern "C" void rohm_body_destroy(rohm_body* bd) { delete bd; }

extern "C" int rohm_body_skin_path(const rohm_body* bd) {
  if (bd == nullptr || bd->vposed == nullptr) return -1;
  return bd->fused_lbs ? 0 : (bd->sparse_ok ? 1 : 2);
}

extern "C" int rohm_body_set_vertex_pitch(rohm_body* bd, int64_t pitch_floats) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  if (pitch_floats == 0) {
    bd->vertex_pitch = 0;
    return ROHM_OK;
  }
  if (!bd->fused_lbs)
    return fail(bd->ctx, ROHM_ERR_STATE, "rohm_body_set_vertex_pitch: only the fused blend + skinning launch writes pitched rows");
  if (pitch_floats < static_cast<int64_t>(bd->V) * 3 || pitch_floats % 4 != 0 || pitch_floats > 0x7fffffff)
    return fail(bd->ctx, ROHM_ERR_INVALID, "rohm_body_set_vertex_pitch: pitch %lld must be a multiple of 4 floats and >= 3 V = %d",
                static_cast<long long>(pitch_floats), bd->V * 3);
  bd->vertex_pitch = pitch_floats;
  return ROHM_OK;
}

// SMPLX.forward as RoHM calls it (jaw / eyes / hands / expression zero).  global_orient [N,3], body_pose [N,63]
// (axis-angle), betas [N,10], transl [N,3] -> joints [N, num_joints<=55, 3] and (optionally) vertices [N, V, 3].
extern "C" int rohm_body_forward(rohm_body* bd, const float* global_orient, const float* body_pose, const float* betas,
                                 const float* transl, int64_t N, float* joints, int num_joints, float* vertices,
                                 void* stream) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = bd->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  if (!global_orient || !body_pose || !betas || !transl || N <= 0 || N > bd->max_frames || num_joints < 0 ||
      num_joints > kJ || (joints == nullptr && vertices == nullptr))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_body_forward: bad arguments (N=%lld, capacity %lld)",
                static_cast<long long>(N), static_cast<long long>(bd->max_frames));
  if (vertices != nullptr && bd->vposed == nullptr)
    return fail(ctx, ROHM_ERR_STATE, "rohm_body_forward: handle was created without vertex support");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool verts = vertices != nullptr;
  fk_full_kernel<<<static_cast<unsigned>((N + kFkWarps - 1) / kFkWarps), 32 * kFkWarps, 0, st>>>(
      global_orient, body_pose, betas, transl, bd->Jt, bd->Jd, static_cast<int>(N), joints, num_joints,
      verts ? bd->A : nullptr, (verts && bd->fused_lbs) ? bd->a_frame_stride : 0, verts ? bd->feat_h : nullptr,
      verts ? bd->feat_l : nullptr, bd->kind == kKindF16 ? 1 : 0);
  ROHM_CUDA(ctx, cudaGetLastError());
  if (verts && bd->fused_lbs) {
    // one launch: blend GEMM with the skinning epilogue (gemm.cu, EPI 4); v_posed stays in registers / shared memory
    GemmParams g = bd->g_skin;
    g.M = static_cast<int>(N);
    g.out = vertices;
    if (bd->vertex_pitch != 0) {
      // pitched output (rohm_body_set_vertex_pitch): rows start on 16-byte boundaries, so the tile leaves through TMA stores
      if ((reinterpret_cast<uintptr_t>(vertices) & 15u) != 0)
        return fail(ctx, ROHM_ERR_INVALID, "rohm_body_forward: a pitched vertex buffer must be 16-byte aligned");
      g.ldo = static_cast<int>(bd->vertex_pitch);
      if (make_store_tmap(&g.st_out, vertices, N, static_cast<int64_t>(bd->V) * 3, bd->vertex_pitch, false, kGemmBlockM) != 0)
        return fail(ctx, ROHM_ERR_CUDA, "rohm_body_forward: vertex store tensor map failed");
      g.st_hi = g.st_out, g.st_lo = g.st_out;
      g.tma_store = 1;
    }
    ROHM_CUDA(ctx, launch_gemm(g, static_cast<int>(N), bd->blend.Np, 96, bd->passes, st, false, bd->kind));
  } else if (verts) {
    // Pipeline over chunks of bd->chunk frames (4608 by default, ROHM_B200_LBS_CHUNK): blend GEMM of chunk i on the caller's
    // stream into v_posed buffer i % 2, skinning of chunk i on a second stream (HBM-bound next to the tensor-bound GEMM of
    // chunk i + 1).  One chunk, or ROHM_B200_LBS_OVERLAP=0, runs everything on the caller's stream with one buffer.
    const int vblocks = (bd->V + 255) / 256;
    int occ = 0;  // resident CTAs per SM (registers / the 42 KB of shared memory decide)
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, skin_kernel, 256, 0) != cudaSuccess || occ < 1) occ = 3;
    const int skin_y = std::max(1, (ctx->sm_count > 0 ? ctx->sm_count : 132) * occ / vblocks);  // one full wave
    const int64_t kChunk = bd->chunk;
    const int64_t chunks = (N + kChunk - 1) / kChunk;
    const bool overlap = bd->skin_stream != nullptr && chunks > 1;
    cudaStream_t ss = overlap ? bd->skin_stream : st;
    for (int64_t c = 0; c < chunks; ++c) {
      const int64_t r0 = c * kChunk;
      const int64_t n = std::min<int64_t>(kChunk, N - r0);
      float* vp = bd->vposed + (overlap ? (c & 1) : 0) * bd->vposed_stride;
      if (overlap && c >= 2) ROHM_CUDA(ctx, cudaStreamWaitEvent(st, bd->skin_done[c & 1], 0));  // buffer free again
      GemmParams g = bd->g_blend;
      g.M = static_cast<int>(n);
      g.seg_row_shift[0] = static_cast<int>(r0);  // A rows of this chunk; output rows are chunk-local
      if (overlap && (c & 1)) g.out = vp, g.st_out = bd->st_out_b, g.st_hi = bd->st_out_b, g.st_lo = bd->st_out_b;
      ROHM_CUDA(ctx, launch_gemm(g, static_cast<int>(n), bd->blend.Np, 128, bd->passes, st, false, bd->kind));
      if (overlap) {
        ROHM_CUDA(ctx, cudaEventRecord(bd->gemm_done[c & 1], st));
        ROHM_CUDA(ctx, cudaStreamWaitEvent(ss, bd->gemm_done[c & 1], 0));
      }
      const float* A = bd->A + r0 * kJ * 12;
      float* vout = vertices + r0 * bd->V * 3;
      if (bd->sparse_ok) {
        const int64_t fblocks = (n + kSkinFrames - 1) / kSkinFrames;
        skin_kernel<<<dim3(vblocks, static_cast<unsigned>(std::min<int64_t>(skin_y, fblocks))), 256, 0, ss>>>(
            vp, bd->blend.Np, A, bd->bone_idx, bd->bone_w, bd->V, n, vout);
      } else {
        skin_dense_kernel<<<dim3(vblocks, static_cast<unsigned>(n)), 256, 0, ss>>>(vp, bd->blend.Np, A, bd->lbs_w_copy, bd->V, vout);
      }
      ROHM_CUDA(ctx, cudaGetLastError());
      if (overlap) ROHM_CUDA(ctx, cudaEventRecord(bd->skin_done[c & 1], ss));
    }
    if (overlap) {  // join: the caller's stream continues after the last skinning kernels
      ROHM_CUDA(ctx, cudaStreamWaitEvent(st, bd->skin_done[0], 0));
      ROHM_CUDA(ctx, cudaStreamWaitEvent(st, bd->skin_done[1], 0));
    }
  }
  return ROHM_OK;
}

// recover_from_repr_smpl(recover_mode='smplx_params') on a normalised representation x ([B, 294, 1, T] or, channels_last,
// [B, T, 294]): joints [B*T, num_joints, 3] and optionally vertices [B*T, V, 3].  With lengths only the clips' own frames are
// gathered, so FK and the blend GEMM + skinning run over total_frames rows and write packed joints / vertices.
extern "C" int rohm_body_from_repr(rohm_body* bd, const float* x, int channels_last, const float* mean, const float* stdv,
                                   int B, int T, const int* lengths, const int* clip_off, int64_t total_frames,
                                   float* joints, int num_joints, float* vertices, void* stream) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = bd->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const bool ragged = lengths != nullptr;
  const int64_t N = static_cast<int64_t>(B) * T;
  const int64_t frames = ragged ? total_frames : N;  // rows FK runs over
  if (!x || !mean || !stdv || B <= 0 || T <= 0 || frames > bd->max_frames ||
      (ragged ? (!clip_off || total_frames < B || total_frames > N || total_frames > INT32_MAX)
              : (clip_off != nullptr || total_frames != 0)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_body_from_repr: bad arguments (B=%d T=%d, %lld frames in the clips, "
                "capacity %lld)", B, T, static_cast<long long>(frames), static_cast<long long>(bd->max_frames));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t total = frames * kBodyJ;
  const int64_t sb = static_cast<int64_t>(kC) * T, sc = channels_last ? 1 : T, stt = channels_last ? kC : 1;
  const auto kernel = ragged ? repr_to_smplx_kernel<true> : repr_to_smplx_kernel<false>;
  kernel<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(x, sb, sc, stt, mean, stdv, B, T, bd->go, bd->bp,
                                                                     bd->betas, bd->transl, clip_off, total_frames);
  ROHM_CUDA(ctx, cudaGetLastError());
  return rohm_body_forward(bd, bd->go, bd->bp, bd->betas, bd->transl, frames, joints, num_joints, vertices, stream);
}

// guide_skating_with_smpl (posenet.py:196-257): grad [B, 294, 1, T] = d(-(loss_smpl + loss_abs))/dx0 with the
// trajectory and contact channels zeroed.  If nothing skates the gradient is all zeros (the reference returns a
// scalar 0 in that case; adding weight*variance*0 is the same update).  loss_out (device float[4], optional) receives
// {sum_abs, count_abs, sum_smpl, count_smpl}.
// The two halves of rohm_skating_guidance, for clip-sharded runs that want the reference's batch-global normalisers
// (posenet.py:230-233, 242-248: loss = sum of masked speeds / number of masked (frame, foot) pairs over the WHOLE batch):
//   rohm_skating_guidance_sums     forward kinematics of both recovery paths + masked loss sums of THIS shard -> sums[4]
//                                  = {sum_abs, count_abs, sum_smpl, count_smpl} (device); per-frame state stays in the handle
//   (caller: all-reduce the 4 floats over the ranks)
//   rohm_skating_guidance_backward VJP with the given (global) sums -> grad of this shard
extern "C" int rohm_skating_guidance_sums(rohm_body* bd, const float* x0, const float* mean, const float* stdv, int B, int T,
                                          float* sums_out, void* stream) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = bd->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const int64_t N = static_cast<int64_t>(B) * T;
  if (!x0 || !mean || !stdv || !sums_out || B <= 0 || T <= 0 || N > bd->max_frames)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_skating_guidance_sums: bad arguments (B*T=%lld, capacity %lld)",
                static_cast<long long>(N), static_cast<long long>(bd->max_frames));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GuideWs ws{bd->foot, bd->gdir, sums_out};
  ROHM_CUDA(ctx, cudaMemsetAsync(sums_out, 0, 4 * sizeof(float), st));
  const unsigned blocks = static_cast<unsigned>((N + 127) / 128);
  guide_forward_kernel<<<blocks, 128, 0, st>>>(x0, mean, stdv, bd->Jt, bd->Jd, B, T, ws);
  guide_loss_kernel<false, false><<<blocks, 128, 0, st>>>(x0, mean, stdv, B, T, ws, nullptr);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_skating_guidance_backward(rohm_body* bd, const float* x0, const float* mean, const float* stdv, int B,
                                              int T, const float* sums, float* grad, void* stream) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = bd->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const int64_t N = static_cast<int64_t>(B) * T;
  if (!x0 || !mean || !stdv || !sums || !grad || B <= 0 || T <= 0 || N > bd->max_frames)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_skating_guidance_backward: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  GuideWs ws{bd->foot, bd->gdir, const_cast<float*>(sums)};
  ROHM_CUDA(ctx, cudaMemsetAsync(grad, 0, sizeof(float) * N * kC, st));
  guide_backward_kernel<false><<<static_cast<unsigned>((N + 127) / 128), 128, 0, st>>>(x0, mean, stdv, bd->Jt, bd->Jd, B, T, ws,
                                                                                      grad, nullptr);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

// lengths (device int[B], or nullptr for clips of T frames): frames at or past lengths[b] add nothing and get a zero gradient.
// per_clip: each clip is normalised by its own counts (sums [B][4] in the handle, B <= B*T fits its capacity).
extern "C" int rohm_skating_guidance(rohm_body* bd, const float* x0, const float* mean, const float* stdv, const int* lengths,
                                     int B, int T, int per_clip, float* grad, float* loss_out, void* stream) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = bd->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const int64_t N = static_cast<int64_t>(B) * T;
  if (!x0 || !mean || !stdv || !grad || B <= 0 || T <= 0 || N > bd->max_frames)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_skating_guidance: bad arguments (B*T=%lld, capacity %lld)",
                static_cast<long long>(N), static_cast<long long>(bd->max_frames));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool clip = per_clip != 0;
  const int64_t nsums = clip ? static_cast<int64_t>(B) * 4 : 4;
  GuideWs ws{bd->foot, bd->gdir, clip ? bd->clip_sums : bd->sums};
  ROHM_CUDA(ctx, cudaMemsetAsync(ws.sums, 0, nsums * sizeof(float), st));
  ROHM_CUDA(ctx, cudaMemsetAsync(grad, 0, sizeof(float) * N * kC, st));
  const unsigned blocks = static_cast<unsigned>((N + 127) / 128);
  guide_forward_kernel<<<blocks, 128, 0, st>>>(x0, mean, stdv, bd->Jt, bd->Jd, B, T, ws);
  const auto loss = lengths != nullptr ? (clip ? guide_loss_kernel<true, true> : guide_loss_kernel<true, false>)
                                       : (clip ? guide_loss_kernel<false, true> : guide_loss_kernel<false, false>);
  loss<<<blocks, 128, 0, st>>>(x0, mean, stdv, B, T, ws, lengths);
  const auto backward = clip ? guide_backward_kernel<true> : guide_backward_kernel<false>;
  backward<<<blocks, 128, 0, st>>>(x0, mean, stdv, bd->Jt, bd->Jd, B, T, ws, grad, lengths);
  ROHM_CUDA(ctx, cudaGetLastError());
  if (loss_out != nullptr)
    ROHM_CUDA(ctx, cudaMemcpyAsync(loss_out, ws.sums, nsums * sizeof(float), cudaMemcpyDeviceToDevice, st));
  return ROHM_OK;
}
