// Kernels either side of the sampling loops (SURVEY.md 8f, rows N1-N4) and the 2-D reprojection guidance (row N2).
//
//   rohm_traj_glue              test_amass_full.py:268-311  TrajNet output -> composite representation -> SMPL-X joints ->
//                               get_repr_smplx (data_loaders/motion_representation.py:187-282) -> the 22 trajectory
//                               channels PoseNet is conditioned on.  The reference does this per clip on the host
//                               (numpy + scipy + two PCIe round trips); here it is three launches on the stream.
//   rohm_pose_to_control_cond   test_amass_full.py:256-258  PoseNet output -> TrajControl condition
//   rohm_build_pose_cond        test_amass_full.py:320-370  PoseNet condition: trajectory block + occlusion masks
//   rohm_rot6d_to_aa            quaternion.py:482-501 + konia_transform.py:317-444,561-631 as a stand-alone entry
//   rohm_joints_from_traj       motion_representation.py:285-371 recover_from_repr_smpl 'joint_abs_traj' / 'joint_rel_traj'
//   rohm_projection_guidance    model/posenet.py:260-317 guide_2d_projection_with_smpl, analytic VJP instead of autograd
#include <cmath>
#include <cstdint>

#include <cooperative_groups.h>

#include "body_internal.h"
#include "kin.cuh"
#include "repr.cuh"

namespace cg = cooperative_groups;

namespace rohm {
namespace {

using namespace kin;

constexpr int kC = 294;
constexpr int kBodyJ = 22;
constexpr int kBetas = 10;
constexpr int kTrajFull = 22;
constexpr int kChAngle = 0, kChAngleVel = 1, kChRootPos = 2, kChRootVel = 4, kChHeight = 6, kChRot6d = 7, kChTrans = 16,
              kChLocalPos = 22, kChBodyPose = 154, kChBetas = 280, kChContact = 290;

// channel of the 294-wide row that TrajNet's k-th output channel overwrites (repr_abs_only: 13 channels,
// test_amass_full.py:272-277; otherwise the first traj_dim channels, :270)
__device__ __forceinline__ int traj_channel(int k, int traj_dim) {
  if (traj_dim != 13) return k;
  return k == 0 ? 0 : (k <= 2 ? k + 1 : (k == 3 ? 6 : (k <= 9 ? k + 3 : k + 6)));
}

// composite[b,t,:] = clean[b,t,:] with the trajectory channels replaced by the TrajNet output (both normalised).
// kLengths: rows are [B, T] and clip b has lengths[b] frames; rows past a clip are written as zeros, their sources not read.
template <bool kLengths>
__global__ void compose_repr_kernel(const float* __restrict__ traj, int traj_dim, const float* __restrict__ clean,
                                    float* __restrict__ out, int64_t rows, const int* __restrict__ lengths, int T) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= rows * kC) return;
  if constexpr (kLengths) {
    const int64_t row = i / kC;
    if (row % T >= lengths[row / T]) {
      out[i] = 0.0f;
      return;
    }
  }
  out[i] = clean[i];
  const int c = static_cast<int>(i % kC);
  const int64_t r = i / kC;
  // inverse map: is c one of the overwritten channels?
  int k = -1;
  if (traj_dim != 13) k = c < traj_dim ? c : -1;
  else if (c == 0) k = 0;
  else if (c == 2 || c == 3) k = c - 1;
  else if (c == 6) k = 3;
  else if (c >= 7 && c <= 12) k = c - 3;
  else if (c >= 16 && c <= 18) k = c - 6;
  if (k >= 0) out[i] = traj[r * traj_dim + k];
}

constexpr int kReprFramesPerCta = 1024;  // frames (threads) per CTA of traj_full_repr_kernel
constexpr int kReprMaxCluster = 8;       // CTAs per clip: clips of up to 8192 frames

// get_repr_smplx, trajectory block only (channels 0..21 of REPR_LIST): one cluster of n = ceil(T / 1024) CTAs per clip, one
// thread per frame; CTA `rank` holds frames [rank * ceil(T / n), ...) and their root quaternions in its shared memory.  The
// clip-wide first NaN frame (rank 0's first_nan) and the quaternions of frames in other CTAs are reached through
// distributed shared memory.  joints: [B, T, 22, 3]; go: [B*T, 3] axis-angle global orient; transl: [B*T, 3]; out:
// [B, T-1, 22] z-scored with the PoseNet dataset statistics.
// kLengths: clip b has len = lengths[b] <= T frames and joints / go / transl hold the clips packed, clip b's frames from row
// clip_off[b].  The cluster shape still follows T (it is a property of the launch), so a CTA whose frames all lie past its
// clip computes nothing but takes part in every cluster barrier.  The NaN search, the wrap-around source of the repair and
// the velocity pairs stop at len; out keeps its padded [B, T-1, 22] shape, rows len-1 .. T-2 are written as zeros.
template <bool kLengths>
__global__ void traj_full_repr_kernel(const float* __restrict__ joints, const float* __restrict__ go,
                                      const float* __restrict__ transl, const float* __restrict__ mean,
                                      const float* __restrict__ stdv, int T, float* __restrict__ out,
                                      const int* __restrict__ lengths, const int* __restrict__ clip_off) {
  extern __shared__ float sm[];
  cg::cluster_group cluster = cg::this_cluster();
  const int ncta = static_cast<int>(cluster.num_blocks()), rank = static_cast<int>(cluster.block_rank());
  const int rows = (T + ncta - 1) / ncta;  // frames per CTA
  float* qw = sm;                    // root quaternion (w, 0, 0, z) per frame of this CTA
  float* qz = sm + rows;
  __shared__ int first_nan;
  // this CTA's shared address p as seen in CTA r (a single CTA is its own cluster)
  auto peer = [&](auto* p, int r) { return ncta > 1 ? cluster.map_shared_rank(p, r) : p; };
  auto sync = [&] { ncta > 1 ? cluster.sync() : __syncthreads(); };
  const int b = blockIdx.x / ncta;
  const int t = rank * rows + threadIdx.x;
  const int len = kLengths ? lengths[b] : T;  // frames of this clip
  // row of the clip's frame 0 in joints / go / transl
  auto row0 = [&] { return kLengths ? static_cast<int64_t>(clip_off[b]) : static_cast<int64_t>(b) * T; };
  const bool mine = threadIdx.x < rows && t < len;  // this thread's frame exists and belongs to this CTA
  if (rank == 0 && threadIdx.x == 0) first_nan = len;
  sync();
  const float* P = joints + (row0() + (mine ? t : 0)) * kBodyJ * 3;
  auto J = [&](const float* base, int j) { return V3{base[j * 3], base[j * 3 + 1], base[j * 3 + 2]}; };
  if (mine) {
    float q0, q1, q3;
    repr::heading_quat(J(P, 1), J(P, 2), J(P, 17), J(P, 16), q0, q1, q3);
    qw[threadIdx.x] = q0, qz[threadIdx.x] = q3;
    if (isnan(q0) || isnan(q1) || isnan(q3)) atomicMin(peer(&first_nan, 0), t);
  }
  sync();
  if (rank == 0 && threadIdx.x == 0) {
    // "several frames have nan values": the reference repairs the FIRST one only, with its predecessor
    // (frame -1 = the last frame when the first frame is the bad one), then pins frame 0 to the identity
    if (first_nan < len) {
      const int dst = first_nan, src = first_nan > 0 ? first_nan - 1 : len - 1;
      peer(qw, dst / rows)[dst % rows] = peer(qw, src / rows)[src % rows];
      peer(qz, dst / rows)[dst % rows] = peer(qz, src / rows)[src % rows];
    }
    qw[0] = 1.0f, qz[0] = 0.0f;
  }
  sync();
  if (mine && t < len - 1) {
    const float* P1 = P + kBodyJ * 3;
    const int64_t f = row0() + t;
    float o[kTrajFull];
    // frame t + 1 is the next CTA's first when t is this CTA's last
    const int u = threadIdx.x + 1 < rows ? threadIdx.x + 1 : 0, ur = threadIdx.x + 1 < rows ? rank : rank + 1;
    const float w0 = qw[threadIdx.x], z0 = qz[threadIdx.x], w1 = peer(qw, ur)[u], z1 = peer(qz, ur)[u];
    auto root = [&](int k) { return J(k == 0 ? P : P1, 0); };
    auto rot = [&](int k) { return repr::rotvec_to_mat({go[(f + k) * 3], go[(f + k) * 3 + 1], go[(f + k) * 3 + 2]}); };
    auto tr = [&](int k, int c) { return transl[(f + k) * 3 + c]; };
    repr::traj_channels(o, w0, z0, w1, z1, root, rot, tr);
    float* dst = out + (static_cast<int64_t>(b) * (T - 1) + t) * kTrajFull;
#pragma unroll
    for (int c = 0; c < kTrajFull; ++c) dst[c] = (o[c] - mean[c]) / stdv[c];
  } else if (kLengths && threadIdx.x < rows && t < T - 1) {
    float* dst = out + (static_cast<int64_t>(b) * (T - 1) + t) * kTrajFull;
#pragma unroll
    for (int c = 0; c < kTrajFull; ++c) dst[c] = 0.0f;
  }
  if (ncta > 1) cluster.sync();  // peers may still read this CTA's quaternions
}

// B clusters of ceil(T / 1024) CTAs; T <= kReprFramesPerCta * kReprMaxCluster (checked by the callers).  lengths / clip_off
// (device int[B] / int[B + 1]) select the instance for packed clips of different lengths.
cudaError_t launch_traj_full_repr(const float* joints, const float* go, const float* transl, const float* mean,
                                  const float* stdv, int B, int T, float* out, cudaStream_t st,
                                  const int* lengths = nullptr, const int* clip_off = nullptr) {
  const int n = (T + kReprFramesPerCta - 1) / kReprFramesPerCta;
  const int rows = (T + n - 1) / n;
  return launch_chain(lengths != nullptr ? traj_full_repr_kernel<true> : traj_full_repr_kernel<false>,
                      dim3(static_cast<unsigned>(B * n)), dim3((rows + 31) / 32 * 32), 2 * rows * sizeof(float), st,
                      ChainAttrs(false, static_cast<unsigned>(n)), joints, go, transl, mean, stdv, T, out, lengths, clip_off);
}

// control_cond[b, t, :] = pose_out[b, 22 + c, 0, min(t, Tp-1)]   (Tp = T-1 frames of PoseNet output; last frame repeated)
// kLengths: clip b has lengths[b] <= Tp pose frames; its own last pose frame is the one repeated (into control frame
// lengths[b]), later control frames are zero and pose_out is not read past the clip.
template <bool kLengths>
__global__ void pose_to_control_kernel(const float* __restrict__ pose_out, int Tp, int T, int traj, int ncond,
                                       float* __restrict__ control, const int* __restrict__ lengths) {
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, t = t0 + tx;
    const int len = kLengths ? lengths[b] : Tp;  // pose frames of this clip; control frames [0, len] are real
    const int ts = t < len ? t : len - 1;
    tile[j][tx] = (c < ncond && t < (kLengths ? len + 1 : T)) ? pose_out[(static_cast<int64_t>(b) * (traj + ncond) + traj + c) * Tp + ts] : 0.0f;
  }
  __syncthreads();
  for (int j = ty; j < 32; j += 8) {
    const int t = t0 + j, c = c0 + tx;
    if (t < T && c < ncond) control[(static_cast<int64_t>(b) * T + t) * ncond + c] = tile[tx][j];
  }
}

// PoseNet condition [B, 294, 1, Tp] from a source in either layout, the trajectory block and the occlusion masks.
// kLengths: clip b has lengths[b] <= Tp frames; later frames are written as zeros, src and traj_full are not read there.
// kVis (video driver, test_prox_egobody.py:302-309): after the occlusion zeroing every channel is multiplied by
// vis_mask[b, t, c] ([B, vis_T, 294], vis_T >= Tp), then the contact channels are zeroed.  A multiply, not a select: the
// reference's -x * 0 = -0, NaN * 1 = NaN and Inf * 0 = NaN are kept.
template <bool kLengths, bool kVis = false>
__global__ void build_pose_cond_kernel(const float* __restrict__ src, int src_channel_major, int src_T,
                                       const float* __restrict__ traj_full, const unsigned char* __restrict__ chan_keep,
                                       const int* __restrict__ frame_lo, const int* __restrict__ frame_hi,
                                       int zero_contact, int Tp, float* __restrict__ out,
                                       const int* __restrict__ lengths, const float* __restrict__ vis_mask = nullptr,
                                       int vis_T = 0) {
  static_assert(!(kLengths && kVis), "the visibility mask applies to whole clips");
  __shared__ float tile[32][33];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int len = kLengths ? lengths[b] : Tp;  // frames of this clip
  // load tile[c][t]
  if (src_channel_major) {
    for (int j = ty; j < 32; j += 8) {
      const int c = c0 + j, t = t0 + tx;
      tile[j][tx] = (c < kC && t < len) ? src[(static_cast<int64_t>(b) * kC + c) * src_T + t] : 0.0f;
    }
  } else {
    for (int j = ty; j < 32; j += 8) {
      const int t = t0 + j, c = c0 + tx;
      tile[tx][j] = (c < kC && t < len) ? src[(static_cast<int64_t>(b) * src_T + t) * kC + c] : 0.0f;
    }
  }
  if constexpr (kVis) {
    // the mask is channels-last: staged through shared memory like a channels-last source, so both reads coalesce
    __shared__ float vtile[32][33];
    for (int j = ty; j < 32; j += 8) {
      const int t = t0 + j, c = c0 + tx;
      vtile[tx][j] = (c < kC && t < Tp) ? vis_mask[(static_cast<int64_t>(b) * vis_T + t) * kC + c] : 0.0f;
    }
    __syncthreads();
    const int lo = frame_lo != nullptr ? frame_lo[b] : 0, hi = frame_hi != nullptr ? frame_hi[b] : 0;
    for (int j = ty; j < 32; j += 8) {
      const int c = c0 + j, t = t0 + tx;
      if (c >= kC || t >= Tp) continue;
      float v = tile[j][tx];
      if (c < kTrajFull) {
        if (traj_full != nullptr) v = traj_full[(static_cast<int64_t>(b) * Tp + t) * kTrajFull + c];
      } else if ((chan_keep != nullptr && chan_keep[c] == 0) || (t >= lo && t < hi)) {
        v = 0.0f;
      }
      v = v * vtile[j][tx];
      if (zero_contact && c >= kChContact) v = 0.0f;
      out[(static_cast<int64_t>(b) * kC + c) * Tp + t] = v;
    }
    return;
  }
  __syncthreads();
  const int lo = frame_lo != nullptr ? frame_lo[b] : 0, hi = frame_hi != nullptr ? frame_hi[b] : 0;
  for (int j = ty; j < 32; j += 8) {
    const int c = c0 + j, t = t0 + tx;
    if (c >= kC || t >= Tp) continue;
    float v = tile[j][tx];
    if (kLengths && t >= len) {
      v = 0.0f;
    } else if (c < kTrajFull) {
      if (traj_full != nullptr) v = traj_full[(static_cast<int64_t>(b) * Tp + t) * kTrajFull + c];
    } else {
      const bool masked = (chan_keep != nullptr && chan_keep[c] == 0) || (t >= lo && t < hi) ||
                          (zero_contact && c >= kChContact);
      if (masked) v = 0.0f;
    }
    out[(static_cast<int64_t>(b) * kC + c) * Tp + t] = v;
  }
}

__global__ void rot6d_to_aa_kernel(const float* __restrict__ r6, int64_t n, float* __restrict__ aa,
                                   float* __restrict__ rotmat) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float x[6];
#pragma unroll
  for (int e = 0; e < 6; ++e) x[e] = r6[i * 6 + e];
  const M3 R = rot6d_to_mat(x);
  if (rotmat != nullptr) {
    float* o = rotmat + i * 9;
    o[0] = R.c0.x, o[1] = R.c1.x, o[2] = R.c2.x, o[3] = R.c0.y, o[4] = R.c1.y, o[5] = R.c2.y;
    o[6] = R.c0.z, o[7] = R.c1.z, o[8] = R.c2.z;
  }
  if (aa != nullptr) {
    const V3 a = mat_to_aa(R);
    aa[i * 3] = a.x, aa[i * 3 + 1] = a.y, aa[i * 3 + 2] = a.z;
  }
}

// recover_from_repr_smpl, 'joint_abs_traj' (mode 0) and 'joint_rel_traj' (mode 1): one thread per clip walks the frames
// (the relative mode is two running sums over time; the absolute mode has no dependency but shares the code).
// x element (b, c, t) at x[b*sb + c*sc + t*st], normalised; joints [B, T, 22, 3].
// kLengths: clip b has lengths[b] <= T frames and joints holds the clips packed ([sum of lengths, 22, 3], clip b from row
// clip_off[b]).  The absolute mode runs one thread per packed frame (total of them), the relative mode keeps one thread
// per clip and stops at the clip's length.
template <bool kLengths>
__global__ void joints_from_traj_kernel(const float* __restrict__ x, int64_t sb, int64_t sc, int64_t st,
                                        const float* __restrict__ mean, const float* __restrict__ stdv, int B, int T,
                                        int mode, float* __restrict__ joints, const int* __restrict__ lengths,
                                        const int* __restrict__ clip_off, int total) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;  // clip, or packed frame (kLengths, absolute mode)
  if (i >= (kLengths && mode == 0 ? total : B)) return;
  const int b = kLengths && mode == 0 ? clip_of_frame(clip_off, B, i) : i;
  const int t_begin = kLengths && mode == 0 ? i - clip_off[b] : 0;
  const int t_end = kLengths ? (mode == 0 ? t_begin + 1 : lengths[b]) : T;
  if (kLengths && t_begin >= lengths[b]) return;
  float ang = 0.0f;            // running root angle (rel)
  float px = 0.0f, py = 0.0f;  // running root position (rel)
  for (int t = t_begin; t < t_end; ++t) {
    auto ch = [&](int c, int tt) { return x[b * sb + c * sc + tt * st] * stdv[c] + mean[c]; };
    float a, rx, ry;
    const float rz = ch(kChHeight, t);
    if (mode == 0) {
      a = ch(kChAngle, t), rx = ch(kChRootPos, t), ry = ch(kChRootPos + 1, t);
    } else {
      // r_rot_ang[t] = sum_{s<t} rot_vel[s];  r_pos[t] = sum_{s<=t} qrot(qinv(q[s]), (vel[s-1].x, vel[s-1].y, 0))
      if (t > 0) ang += ch(kChAngleVel, t - 1);
      a = ang;
      if (t > 0) {
        float sn, cs;
        sincosf(a, &sn, &cs);
        const V3 v = {ch(kChRootVel, t - 1), ch(kChRootVel + 1, t - 1), 0.0f};
        const V3 qv = {0.0f, 0.0f, -sn};
        const V3 uv = cross(qv, v);
        const V3 uuv = cross(qv, uv);
        px += v.x + 2.0f * (cs * uv.x + uuv.x);
        py += v.y + 2.0f * (cs * uv.y + uuv.y);
      }
      rx = px, ry = py;
    }
    float sn, cs;
    sincosf(a, &sn, &cs);
    float* o = joints + (kLengths ? static_cast<int64_t>(clip_off[b]) + t : static_cast<int64_t>(b) * T + t) * kBodyJ * 3;
    o[0] = rx, o[1] = ry, o[2] = rz;
    for (int j = 1; j < kBodyJ; ++j) {
      const V3 v = {ch(kChLocalPos + j * 3, t), ch(kChLocalPos + j * 3 + 1, t), ch(kChLocalPos + j * 3 + 2, t)};
      const V3 qv = {0.0f, 0.0f, -sn};
      const V3 uv = cross(qv, v);
      const V3 uuv = cross(qv, uv);
      o[j * 3] = v.x + 2.0f * (cs * uv.x + uuv.x) + rx;
      o[j * 3 + 1] = v.y + 2.0f * (cs * uv.y + uuv.y) + ry;
      o[j * 3 + 2] = v.z + 2.0f * (cs * uv.z + uuv.z);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// 2-D reprojection guidance (posenet.py:260-317)
// ---------------------------------------------------------------------------------------------------------------
// loss = mean_{b,t,j in sel,c} |proj(joints_smplx)[b,t,j,c] - kp[b,t,j,c]| * conf[b,t,j];  grad = d(-loss)/dx0 with the
// trajectory channels [0,22) and the contact channels zeroed.  One thread per frame: forward kinematics of the 22 body
// joints (local rotations through the reference's 6D -> R -> axis-angle -> R round trip), projection, then the reverse
// sweep over the kinematic tree (leaf to root) that accumulates position gradients, world-rotation gradients and the
// rest-offset (betas) gradients in one pass.
struct ProjParams {
  const float* x;        // [B, 294, 1, T] normalised
  const float* mean;
  const float* stdv;
  const float* Jt;
  const float* Jd;
  const int* parents;
  const float* cam;      // [B, 12]: rows of the 3x4 canonical -> camera transform
  const float* focal;    // [B, 2]
  const float* center;   // [B, 2]
  const float* kp;       // [B, kpT, 22, 3]: (u, v, confidence)
  int kpT;
  int B, T;
  float* grad;           // [B, 294, 1, T]
  float* loss_sum;       // optional accumulator (sum of |.|*conf over the selected joints): [1], per-clip normalisers [B]
  const int* lengths;    // [B] real frames per clip (kLengths instance only)
};

// kPerClip: the mean runs over clip b's own n_b frames (n_b = lengths[b] with kLengths, else T), so clip b's gradient is
// that of the clip run as a one-clip batch of n_b frames.  kLengths (with kPerClip only): frames at or past lengths[b] are
// never read and keep the cleared zero gradient.
template <bool kPerClip, bool kLengths>
__global__ void __launch_bounds__(64) projection_guidance_kernel(const ProjParams p) {
  static_assert(kPerClip || !kLengths, "a lengths instance normalises per clip");
  const int64_t f = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t frames = static_cast<int64_t>(p.B) * p.T;
  if (f >= frames) return;
  const int b = static_cast<int>(f / p.T), t = static_cast<int>(f % p.T);
  const int T = p.T;
  const int n = kLengths ? p.lengths[b] : T;
  if (kLengths && t >= n) return;
  auto ch = [&](int c) { return p.x[(static_cast<int64_t>(b) * kC + c) * T + t] * p.stdv[c] + p.mean[c]; };
  auto put = [&](int c, float g) { p.grad[(static_cast<int64_t>(b) * kC + c) * T + t] = g * p.stdv[c]; };
  float be[kBetas], gbe[kBetas];
#pragma unroll
  for (int l = 0; l < kBetas; ++l) be[l] = ch(kChBetas + l), gbe[l] = 0.0f;
  auto restJ = [&](int j) {
    V3 J = {p.Jt[j * 3], p.Jt[j * 3 + 1], p.Jt[j * 3 + 2]};
#pragma unroll
    for (int l = 0; l < kBetas; ++l) {
      J.x = fmaf(p.Jd[j * 30 + l], be[l], J.x);
      J.y = fmaf(p.Jd[j * 30 + 10 + l], be[l], J.y);
      J.z = fmaf(p.Jd[j * 30 + 20 + l], be[l], J.z);
    }
    return J;
  };
  auto acc_beta = [&](int j, V3 g, float sign) {
#pragma unroll
    for (int l = 0; l < kBetas; ++l)
      gbe[l] += sign * (p.Jd[j * 30 + l] * g.x + p.Jd[j * 30 + 10 + l] * g.y + p.Jd[j * 30 + 20 + l] * g.z);
  };
  M3 W[kBodyJ];   // world rotations
  M3 Rl[kBodyJ];  // local rotations
  V3 d[kBodyJ];   // rest offsets J_j - J_parent (d[0] = J_0)
  V3 pos[kBodyJ];
  V3 Jrest[kBodyJ];
  const V3 tr = {ch(kChTrans), ch(kChTrans + 1), ch(kChTrans + 2)};
  for (int j = 0; j < kBodyJ; ++j) {
    float r6[6];
    const int c0 = (j == 0) ? kChRot6d : kChBodyPose + (j - 1) * 6;
#pragma unroll
    for (int e = 0; e < 6; ++e) r6[e] = ch(c0 + e);
    Rl[j] = rodrigues(mat_to_aa(rot6d_to_mat(r6)));
    Jrest[j] = restJ(j);
    const int par = p.parents[j];
    if (j == 0 || par < 0) {
      W[j] = Rl[j], d[j] = Jrest[j], pos[j] = Jrest[j];
    } else {
      d[j] = Jrest[j] - Jrest[par];
      pos[j] = pos[par] + mul(W[par], d[j]);
      W[j] = mul(W[par], Rl[j]);
    }
  }
  // projection and dL/dposition of the selected joints
  V3 gp[kBodyJ];
#pragma unroll
  for (int j = 0; j < kBodyJ; ++j) gp[j] = {0.f, 0.f, 0.f};
  const float* cm = p.cam + static_cast<int64_t>(b) * 12;
  const float fx = p.focal[b * 2], fy = p.focal[b * 2 + 1], cx = p.center[b * 2], cy = p.center[b * 2 + 1];
  // d(-mean)/d term; per clip the same expression with B = 1 and T = n_b
  const float scale = kPerClip ? -1.0f / (static_cast<float>(1) * static_cast<float>(n) * 10.0f * 2.0f)
                               : -1.0f / (static_cast<float>(p.B) * static_cast<float>(p.T) * 10.0f * 2.0f);
  const int sel[10] = {16, 18, 20, 17, 19, 21, 4, 5, 7, 8};
  float lsum = 0.0f;
#pragma unroll
  for (int s = 0; s < 10; ++s) {
    const int j = sel[s];
    const V3 pj = pos[j] + tr;
    const float X = cm[0] * pj.x + cm[1] * pj.y + cm[2] * pj.z + cm[3];
    const float Y = cm[4] * pj.x + cm[5] * pj.y + cm[6] * pj.z + cm[7];
    const float Z = cm[8] * pj.x + cm[9] * pj.y + cm[10] * pj.z + cm[11];
    const float u = fx * (X / Z) + cx, v = fy * (Y / Z) + cy;
    const float* k = p.kp + ((static_cast<int64_t>(b) * p.kpT + t) * kBodyJ + j) * 3;
    const float conf = k[2];
    const float du = u - k[0], dv = v - k[1];
    lsum += (fabsf(du) + fabsf(dv)) * conf;
    const float gu = (du > 0.f ? 1.f : (du < 0.f ? -1.f : 0.f)) * conf * scale;
    const float gv = (dv > 0.f ? 1.f : (dv < 0.f ? -1.f : 0.f)) * conf * scale;
    // d(u, v)/d(X, Y, Z)
    const float gX = gu * fx / Z, gY = gv * fy / Z, gZ = -(gu * fx * X + gv * fy * Y) / (Z * Z);
    gp[j] = {cm[0] * gX + cm[4] * gY + cm[8] * gZ, cm[1] * gX + cm[5] * gY + cm[9] * gZ,
             cm[2] * gX + cm[6] * gY + cm[10] * gZ};
  }
  if (p.loss_sum != nullptr && lsum != 0.0f) atomicAdd(kPerClip ? p.loss_sum + b : p.loss_sum, lsum);
  // reverse sweep
  M3 GW[kBodyJ];
#pragma unroll
  for (int j = 0; j < kBodyJ; ++j) GW[j] = {{0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}, {0.f, 0.f, 0.f}};
  for (int j = kBodyJ - 1; j >= 1; --j) {
    const int par = p.parents[j];
    const V3 g = gp[j];
    gp[par] = gp[par] + g;
    const V3 gd = mulT(W[par], g);  // dL/dd_j
    acc_beta(j, gd, 1.0f);
    acc_beta(par, gd, -1.0f);
    // local rotation gradient and its 6-D pull-back
    const M3 GR = {mulT(W[par], GW[j].c0), mulT(W[par], GW[j].c1), mulT(W[par], GW[j].c2)};
    float r6[6], gx[6];
    const int c0 = kChBodyPose + (j - 1) * 6;
#pragma unroll
    for (int e = 0; e < 6; ++e) r6[e] = ch(c0 + e);
    rot6d_backward(r6, GR, gx);
#pragma unroll
    for (int e = 0; e < 6; ++e) put(c0 + e, gx[e]);
    // GW[par] += g d_j^T + GW[j] R_j^T      (outer product u v^T by columns: column c = v_c u)
    const M3& Rj = Rl[j];
    const M3& G = GW[j];
    GW[par].c0 = GW[par].c0 + d[j].x * g + (Rj.c0.x * G.c0 + Rj.c1.x * G.c1 + Rj.c2.x * G.c2);
    GW[par].c1 = GW[par].c1 + d[j].y * g + (Rj.c0.y * G.c0 + Rj.c1.y * G.c1 + Rj.c2.y * G.c2);
    GW[par].c2 = GW[par].c2 + d[j].z * g + (Rj.c0.z * G.c0 + Rj.c1.z * G.c1 + Rj.c2.z * G.c2);
  }
  acc_beta(0, gp[0], 1.0f);
#pragma unroll
  for (int l = 0; l < kBetas; ++l) put(kChBetas + l, gbe[l]);
}

}  // namespace
}  // namespace rohm

using namespace rohm;

extern "C" int rohm_traj_glue(rohm_body* bd, const float* traj_out, int traj_dim, const float* repr_clean,
                              const float* traj_mean, const float* traj_std, const float* pose_mean,
                              const float* pose_std, int B, int T, const int* lengths, const int* clip_off,
                              int64_t total_frames, float* composite_out, float* traj_full_out, void* stream) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = bd->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const bool ragged = lengths != nullptr;
  const int64_t N = static_cast<int64_t>(B) * T;
  const int64_t frames = ragged ? total_frames : N;  // frames FK runs over
  if (!traj_out || !repr_clean || !traj_mean || !traj_std || !pose_mean || !pose_std || !composite_out || !traj_full_out ||
      B <= 0 || T < 2 || frames > bd->max_frames || (traj_dim != 13 && (traj_dim < 1 || traj_dim > kTrajFull)) ||
      (ragged ? (!clip_off || total_frames < 2 * static_cast<int64_t>(B) || total_frames > N)
              : (clip_off != nullptr || total_frames != 0)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_traj_glue: bad arguments (B=%d T=%d traj_dim=%d, %lld frames in the clips, "
                "capacity %lld frames)", B, T, traj_dim, static_cast<long long>(frames),
                static_cast<long long>(bd->max_frames));
  if (T > kReprFramesPerCta * kReprMaxCluster)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_traj_glue: T=%d frames exceeds %d (one cluster of at most %d CTAs of %d frames "
                "per clip)", T, kReprFramesPerCta * kReprMaxCluster, kReprMaxCluster, kReprFramesPerCta);
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int64_t total = N * kC;
  const auto compose = ragged ? compose_repr_kernel<true> : compose_repr_kernel<false>;
  compose<<<static_cast<unsigned>((total + 255) / 256), 256, 0, st>>>(traj_out, traj_dim, repr_clean, composite_out, N,
                                                                     lengths, T);
  ROHM_CUDA(ctx, cudaGetLastError());
  // with lengths, FK over the clips' own frames only: packed joints in jwork, packed global orientations / translations in
  // the handle
  int rc = rohm_body_from_repr(bd, composite_out, 1, traj_mean, traj_std, B, T, lengths, clip_off, total_frames, bd->jwork,
                               kBodyJ, nullptr, stream);
  if (rc != ROHM_OK) return rc;
  ROHM_CUDA(ctx, launch_traj_full_repr(bd->jwork, bd->go, bd->transl, pose_mean, pose_std, B, T, traj_full_out, st, lengths,
                                       clip_off));
  return ROHM_OK;
}

extern "C" int rohm_traj_repr_from_joints(rohm_ctx* ctx, const float* joints, const float* global_orient_aa,
                                          const float* transl, const float* mean, const float* stdv, int B, int T,
                                          const int* lengths, const int* clip_off, float* traj_full_out, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!joints || !global_orient_aa || !transl || !mean || !stdv || !traj_full_out || B <= 0 || T < 2 ||
      (lengths == nullptr) != (clip_off == nullptr))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_traj_repr_from_joints: bad arguments");
  if (T > kReprFramesPerCta * kReprMaxCluster)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_traj_repr_from_joints: T=%d frames exceeds %d (one cluster of at most %d CTAs "
                "of %d frames per clip)", T, kReprFramesPerCta * kReprMaxCluster, kReprMaxCluster, kReprFramesPerCta);
  ROHM_CUDA(ctx, launch_traj_full_repr(joints, global_orient_aa, transl, mean, stdv, B, T, traj_full_out,
                                       static_cast<cudaStream_t>(stream), lengths, clip_off));
  return ROHM_OK;
}

// With lengths the clips' control frames end one past their pose frames, so T must exceed Tp.
extern "C" int rohm_pose_to_control_cond(rohm_ctx* ctx, const float* pose_out, int B, int Tp, int T, int traj_feats,
                                         int cond_feats, const int* lengths, float* control_cond, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!pose_out || !control_cond || B <= 0 || Tp <= 0 || (lengths != nullptr ? T <= Tp : T < Tp) || traj_feats < 0 ||
      cond_feats <= 0 || B > 65535)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_pose_to_control_cond: bad arguments");
  dim3 grid((T + 31) / 32, (cond_feats + 31) / 32, B);
  const auto kernel = lengths != nullptr ? pose_to_control_kernel<true> : pose_to_control_kernel<false>;
  kernel<<<grid, dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(pose_out, Tp, T, traj_feats, cond_feats, control_cond,
                                                                      lengths);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_build_pose_cond(rohm_ctx* ctx, const float* src, int src_channel_major, int src_T,
                                    const float* traj_full, const unsigned char* chan_keep, const int* frame_lo,
                                    const int* frame_hi, int zero_contact, int B, int Tp, const int* lengths,
                                    const float* vis_mask, int vis_T, float* cond_out, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!src || !cond_out || B <= 0 || Tp <= 0 || src_T < Tp || B > 65535 || ((frame_lo == nullptr) != (frame_hi == nullptr)) ||
      (vis_mask != nullptr && (vis_T < Tp || lengths != nullptr)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_build_pose_cond: bad arguments");
  dim3 grid((Tp + 31) / 32, (kC + 31) / 32, B);
  const auto kernel = vis_mask != nullptr ? build_pose_cond_kernel<false, true>
                      : lengths != nullptr ? build_pose_cond_kernel<true> : build_pose_cond_kernel<false>;
  kernel<<<grid, dim3(32, 8), 0, static_cast<cudaStream_t>(stream)>>>(
      src, src_channel_major, src_T, traj_full, chan_keep, frame_lo, frame_hi, zero_contact, Tp, cond_out, lengths,
      vis_mask, vis_T);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_rot6d_to_aa(rohm_ctx* ctx, const float* rot6d, int64_t n, float* aa, float* rotmat, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!rot6d || n < 0 || (aa == nullptr && rotmat == nullptr))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_rot6d_to_aa: bad arguments");
  if (n == 0) return ROHM_OK;
  rot6d_to_aa_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(rot6d, n, aa,
                                                                                                           rotmat);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

// With lengths the absolute mode runs one thread per packed frame (frames are independent); otherwise one thread per clip.
extern "C" int rohm_joints_from_traj(rohm_ctx* ctx, const float* x, int channels_last, const float* mean,
                                     const float* stdv, int B, int T, const int* lengths, const int* clip_off,
                                     int64_t total_frames, int relative, float* joints, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  const bool ragged = lengths != nullptr;
  if (!x || !mean || !stdv || !joints || B <= 0 || T <= 0 ||
      (ragged ? (!clip_off || total_frames < B || total_frames > static_cast<int64_t>(B) * T || total_frames > INT32_MAX)
              : (clip_off != nullptr || total_frames != 0)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_joints_from_traj: bad arguments");
  const int64_t sb = static_cast<int64_t>(kC) * T, sc = channels_last ? 1 : T, stt = channels_last ? kC : 1;
  const bool per_frame = ragged && !relative;
  const int64_t threads = per_frame ? total_frames : B;
  const int block = per_frame ? 128 : 32;
  const auto kernel = ragged ? joints_from_traj_kernel<true> : joints_from_traj_kernel<false>;
  kernel<<<static_cast<unsigned>((threads + block - 1) / block), block, 0, static_cast<cudaStream_t>(stream)>>>(
      x, sb, sc, stt, mean, stdv, B, T, relative ? 1 : 0, joints, lengths, clip_off, static_cast<int>(total_frames));
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

// Lengths are defined for per-clip normalisers only: a batch-wide mean over clips of different lengths is not what a
// one-clip reference run computes for any of them.
extern "C" int rohm_projection_guidance(rohm_body* bd, const float* x0, const float* mean, const float* stdv,
                                        const int* lengths, int B, int T, int per_clip, const float* cam_affine,
                                        const float* focal, const float* center, const float* keypoints_2d, int kp_frames,
                                        float* grad, float* loss_out, void* stream) {
  if (bd == nullptr) return ROHM_ERR_INVALID;
  rohm_ctx* ctx = bd->ctx;
  rohm::DeviceGuard device_guard__(ctx);
  const int64_t N = static_cast<int64_t>(B) * T;
  if (!x0 || !mean || !stdv || !cam_affine || !focal || !center || !keypoints_2d || !grad || B <= 0 || T <= 0 ||
      kp_frames < T)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_projection_guidance: bad arguments");
  if (lengths != nullptr && per_clip == 0)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_projection_guidance: lengths need per-clip normalisers (per_clip = 1)");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool clip = per_clip != 0;
  ROHM_CUDA(ctx, cudaMemsetAsync(grad, 0, sizeof(float) * N * kC, st));
  if (loss_out != nullptr) ROHM_CUDA(ctx, cudaMemsetAsync(loss_out, 0, sizeof(float) * (clip ? B : 1), st));
  ProjParams p{x0, mean, stdv, bd->Jt, bd->Jd, bd->parents_dev, cam_affine, focal, center, keypoints_2d, kp_frames, B, T,
               grad, loss_out, lengths};
  const auto kernel = lengths != nullptr ? projection_guidance_kernel<true, true>
                                         : (clip ? projection_guidance_kernel<true, false>
                                                 : projection_guidance_kernel<false, false>);
  kernel<<<static_cast<unsigned>((N + 63) / 64), 64, 0, st>>>(p);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}
