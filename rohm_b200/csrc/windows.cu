// Sliding-window batching of whole recordings (SURVEY.md 8f, row N4): what the reference's data loaders do on the host,
// one clip at a time, before the rounds, and the inverse of its canonical frame after them.
//
//   rohm_window_encode    dataloader_video.py:160-183 / dataloader_amass.py:105-131 (windows of clip_len frames, stride
//                         clip_len - overlap), motion_representation.py:47-110 cano_seq_smplx + other_utils.py:189-240
//                         update_globalRT_for_smplx (canonical frame and SMPL-X global R/T), motion_representation.py:187-282
//                         get_repr_smplx + :23-44 foot_detect (the 294 channels), dataloader_amass.py:328-329 (z-score)
//   rohm_window_to_world  eval_prox_egobody.py:177-182 (points_coord_trans with the inverse of transf_matrix), scattered
//                         into the recordings' frames
//   rohm_window_param_noise       dataloader_amass.py:156-192 (input noise on the canonical SMPL-X parameters, sep_noise
//                                 False): transl and betas + n, rotations through scipy's 'zxy' Euler angles + n (degrees)
//   rohm_window_encode_canonical  dataloader_amass.py:212-215 (get_repr_smplx of the noisy canonical window, not
//                                 re-canonicalised) and :328-329 (z-score)
//   rohm_window_encode_video      dataloader_video.py:95-183 / :184-370 (camera-frame fits to the scene frame, windows),
//                                 :373-403 (cano_seq_smplx / cano_seq_smplx_egobody, get_repr_smplx), :421-436 (z-score,
//                                 canonical joints and parameters, scene joints, transf_matrix); EgoBody's y-up scene
//                                 enters through the fixed rotation Q = Rx(+90 deg) folded into the camera (DESIGN §4.14)
//   rohm_window_keypoints         dataloader_video.py:441-484 (BODY_25 -> SMPL topology, PROX's flip + cv2.undistortPoints
//                                 + flip back, mask_joint_vis, mask_vec_vis)
//   rohm_window_scene_joints      dataloader_video.py:312-314 (ground-truth joints in the scene frame, per window frame)
#include <cfloat>
#include <cmath>
#include <cstdint>
#include <vector>

#include "common.h"
#include "kin.cuh"
#include "repr.cuh"

namespace rohm {
namespace {

using namespace kin;

constexpr int kC = 294;
constexpr int kJ = 22;
constexpr int kBetas = 10;
constexpr int kPoseJ = 21;
constexpr int kMaxClip = 160;  // frames per window: one thread per frame in one CTA
constexpr int kChLocalPos = 22, kChLocalVel = 88, kChBodyPose = 154, kChBetas = 280, kChContact = 290;
constexpr float kFootVel = 5e-5f;  // get_repr_smplx feet_vel_thre: squared displacement per frame
// a noisy canonical parameter row: global_orient 3 | transl 3 | betas 10 | body_pose 63 (axis-angle)
constexpr int kRowGo = 0, kRowTransl = 3, kRowBetas = 6, kRowPose = 16, kRow = 79;

// A window's canonical frame, cano_seq_smplx: the canonical x and y axes in world coordinates (a, b), the frame-0 root XY
// (ox, oy) and the floor height fl.
struct CanoFrame {
  float ax, ay, bx, by, ox, oy, fl;
  // Rt (p - o) for a world point, Rt v for a world direction
  __device__ __forceinline__ V3 to_cano(V3 p) const {
    const float dx = p.x - ox, dy = p.y - oy;
    return V3{ax * dx + ay * dy, bx * dx + by * dy, p.z - fl};
  }
  __device__ __forceinline__ V3 rot_cano(V3 v) const { return V3{ax * v.x + ay * v.y, bx * v.x + by * v.y, v.z}; }
};

// update_globalRT_for_smplx: R' = Rt R; T' = Rt (T + delta_T - o) - delta_T with delta_T = pelvis - T, i.e. component c of
// the canonical pelvis - pelvis + T.  The encoder and the input noise both take the canonical R/T from here.
__device__ __forceinline__ M3 cano_global_rot(const CanoFrame& F, const float* go) {
  const M3 R = repr::rotvec_to_mat({go[0], go[1], go[2]});
  return M3{F.rot_cano(R.c0), F.rot_cano(R.c1), F.rot_cano(R.c2)};
}
__device__ __forceinline__ float cano_transl(float cano_pelvis, float pelvis, float transl) {
  return cano_pelvis - (pelvis - transl);
}

// A recording's camera -> z-up scene map [A | b], rows of 4 floats.  Every product and sum is one fmaf onto the exact
// zero of the innermost term's start, so an identity camera returns its input exactly.
__device__ __forceinline__ V3 cam_point(const float* c, V3 p) {
  return V3{fmaf(c[0], p.x, fmaf(c[1], p.y, fmaf(c[2], p.z, c[3]))),
            fmaf(c[4], p.x, fmaf(c[5], p.y, fmaf(c[6], p.z, c[7]))),
            fmaf(c[8], p.x, fmaf(c[9], p.y, fmaf(c[10], p.z, c[11])))};
}
__device__ __forceinline__ V3 cam_dir(const float* c, V3 v) {
  return V3{fmaf(c[0], v.x, fmaf(c[1], v.y, fmaf(c[2], v.z, 0.0f))),
            fmaf(c[4], v.x, fmaf(c[5], v.y, fmaf(c[6], v.z, 0.0f))),
            fmaf(c[8], v.x, fmaf(c[9], v.y, fmaf(c[10], v.z, 0.0f)))};
}
// cano_global_rot for a rotation in a recording's camera frame: F R_c2w R_cam.  F's products are written out with the
// fused multiply-adds the compiler chose for cano_global_rot in the world instance (column 0 fuses the product with
// the y component, columns 1 and 2 the one with x), so that an identity camera gives that instance's bits.
__device__ __forceinline__ M3 cano_global_rot_cam(const CanoFrame& F, const float* cam, const float* go) {
  const M3 R = repr::rotvec_to_mat({go[0], go[1], go[2]});
  const V3 a = cam_dir(cam, R.c0), b = cam_dir(cam, R.c1), c = cam_dir(cam, R.c2);
  auto fuse_y = [&](V3 v) {
    return V3{__fmaf_rn(F.ay, v.y, __fmul_rn(F.ax, v.x)), __fmaf_rn(F.by, v.y, __fmul_rn(F.bx, v.x)), v.z};
  };
  auto fuse_x = [&](V3 v) {
    return V3{__fmaf_rn(F.ax, v.x, __fmul_rn(F.ay, v.y)), __fmaf_rn(F.bx, v.x, __fmul_rn(F.by, v.y)), v.z};
  };
  return M3{fuse_y(a), fuse_x(b), fuse_x(c)};
}

// The camera instance's extra inputs and outputs (all null for the other instances).  cam [R,12]: each recording's
// camera -> z-up scene map (for a y-up scene, Q = Rx(+90 deg) times camera -> scene); floor [R]: a preset floor height,
// 0 for the window minimum (the reference's `if preset_floor_height:`); y_up: the scene is y-up (EgoBody), so scene
// points are Q^T of the z-up ones and transf is T_z Q.  Outputs per window frame, including the last: cano_joints and
// scene_joints [W*clip_len,22,3], cano_params [W*clip_len,79] (rows as rohm_window_param_noise writes them).
struct CamIn {
  const float* cam;
  const float* floor;
  int y_up;
  float* cano_joints;
  float* scene_joints;
  float* cano_params;
};

// ---- scipy.spatial.transform.Rotation in float64 (scipy 1.18.1, _rotation_xp.py) ----
// Quaternions are scalar-last (x, y, z, w) like scipy's.
struct Q4 {
  double x, y, z, w;
};

// from_matrix (Shepperd: the largest of the diagonal and the trace picks the stable formula; scipy's order of the
// comparisons, the first maximum wins), then normalised.  m(i, j) is row i, column j.  One branch per choice, so the
// quaternion stays in registers.
template <class M>
__device__ __forceinline__ Q4 quat_from_matrix(M m) {
  const double d0 = m(0, 0), d1 = m(1, 1), d2 = m(2, 2), tr = d0 + d1 + d2;
  int c = 0;  // argmax over (d0, d1, d2, tr)
  double best = d0;
  if (d1 > best) c = 1, best = d1;
  if (d2 > best) c = 2, best = d2;
  if (tr > best) c = 3;
  Q4 q;
  if (c == 0) {
    q = {1.0 - tr + 2.0 * d0, m(1, 0) + m(0, 1), m(2, 0) + m(0, 2), m(2, 1) - m(1, 2)};
  } else if (c == 1) {
    q = {m(0, 1) + m(1, 0), 1.0 - tr + 2.0 * d1, m(2, 1) + m(1, 2), m(0, 2) - m(2, 0)};
  } else if (c == 2) {
    q = {m(0, 2) + m(2, 0), m(1, 2) + m(2, 1), 1.0 - tr + 2.0 * d2, m(1, 0) - m(0, 1)};
  } else {
    q = {m(2, 1) - m(1, 2), m(0, 2) - m(2, 0), m(1, 0) - m(0, 1), 1.0 + tr};
  }
  const double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}

// as_rotvec: the quaternion in scipy's canonical sign (w > 0; at w == 0 the first non-zero of x, y, z positive), angle = 2 atan2(|v|, w), scale = 2 + angle^2/12 +
// 7 angle^4/2880 for angle <= 1e-3, angle / sin(angle/2) otherwise
__device__ __forceinline__ void rotvec_from_quat(Q4 q, float* out) {
  const bool flip = q.w < 0.0 || (q.w == 0.0 && (q.x < 0.0 || (q.x == 0.0 && (q.y < 0.0 || (q.y == 0.0 && q.z < 0.0)))));
  if (flip) q = {-q.x, -q.y, -q.z, -q.w};
  const double n = sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
  const double a = 2.0 * atan2(n, q.w), a2 = a * a;
  const double sc = a <= 1e-3 ? 2.0 + a2 / 12.0 + 7.0 * a2 * a2 / 2880.0 : a / sin(0.5 * a);
  out[0] = static_cast<float>(sc * q.x), out[1] = static_cast<float>(sc * q.y), out[2] = static_cast<float>(sc * q.z);
}

// the instances of window_encode_kernel: what its joints and parameters are
constexpr int kWorldIn = 0, kCanonicalIn = 1, kCameraIn = 2;

// One CTA per window, one thread per window frame.  (1) the floor height (min z over the window's clip_len x 22 joints),
// the frame-0 root XY and the frame-0 heading from hips + shoulders give transf = [Rt | -Rt o]; (2) each thread
// canonicalises its frame's joints into shared memory and takes their root heading quaternion; (3) the first NaN
// heading is repaired and frame 0 pinned to the identity, as traj_full_repr_kernel does over a clip; (4) frame t < clip_len
// - 1 writes row t: the 22 trajectory channels through repr::traj_channels with the canonical SMPL-X global R/T, then local
// positions, local velocities, body-pose 6-D, betas and foot contacts, z-scored twice (TrajNet and PoseNet statistics).
// Input rows are the packed recording frames rec_off[win_rec[w]] + win_start[w] + t; nothing outside a window is read.
//
// kCanonical: the window's frames are already canonical (the noisy windows, which the reference does not re-canonicalise):
// joints are window-major rows w * clip_len + t, the parameters are kRow-wide rows of that layout (go, transl, betas and
// body_pose point into one row array), (1) is skipped, nothing is written to transf, and the SMPL-X R/T are used as given.
//
// kCameraIn: joints and parameters are in each recording's camera frame (the video loader's per-frame fits): (0) each
// thread maps its frame's joints by the recording's camera (cam_point) into shared memory and writes them, in the scene
// frame, to cam.scene_joints; (1) takes the preset floor unless it is 0 and reads the frame from shared memory; the
// global rotation is F R_c2w R_cam and the translation cano_pelvis - (pelvis_cam - transl_cam) (delta_T of
// update_globalRT_for_smplx is the same in the camera and the scene frame); every frame writes its canonical joints and
// SMPL-X parameters (global_orient by scipy's from_matrix / as_rotvec in float64).
template <int kIn>
__global__ void __launch_bounds__(kMaxClip) window_encode_kernel(
    const float* __restrict__ joints, const float* __restrict__ go, const float* __restrict__ transl,
    const float* __restrict__ betas, const float* __restrict__ body_pose, const int* __restrict__ win_rec,
    const int* __restrict__ win_start, const int* __restrict__ rec_off, int clip_len, const float* __restrict__ tmean,
    const float* __restrict__ tstd, const float* __restrict__ pmean, const float* __restrict__ pstd,
    float* __restrict__ transf, float* __restrict__ out_traj, float* __restrict__ out_pose, const CamIn cam) {
  constexpr bool kCanonical = kIn == kCanonicalIn, kCamera = kIn == kCameraIn;
  constexpr int kGoS = kCanonical ? kRow : 3, kTrS = kCanonical ? kRow : 3, kBeS = kCanonical ? kRow : kBetas,
                kBpS = kCanonical ? kRow : kPoseJ * 3;
  __shared__ float cj[kMaxClip * kJ * 3];  // canonical joints of the window's frames
  __shared__ float qw[kMaxClip], qz[kMaxClip];
  __shared__ float wmin[kMaxClip / 32];
  __shared__ float frame[7];  // x axis (xy), y axis (xy), origin (x, y, floor)
  __shared__ int first_nan;
  const int w = blockIdx.x, t = threadIdx.x;
  const bool mine = t < clip_len;
  const int64_t f = kCanonical ? static_cast<int64_t>(w) * clip_len + (mine ? t : 0)
                               : static_cast<int64_t>(rec_off[win_rec[w]]) + win_start[w] + (mine ? t : 0);
  const float* P = joints + f * kJ * 3;
  auto J = [&](const float* base, int j) { return V3{base[j * 3], base[j * 3 + 1], base[j * 3 + 2]}; };
  CanoFrame F;
  const float* A = nullptr;  // the recording's camera (kCameraIn)

  if constexpr (kCanonical) {
    if (t == 0) first_nan = clip_len;
    __syncthreads();
    if (mine)
      for (int j = 0; j < kJ * 3; ++j) cj[t * kJ * 3 + j] = P[j];
  } else {
    // (1) canonical frame; the camera instance first maps its frame's joints into the z-up scene frame, in shared memory,
    // and reads the frame from there
    const float* S = P;
    float m = INFINITY;
    if constexpr (kCamera) {
      A = cam.cam + static_cast<int64_t>(win_rec[w]) * 12;
      S = cj;
      if (mine) {
        float* D = cj + t * kJ * 3;
        float* o = cam.scene_joints + (static_cast<int64_t>(w) * clip_len + t) * kJ * 3;
        for (int j = 0; j < kJ; ++j) {
          const V3 p = cam_point(A, J(P, j));
          D[j * 3] = p.x, D[j * 3 + 1] = p.y, D[j * 3 + 2] = p.z;
          m = fminf(m, p.z);
          o[j * 3] = p.x, o[j * 3 + 1] = cam.y_up ? p.z : p.y, o[j * 3 + 2] = cam.y_up ? -p.y : p.z;
        }
      }
    } else {
      if (mine)
        for (int j = 0; j < kJ; ++j) m = fminf(m, P[j * 3 + 2]);
    }
    for (int s = 16; s > 0; s >>= 1) m = fminf(m, __shfl_xor_sync(0xffffffffu, m, s));
    if ((t & 31) == 0) wmin[t >> 5] = m;
    if (t == 0) first_nan = clip_len;
    __syncthreads();
    if (t == 0) {
      float fl = wmin[0];
      for (int i = 1; i < static_cast<int>(blockDim.x) / 32; ++i) fl = fminf(fl, wmin[i]);
      if constexpr (kCamera) {  // the reference's `if preset_floor_height:`: a preset 0 takes the window minimum
        const float pre = cam.floor[win_rec[w]];
        if (pre != 0.0f) fl = pre;
      }
      // cano_seq_smplx: x = (r_hip - l_hip) + (sdr_r - sdr_l) = (2 - 1) + (17 - 16) without its up component, y = z x x
      V3 x = (J(S, 2) - J(S, 1)) + (J(S, 17) - J(S, 16));
      x.z = 0.0f;
      x = (1.0f / sqrtf(dot(x, x))) * x;
      V3 y = {-x.y, x.x, 0.0f};
      y = (1.0f / sqrtf(dot(y, y))) * y;
      const float ox = S[0], oy = S[1];
      frame[0] = x.x, frame[1] = x.y, frame[2] = y.x, frame[3] = y.y, frame[4] = ox, frame[5] = oy, frame[6] = fl;
      float* M = transf + static_cast<int64_t>(w) * 16;
      M[0] = x.x, M[1] = x.y, M[2] = 0.0f, M[3] = -(x.x * ox + x.y * oy);
      M[4] = y.x, M[5] = y.y, M[6] = 0.0f, M[7] = -(y.x * ox + y.y * oy);
      M[8] = 0.0f, M[9] = 0.0f, M[10] = 1.0f, M[11] = -fl;
      M[12] = 0.0f, M[13] = 0.0f, M[14] = 0.0f, M[15] = 1.0f;
      if constexpr (kCamera)
        if (cam.y_up)  // T_z Q: columns (c0, c2, -c1, c3)
          for (int i = 0; i < 3; ++i) {
            const float c1 = M[i * 4 + 1];
            M[i * 4 + 1] = M[i * 4 + 2], M[i * 4 + 2] = -c1;
          }
    }
    __syncthreads();
    F = CanoFrame{frame[0], frame[1], frame[2], frame[3], frame[4], frame[5], frame[6]};
  }

  // (2) canonical joints and headings
  float* C0 = cj + t * kJ * 3;
  if (mine) {
    if constexpr (kCamera) {
      const int64_t row = static_cast<int64_t>(w) * clip_len + t;
      float* oj = cam.cano_joints + row * kJ * 3;
      for (int j = 0; j < kJ; ++j) {
        const V3 c = F.to_cano(J(C0, j));
        C0[j * 3] = c.x, C0[j * 3 + 1] = c.y, C0[j * 3 + 2] = c.z;
        oj[j * 3] = c.x, oj[j * 3 + 1] = c.y, oj[j * 3 + 2] = c.z;
      }
      float* o = cam.cano_params + row * kRow;
      const M3 R = cano_global_rot_cam(F, A, go + f * 3);
      auto m = [&](int a, int b) {
        const V3 col = b == 0 ? R.c0 : (b == 1 ? R.c1 : R.c2);
        return static_cast<double>(a == 0 ? col.x : (a == 1 ? col.y : col.z));
      };
      rotvec_from_quat(quat_from_matrix(m), o + kRowGo);
      for (int c = 0; c < 3; ++c) o[kRowTransl + c] = cano_transl(C0[c], P[c], transl[f * 3 + c]);
      for (int l = 0; l < kBetas; ++l) o[kRowBetas + l] = betas[f * kBetas + l];
      for (int k = 0; k < kPoseJ * 3; ++k) o[kRowPose + k] = body_pose[f * kPoseJ * 3 + k];
    } else if constexpr (!kCanonical)
      for (int j = 0; j < kJ; ++j) {
        const V3 c = F.to_cano(J(P, j));
        C0[j * 3] = c.x, C0[j * 3 + 1] = c.y, C0[j * 3 + 2] = c.z;
      }
    float q0, q1, q3;
    repr::heading_quat(J(C0, 1), J(C0, 2), J(C0, 17), J(C0, 16), q0, q1, q3);
    qw[t] = q0, qz[t] = q3;
    if (isnan(q0) || isnan(q1) || isnan(q3)) atomicMin(&first_nan, t);
  }
  __syncthreads();
  // (3) the reference repairs the first NaN heading only, with its predecessor (the last frame for frame 0)
  if (t == 0) {
    if (first_nan < clip_len) {
      const int dst = first_nan, src = first_nan > 0 ? first_nan - 1 : clip_len - 1;
      qw[dst] = qw[src], qz[dst] = qz[src];
    }
    qw[0] = 1.0f, qz[0] = 0.0f;
  }
  __syncthreads();
  if (t >= clip_len - 1) return;

  // (4) row t
  const float* C1 = C0 + kJ * 3;
  const float w0 = qw[t], z0 = qz[t], w1 = qw[t + 1], z1 = qz[t + 1];
  const int64_t row = static_cast<int64_t>(w) * (clip_len - 1) + t;
  float* dt = out_traj + row * kC;
  float* dp = out_pose + row * kC;
  auto put = [&](int c, float v) {
    dt[c] = (v - tmean[c]) / tstd[c];
    dp[c] = (v - pmean[c]) / pstd[c];
  };
  float o[repr::kTrajFull];
  {
    auto root = [&](int k) { return J(k == 0 ? C0 : C1, 0); };
    auto rot = [&](int k) {
      if constexpr (kCanonical) {
        const float* a = go + (f + k) * kGoS;
        return repr::rotvec_to_mat({a[0], a[1], a[2]});
      } else if constexpr (kCamera) {
        return cano_global_rot_cam(F, A, go + (f + k) * 3);
      } else {
        return cano_global_rot(F, go + (f + k) * 3);
      }
    };
    auto tr = [&](int k, int c) {
      if constexpr (kCanonical) {
        return transl[(f + k) * kTrS + c];
      } else {
        return cano_transl((k == 0 ? C0 : C1)[c], P[k * kJ * 3 + c], transl[(f + k) * 3 + c]);
      }
    };
    repr::traj_channels(o, w0, z0, w1, z1, root, rot, tr);
  }
#pragma unroll
  for (int c = 0; c < repr::kTrajFull; ++c) put(c, o[c]);
  const V3 r0 = J(C0, 0);
  for (int j = 0; j < kJ; ++j) {
    const V3 c0 = J(C0, j), c1 = J(C1, j);
    const V3 lp = repr::qrot_z(w0, z0, {c0.x - r0.x, c0.y - r0.y, c0.z});
    const V3 lv = repr::qrot_z(w0, z0, c1 - c0);
    put(kChLocalPos + j * 3, lp.x), put(kChLocalPos + j * 3 + 1, lp.y), put(kChLocalPos + j * 3 + 2, lp.z);
    put(kChLocalVel + j * 3, lv.x), put(kChLocalVel + j * 3 + 1, lv.y), put(kChLocalVel + j * 3 + 2, lv.z);
  }
  for (int k = 0; k < kPoseJ; ++k) {
    const float* a = body_pose + f * kBpS + k * 3;
    const M3 R = repr::rotvec_to_mat({a[0], a[1], a[2]});
    const int c = kChBodyPose + k * 6;
    put(c, R.c0.x), put(c + 1, R.c1.x), put(c + 2, R.c0.y), put(c + 3, R.c1.y), put(c + 4, R.c0.z), put(c + 5, R.c1.z);
  }
  for (int l = 0; l < kBetas; ++l) put(kChBetas + l, betas[f * kBeS + l]);
  // foot_detect (up axis z): left feet 7, 10 then right feet 8, 11; height factors 0.18 (ankles), 0.15 (toes)
  for (int s = 0; s < 4; ++s) {
    const int j = (s & 1 ? 10 : 7) + (s >> 1);
    const float thr = s & 1 ? 0.15f : 0.18f;
    const V3 d = J(C1, j) - J(C0, j);
    const bool contact = d.x * d.x + d.y * d.y + d.z * d.z < kFootVel && C0[j * 3 + 2] < thr;
    put(kChContact + s, contact ? 1.0f : 0.0f);
  }
}

// ---- the rest of scipy's Rotation the noise needs (Q4, quat_from_matrix and rotvec_from_quat are above) ----

// from_rotvec: angle = |r|; scale = 0.5 - angle^2/48 + angle^4/3840 for angle <= 1e-3, sin(angle/2)/angle otherwise
__device__ __forceinline__ Q4 quat_from_rotvec(double rx, double ry, double rz) {
  const double a2 = rx * rx + ry * ry + rz * rz, a = sqrt(a2);
  const double sc = a <= 1e-3 ? 0.5 - a2 / 48.0 + a2 * a2 / 3840.0 : sin(0.5 * a) / a;
  return {sc * rx, sc * ry, sc * rz, cos(0.5 * a)};
}

// scipy's wrap of an Euler angle: one turn added or taken away where it lies outside [-pi, pi] (an exact +-pi stays)
__device__ __forceinline__ double wrap_pi(double a) {
  return a < -M_PI ? a + 2.0 * M_PI : (a > M_PI ? a - 2.0 * M_PI : a);
}

// as_euler('zxy') (extrinsic z, then x, then y) by Bernardes & Viollet's quaternion method, the algorithm scipy uses
// since 1.10 (scipy 1.8.0, which the reference pins, goes through the matrix; both agree away from the lock): axes
// (i, j, k) = (z, x, y), sign +1, a = w - x, b = z + y, c = x + w, d = y - z.  The middle angle is 2 atan2(|(c, d)|,
// |(a, b)|) - pi/2 in [-pi/2, pi/2].  Within 1e-7 rad of the lock (middle angle +-pi/2) the third angle is 0 and the first
// carries the whole rotation about the vertical: 2 atan2(b, a) at -pi/2, -2 atan2(d, c) at +pi/2 - scipy's rule and
// threshold.  Every angle is then brought into [-pi, pi] as wrap_pi does.
__device__ __forceinline__ void euler_zxy(const Q4& q, double e[3]) {
  const double a = q.w - q.x, b = q.z + q.y, c = q.x + q.w, d = q.y - q.z;
  const double hs = atan2(b, a), hd = atan2(d, c);
  const double th = 2.0 * atan2(hypot(c, d), hypot(a, b));
  const bool lock0 = fabs(th) <= 1e-7, lock1 = fabs(th - M_PI) <= 1e-7;
  if (lock0 || lock1) {
    e[0] = lock0 ? 2.0 * hs : -2.0 * hd;
    e[2] = 0.0;
  } else {
    e[0] = hs - hd;
    e[2] = hs + hd;
  }
  e[1] = th - 0.5 * M_PI;
  for (int i = 0; i < 3; ++i) e[i] = wrap_pi(e[i]);
}

// from_euler('zxy', e): q = q_y(e2) q_x(e1) q_z(e0), elementary q_axis(t) = (sin(t/2) axis, cos(t/2))
__device__ __forceinline__ Q4 quat_from_euler_zxy(const double e[3]) {
  double sz, cz, sx, cx, sy, cy;
  sincos(0.5 * e[0], &sz, &cz);
  sincos(0.5 * e[1], &sx, &cx);
  sincos(0.5 * e[2], &sy, &cy);
  // q_x q_z = (sx cz, -sx sz... ): (cx, sx, 0, 0) * (cz, 0, 0, sz) in (w, x, y, z)
  const double w1 = cx * cz, x1 = sx * cz, y1 = -sx * sz, z1 = cx * sz;
  // q_y * q1 with q_y = (cy, 0, sy, 0)
  return {cy * x1 + sy * z1, cy * y1 + sy * w1, cy * z1 - sy * x1, cy * w1 - sy * y1};
}

// One rotation + n degrees of zxy Euler noise, in float64: the reference's as_euler('zxy', degrees=True) + n ->
// from_euler('zxy', degrees=True) -> as_rotvec.
__device__ __forceinline__ void add_euler_noise(const Q4& q, const float* n_deg, float* out) {
  double e[3];
  euler_zxy(q, e);
  constexpr double kDeg = M_PI / 180.0;
  for (int i = 0; i < 3; ++i) e[i] += static_cast<double>(n_deg[i]) * kDeg;
  rotvec_from_quat(quat_from_euler_zxy(e), out);
}

// One thread per (window, frame, rotation): rotation 0 is the canonical global orientation (that thread also writes the
// canonical translation and the betas, each + n), rotations 1..21 the body-pose joints.  The canonical R/T come from the
// encoder's own functions (cano_global_rot, cano_transl) on the window's frame, rebuilt from transf and the window's
// frame-0 root, so the clean parameters under the noise are those the clean rows were encoded from.  Noise arrays are
// window-major [W, clip_len, .]; out is [W * clip_len, kRow].
__global__ void window_param_noise_kernel(const float* __restrict__ joints, const float* __restrict__ go,
                                          const float* __restrict__ transl, const float* __restrict__ betas,
                                          const float* __restrict__ body_pose, const int* __restrict__ win_rec,
                                          const int* __restrict__ win_start, const int* __restrict__ rec_off,
                                          const float* __restrict__ transf, int W, int clip_len,
                                          const float* __restrict__ n_transl, const float* __restrict__ n_betas,
                                          const float* __restrict__ n_go, const float* __restrict__ n_pose,
                                          float* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(W) * clip_len * (kPoseJ + 1)) return;
  const int r = static_cast<int>(i % (kPoseJ + 1));
  const int64_t row = i / (kPoseJ + 1);  // w * clip_len + t
  const int w = static_cast<int>(row / clip_len), t = static_cast<int>(row % clip_len);
  const int64_t f0 = static_cast<int64_t>(rec_off[win_rec[w]]) + win_start[w], f = f0 + t;
  float* o = out + row * kRow;
  if (r > 0) {
    const float* a = body_pose + f * kPoseJ * 3 + (r - 1) * 3;
    add_euler_noise(quat_from_rotvec(a[0], a[1], a[2]), n_pose + (row * kPoseJ + (r - 1)) * 3, o + kRowPose + (r - 1) * 3);
    return;
  }
  const float* M = transf + static_cast<int64_t>(w) * 16;
  const float* P0 = joints + f0 * kJ * 3;
  const CanoFrame F{M[0], M[1], M[4], M[5], P0[0], P0[1], -M[11]};
  const float* P = joints + f * kJ * 3;
  const V3 pelvis = F.to_cano({P[0], P[1], P[2]});
  const float cp[3] = {pelvis.x, pelvis.y, pelvis.z};
  for (int c = 0; c < 3; ++c) o[kRowTransl + c] = cano_transl(cp[c], P[c], transl[f * 3 + c]) + n_transl[row * 3 + c];
  for (int l = 0; l < kBetas; ++l) o[kRowBetas + l] = betas[f * kBetas + l] + n_betas[row * kBetas + l];
  const M3 R = cano_global_rot(F, go + f * 3);
  auto m = [&](int a, int b) {
    const V3 col = b == 0 ? R.c0 : (b == 1 ? R.c1 : R.c2);
    return static_cast<double>(a == 0 ? col.x : (a == 1 ? col.y : col.z));
  };
  add_euler_noise(quat_from_matrix(m), n_go + row * 3, o + kRowGo);
}

// One thread per (window, pose frame, joint): p = R^T (c - t) for transf = [R | t], written to recording frame
// rec_off[win_rec[w]] + win_start[w] + pose frame, which is marked covered.
__global__ void window_to_world_kernel(const float* __restrict__ joints, const int* __restrict__ win_rec,
                                       const int* __restrict__ win_start, const int* __restrict__ rec_off,
                                       const float* __restrict__ transf, int W, int pose_frames, float* __restrict__ world,
                                       unsigned char* __restrict__ covered) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(W) * pose_frames * kJ) return;
  const int j = static_cast<int>(i % kJ);
  const int64_t r = i / kJ;
  const int w = static_cast<int>(r / pose_frames), t = static_cast<int>(r % pose_frames);
  const float* M = transf + static_cast<int64_t>(w) * 16;
  const float* c = joints + i * 3;
  const V3 d = {c[0] - M[3], c[1] - M[7], c[2] - M[11]};
  const int64_t fr = static_cast<int64_t>(rec_off[win_rec[w]]) + win_start[w] + t;
  float* o = world + (fr * kJ + j) * 3;
  o[0] = M[0] * d.x + M[4] * d.y + M[8] * d.z;
  o[1] = M[1] * d.x + M[5] * d.y + M[9] * d.z;
  o[2] = M[2] * d.x + M[6] * d.y + M[10] * d.z;
  if (j == 0) covered[fr] = 1;
}

// dataloader_video.py:50: the OpenPose BODY_25 keypoint of each of the 22 SMPL joints
__constant__ int kBody25ToSmpl[kJ] = {8, 12, 9, 8, 13, 10, 8, 14, 11, 1, 20, 23, 1, 5, 2, 0, 5, 2, 6, 3, 7, 4};
constexpr double kFlipX = 1919.0;  // dataloader_video.py:445: x -> 1920 - 1 - x (PROX's mirrored colour frames)

// cv2.undistortPoints(src, K, k, P=K) for one point, float64, in OpenCV's order of operations (undistort.dispatch.cpp
// cvUndistortPointsInternal, 4.13): 5 fixed iterations (the default criteria count iterations only); a negative icdist
// keeps the input point; no tilt (the identity tilt map leaves x, y unchanged); then P.  Every product and sum is a
// separately rounded _rn operation, as the host code computes it without fused multiply-adds.
__device__ __forceinline__ void undistort_point(const double* K, const double* k, double& x, double& y) {
  auto mul = [](double a, double b) { return __dmul_rn(a, b); };
  auto add = [](double a, double b) { return __dadd_rn(a, b); };
  auto sub = [](double a, double b) { return __dsub_rn(a, b); };
  const double fx = K[0], fy = K[4], cx = K[2], cy = K[5];
  const double ifx = 1.0 / fx, ify = 1.0 / fy;
  const double u = x, v = y;
  x = mul(sub(x, cx), ifx);
  y = mul(sub(y, cy), ify);
  const double x0 = x, y0 = y;
  for (int it = 0; it < 5; ++it) {
    const double r2 = add(mul(x, x), mul(y, y));
    const double num = add(1.0, mul(add(mul(add(mul(k[7], r2), k[6]), r2), k[5]), r2));
    const double den = add(1.0, mul(add(mul(add(mul(k[4], r2), k[1]), r2), k[0]), r2));
    const double icdist = num / den;
    if (icdist < 0) {
      x = mul(sub(u, cx), ifx);
      y = mul(sub(v, cy), ify);
      break;
    }
    const double dx = add(add(add(mul(mul(mul(2.0, k[2]), x), y), mul(k[3], add(r2, mul(mul(2.0, x), x)))), mul(k[8], r2)),
                          mul(mul(k[9], r2), r2));
    const double dy = add(add(add(mul(k[2], add(r2, mul(mul(2.0, y), y))), mul(mul(mul(2.0, k[3]), x), y)), mul(k[10], r2)),
                          mul(mul(k[11], r2), r2));
    x = mul(sub(x0, dx), icdist);
    y = mul(sub(y0, dy), icdist);
  }
  const double xx = add(add(mul(K[0], x), mul(K[1], y)), K[2]);
  const double yy = add(add(mul(K[3], x), mul(K[4], y)), K[5]);
  const double ww = 1.0 / add(add(mul(K[6], x), mul(K[7], y)), K[8]);
  x = mul(xx, ww);
  y = mul(yy, ww);
}

// mask_joint_vis of one joint: (conf > 0.2) * depth mask, the comparison in float64 where the recording's keypoint array
// is float64 (a frame without a person made it so), in float32 otherwise
__device__ __forceinline__ float joint_vis(const float* kp25, const float* depth, int64_t f, int j, bool conf64) {
  const float c = kp25[(f * 25 + kBody25ToSmpl[j]) * 3 + 2];
  const bool seen = conf64 ? static_cast<double>(c) > 0.2 : c > 0.2f;
  return seen ? depth[f * 25 + j] : 0.0f;
}

// One thread per (window, frame, joint): the keypoint in SMPL topology (PROX: un-flipped, undistorted, flipped back),
// mask_joint_vis, and the joint's columns of the 294-wide mask_vec_vis row (local positions and velocities x3, body pose
// x6 from joint 1); joint 0 also writes the trajectory, betas and foot-contact columns.
__global__ void window_keypoints_kernel(const float* __restrict__ kp25, const float* __restrict__ depth,
                                        const unsigned char* __restrict__ kp64, const double* __restrict__ cam_mtx,
                                        const double* __restrict__ dist, int undistort, const int* __restrict__ rec_off,
                                        const int* __restrict__ win_rec, const int* __restrict__ win_start, int W,
                                        int clip_len, float* __restrict__ kp_out, float* __restrict__ vis_out,
                                        float* __restrict__ vec_out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(W) * clip_len * kJ) return;
  const int j = static_cast<int>(i % kJ);
  const int64_t row = i / kJ;
  const int w = static_cast<int>(row / clip_len), t = static_cast<int>(row % clip_len);
  const int rec = win_rec[w];
  const int64_t f = static_cast<int64_t>(rec_off[rec]) + win_start[w] + t;
  const bool wide = kp64[rec] != 0;
  const float* p = kp25 + (f * 25 + kBody25ToSmpl[j]) * 3;
  float* o = kp_out + i * 3;
  if (undistort) {
    double x = wide ? kFlipX - static_cast<double>(p[0]) : static_cast<double>(__fsub_rn(1919.0f, p[0]));
    double y = p[1];
    undistort_point(cam_mtx + static_cast<int64_t>(rec) * 9, dist + static_cast<int64_t>(rec) * 14, x, y);
    o[0] = static_cast<float>(kFlipX - x), o[1] = static_cast<float>(y);
  } else {
    o[0] = p[0], o[1] = p[1];
  }
  o[2] = p[2];
  const float v = joint_vis(kp25, depth, f, j, wide);
  vis_out[i] = v;
  float* r = vec_out + row * kC;
  for (int c = 0; c < 3; ++c) r[kChLocalPos + j * 3 + c] = v, r[kChLocalVel + j * 3 + c] = v;
  if (j > 0)
    for (int c = 0; c < 6; ++c) r[kChBodyPose + (j - 1) * 6 + c] = v;
  if (j == 0) {
    for (int c = 0; c < repr::kTrajFull; ++c) r[c] = 1.0f;
    for (int c = 0; c < kBetas; ++c) r[kChBetas + c] = 1.0f;
    const bool left = joint_vis(kp25, depth, f, 7, wide) == 1.0f && joint_vis(kp25, depth, f, 10, wide) == 1.0f;
    const bool right = joint_vis(kp25, depth, f, 8, wide) == 1.0f && joint_vis(kp25, depth, f, 11, wide) == 1.0f;
    r[kChContact] = r[kChContact + 1] = left ? 1.0f : 0.0f;
    r[kChContact + 2] = r[kChContact + 3] = right ? 1.0f : 0.0f;
  }
}

// One thread per (window, frame, joint): the recording's camera applied to joints (packed recording frames), gathered
// into window-major rows [W*clip_len, 22, 3].
__global__ void window_scene_joints_kernel(const float* __restrict__ joints, const float* __restrict__ cam,
                                           const int* __restrict__ rec_off, const int* __restrict__ win_rec,
                                           const int* __restrict__ win_start, int W, int clip_len,
                                           float* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= static_cast<int64_t>(W) * clip_len * kJ) return;
  const int j = static_cast<int>(i % kJ);
  const int64_t row = i / kJ;
  const int w = static_cast<int>(row / clip_len), t = static_cast<int>(row % clip_len);
  const int rec = win_rec[w];
  const int64_t f = static_cast<int64_t>(rec_off[rec]) + win_start[w] + t;
  const float* p = joints + (f * kJ + j) * 3;
  const V3 q = cam_point(cam + static_cast<int64_t>(rec) * 12, V3{p[0], p[1], p[2]});
  out[i * 3] = q.x, out[i * 3 + 1] = q.y, out[i * 3 + 2] = q.z;
}

// The reference loop: window k of a recording starts at k * (clip_len - overlap) and is cut while it ends inside the
// recording; a recording shorter than clip_len gives none.  Host arrays; returns ROHM_OK or the failure.
int cut_windows(rohm_ctx* ctx, const char* name, const int* rec_off_host, int R, int clip_len, int overlap,
                std::vector<int>& tab_rec, std::vector<int>& tab_start) {
  if (clip_len < 3 || clip_len > kMaxClip || overlap < 0 || overlap > 2)
    return fail(ctx, ROHM_ERR_INVALID, "%s: clip_len=%d overlap=%d; windows of 3 to %d frames with an "
                "overlap of 0 to 2 frames (so that no recording frame lies in two windows' pose frames)", name, clip_len,
                overlap, kMaxClip);
  const int stride = clip_len - overlap;
  for (int r = 0; r < R; ++r) {
    const int n = rec_off_host[r + 1] - rec_off_host[r];
    if (rec_off_host[r] < 0 || n < 0)
      return fail(ctx, ROHM_ERR_INVALID, "%s: recording offsets must be non-negative and non-decreasing "
                  "(rec_off[%d] = %d, rec_off[%d] = %d)", name, r, rec_off_host[r], r + 1, rec_off_host[r + 1]);
    for (int s = 0; s + clip_len <= n; s += stride) tab_rec.push_back(r), tab_start.push_back(s);
  }
  return ROHM_OK;
}

}  // namespace
}  // namespace rohm

using namespace rohm;

extern "C" int rohm_window_encode(rohm_ctx* ctx, const float* global_orient, const float* transl, const float* betas,
                                  const float* body_pose, const float* joints, const int* rec_off_host,
                                  const int* rec_off, int R, int clip_len,
                                  int overlap, const float* traj_mean, const float* traj_std, const float* pose_mean,
                                  const float* pose_std, int max_windows, int* n_windows, int* win_rec, int* win_start,
                                  float* transf, float* repr_traj, float* repr_pose, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!global_orient || !transl || !betas || !body_pose || !joints || !rec_off || !traj_mean || !traj_std || !pose_mean ||
      !pose_std || !rec_off_host || !n_windows || !win_rec || !win_start || !transf || !repr_traj || !repr_pose || R <= 0 || max_windows < 0)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_encode: bad arguments");
  std::vector<int> tab_rec, tab_start;
  if (const int rc = cut_windows(ctx, "rohm_window_encode", rec_off_host, R, clip_len, overlap, tab_rec, tab_start))
    return rc;
  const int W = static_cast<int>(tab_rec.size());
  *n_windows = W;
  if (W > max_windows)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_encode: %d windows exceed the %d the outputs hold", W, max_windows);
  if (W == 0) return ROHM_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ROHM_CUDA(ctx, cudaMemcpyAsync(win_rec, tab_rec.data(), sizeof(int) * W, cudaMemcpyHostToDevice, st));
  ROHM_CUDA(ctx, cudaMemcpyAsync(win_start, tab_start.data(), sizeof(int) * W, cudaMemcpyHostToDevice, st));
  window_encode_kernel<kWorldIn><<<W, (clip_len + 31) / 32 * 32, 0, st>>>(
      joints, global_orient, transl, betas, body_pose, win_rec, win_start, rec_off, clip_len, traj_mean, traj_std,
      pose_mean, pose_std, transf, repr_traj, repr_pose, CamIn{});
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_window_param_noise(rohm_ctx* ctx, const float* global_orient, const float* transl,
                                       const float* betas, const float* body_pose, const float* joints, const int* rec_off,
                                       const int* win_rec, const int* win_start, const float* transf, int W, int clip_len,
                                       const float* noise_transl, const float* noise_betas, const float* noise_global_orient,
                                       const float* noise_body_pose, float* noisy_params, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (W < 0 || clip_len < 3 || clip_len > kMaxClip ||
      (W > 0 && (!global_orient || !transl || !betas || !body_pose || !joints || !rec_off || !win_rec || !win_start ||
                 !transf || !noise_transl || !noise_betas || !noise_global_orient || !noise_body_pose || !noisy_params)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_param_noise: bad arguments");
  const int64_t n = static_cast<int64_t>(W) * clip_len * (kPoseJ + 1);
  if (n == 0) return ROHM_OK;
  window_param_noise_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      joints, global_orient, transl, betas, body_pose, win_rec, win_start, rec_off, transf, W, clip_len, noise_transl,
      noise_betas, noise_global_orient, noise_body_pose, noisy_params);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_window_encode_canonical(rohm_ctx* ctx, const float* params, const float* joints, int W, int clip_len,
                                            const float* traj_mean, const float* traj_std, const float* pose_mean,
                                            const float* pose_std, float* repr_traj, float* repr_pose, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (W < 0 || clip_len < 3 || clip_len > kMaxClip ||
      (W > 0 && (!params || !joints || !traj_mean || !traj_std || !pose_mean || !pose_std || !repr_traj || !repr_pose)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_encode_canonical: bad arguments");
  if (W == 0) return ROHM_OK;
  window_encode_kernel<kCanonicalIn><<<W, (clip_len + 31) / 32 * 32, 0, static_cast<cudaStream_t>(stream)>>>(
      joints, params + kRowGo, params + kRowTransl, params + kRowBetas, params + kRowPose, nullptr, nullptr, nullptr,
      clip_len, traj_mean, traj_std, pose_mean, pose_std, nullptr, repr_traj, repr_pose, CamIn{});
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_window_to_world(rohm_ctx* ctx, const float* joints, const int* win_rec, const int* win_start,
                                    const float* transf, int W, int clip_len, const int* rec_off, int64_t total_frames,
                                    float* world, unsigned char* covered, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!world || !covered || !rec_off || W < 0 || clip_len < 3 || clip_len > kMaxClip || total_frames < 0 ||
      (W > 0 && (!joints || !win_rec || !win_start || !transf)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_to_world: bad arguments");
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (total_frames == 0) return ROHM_OK;
  ROHM_CUDA(ctx, cudaMemsetAsync(world, 0, sizeof(float) * total_frames * kJ * 3, st));
  ROHM_CUDA(ctx, cudaMemsetAsync(covered, 0, static_cast<size_t>(total_frames), st));
  const int64_t n = static_cast<int64_t>(W) * (clip_len - 2) * kJ;
  if (n == 0) return ROHM_OK;
  window_to_world_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, st>>>(joints, win_rec, win_start, rec_off, transf,
                                                                                W, clip_len - 2, world, covered);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_window_encode_video(rohm_ctx* ctx, const float* global_orient, const float* transl,
                                        const float* betas, const float* body_pose, const float* joints,
                                        const int* rec_off_host, const int* rec_off, int R, int clip_len, int overlap,
                                        const float* cam, const float* floor, int y_up, const float* traj_mean,
                                        const float* traj_std, const float* pose_mean, const float* pose_std,
                                        int max_windows, int* n_windows, int* win_rec, int* win_start, float* transf,
                                        float* repr_traj, float* repr_pose, float* cano_joints, float* scene_joints,
                                        float* cano_params, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!global_orient || !transl || !betas || !body_pose || !joints || !rec_off || !cam || !floor || !traj_mean ||
      !traj_std || !pose_mean || !pose_std || !rec_off_host || !n_windows || !win_rec || !win_start || !transf ||
      !repr_traj || !repr_pose || !cano_joints || !scene_joints || !cano_params || R <= 0 || max_windows < 0 ||
      (y_up != 0 && y_up != 1))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_encode_video: bad arguments");
  std::vector<int> tab_rec, tab_start;
  if (const int rc = cut_windows(ctx, "rohm_window_encode_video", rec_off_host, R, clip_len, overlap, tab_rec, tab_start))
    return rc;
  const int W = static_cast<int>(tab_rec.size());
  *n_windows = W;
  if (W > max_windows)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_encode_video: %d windows exceed the %d the outputs hold", W,
                max_windows);
  if (W == 0) return ROHM_OK;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ROHM_CUDA(ctx, cudaMemcpyAsync(win_rec, tab_rec.data(), sizeof(int) * W, cudaMemcpyHostToDevice, st));
  ROHM_CUDA(ctx, cudaMemcpyAsync(win_start, tab_start.data(), sizeof(int) * W, cudaMemcpyHostToDevice, st));
  window_encode_kernel<kCameraIn><<<W, (clip_len + 31) / 32 * 32, 0, st>>>(
      joints, global_orient, transl, betas, body_pose, win_rec, win_start, rec_off, clip_len, traj_mean, traj_std,
      pose_mean, pose_std, transf, repr_traj, repr_pose, CamIn{cam, floor, y_up, cano_joints, scene_joints, cano_params});
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_window_keypoints(rohm_ctx* ctx, const float* keypoints25, const float* depth_mask,
                                     const unsigned char* conf64, const double* camera_mtx, const double* dist,
                                     int undistort, const int* rec_off, const int* win_rec, const int* win_start, int W,
                                     int clip_len, float* keypoints, float* mask_joint_vis, float* mask_vec_vis,
                                     void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (W < 0 || clip_len < 3 || clip_len > kMaxClip || (undistort != 0 && undistort != 1) ||
      (W > 0 && (!keypoints25 || !depth_mask || !conf64 || !rec_off || !win_rec || !win_start || !keypoints ||
                 !mask_joint_vis || !mask_vec_vis || (undistort && (!camera_mtx || !dist)))))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_keypoints: bad arguments");
  const int64_t n = static_cast<int64_t>(W) * clip_len * kJ;
  if (n == 0) return ROHM_OK;
  window_keypoints_kernel<<<static_cast<unsigned>((n + 127) / 128), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      keypoints25, depth_mask, conf64, camera_mtx, dist, undistort, rec_off, win_rec, win_start, W, clip_len, keypoints,
      mask_joint_vis, mask_vec_vis);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_window_scene_joints(rohm_ctx* ctx, const float* joints, const float* cam, const int* rec_off,
                                        const int* win_rec, const int* win_start, int W, int clip_len, float* out,
                                        void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (W < 0 || clip_len < 3 || clip_len > kMaxClip ||
      (W > 0 && (!joints || !cam || !rec_off || !win_rec || !win_start || !out)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_window_scene_joints: bad arguments");
  const int64_t n = static_cast<int64_t>(W) * clip_len * kJ;
  if (n == 0) return ROHM_OK;
  window_scene_joints_kernel<<<static_cast<unsigned>((n + 255) / 256), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      joints, cam, rec_off, win_rec, win_start, W, clip_len, out);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}
