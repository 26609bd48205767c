// get_repr_smplx (data_loaders/motion_representation.py:187-282) per frame: the pieces shared by the glue's trajectory
// encoder (glue.cu traj_full_repr_kernel, between rounds) and the window encoder (windows.cu rohm_window_encode, on the
// way in), so that both compute the 22 trajectory channels with the same instructions.
#pragma once
#include "kin.cuh"

namespace rohm {
namespace repr {

using namespace kin;

constexpr int kTrajFull = 22;
constexpr int kChAngle = 0, kChAngleVel = 1, kChRootPos = 2, kChRootVel = 4, kChHeight = 6, kChRot6d = 7, kChRotVel = 13,
              kChTrans = 16, kChTransVel = 19;

// scipy Rotation.from_rotvec(r).as_matrix() (rotvec -> unit quaternion -> matrix), fp32
__device__ __forceinline__ M3 rotvec_to_mat(V3 r) {
  const float a2 = dot(r, r);
  const float a = sqrtf(a2);
  float sc, qw;
  if (a <= 1e-3f) {
    sc = 0.5f - a2 / 48.0f + a2 * a2 / 3840.0f;
    qw = cosf(0.5f * a);
  } else {
    float sn;
    sincosf(0.5f * a, &sn, &qw);
    sc = sn / a;
  }
  const float x = sc * r.x, y = sc * r.y, z = sc * r.z, w = qw;
  const float x2 = x * x, y2 = y * y, z2 = z * z, w2 = w * w;
  const float xy = x * y, zw = z * w, xz = x * z, yw = y * w, yz = y * z, xw = x * w;
  M3 R;
  R.c0 = {x2 - y2 - z2 + w2, 2.0f * (xy + zw), 2.0f * (xz - yw)};
  R.c1 = {2.0f * (xy - zw), -x2 + y2 - z2 + w2, 2.0f * (yz + xw)};
  R.c2 = {2.0f * (xz + yw), 2.0f * (yz - xw), -x2 - y2 + z2 + w2};
  return R;
}

// Root heading of one frame, qbetween(forward, (0, 1, 0)) = (q0, q1, 0, q3), from the joints the reference unpacks as
// (l_hip, r_hip, sdr_r, sdr_l) = (2, 1, 17, 16): across = (joint 1 - joint 2) + (joint 17 - joint 16).  NaN when the
// across vector has no horizontal part (the frames the reference repairs).
__device__ __forceinline__ void heading_quat(V3 j1, V3 j2, V3 j17, V3 j16, float& q0, float& q1, float& q3) {
  V3 across = (j1 - j2) + (j17 - j16);
  across = (1.0f / sqrtf(dot(across, across))) * across;
  V3 fwd = {-across.y, across.x, 0.0f};  // cross((0,0,1), across)
  fwd = (1.0f / sqrtf(dot(fwd, fwd))) * fwd;
  // qbetween(fwd, (0,1,0)): v = fwd x target = (-f.z, 0, f.x), w = |f||t| + f.t
  const float vx = -fwd.z, vz = fwd.x;
  const float w = sqrtf(dot(fwd, fwd) * 1.0f) + fwd.y;
  const float n = sqrtf(w * w + vx * vx + vz * vz);
  q0 = w / n, q1 = vx / n, q3 = vz / n;
}

// qrot((w, 0, 0, z), v): rotation about the up axis by a repaired heading quaternion
__device__ __forceinline__ V3 qrot_z(float w, float z, V3 v) {
  const V3 qv = {0.0f, 0.0f, z};
  const V3 uv = cross(qv, v);
  const V3 uuv = cross(qv, uv);
  return v + 2.0f * (w * uv + uuv);
}

// Channels [0, 22) of frame t (un-normalised, REPR_LIST order): heading quaternions (w0, z0) of frame t and (w1, z1) of
// frame t + 1 after the NaN repair; root(k) and rot(k) give the root joint (V3) and the global-orientation matrix (M3) of
// frame t + k, and tr(k, c) component c of its translation.  The callers' loads are issued where these functors are called.
template <class Root, class Rot, class Tr>
__device__ __forceinline__ void traj_channels(float* o, float w0, float z0, float w1, float z1, Root root, Rot rot, Tr tr) {
  o[kChAngle] = atan2f(z0, w0);
  // q[t+1] * conj(q[t]) for rotations about z
  o[kChAngleVel] = atan2f(w0 * z1 - z0 * w1, w1 * w0 + z1 * z0);
  const V3 r0 = root(0), r1 = root(1);
  o[kChRootPos] = r0.x, o[kChRootPos + 1] = r0.y;
  {
    // qrot(q[t+1], r1 - r0), qvec = (0, 0, z1)
    const V3 v = r1 - r0;
    const V3 qv = {0.0f, 0.0f, z1};
    const V3 uv = cross(qv, v);
    const V3 uuv = cross(qv, uv);
    o[kChRootVel] = v.x + 2.0f * (w1 * uv.x + uuv.x);
    o[kChRootVel + 1] = v.y + 2.0f * (w1 * uv.y + uuv.y);
  }
  o[kChHeight] = r0.z;
  const M3 R0 = rot(0), R1 = rot(1);
  // rot6d = R[:, :2] row-major
  o[kChRot6d] = R0.c0.x, o[kChRot6d + 1] = R0.c1.x, o[kChRot6d + 2] = R0.c0.y, o[kChRot6d + 3] = R0.c1.y;
  o[kChRot6d + 4] = R0.c0.z, o[kChRot6d + 5] = R0.c1.z;
  {
    // estimate_angular_velocity_np: w_mat = dR R^T; entries (i,j) = sum_k dR[i][k] R[j][k]
    const M3 dR = {R1.c0 - R0.c0, R1.c1 - R0.c1, R1.c2 - R0.c2};
    auto rowd = [&](int i) { return i == 0 ? V3{dR.c0.x, dR.c1.x, dR.c2.x} : (i == 1 ? V3{dR.c0.y, dR.c1.y, dR.c2.y} : V3{dR.c0.z, dR.c1.z, dR.c2.z}); };
    auto rowr = [&](int i) { return i == 0 ? V3{R0.c0.x, R0.c1.x, R0.c2.x} : (i == 1 ? V3{R0.c0.y, R0.c1.y, R0.c2.y} : V3{R0.c0.z, R0.c1.z, R0.c2.z}); };
    auto wm = [&](int i, int j) { return dot(rowd(i), rowr(j)); };
    o[kChRotVel] = (-wm(1, 2) + wm(2, 1)) / 2.0f;
    o[kChRotVel + 1] = (wm(0, 2) - wm(2, 0)) / 2.0f;
    o[kChRotVel + 2] = (-wm(0, 1) + wm(1, 0)) / 2.0f;
  }
  for (int k = 0; k < 3; ++k) {
    const float a = tr(0, k), c = tr(1, k);
    o[kChTrans + k] = a;
    o[kChTransVel + k] = c - a;
  }
}

}  // namespace repr
}  // namespace rohm
