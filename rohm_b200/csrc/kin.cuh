// Device-side rotation / kinematics helpers shared by the body-model, guidance and glue kernels.  Each function names the
// reference code it restates:
//   rot6d_to_mat      data_loaders/common/quaternion.py:482-501 (rot6d_to_rotmat: Gram-Schmidt, F.normalize eps 1e-12)
//   mat_to_aa         utils/konia_transform.py:317-340, 350-444, 561-631 (rotation matrix -> quaternion -> axis-angle)
//   rodrigues         third-party smplx==0.1.28 lbs.py batch_rodrigues (eps added to the vector before the norm)
#pragma once
#include <cuda_runtime.h>

namespace rohm {
namespace kin {

struct V3 {
  float x, y, z;
};
__device__ __forceinline__ V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3 operator*(float s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
__device__ __forceinline__ float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
__device__ __forceinline__ V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
struct M3 {  // columns
  V3 c0, c1, c2;
};
__device__ __forceinline__ V3 mul(const M3& R, V3 v) { return v.x * R.c0 + v.y * R.c1 + v.z * R.c2; }
__device__ __forceinline__ V3 mulT(const M3& R, V3 v) { return {dot(R.c0, v), dot(R.c1, v), dot(R.c2, v)}; }
__device__ __forceinline__ M3 mul(const M3& A, const M3& B) { return {mul(A, B.c0), mul(A, B.c1), mul(A, B.c2)}; }

// rot6d (row-major 3x2: a1 = x[0,2,4], a2 = x[1,3,5]) -> rotation matrix with columns b1, b2, b3.
__device__ __forceinline__ M3 rot6d_to_mat(const float* x, float* n1 = nullptr, float* n2 = nullptr, float* s = nullptr) {
  const V3 a1 = {x[0], x[2], x[4]}, a2 = {x[1], x[3], x[5]};
  const float l1 = fmaxf(sqrtf(dot(a1, a1)), 1e-12f);
  const V3 b1 = (1.0f / l1) * a1;
  const float d = dot(b1, a2);
  const V3 u2 = a2 - d * b1;
  const float l2 = fmaxf(sqrtf(dot(u2, u2)), 1e-12f);
  const V3 b2 = (1.0f / l2) * u2;
  if (n1) *n1 = l1, *n2 = l2, *s = d;
  return {b1, b2, cross(b1, b2)};
}

// VJP of rot6d_to_mat: G = dL/dR (columns g1, g2, g3) -> dL/dx[6].
__device__ __forceinline__ void rot6d_backward(const float* x, const M3& G, float* gx) {
  float l1, l2, s;
  const M3 R = rot6d_to_mat(x, &l1, &l2, &s);
  const V3 a2 = {x[1], x[3], x[5]};
  V3 gb1 = G.c0 + cross(R.c1, G.c2);   // b3 = b1 x b2
  V3 gb2 = G.c1 + cross(G.c2, R.c0);
  const V3 gu2 = (1.0f / l2) * (gb2 - dot(gb2, R.c1) * R.c1);
  const V3 ga2 = gu2 - dot(R.c0, gu2) * R.c0;
  gb1 = gb1 - s * gu2 - dot(gu2, R.c0) * a2;
  const V3 ga1 = (1.0f / l1) * (gb1 - dot(gb1, R.c0) * R.c0);
  gx[0] = ga1.x, gx[2] = ga1.y, gx[4] = ga1.z;
  gx[1] = ga2.x, gx[3] = ga2.y, gx[5] = ga2.z;
}

// rotation matrix -> axis-angle through the reference's quaternion route (kornia WXYZ, eps = 1e-6 everywhere)
__device__ __forceinline__ float safe_div(float n, float d) { return n / (fabsf(d) < 1e-6f ? d + 1e-6f : d); }
__device__ __forceinline__ float safe_atan2(float y, float x) {
  if (fabsf(y) < 1e-6f && fabsf(x) < 1e-6f) y += 1e-6f;
  return atan2f(y, x);
}
__device__ __forceinline__ V3 mat_to_aa(const M3& R) {
  const float m00 = R.c0.x, m10 = R.c0.y, m20 = R.c0.z, m01 = R.c1.x, m11 = R.c1.y, m21 = R.c1.z, m02 = R.c2.x,
              m12 = R.c2.y, m22 = R.c2.z;
  const float trace = m00 + m11 + m22;
  float qw, qx, qy, qz;
  if (trace > 0.0f) {
    const float sq = sqrtf(fmaxf(trace + 1.0f, 1e-6f)) * 2.0f;
    qw = 0.25f * sq, qx = safe_div(m21 - m12, sq), qy = safe_div(m02 - m20, sq), qz = safe_div(m10 - m01, sq);
  } else if (m00 > m11 && m00 > m22) {
    const float sq = sqrtf(fmaxf(1.0f + m00 - m11 - m22, 1e-6f)) * 2.0f;
    qw = safe_div(m21 - m12, sq), qx = 0.25f * sq, qy = safe_div(m01 + m10, sq), qz = safe_div(m02 + m20, sq);
  } else if (m11 > m22) {
    const float sq = sqrtf(fmaxf(1.0f + m11 - m00 - m22, 1e-6f)) * 2.0f;
    qw = safe_div(m02 - m20, sq), qx = safe_div(m01 + m10, sq), qy = 0.25f * sq, qz = safe_div(m12 + m21, sq);
  } else {
    const float sq = sqrtf(fmaxf(1.0f + m22 - m00 - m11, 1e-6f)) * 2.0f;
    qw = safe_div(m10 - m01, sq), qx = safe_div(m02 + m20, sq), qy = safe_div(m12 + m21, sq), qz = 0.25f * sq;
  }
  const float s2 = qx * qx + qy * qy + qz * qz;
  const float sn = sqrtf(fmaxf(s2, 1e-6f));
  const float two_theta = 2.0f * (qw < 0.0f ? safe_atan2(-sn, -qw) : safe_atan2(sn, qw));
  const float k = s2 > 0.0f ? safe_div(two_theta, sn) : 2.0f;
  return {qx * k, qy * k, qz * k};
}
// smplx batch_rodrigues: the 1e-8 is added to the VECTOR before the norm
__device__ __forceinline__ M3 rodrigues(V3 r) {
  const V3 e = {r.x + 1e-8f, r.y + 1e-8f, r.z + 1e-8f};
  const float ang = sqrtf(dot(e, e));
  const V3 k = (1.0f / ang) * r;
  float sn, cs;
  sincosf(ang, &sn, &cs);
  const float c1 = 1.0f - cs;
  // I + sin K + (1 - cos) K^2
  M3 R;
  R.c0 = {1.0f + c1 * (-k.z * k.z - k.y * k.y), sn * k.z + c1 * k.x * k.y, -sn * k.y + c1 * k.x * k.z};
  R.c1 = {-sn * k.z + c1 * k.x * k.y, 1.0f + c1 * (-k.z * k.z - k.x * k.x), sn * k.x + c1 * k.y * k.z};
  R.c2 = {sn * k.y + c1 * k.x * k.z, -sn * k.x + c1 * k.y * k.z, 1.0f + c1 * (-k.y * k.y - k.x * k.x)};
  return R;
}


// Packed frame f of a batch of clips with different lengths -> its clip b: clip_off (int[B + 1], the exclusive prefix sum of
// the clips' lengths) has clip_off[b] <= f < clip_off[b + 1].  A binary search per thread (log2 B reads of a table every
// thread of the launch shares, L1-resident) instead of a frame -> clip map, which would cost a scan launch and a 4-byte read
// per frame for tables of a handful of clips.
__device__ __forceinline__ int clip_of_frame(const int* __restrict__ clip_off, int B, int f) {
  int lo = 0, hi = B;
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (clip_off[mid] <= f) lo = mid;
    else hi = mid;
  }
  return lo;
}

}  // namespace kin
}  // namespace rohm
