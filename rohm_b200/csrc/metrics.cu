// Evaluation metrics of the reconstruction, one CTA per clip or window (SURVEY.md 8g):
//
//   rohm_eval_amass   eval_amass_full.py:71-147: per (frame, joint) global MPJPE, contact-label matches, foot skating of
//                     the clean and the reconstructed joints over the clean clip's lowest z, acceleration error, toe
//                     penetration; per clip float64 sums and int64 counts
//   rohm_eval_video   eval_prox_egobody.py:172-272: the reconstruction mapped back to the scene by the inverse of each
//                     window's transf_matrix, foot skating over the recording's floor, ||acc||, toe penetration and, with
//                     ground truth (EgoBody), acceleration error, global / root-relative MPJPE and the visibility-weighted
//                     MPJPE sums; per window float64 sums and int64 counts
//   rohm_eval_reduce  the per-item sums of one of the above, per group (recording) in the given item order, then over
//                     the groups in order
//
// The per-frame values are the reference's float32 numpy values: every product, sum and square root is rounded on its
// own (no contraction into FMA) in numpy's order of operations -- a norm over 3 channels is sqrt((s0 + s1) + s2), a mean
// over 22 joints numpy's 8-accumulator pairwise sum divided by 22 -- except the scene transform, whose float32 matrix
// product is the FMA chain of the FMA BLAS kernels numpy calls (DESIGN §4.16).  The sums are float64 in a fixed order
// (strided per thread, then a fixed tree), so every result is the same in any batch and on every run.
#include <cmath>
#include <cstdint>

#include "common.h"

namespace rohm {
namespace {

constexpr int kJ = 22;
constexpr int kThreads = 128;
constexpr float kFps = 30.0f, kFps2 = 900.0f;
constexpr float kVel = 0.1f, kHeightAnkle = 0.15f, kHeightToe = 0.1f, kPene = -0.05f;
// left ankle, left toe, right ankle, right toe (the contact channels' order)
__device__ __forceinline__ int foot(int f) { return f == 0 ? 7 : f == 1 ? 10 : f == 2 ? 8 : 11; }

// per-clip outputs of the AMASS pass
constexpr int kAmassSums = 5;    // mpjpe, mpjpe visible, mpjpe occluded, accel error, pene dist
constexpr int kAmassCounts = 11; // mpjpe n, vis n, occ n, contact matches, contact n, skate gt, skate rec, skate n,
                                 // accel n, pene freq, pene n
// per-window outputs of the video pass
constexpr int kVideoSums = 10;   // acc, acc error, gmpjpe, mpjpe, vis num, vis den, occ num, occ den, pene freq, pene dist
constexpr int kVideoCounts = 1;  // skating frames

__device__ __forceinline__ float fnan() { return __int_as_float(0x7fffffff); }
// np.min: NaN propagates (fminf would drop it)
__device__ __forceinline__ float nanmin(float a, float b) { return (a != a || b != b) ? fnan() : fminf(a, b); }
__device__ __forceinline__ float sq(float a) { return __fmul_rn(a, a); }
// np.linalg.norm over 3 float32 channels: sqrt((s0 + s1) + s2)
__device__ __forceinline__ float norm3(float a, float b, float c) {
  return __fsqrt_rn(__fadd_rn(__fadd_rn(sq(a), sq(b)), sq(c)));
}
__device__ __forceinline__ float norm2(float a, float b) { return __fsqrt_rn(__fadd_rn(sq(a), sq(b))); }
// (x[t+2] - 2 x[t+1] + x[t]) * fps^2, evaluated left to right as numpy does
__device__ __forceinline__ float accel(float x0, float x1, float x2) {
  return __fmul_rn(__fadd_rn(__fsub_rn(x2, __fmul_rn(2.0f, x1)), x0), kFps2);
}
// np.mean over 22 float32 values: numpy's pairwise sum (8 accumulators, then the tail in order), divided by 22
__device__ __forceinline__ float mean22(const float* v) {
  float r[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) r[j] = __fadd_rn(v[j], v[8 + j]);
  float s = __fadd_rn(__fadd_rn(__fadd_rn(r[0], r[1]), __fadd_rn(r[2], r[3])),
                      __fadd_rn(__fadd_rn(r[4], r[5]), __fadd_rn(r[6], r[7])));
#pragma unroll
  for (int j = 16; j < kJ; ++j) s = __fadd_rn(s, v[j]);
  return __fdiv_rn(s, 22.0f);
}

// Block sum of n float64 / int64 values per thread in a fixed order: warp tree, then the warps in order.
template <int N, typename T>
__device__ void block_sum(T (&v)[N], T* out) {
  __shared__ T part[kThreads / 32][N];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < N; ++k) {
    T x = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if (lane == 0) part[warp][k] = x;
  }
  __syncthreads();
  if (threadIdx.x < N) {
    T s = part[0][threadIdx.x];
    for (int w = 1; w < kThreads / 32; ++w) s += part[w][threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

// The skating rule for one frame pair of the 4 foot joints: horizontal speed (a, b) and height h per joint.
__device__ __forceinline__ bool skates(const float (&v)[4], const float (&h)[4]) {
  const bool left = v[0] > kVel && v[1] > kVel && h[0] < kHeightAnkle && h[1] < kHeightToe;
  const bool right = v[2] > kVel && v[3] > kVel && h[2] < kHeightAnkle && h[3] < kHeightToe;
  return left && right;
}

__global__ void __launch_bounds__(kThreads) eval_amass_kernel(
    const float* __restrict__ gt, const float* __restrict__ rec, const float* __restrict__ repr_clean,
    const float* __restrict__ repr_rec, int repr_width, const int64_t* __restrict__ frame_off, unsigned occ_joints,
    int occ_lo, int occ_hi, float* __restrict__ h0_out, float* __restrict__ mpjpe, float* __restrict__ accerr,
    unsigned char* __restrict__ skate_gt, unsigned char* __restrict__ skate_rec, unsigned char* __restrict__ contact,
    unsigned char* __restrict__ pene_freq, float* __restrict__ pene_dist, double* __restrict__ sums,
    int64_t* __restrict__ counts) {
  const int b = blockIdx.x;
  const int64_t r0 = frame_off[b];
  const int T = static_cast<int>(frame_off[b + 1] - r0);
  const float* G = gt + r0 * kJ * 3;
  const float* P = rec + r0 * kJ * 3;

  // pass 1: h0 = np.min of the clean clip's z over every frame and joint
  __shared__ float s_h0[kThreads / 32];
  float m = INFINITY;
  for (int i = threadIdx.x; i < T * kJ; i += kThreads) m = nanmin(m, G[i * 3 + 2]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = nanmin(m, __shfl_down_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) s_h0[threadIdx.x >> 5] = m;
  __syncthreads();
  float h0 = s_h0[0];
  for (int w = 1; w < kThreads / 32; ++w) h0 = nanmin(h0, s_h0[w]);
  if (threadIdx.x == 0) h0_out[b] = h0;

  // pass 2: per-frame values and this thread's float64 sums / int64 counts
  const int lo = min(occ_lo, T), hi = max(lo, min(occ_hi, T));
  double s[kAmassSums] = {0.0, 0.0, 0.0, 0.0, 0.0};
  int64_t c[kAmassCounts] = {};
  for (int t = threadIdx.x; t < T; t += kThreads) {
    const int64_t row = r0 + t;
    const float* g = G + t * kJ * 3;
    const float* p = P + t * kJ * 3;
    const bool occ_frame = t >= lo && t < hi;
    for (int j = 0; j < kJ; ++j) {
      const float e = norm3(__fsub_rn(g[3 * j], p[3 * j]), __fsub_rn(g[3 * j + 1], p[3 * j + 1]),
                            __fsub_rn(g[3 * j + 2], p[3 * j + 2]));
      mpjpe[row * kJ + j] = e;
      s[0] += e;
      if (occ_frame && ((occ_joints >> j) & 1u)) s[2] += e; else s[1] += e;
    }
    // contact labels: the reconstruction's thresholded at 0.5 (NaN stays NaN), compared with the raw clean label
    for (int k = 0; k < 4; ++k) {
      const float lr = repr_rec[row * repr_width + repr_width - 4 + k];
      const float lc = repr_clean[row * repr_width + repr_width - 4 + k];
      const float bin = lr > 0.5f ? 1.0f : (lr <= 0.5f ? 0.0f : lr);
      const bool eq = lc == bin;
      contact[row * 4 + k] = eq;
      c[3] += eq;
    }
    for (int i = 0; i < 2; ++i) {
      float d = __fsub_rn(p[3 * (10 + i) + 2], h0);
      const bool f = d < kPene;
      pene_freq[row * 2 + i] = f;
      c[9] += f;
      if (d >= 0.0f) d = 0.0f;
      pene_dist[row * 2 + i] = d;
      s[4] += d;
    }
    if (t + 1 < T) {
      bool sk[2];
      for (int which = 0; which < 2; ++which) {
        const float* x = which ? p : g;
        float v[4], h[4];
        for (int f = 0; f < 4; ++f) {
          const float* a = x + 3 * foot(f);
          const float* a1 = a + kJ * 3;
          v[f] = __fmul_rn(norm2(__fsub_rn(a1[0], a[0]), __fsub_rn(a1[1], a[1])), kFps);
          h[f] = __fsub_rn(a[2], h0);
        }
        sk[which] = skates(v, h);
      }
      skate_gt[row] = sk[0];
      skate_rec[row] = sk[1];
      c[5] += sk[0];
      c[6] += sk[1];
    } else {
      skate_gt[row] = 0;
      skate_rec[row] = 0;
    }
    if (t + 2 < T) {
      for (int j = 0; j < kJ; ++j) {
        float d[3];
        for (int k = 0; k < 3; ++k) {
          const int i = 3 * j + k;
          d[k] = __fsub_rn(accel(p[i], p[i + kJ * 3], p[i + 2 * kJ * 3]), accel(g[i], g[i + kJ * 3], g[i + 2 * kJ * 3]));
        }
        const float e = norm3(d[0], d[1], d[2]);
        accerr[row * kJ + j] = e;
        s[3] += e;
      }
    } else {
      for (int j = 0; j < kJ; ++j) accerr[row * kJ + j] = 0.0f;
    }
  }
  block_sum(s, sums + static_cast<int64_t>(b) * kAmassSums);
  if (threadIdx.x == 0) {
    const int n_occ_j = __popc(occ_joints & ((1u << kJ) - 1u));
    c[0] = static_cast<int64_t>(T) * kJ;
    c[2] = static_cast<int64_t>(hi - lo) * n_occ_j;
    c[1] = c[0] - c[2];
    c[4] = static_cast<int64_t>(T) * 4;
    c[7] = T > 1 ? T - 1 : 0;
    c[8] = static_cast<int64_t>(T > 2 ? T - 2 : 0) * kJ;
    c[10] = static_cast<int64_t>(T) * 2;
  }
  // fixed-index counts are set by thread 0 only; the data counts (3, 5, 6, 9) are summed over the block
  block_sum(c, counts + static_cast<int64_t>(b) * kAmassCounts);
}

// numpy's float32 inv: LU in float64, rounded to float32 (Gauss-Jordan with partial pivoting here)
__device__ void inverse4_f64(const float* a, float* out) {
  double m[4][8];
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) {
      m[i][j] = a[i * 4 + j];
      m[i][4 + j] = i == j ? 1.0 : 0.0;
    }
  for (int c = 0; c < 4; ++c) {
    int piv = c;
    for (int i = c + 1; i < 4; ++i)
      if (fabs(m[i][c]) > fabs(m[piv][c])) piv = i;
    if (piv != c)
      for (int j = 0; j < 8; ++j) {
        const double t = m[c][j];
        m[c][j] = m[piv][j];
        m[piv][j] = t;
      }
    const double inv = 1.0 / m[c][c];
    for (int j = 0; j < 8; ++j) m[c][j] *= inv;
    for (int i = 0; i < 4; ++i)
      if (i != c) {
        const double f = m[i][c];
        for (int j = 0; j < 8; ++j) m[i][j] -= f * m[c][j];
      }
  }
  for (int i = 0; i < 4; ++i)
    for (int j = 0; j < 4; ++j) out[i * 4 + j] = static_cast<float>(m[i][4 + j]);
}

// points_coord_trans(x, M): x.dot(M[:3,:3].T) + M[:3,3] with numpy's float32 BLAS product (FMA chain over k)
__device__ __forceinline__ float scene_coord(const float* M, const float* x, int i) {
  const float* r = M + 4 * i;
  return __fadd_rn(__fmaf_rn(x[2], r[2], __fmaf_rn(x[1], r[1], __fmul_rn(x[0], r[0]))), r[3]);
}

__device__ __forceinline__ void scene_joint(const float* M, const float* x, float* y) {
  y[0] = scene_coord(M, x, 0);
  y[1] = scene_coord(M, x, 1);
  y[2] = scene_coord(M, x, 2);
}

__global__ void __launch_bounds__(kThreads) eval_video_kernel(
    const float* __restrict__ rec, int T, const float* __restrict__ transf, const float* __restrict__ gt, int gt_frames,
    const float* __restrict__ mask_vis, int mask_frames, const int* __restrict__ win_rec,
    const float* __restrict__ floor, int y_up, unsigned char* __restrict__ skate, float* __restrict__ acc,
    float* __restrict__ accerr, float* __restrict__ gmpjpe, float* __restrict__ mpjpe, float* __restrict__ pene_freq,
    float* __restrict__ pene_dist, double* __restrict__ sums, int64_t* __restrict__ counts) {
  const int w = blockIdx.x;
  __shared__ float M[16];
  if (threadIdx.x == 0) inverse4_f64(transf + static_cast<int64_t>(w) * 16, M);
  __syncthreads();
  const float fl = floor[win_rec[w]];
  const int up = y_up ? 1 : 2, hx = 0, hy = y_up ? 2 : 1;
  const float* P = rec + static_cast<int64_t>(w) * T * kJ * 3;
  const float* G = gt ? gt + static_cast<int64_t>(w) * gt_frames * kJ * 3 : nullptr;
  const float* mv = mask_vis ? mask_vis + static_cast<int64_t>(w) * mask_frames * kJ : nullptr;
  const int64_t wrow = static_cast<int64_t>(w) * T;
  double s[kVideoSums] = {};
  int64_t c[kVideoCounts] = {};
  for (int t = threadIdx.x; t < T; t += kThreads) {
    const int64_t row = wrow + t;
    const float* x = P + static_cast<int64_t>(t) * kJ * 3;  // canonical joints of frame t; t + 1 is x + kJ * 3
    float q[3];
    // toe penetration: per frame, the mean over the two toes of d < -0.05 and of min(d, 0)
    float d[2];
    int n_pene = 0;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      d[i] = __fsub_rn(scene_coord(M, x + 3 * (10 + i), up), fl);
      n_pene += d[i] < kPene;
      if (d[i] >= 0.0f) d[i] = 0.0f;
    }
    const float pf = 0.5f * n_pene, pd = __fmul_rn(__fadd_rn(d[0], d[1]), 0.5f);
    pene_freq[row] = pf;
    pene_dist[row] = pd;
    s[8] += pf;
    s[9] += pd;
    if (t + 1 < T) {
      float v[4], h[4];
#pragma unroll
      for (int f = 0; f < 4; ++f) {
        float q1[3];
        scene_joint(M, x + 3 * foot(f), q);
        scene_joint(M, x + kJ * 3 + 3 * foot(f), q1);
        v[f] = __fmul_rn(norm2(__fsub_rn(q1[hx], q[hx]), __fsub_rn(q1[hy], q[hy])), kFps);
        h[f] = __fsub_rn(q[up], fl);
      }
      const bool sk = skates(v, h);
      skate[wrow - w + t] = sk;  // [W, T-1]
      c[0] += sk;
    }
    if (t + 2 < T) {
      float an[kJ], ae[kJ];
#pragma unroll
      for (int j = 0; j < kJ; ++j) {
        float q1[3], q2[3], a[3], e[3];
        scene_joint(M, x + 3 * j, q);
        scene_joint(M, x + kJ * 3 + 3 * j, q1);
        scene_joint(M, x + 2 * kJ * 3 + 3 * j, q2);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          a[k] = accel(q[k], q1[k], q2[k]);
          if (G) {
            const float* g = G + (static_cast<int64_t>(t) * kJ + j) * 3 + k;
            e[k] = __fsub_rn(a[k], accel(g[0], g[kJ * 3], g[2 * kJ * 3]));
          } else {
            e[k] = 0.0f;
          }
        }
        an[j] = norm3(a[0], a[1], a[2]);
        ae[j] = norm3(e[0], e[1], e[2]);
      }
      const int64_t arow = static_cast<int64_t>(w) * (T - 2) + t;  // [W, T-2]
      const float am = mean22(an);
      acc[arow] = am;
      s[0] += am;
      if (G) {
        const float em = mean22(ae);
        accerr[arow] = em;
        s[1] += em;
      }
    }
    if (G) {
      const float* g = G + static_cast<int64_t>(t) * kJ * 3;
      float q0[3];
      scene_joint(M, x, q0);
      for (int j = 0; j < kJ; ++j) {
        const float* gj = g + 3 * j;
        scene_joint(M, x + 3 * j, q);
        const float eg = norm3(__fsub_rn(gj[0], q[0]), __fsub_rn(gj[1], q[1]), __fsub_rn(gj[2], q[2]));
        // root-relative: (G_j - G_0) - (P_j - P_0)
        float dl[3];
#pragma unroll
        for (int k = 0; k < 3; ++k) dl[k] = __fsub_rn(__fsub_rn(gj[k], g[k]), __fsub_rn(q[k], q0[k]));
        const float el = norm3(dl[0], dl[1], dl[2]);
        gmpjpe[row * kJ + j] = eg;
        mpjpe[row * kJ + j] = el;
        s[2] += eg;
        s[3] += el;
        if (mv) {
          const float m = mv[static_cast<int64_t>(t) * kJ + j], om = __fsub_rn(1.0f, m);
          s[4] += __fmul_rn(el, m);
          s[5] += m;
          s[6] += __fmul_rn(el, om);
          s[7] += om;
        }
      }
    }
  }
  block_sum(s, sums + static_cast<int64_t>(w) * kVideoSums);
  block_sum(c, counts + static_cast<int64_t>(w) * kVideoCounts);
}

// One thread per column: group g sums items order[group_off[g] .. group_off[g+1]) in that order; row G is the sum of
// the G group rows in order.
__global__ void eval_reduce_kernel(const double* __restrict__ sums, int ks, const int64_t* __restrict__ counts, int kc,
                                   const int* __restrict__ order, const int* __restrict__ group_off, int n_groups,
                                   double* __restrict__ out_sums, int64_t* __restrict__ out_counts) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= ks + kc) return;
  if (k < ks) {
    double all = 0.0;
    for (int g = 0; g < n_groups; ++g) {
      double a = 0.0;
      for (int i = group_off[g]; i < group_off[g + 1]; ++i) a += sums[static_cast<int64_t>(order[i]) * ks + k];
      out_sums[static_cast<int64_t>(g) * ks + k] = a;
      all += a;
    }
    out_sums[static_cast<int64_t>(n_groups) * ks + k] = all;
  } else {
    const int q = k - ks;
    int64_t all = 0;
    for (int g = 0; g < n_groups; ++g) {
      int64_t a = 0;
      for (int i = group_off[g]; i < group_off[g + 1]; ++i) a += counts[static_cast<int64_t>(order[i]) * kc + q];
      out_counts[static_cast<int64_t>(g) * kc + q] = a;
      all += a;
    }
    out_counts[static_cast<int64_t>(n_groups) * kc + q] = all;
  }
}

}  // namespace
}  // namespace rohm

using namespace rohm;

extern "C" int rohm_eval_amass(rohm_ctx* ctx, const float* gt, const float* rec, const float* repr_clean,
                               const float* repr_rec, int repr_width, const int64_t* frame_off, int B,
                               unsigned occ_joints, int occ_lo, int occ_hi, float* h0, float* mpjpe, float* accerr,
                               unsigned char* skate_gt, unsigned char* skate_rec, unsigned char* contact,
                               unsigned char* pene_freq, float* pene_dist, double* sums, int64_t* counts,
                               void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (B < 0 || repr_width < 4 || occ_lo < 0 || occ_hi < occ_lo ||
      (B > 0 && (!gt || !rec || !repr_clean || !repr_rec || !frame_off || !h0 || !mpjpe || !accerr || !skate_gt ||
                 !skate_rec || !contact || !pene_freq || !pene_dist || !sums || !counts)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_eval_amass: bad arguments");
  if (B == 0) return ROHM_OK;
  eval_amass_kernel<<<B, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      gt, rec, repr_clean, repr_rec, repr_width, frame_off, occ_joints, occ_lo, occ_hi, h0, mpjpe, accerr, skate_gt,
      skate_rec, contact, pene_freq, pene_dist, sums, counts);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_eval_video(rohm_ctx* ctx, const float* rec, int T, const float* transf, const float* gt,
                               int gt_frames, const float* mask_vis, int mask_frames, const int* win_rec,
                               const float* floor, int W, int y_up, unsigned char* skate, float* acc, float* accerr,
                               float* gmpjpe, float* mpjpe, float* pene_freq, float* pene_dist, double* sums,
                               int64_t* counts, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  const bool with_gt = gt != nullptr;
  if (W < 0 || T < 3 || (with_gt && (gt_frames < T || !accerr || !gmpjpe || !mpjpe)) ||
      (mask_vis && (!with_gt || mask_frames < T)) ||
      (W > 0 && (!rec || !transf || !win_rec || !floor || !skate || !acc || !pene_freq || !pene_dist || !sums ||
                 !counts)))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_eval_video: bad arguments");
  if (W == 0) return ROHM_OK;
  eval_video_kernel<<<W, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      rec, T, transf, gt, gt_frames, mask_vis, mask_frames, win_rec, floor, y_up, skate, acc, accerr, gmpjpe, mpjpe,
      pene_freq, pene_dist, sums, counts);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_eval_reduce(rohm_ctx* ctx, const double* sums, int ks, const int64_t* counts, int kc,
                                const int* order, const int* group_off, int n_groups, double* out_sums,
                                int64_t* out_counts, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (ks < 0 || kc < 0 || ks + kc == 0 || n_groups < 0 || !group_off || !out_sums || !out_counts ||
      (ks > 0 && !sums) || (kc > 0 && !counts))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_eval_reduce: bad arguments");
  const int n = ks + kc;
  eval_reduce_kernel<<<(n + 31) / 32, 32, 0, static_cast<cudaStream_t>(stream)>>>(
      sums, ks, counts, kc, order, group_off, n_groups, out_sums, out_counts);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}
