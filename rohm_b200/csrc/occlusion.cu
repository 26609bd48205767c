// The PROX joint occlusion masks (utils/get_occlusion_mask.py:55-144, DESIGN §4.17): a depth map of the scene mesh per
// camera, and per frame the depth of the posed body mesh at each of its 25 projected joints.  Only the pixel-centre rays
// are ever tested, so neither kernel rasterises in the GL sense: both call ray_depth, one float64 ray-triangle test.
//
//   rohm_scene_depth       the scene mesh rendered alone (pyrender OffscreenRenderer depth, one camera)
//   rohm_joint_occlusion   cv2.projectPoints of joints 0..24, the body mesh's depth at those pixels, and the mask rule
//
// Geometry is float64 with every product, sum and quotient a separately rounded _rn operation in the order written
// here, so the compiler cannot contract any of it into fused multiply-adds and the numpy restatement
// (oracle/occlusion_oracle.py) computes the same bits.
#include <algorithm>
#include <cfloat>
#include <climits>
#include <cmath>
#include <cstdint>

#include "common.h"

namespace rohm {
namespace {

constexpr int kJoints = 25;                     // joints[0:25] of the reference script
constexpr unsigned long long kNoHit = ~0ull;    // above every positive double's bit pattern
constexpr int64_t kLargeBox = 1024;             // screen boxes of more pixels go to the one-CTA-per-triangle pass
constexpr int kThreads = 256;

__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ double quo(double a, double b) { return __ddiv_rn(a, b); }

struct D3 {
  double x, y, z;
};

// The render camera: pinhole intrinsics, clip range and viewport.
struct Cam {
  double fx, fy, cx, cy, znear, zfar;
  int width, height;
};

// The ray through the centre of pixel (x, y): d = ((x + 0.5 - cx) / fx, (y + 0.5 - cy) / fy, 1), so its hit parameter t
// is the camera-frame z of the hit (pyrender's linear depth).
__device__ __forceinline__ double ray_dx(int x, const Cam& k) { return quo(sub(add(x, 0.5), k.cx), k.fx); }
__device__ __forceinline__ double ray_dy(int y, const Cam& k) { return quo(sub(add(y, 0.5), k.cy), k.fy); }

// Möller-Trumbore from the camera centre, for both kernels.  e1 = v1 - v0, e2 = v2 - v0, p = d x e2, det = e1.p; a
// triangle is front-facing for the ray iff det > 0 (GL's counter-clockwise front face seen through diag(1,-1,-1)), and
// det <= 0 or NaN rejects it.  s = -v0, u' = s.p, q = s x e1, v' = d.q, t' = e2.q; the hit is inclusive: u' >= 0,
// v' >= 0, u' + v' <= det (edges and vertices count).  z = t' / det, accepted in [znear, zfar].  Dots are
// ((a.x b.x + a.y b.y) + a.z b.z); products with the ray's unit z are exact and left out.
__device__ __forceinline__ bool ray_depth(double dx, double dy, D3 v0, D3 v1, D3 v2, const Cam& k, double& z) {
  const D3 e1{sub(v1.x, v0.x), sub(v1.y, v0.y), sub(v1.z, v0.z)};
  const D3 e2{sub(v2.x, v0.x), sub(v2.y, v0.y), sub(v2.z, v0.z)};
  const D3 p{sub(mul(dy, e2.z), e2.y), sub(e2.x, mul(dx, e2.z)), sub(mul(dx, e2.y), mul(dy, e2.x))};
  const double det = add(add(mul(e1.x, p.x), mul(e1.y, p.y)), mul(e1.z, p.z));
  if (!(det > 0.0)) return false;
  const D3 s{-v0.x, -v0.y, -v0.z};
  const double u = add(add(mul(s.x, p.x), mul(s.y, p.y)), mul(s.z, p.z));
  if (!(u >= 0.0)) return false;
  const D3 q{sub(mul(s.y, e1.z), mul(s.z, e1.y)), sub(mul(s.z, e1.x), mul(s.x, e1.z)), sub(mul(s.x, e1.y), mul(s.y, e1.x))};
  const double v = add(add(mul(dx, q.x), mul(dy, q.y)), q.z);
  if (!(v >= 0.0) || !(add(u, v) <= det)) return false;
  const double t = quo(add(add(mul(e2.x, q.x), mul(e2.y, q.y)), mul(e2.z, q.z)), det);
  if (!(t >= k.znear && t <= k.zfar)) return false;
  z = t;
  return true;
}

// The triangle's conservative screen box in pixel indices [x0, x1] x [y0, y1], clipped to the viewport: the vertices
// with z >= znear and the znear crossings of its edges (p + (q - p) s, s = (znear - p.z) / (q.z - p.z)) projected as
// u = fx (x / z) + cx, then floor(umin - 0.5) - 1 .. ceil(umax - 0.5) + 1 (pixel x's centre is u = x + 0.5, plus one
// pixel of padding).  False for a triangle with a non-finite coordinate, wholly nearer than znear, wholly beyond zfar,
// or off screen.  Any pixel whose centre ray ray_depth accepts lies inside it.
__device__ __forceinline__ bool screen_box(D3 a, D3 b, D3 c, const Cam& k, int& x0, int& y0, int& x1, int& y1) {
  if (!(isfinite(a.x) && isfinite(a.y) && isfinite(a.z) && isfinite(b.x) && isfinite(b.y) && isfinite(b.z) &&
        isfinite(c.x) && isfinite(c.y) && isfinite(c.z)))
    return false;
  if (a.z < k.znear && b.z < k.znear && c.z < k.znear) return false;
  if (a.z > k.zfar && b.z > k.zfar && c.z > k.zfar) return false;
  double umin = INFINITY, umax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
  auto take = [&](double x, double y, double z) {
    const double u = add(mul(k.fx, quo(x, z)), k.cx), v = add(mul(k.fy, quo(y, z)), k.cy);
    umin = fmin(umin, u), umax = fmax(umax, u), vmin = fmin(vmin, v), vmax = fmax(vmax, v);
  };
  auto edge = [&](D3 p, D3 q) {
    if ((p.z < k.znear) == (q.z < k.znear)) return;
    const double s = quo(sub(k.znear, p.z), sub(q.z, p.z));
    take(add(p.x, mul(sub(q.x, p.x), s)), add(p.y, mul(sub(q.y, p.y), s)), k.znear);
  };
  if (a.z >= k.znear) take(a.x, a.y, a.z);
  if (b.z >= k.znear) take(b.x, b.y, b.z);
  if (c.z >= k.znear) take(c.x, c.y, c.z);
  edge(a, b), edge(b, c), edge(c, a);
  const double lx = fmax(sub(floor(sub(umin, 0.5)), 1.0), 0.0);
  const double hx = fmin(add(ceil(sub(umax, 0.5)), 1.0), static_cast<double>(k.width - 1));
  const double ly = fmax(sub(floor(sub(vmin, 0.5)), 1.0), 0.0);
  const double hy = fmin(add(ceil(sub(vmax, 0.5)), 1.0), static_cast<double>(k.height - 1));
  if (!(lx <= hx && ly <= hy)) return false;
  x0 = static_cast<int>(lx), x1 = static_cast<int>(hx), y0 = static_cast<int>(ly), y1 = static_cast<int>(hy);
  return true;
}

__device__ __forceinline__ unsigned long long depth_key(double z) {
  return static_cast<unsigned long long>(__double_as_longlong(z));  // z > 0: the bit patterns order as the values
}
__device__ __forceinline__ float key_depth(unsigned long long key) {
  return key == kNoHit ? 0.0f : __double2float_rn(__longlong_as_double(static_cast<long long>(key)));
}

// world -> camera [R | t], rows of 4
struct Rt {
  double m[12];
};

// One thread per scene vertex: x_c = ((R00 X + R01 Y) + R02 Z) + t0, ... in float64.
__global__ void scene_to_camera_kernel(const float* __restrict__ v, int64_t n, const Rt rt, double* __restrict__ out) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double X = v[i * 3], Y = v[i * 3 + 1], Z = v[i * 3 + 2];
  for (int r = 0; r < 3; ++r) {
    const double* m = rt.m + r * 4;
    out[i * 3 + r] = add(add(add(mul(m[0], X), mul(m[1], Y)), mul(m[2], Z)), m[3]);
  }
}

__device__ __forceinline__ D3 cam_vertex(const double* cv, int i) {
  return D3{cv[static_cast<int64_t>(i) * 3], cv[static_cast<int64_t>(i) * 3 + 1], cv[static_cast<int64_t>(i) * 3 + 2]};
}

// Every pixel centre of the box run through ray_depth, the nearest hit kept by 64-bit atomicMin (order-independent).
__device__ __forceinline__ void raster_box(D3 a, D3 b, D3 c, const Cam& k, int x0, int y0, int x1, int y1, int64_t first,
                                           int64_t step, unsigned long long* keys) {
  const int64_t w = x1 - x0 + 1, n = w * (y1 - y0 + 1);
  for (int64_t p = first; p < n; p += step) {
    const int x = x0 + static_cast<int>(p % w), y = y0 + static_cast<int>(p / w);
    double z;
    if (ray_depth(ray_dx(x, k), ray_dy(y, k), a, b, c, k, z))
      atomicMin(keys + static_cast<int64_t>(y) * k.width + x, depth_key(z));
  }
}

// One thread per triangle: boxes of up to kLargeBox pixels are rastered here, larger ones listed for the next launch.
__global__ void __launch_bounds__(kThreads) scene_raster_kernel(const double* __restrict__ cv, const int* __restrict__ faces,
                                                                int64_t F, const Cam k, unsigned long long* keys,
                                                                int* __restrict__ large, int* __restrict__ n_large) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= F) return;
  const D3 a = cam_vertex(cv, faces[i * 3]), b = cam_vertex(cv, faces[i * 3 + 1]), c = cam_vertex(cv, faces[i * 3 + 2]);
  int x0, y0, x1, y1;
  if (!screen_box(a, b, c, k, x0, y0, x1, y1)) return;
  if (static_cast<int64_t>(x1 - x0 + 1) * (y1 - y0 + 1) > kLargeBox) {
    large[atomicAdd(n_large, 1)] = static_cast<int>(i);
    return;
  }
  raster_box(a, b, c, k, x0, y0, x1, y1, 0, 1, keys);
}

// The listed large triangles, one CTA at a time per triangle, its threads striding over the box.
__global__ void __launch_bounds__(kThreads) scene_raster_large_kernel(const double* __restrict__ cv,
                                                                      const int* __restrict__ faces,
                                                                      const int* __restrict__ large,
                                                                      const int* __restrict__ n_large, const Cam k,
                                                                      unsigned long long* keys) {
  const int n = *n_large;
  for (int j = blockIdx.x; j < n; j += gridDim.x) {
    const int64_t i = large[j];
    const D3 a = cam_vertex(cv, faces[i * 3]), b = cam_vertex(cv, faces[i * 3 + 1]), c = cam_vertex(cv, faces[i * 3 + 2]);
    int x0, y0, x1, y1;
    if (screen_box(a, b, c, k, x0, y0, x1, y1)) raster_box(a, b, c, k, x0, y0, x1, y1, threadIdx.x, blockDim.x, keys);
  }
}

__global__ void scene_depth_finish_kernel(const unsigned long long* __restrict__ keys, int64_t n, float* __restrict__ depth) {
  const int64_t i = static_cast<int64_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) depth[i] = key_depth(keys[i]);
}

// cv2.projectPoints(P, rvec = 0, tvec = 0, K, k) for one point, in OpenCV's order of operations (calib3d
// cvProjectPoints2Internal, 4.13; the identity rotation's zero products kept, so a non-finite coordinate makes both
// outputs NaN as there): z' = z ? 1/z : 1; x' = x z', y' = y z'; r2 = x'^2 + y'^2, r4 = r2^2, r6 = r4 r2; radial
// (1 + k0 r2 + k1 r4 + k4 r6) / (1 + k5 r2 + k6 r4 + k7 r6), tangential and thin-prism terms; the identity tilt map;
// u = xd fx + cx, v = yd fy + cy, rounded to float32 as cv2 returns them for float32 object points.  k holds 14
// coefficients, zero-padded.
__device__ __forceinline__ void project_point(float X32, float Y32, float Z32, const double* K, const double* k, float& u,
                                              float& v) {
  const double X = X32, Y = Y32, Z = Z32;
  double x = add(add(add(mul(1.0, X), mul(0.0, Y)), mul(0.0, Z)), 0.0);
  double y = add(add(add(mul(0.0, X), mul(1.0, Y)), mul(0.0, Z)), 0.0);
  double z = add(add(add(mul(0.0, X), mul(0.0, Y)), mul(1.0, Z)), 0.0);
  z = z != 0.0 ? quo(1.0, z) : 1.0;
  x = mul(x, z), y = mul(y, z);
  const double r2 = add(mul(x, x), mul(y, y)), r4 = mul(r2, r2), r6 = mul(r4, r2);
  const double a1 = mul(mul(2.0, x), y), a2 = add(r2, mul(mul(2.0, x), x)), a3 = add(r2, mul(mul(2.0, y), y));
  const double cdist = add(add(add(1.0, mul(k[0], r2)), mul(k[1], r4)), mul(k[4], r6));
  const double icdist2 = quo(1.0, add(add(add(1.0, mul(k[5], r2)), mul(k[6], r4)), mul(k[7], r6)));
  const double xd0 = add(add(add(add(mul(mul(x, cdist), icdist2), mul(k[2], a1)), mul(k[3], a2)), mul(k[8], r2)),
                         mul(k[9], r4));
  const double yd0 = add(add(add(add(mul(mul(y, cdist), icdist2), mul(k[2], a3)), mul(k[3], a1)), mul(k[10], r2)),
                         mul(k[11], r4));
  const double t0 = add(add(mul(1.0, xd0), mul(0.0, yd0)), mul(0.0, 1.0));
  const double t1 = add(add(mul(0.0, xd0), mul(1.0, yd0)), mul(0.0, 1.0));
  const double t2 = add(add(mul(0.0, xd0), mul(0.0, yd0)), mul(1.0, 1.0));
  const double ip = t2 != 0.0 ? quo(1.0, t2) : 1.0;
  const double xd = mul(ip, t0), yd = mul(ip, t1);
  u = __double2float_rn(add(mul(xd, K[0]), K[2]));
  v = __double2float_rn(add(mul(yd, K[4]), K[5]));
}

// numpy's astype(int) of a float32 coordinate as an int32 pixel: the truncation toward zero where it is finite and
// below 2^31 in magnitude, INT_MIN (x86's indefinite integer) otherwise.
__device__ __forceinline__ int trunc_pixel(float c) {
  return isfinite(c) && fabsf(c) < 2147483648.0f ? static_cast<int>(c) : INT_MIN;
}

// One CTA per frame.  Threads 0..24 project the frame's joints with its recording's camera; a joint lies on screen iff
// its truncated pixel is in [0, W) x [0, H), i.e. -1 < u < W and -1 < v < H (NaN and +-inf fail).  The threads then
// stride over the faces: each gathers its triangle from the frame's (pitched) vertex row, skips it unless an on-screen
// joint's pixel lies in its screen box, and keeps the nearest ray_depth hit per joint by shared 64-bit atomicMin.
// Finally mask = 0 iff the joint is on screen, its scene depth is not 0 and float64(body - scene) > 0.1, the float32
// difference compared in float64 as numpy 1.22 compares a float32 scalar with a Python float.
__global__ void __launch_bounds__(kThreads) joint_occlusion_kernel(
    const float* __restrict__ joints, int joints_per_frame, const float* __restrict__ verts, int64_t vertex_pitch,
    const int* __restrict__ faces, int F, const int* __restrict__ frame_rec, const double* __restrict__ camera_mtx,
    const double* __restrict__ dist, const float* __restrict__ maps, const int* __restrict__ map_of_rec, const Cam k,
    float* __restrict__ mask, int* __restrict__ pixel, float* __restrict__ depth_body, float* __restrict__ depth_scene) {
  __shared__ double rdx[kJoints], rdy[kJoints];
  __shared__ int px[kJoints], py[kJoints];
  __shared__ unsigned long long key[kJoints];
  __shared__ unsigned on_screen;
  const int64_t f = blockIdx.x;
  const int t = threadIdx.x;
  const int rec = frame_rec[f];
  if (t < 32) {
    bool in = false;
    if (t < kJoints) {
      const float* P = joints + (f * joints_per_frame + t) * 3;
      float u, v;
      project_point(P[0], P[1], P[2], camera_mtx + static_cast<int64_t>(rec) * 9, dist + static_cast<int64_t>(rec) * 14,
                    u, v);
      in = u > -1.0f && u < static_cast<float>(k.width) && v > -1.0f && v < static_cast<float>(k.height);
      const int x = trunc_pixel(u), y = trunc_pixel(v);
      px[t] = x, py[t] = y, key[t] = kNoHit;
      if (in) rdx[t] = ray_dx(x, k), rdy[t] = ray_dy(y, k);
      if (pixel != nullptr) pixel[(f * kJoints + t) * 2] = x, pixel[(f * kJoints + t) * 2 + 1] = y;
    }
    const unsigned ballot = __ballot_sync(0xffffffffu, in);
    if (t == 0) on_screen = ballot;
  }
  __syncthreads();
  const unsigned live = on_screen;
  if (live != 0) {
    const float* V = verts + f * vertex_pitch;
    for (int i = t; i < F; i += blockDim.x) {
      auto vert = [&](int j) {
        const float* p = V + static_cast<int64_t>(faces[i * 3 + j]) * 3;
        return D3{p[0], p[1], p[2]};
      };
      const D3 a = vert(0), b = vert(1), c = vert(2);
      int x0, y0, x1, y1;
      if (!screen_box(a, b, c, k, x0, y0, x1, y1)) continue;
      for (unsigned m = live; m != 0; m &= m - 1) {
        const int j = __ffs(m) - 1;
        if (px[j] < x0 || px[j] > x1 || py[j] < y0 || py[j] > y1) continue;
        double z;
        if (ray_depth(rdx[j], rdy[j], a, b, c, k, z)) atomicMin(key + j, depth_key(z));
      }
    }
  }
  __syncthreads();
  if (t < kJoints) {
    const bool in = (live >> t) & 1u;
    const float db = in ? key_depth(key[t]) : 0.0f;
    const float ds = in ? maps[(static_cast<int64_t>(map_of_rec[rec]) * k.height + py[t]) * k.width + px[t]] : 0.0f;
    const bool occluded = in && ds != 0.0f && static_cast<double>(__fsub_rn(db, ds)) > 0.1;
    mask[f * kJoints + t] = occluded ? 0.0f : 1.0f;
    if (depth_body != nullptr) depth_body[f * kJoints + t] = db;
    if (depth_scene != nullptr) depth_scene[f * kJoints + t] = ds;
  }
}

bool camera_ok(double fx, double fy, double cx, double cy, int width, int height, double znear, double zfar) {
  return std::isfinite(fx) && std::isfinite(fy) && std::isfinite(cx) && std::isfinite(cy) && fx != 0.0 && fy != 0.0 &&
         width > 0 && height > 0 && std::isfinite(znear) && std::isfinite(zfar) && znear > 0.0 && zfar >= znear;
}

// the scene pass's workspace: camera-frame vertices, the depth keys, the large-triangle list and its count
struct SceneWorkspace {
  double* cam_verts;
  unsigned long long* keys;
  int* large;
  int* n_large;
  int64_t bytes;
};

SceneWorkspace scene_workspace(void* base, int64_t n_verts, int64_t n_faces, int width, int height) {
  char* p = static_cast<char*>(base);
  SceneWorkspace w{};
  int64_t off = 0;
  auto take = [&](int64_t n) {
    char* q = p == nullptr ? nullptr : p + off;
    off += round_up(n, 256);
    return q;
  };
  w.cam_verts = reinterpret_cast<double*>(take(n_verts * 3 * static_cast<int64_t>(sizeof(double))));
  w.keys = reinterpret_cast<unsigned long long*>(take(static_cast<int64_t>(width) * height * 8));
  w.large = reinterpret_cast<int*>(take(n_faces * static_cast<int64_t>(sizeof(int))));
  w.n_large = reinterpret_cast<int*>(take(sizeof(int)));
  w.bytes = off;
  return w;
}

}  // namespace
}  // namespace rohm

using namespace rohm;

extern "C" int64_t rohm_scene_depth_workspace_bytes(int64_t n_verts, int64_t n_faces, int width, int height) {
  if (n_verts < 0 || n_faces < 0 || width <= 0 || height <= 0) return -1;
  return scene_workspace(nullptr, n_verts, n_faces, width, height).bytes;
}

extern "C" int rohm_scene_depth(rohm_ctx* ctx, const float* vertices, int64_t n_verts, const int* faces, int64_t n_faces,
                                const double* world2cam_host, double fx, double fy, double cx, double cy, int width,
                                int height, double znear, double zfar, void* workspace, int64_t workspace_bytes,
                                float* depth, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (!world2cam_host || !depth || !workspace || n_verts < 0 || n_faces < 0 || n_faces > INT_MAX ||
      (n_verts > 0 && !vertices) || (n_faces > 0 && !faces) || !camera_ok(fx, fy, cx, cy, width, height, znear, zfar))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_scene_depth: bad arguments");
  const SceneWorkspace ws = scene_workspace(workspace, n_verts, n_faces, width, height);
  if (workspace_bytes < ws.bytes)
    return fail(ctx, ROHM_ERR_INVALID, "rohm_scene_depth: the workspace holds %lld bytes, %lld are needed",
                static_cast<long long>(workspace_bytes), static_cast<long long>(ws.bytes));
  Rt rt;
  for (int i = 0; i < 12; ++i) rt.m[i] = world2cam_host[i];
  const Cam k{fx, fy, cx, cy, znear, zfar, width, height};
  const int64_t pixels = static_cast<int64_t>(width) * height;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  ROHM_CUDA(ctx, cudaMemsetAsync(ws.keys, 0xff, sizeof(unsigned long long) * pixels, st));
  ROHM_CUDA(ctx, cudaMemsetAsync(ws.n_large, 0, sizeof(int), st));
  if (n_verts > 0) {
    scene_to_camera_kernel<<<static_cast<unsigned>((n_verts + 255) / 256), 256, 0, st>>>(vertices, n_verts, rt,
                                                                                          ws.cam_verts);
    ROHM_CUDA(ctx, cudaGetLastError());
  }
  if (n_faces > 0) {
    scene_raster_kernel<<<static_cast<unsigned>((n_faces + kThreads - 1) / kThreads), kThreads, 0, st>>>(
        ws.cam_verts, faces, n_faces, k, ws.keys, ws.large, ws.n_large);
    ROHM_CUDA(ctx, cudaGetLastError());
    const int64_t ctas = std::min<int64_t>(n_faces, 8LL * (ctx->sm_count > 0 ? ctx->sm_count : 132));
    scene_raster_large_kernel<<<static_cast<unsigned>(ctas), kThreads, 0, st>>>(ws.cam_verts, faces, ws.large,
                                                                                 ws.n_large, k, ws.keys);
    ROHM_CUDA(ctx, cudaGetLastError());
  }
  scene_depth_finish_kernel<<<static_cast<unsigned>((pixels + 255) / 256), 256, 0, st>>>(ws.keys, pixels, depth);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}

extern "C" int rohm_joint_occlusion(rohm_ctx* ctx, const float* joints, int joints_per_frame, const float* vertices,
                                    int64_t vertex_pitch, const int* faces, int n_faces, const int* frame_rec, int N,
                                    const double* camera_mtx, const double* dist, const float* depth_maps,
                                    const int* map_of_rec, double fx, double fy, double cx, double cy, int width,
                                    int height, double znear, double zfar, float* mask, int* pixel, float* depth_body,
                                    float* depth_scene, void* stream) {
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  rohm::DeviceGuard device_guard__(ctx);
  if (N < 0 || n_faces < 0 || joints_per_frame < kJoints || vertex_pitch < 0 ||
      !camera_ok(fx, fy, cx, cy, width, height, znear, zfar) ||
      (N > 0 && (!joints || !frame_rec || !camera_mtx || !dist || !depth_maps || !map_of_rec || !mask ||
                 (n_faces > 0 && (!vertices || !faces)))))
    return fail(ctx, ROHM_ERR_INVALID, "rohm_joint_occlusion: bad arguments");
  if (N == 0) return ROHM_OK;
  joint_occlusion_kernel<<<N, kThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      joints, joints_per_frame, vertices, vertex_pitch, faces, n_faces, frame_rec, camera_mtx, dist, depth_maps,
      map_of_rec, Cam{fx, fy, cx, cy, znear, zfar, width, height}, mask, pixel, depth_body, depth_scene);
  ROHM_CUDA(ctx, cudaGetLastError());
  return ROHM_OK;
}
