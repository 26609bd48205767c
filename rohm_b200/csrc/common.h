// Shared host-side plumbing for the C-ABI library: context, error reporting, device buffers.
#pragma once
#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "../../include/rohm_b200.h"

struct rohm_ctx {
  int device = 0;
  int sm_count = 0;
  std::string err;
};

namespace rohm {

inline int fail(rohm_ctx* ctx, int status, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  if (ctx != nullptr) ctx->err = buf;
  return status;
}

#define ROHM_CUDA(ctx, call)                                                                                  \
  do {                                                                                                        \
    cudaError_t e__ = (call);                                                                                 \
    if (e__ != cudaSuccess)                                                                                   \
      return ::rohm::fail((ctx), ROHM_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e__), __FILE__, \
                          __LINE__);                                                                          \
  } while (0)

inline int64_t round_up(int64_t x, int64_t m) { return (x + m - 1) / m * m; }

// Makes ctx->device the calling thread's current device for the lifetime of the guard and restores the previous one
// afterwards: every entry point launches on the device its context was created for, whatever the caller's current
// device is (a process that drives several GPUs), and never changes it as a side effect.
class DeviceGuard {
 public:
  explicit DeviceGuard(const rohm_ctx* ctx) {
    if (ctx != nullptr && cudaGetDevice(&prev_) == cudaSuccess && prev_ != ctx->device) {
      restore_ = cudaSetDevice(ctx->device) == cudaSuccess;
    }
  }
  ~DeviceGuard() {
    if (restore_) cudaSetDevice(prev_);
  }
  DeviceGuard(const DeviceGuard&) = delete;
  DeviceGuard& operator=(const DeviceGuard&) = delete;

 private:
  int prev_ = -1;
  bool restore_ = false;
};

// Launch attributes of launch_chain: programmatic dependent launch, and a thread-block cluster of `cluster` CTAs along x
// (1: no cluster attribute; the grid's x dimension must be a multiple of it).
struct ChainAttrs {
  ChainAttrs(bool pdl_, unsigned cluster_ = 1) : pdl(pdl_), cluster(cluster_) {}  // implicit: a bare bool is PDL only
  bool pdl;
  unsigned cluster;
};

// Kernel launch with the programmatic-dependent-launch attribute (the kernel must call griddepcontrol.wait before it
// touches memory, which every kernel launched through here does) and optionally a cluster dimension.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_chain(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, ChainAttrs at,
                                Args... args) {
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cudaLaunchAttribute attr[2];
  unsigned na = 0;
  if (at.pdl) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  if (at.cluster > 1) {
    attr[na].id = cudaLaunchAttributeClusterDimension;
    attr[na].val.clusterDim.x = at.cluster;
    attr[na].val.clusterDim.y = 1;
    attr[na].val.clusterDim.z = 1;
    ++na;
  }
  cfg.attrs = attr;
  cfg.numAttrs = na;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

// Owns a set of cudaMalloc'ed buffers; frees them on destruction.
class DevicePool {
 public:
  ~DevicePool() {
    for (void* p : ptrs_) cudaFree(p);
  }
  // Zero-initialised fp32 buffer of n elements (nullptr on failure, error kept in last_error()).
  float* floats(int64_t n) { return static_cast<float*>(bytes(n * static_cast<int64_t>(sizeof(float)))); }
  void* bytes(int64_t n) {
    void* p = nullptr;
    if (n <= 0) n = 16;
    last_ = cudaMalloc(&p, static_cast<size_t>(n));
    if (last_ != cudaSuccess) return nullptr;
    last_ = cudaMemset(p, 0, static_cast<size_t>(n));
    if (last_ != cudaSuccess) return nullptr;
    ptrs_.push_back(p);
    total_ += n;
    return p;
  }
  cudaError_t last_error() const { return last_; }
  int64_t total_bytes() const { return total_; }

 private:
  std::vector<void*> ptrs_;
  cudaError_t last_ = cudaSuccess;
  int64_t total_ = 0;
};

// A weight matrix [N, K] repacked for the GEMM: zero-padded to [Np, Kp] and split into a hi / lo pair: TF32 values in
// fp32 containers (kind 0) or fp16 values of w * scale (kind 1, scale a power of two; see gemm.cuh GemmKind).
struct PackedWeight {
  float* hi = nullptr;
  float* lo = nullptr;
  int N = 0, K = 0, Np = 0, Kp = 0, block_n = 0;
  int kind = 0;
  float scale = 1.0f;
};

}  // namespace rohm
