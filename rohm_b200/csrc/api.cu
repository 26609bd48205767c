// C-ABI: context management.  The per-subsystem entry points live next to their kernels
// (sampler.cu, posenet.cu, trajnet.cu, body.cu).
#include <new>

#include "common.h"

extern "C" int rohm_version(void) { return 108; }

extern "C" int rohm_ctx_create(int device, rohm_ctx** out) {
  if (out == nullptr) return ROHM_ERR_INVALID;
  *out = nullptr;
  int count = 0;
  if (cudaGetDeviceCount(&count) != cudaSuccess || count <= 0 || device < 0 || device >= count) return ROHM_ERR_NO_DEVICE;
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) return ROHM_ERR_CUDA;
  if (prop.major != 9 || prop.minor != 0) return ROHM_ERR_NO_DEVICE;  // kernels are sm_90a only
  rohm_ctx* ctx = new (std::nothrow) rohm_ctx();
  if (ctx == nullptr) return ROHM_ERR_INVALID;
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  {
    // initialise the device's primary context without leaving the caller's current device changed
    rohm::DeviceGuard guard(ctx);
    if (cudaFree(nullptr) != cudaSuccess) {
      delete ctx;
      return ROHM_ERR_CUDA;
    }
  }
  *out = ctx;
  return ROHM_OK;
}

extern "C" void rohm_ctx_destroy(rohm_ctx* ctx) { delete ctx; }

extern "C" const char* rohm_last_error(const rohm_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
