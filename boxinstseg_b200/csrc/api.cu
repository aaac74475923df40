// Library identity, error reporting and small host utilities of the C ABI.
#include <cstring>

#include "common.cuh"

namespace bxs {
namespace {
thread_local char g_err[256] = "";
}  // namespace

void set_last_error(cudaError_t e) {
  std::strncpy(g_err, cudaGetErrorString(e), sizeof(g_err) - 1);
  g_err[sizeof(g_err) - 1] = 0;
}

int sm_count() {
  static thread_local int cached_dev = -1, cached = 0;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (dev != cached_dev) {
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) != cudaSuccess) return 132;
    cached = p.multiProcessorCount;
    cached_dev = dev;
  }
  return cached;
}
}  // namespace bxs

extern "C" int bxs_version(void) { return 100; }   // 0.1.0
extern "C" const char* bxs_last_error(void) { return bxs::g_err; }

extern "C" int bxs_device_sm_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess || n == 0) return BXS_ERR_NO_DEVICE;
  return bxs::sm_count();
}
