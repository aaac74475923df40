// Library identity, error reporting and small host utilities of the C ABI.
#include <cstring>

#include "common.cuh"

namespace bxs {
namespace {
thread_local char g_err[256] = "";
__global__ void fill_kernel(uint4* p, int64_t n, unsigned v) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    p[i] = make_uint4(v, v, v, v);
}
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

extern "C" int bxs_flush_l2(void* scratch, int64_t bytes, bxs_stream_t stream) {
  if (!scratch || bytes < 16) return BXS_ERR_INVALID_ARG;
  static unsigned tick = 0;
  bxs::fill_kernel<<<bxs::sm_count() * 8, 256, 0, bxs::as_stream(stream)>>>((uint4*)scratch, bytes / 16, ++tick);
  return bxs::check_launch();
}
