// Shared device/host helpers for the boxseg_b200 kernels (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/boxseg_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "boxseg_b200 is written for sm_90a (H100) only"
#endif

namespace bxs {

constexpr int kWarp = 32;
constexpr unsigned kFull = 0xffffffffu;

void set_last_error(cudaError_t e);

inline int check_launch() {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_last_error(e);
    return BXS_ERR_LAUNCH;
  }
  return BXS_OK;
}

inline cudaStream_t as_stream(bxs_stream_t s) { return reinterpret_cast<cudaStream_t>(s); }

inline int64_t ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

int sm_count();

// ---------------------------------------------------------------------------------------
// numerics
// ---------------------------------------------------------------------------------------
// (log sigmoid(x), log sigmoid(-x)) sharing one softplus term: L = log1p(exp(-|x|)),
// log s(x) = min(x,0) - L, log s(-x) = min(-x,0) - L.  No cancellation anywhere.
template <typename T>
__device__ __forceinline__ void log_sigmoid_pair(T x, T& lp, T& lm) {
  T ax = x < T(0) ? -x : x;
  T L = log1p(exp(-ax));
  lp = (x < T(0) ? x : T(0)) - L;
  lm = (x < T(0) ? T(0) : -x) - L;
}
template <>
__device__ __forceinline__ void log_sigmoid_pair<float>(float x, float& lp, float& lm) {
  float L = log1pf(expf(-fabsf(x)));
  lp = fminf(x, 0.f) - L;
  lm = fminf(-x, 0.f) - L;
}

// -log( s(a)s(b) + s(-a)s(-b) ) in log space; `has_b == false` models the reference's padded
// neighbour (both class log-probabilities replaced by 0).  pairwise.cu:38-50.
template <typename T>
__device__ __forceinline__ T pair_nlog_logspace(T a, T b, bool has_b) {
  T lpa, lma, lpb = T(0), lmb = T(0);
  log_sigmoid_pair(a, lpa, lma);
  if (has_b) log_sigmoid_pair(b, lpb, lmb);
  T e1 = lpa + lpb, e0 = lma + lmb;
  T mx = e1 > e0 ? e1 : e0;
  T df = e1 > e0 ? e1 - e0 : e0 - e1;
  return -(mx + log1p(exp(-df)));
}

// d/da of the above given the forward value `pl`.  pairwise.cu:52-66.
template <typename T>
__device__ __forceinline__ T pair_nlog_grad_a_logspace(T a, T b, bool has_b, T pl) {
  T lpa, lma, lpb = T(0), lmb = T(0);
  log_sigmoid_pair(a, lpa, lma);
  if (has_b) log_sigmoid_pair(b, lpb, lmb);
  return -(exp(lpb) - exp(lmb)) * exp(lpa + lma + pl);
}

__device__ __forceinline__ float rcp_approx(float v) {      // MUFU.RCP, ~1 ulp
  float o;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(o) : "f"(v));
  return o;
}

// sigmoid pair (s, n) = (sigmoid(x), sigmoid(-x)), both accurate to a few ulp relative (no 1 - s cancellation).
__device__ __forceinline__ void sigmoid_pair(float x, float& s, float& n) {
  float e = __expf(-fabsf(x));
  float big = rcp_approx(1.f + e);
  float small = e * big;
  s = x >= 0.f ? big : small;
  n = x >= 0.f ? small : big;
}

__device__ __forceinline__ float sigmoid_fast(float x) { return __frcp_rn(1.f + __expf(-x)); }

// ---------------------------------------------------------------------------------------
// warp / block reductions (fixed order -> run-to-run deterministic)
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}
__device__ __forceinline__ int warp_sum(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
  return v;
}

// block-wide sum; result valid in thread 0.  `scratch` must hold blockDim.x/32 elements.
template <typename T>
__device__ __forceinline__ T block_sum(T v, T* scratch) {
  v = warp_sum(v);
  int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) scratch[wid] = v;
  __syncthreads();
  T r = T(0);
  if (wid == 0) {
    int nw = (blockDim.x + 31) >> 5;
    r = lane < nw ? scratch[lane] : T(0);
    r = warp_sum(r);
  }
  return r;
}

}  // namespace bxs
