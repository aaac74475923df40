// Shared device/host helpers for the boxseg_b200 kernels (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>
#include <map>
#include <utility>

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
// launch configuration
// ---------------------------------------------------------------------------------------
namespace {    // one memo per source file, which launches only its own kernels; nothing exported from the library
struct KernelState {
  size_t smem_allowed = 0;             // dynamic shared memory opted in to
  int occ_threads = -1, occ = 0;       // last occupancy query and its answer
  size_t occ_smem = 0;
};
// Keyed by the kernel's address, not its type: instantiations with the same signature share a type.  Per thread, so
// no lock; another thread repeats an opt-in or a query, which is harmless.
inline KernelState& kernel_state(const void* kern) {
  static thread_local std::map<std::pair<const void*, int>, KernelState> states;
  int dev = 0;
  cudaGetDevice(&dev);
  return states[{kern, dev}];
}

// Lets `kern` use up to `smem` bytes of dynamic shared memory on the current device (a launch above 48 KB needs it).
// Remembered per (kernel, device): a later call asking for no more skips the driver.  Returns BXS_OK, or
// BXS_ERR_LAUNCH with bxs_last_error() set.
inline int opt_in_smem(const void* kern, size_t smem) {
  KernelState& s = kernel_state(kern);
  if (smem <= s.smem_allowed) return BXS_OK;
  const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_last_error(e);
    return BXS_ERR_LAUNCH;
  }
  s.smem_allowed = smem;
  return BXS_OK;
}

// CTAs of `kern` resident per SM at `threads` threads and `smem` bytes of dynamic shared memory on the current device,
// remembered per (kernel, device) for the last (threads, smem) asked.  0 when none fit or the query fails (then with
// bxs_last_error() set).
inline int max_active_ctas(const void* kern, int threads, size_t smem) {
  KernelState& s = kernel_state(kern);
  if (threads != s.occ_threads || smem != s.occ_smem) {
    int occ = 0;
    const cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem);
    if (e != cudaSuccess) {
      cudaGetLastError();
      set_last_error(e);
      return 0;
    }
    s.occ_threads = threads;
    s.occ_smem = smem;
    s.occ = occ;
  }
  return s.occ;
}

template <typename... A>
inline int opt_in_smem(void (*kern)(A...), size_t smem) {
  return opt_in_smem(reinterpret_cast<const void*>(kern), smem);
}
template <typename... A>
inline int max_active_ctas(void (*kern)(A...), int threads, size_t smem) {
  return max_active_ctas(reinterpret_cast<const void*>(kern), threads, smem);
}
}  // namespace

// 1-D grid of a grid-stride kernel: ceil(total / block) CTAs, at least 1, at most `ctas_per_sm` per SM
inline int grid_for(int64_t total, int block, int ctas_per_sm = 8) {
  const int64_t g = ceil_div(total, block), cap = (int64_t)sm_count() * ctas_per_sm;
  return (int)std::max<int64_t>(1, std::min(g, cap));
}

// ---------------------------------------------------------------------------------------
// workspaces
// ---------------------------------------------------------------------------------------
inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

// Hands out consecutive pieces of a workspace, each starting 256-byte aligned.  With a null base it only measures:
// `off` after the last piece is the size the workspace needs.
struct Carver {
  char* base;
  size_t off = 0;
  explicit Carver(void* b) : base(static_cast<char*>(b)) {}
  char* take(size_t bytes) {
    char* r = base + off;
    off = align_up(off + bytes);
    return r;
  }
};

// ---------------------------------------------------------------------------------------
// PTX: shared-memory addresses, mbarriers, 1-D bulk copy (TMA engine) and their fences
// ---------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred P1;\n\t"
      "LAB_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%0], %1;\n\t"
      "@P1 bra DONE;\n\t"
      "bra LAB_WAIT;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// makes initialised mbarriers visible to the other threads and to the async proxy
__device__ __forceinline__ void fence_mbarrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// orders this thread's generic-proxy shared-memory accesses before later async-proxy (bulk copy) ones
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// `bytes` contiguous bytes global -> shared, completing on `bar` (no tensor map needed)
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}

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
