// Momentum (EMA) update of a teacher's state from a student's, the loop of SingleStageWSInsTeacherDetector.momentum_update
// (mmdet/models/detectors/single_stage_ts.py:118-131) in one launch: t <- fl(fl(s * a) + fl(t * b)) for every element of
// every (teacher, student) region of a table, with a = 1 - m and b = m.
//
// The table travels by value in the kernel parameters (no host-to-device copy, so a call can be captured in a CUDA graph):
// up to EMA_MAX entries per launch.  Each entry is cut into chunks of EMA_CHUNK_BYTES of its own elements; CTA c finds its
// entry by a binary search of the chunk prefix, so a CTA's chunk has one dtype and the dtype switch is uniform.  A chunk
// whose two regions are 16-byte aligned streams 16-byte vectors, four per thread in flight; any other chunk takes the
// scalar path.  Every element is read and written by exactly one thread: no atomics, and a student region may alias its
// own teacher region element for element.
//
// Roundings are those of torch's `cur * (1. - m) + self * m` followed by load_state_dict's copy_: float32 in float32 with
// the Python scalars cast to float; float16 / bfloat16 with each product and the sum computed in float and rounded to the
// dtype; float64 in double; integer and bool entries promoted to float32 (round to nearest), combined in float32 and
// converted back as torch converts (toward zero; uint8 through int64; bool as != 0).  No fused multiply-add anywhere.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include <vector>

#include "common.cuh"

namespace bxs {
namespace {

constexpr int EMA_NT = 256;                       // threads per CTA
constexpr int EMA_UNROLL = 4;                     // 16-byte vectors of each region in flight per thread
constexpr int64_t EMA_CHUNK_BYTES = 64 * 1024;    // teacher bytes per CTA (the last chunk of an entry may be shorter)
constexpr int EMA_MAX = 1024;                     // table entries per launch

struct EmaTable {                                 // by value in the kernel parameters
  void* t[EMA_MAX];
  const void* s[EMA_MAX];
  int64_t n[EMA_MAX];
  int32_t chunk0[EMA_MAX + 1];                    // first chunk of each entry; chunk0[count] = the launch's chunks
  uint8_t dtype[EMA_MAX];
  int count;
  double a, b;
};
static_assert(sizeof(EmaTable) <= 32764, "the table must fit the 32 KB kernel-parameter limit");

__host__ __device__ int elem_bytes(int dtype) {
  switch (dtype) {
    case BXS_EMA_F32: case BXS_EMA_I32: return 4;
    case BXS_EMA_F16: case BXS_EMA_BF16: case BXS_EMA_I16: return 2;
    case BXS_EMA_F64: case BXS_EMA_I64: return 8;
    case BXS_EMA_I8: case BXS_EMA_U8: case BXS_EMA_BOOL: return 1;
    default: return 0;
  }
}

__device__ __forceinline__ float ema_f32(float s, float t, float a, float b) {
  return __fadd_rn(__fmul_rn(s, a), __fmul_rn(t, b));
}

// One element of each dtype: the student's value, the teacher's value, the scalars -> the teacher's new value.
template <typename T> struct Ema;
template <> struct Ema<float> {
  __device__ static float f(float s, float t, double a, double b) { return ema_f32(s, t, (float)a, (float)b); }
};
template <> struct Ema<double> {
  __device__ static double f(double s, double t, double a, double b) { return __dadd_rn(__dmul_rn(s, a), __dmul_rn(t, b)); }
};
template <> struct Ema<__half> {
  __device__ static __half f(__half s, __half t, double a, double b) {
    const __half p = __float2half_rn(__fmul_rn(__half2float(s), (float)a));
    const __half q = __float2half_rn(__fmul_rn(__half2float(t), (float)b));
    return __float2half_rn(__fadd_rn(__half2float(p), __half2float(q)));
  }
};
template <> struct Ema<__nv_bfloat16> {
  __device__ static __nv_bfloat16 f(__nv_bfloat16 s, __nv_bfloat16 t, double a, double b) {
    const __nv_bfloat16 p = __float2bfloat16_rn(__fmul_rn(__bfloat162float(s), (float)a));
    const __nv_bfloat16 q = __float2bfloat16_rn(__fmul_rn(__bfloat162float(t), (float)b));
    return __float2bfloat16_rn(__fadd_rn(__bfloat162float(p), __bfloat162float(q)));
  }
};
template <> struct Ema<int64_t> {
  __device__ static int64_t f(int64_t s, int64_t t, double a, double b) {
    return __float2ll_rz(ema_f32(__ll2float_rn(s), __ll2float_rn(t), (float)a, (float)b));
  }
};
template <> struct Ema<int32_t> {
  __device__ static int32_t f(int32_t s, int32_t t, double a, double b) {
    return __float2int_rz(ema_f32(__int2float_rn(s), __int2float_rn(t), (float)a, (float)b));
  }
};
template <> struct Ema<int16_t> {
  __device__ static int16_t f(int16_t s, int16_t t, double a, double b) {
    return static_cast<int16_t>(ema_f32((float)s, (float)t, (float)a, (float)b));
  }
};
template <> struct Ema<int8_t> {
  __device__ static int8_t f(int8_t s, int8_t t, double a, double b) {
    return static_cast<int8_t>(ema_f32((float)s, (float)t, (float)a, (float)b));
  }
};
template <> struct Ema<uint8_t> {
  __device__ static uint8_t f(uint8_t s, uint8_t t, double a, double b) {
    return static_cast<uint8_t>(static_cast<int64_t>(ema_f32((float)s, (float)t, (float)a, (float)b)));
  }
};
struct EmaBool {};                                // bool entries: bytes that are 0 or 1
template <> struct Ema<EmaBool> {
  __device__ static uint8_t f(uint8_t s, uint8_t t, double a, double b) {
    return ema_f32(s ? 1.f : 0.f, t ? 1.f : 0.f, (float)a, (float)b) != 0.f;
  }
};

template <typename T> struct Storage { using type = T; };
template <> struct Storage<EmaBool> { using type = uint8_t; };

// Elements [begin, end) of one entry; begin is a multiple of the chunk length, so a 16-byte aligned region stays aligned.
// Not inlined: the ten dtypes' bodies inlined into one kernel need 173 registers, each alone fits in 64.
template <typename T>
__device__ __noinline__ void ema_chunk(void* tp, const void* sp, int64_t begin, int64_t end, double a, double b) {
  using S = typename Storage<T>::type;
  constexpr int V = 16 / sizeof(S);
  S* t = static_cast<S*>(tp);
  const S* s = static_cast<const S*>(sp);
  if (((reinterpret_cast<uintptr_t>(t) | reinterpret_cast<uintptr_t>(s)) & 15) == 0) {
    uint4* tv = reinterpret_cast<uint4*>(t + begin);
    const uint4* sv = reinterpret_cast<const uint4*>(s + begin);
    const int64_t nv = (end - begin) / V;
    for (int64_t i0 = threadIdx.x; i0 < nv; i0 += (int64_t)EMA_UNROLL * EMA_NT) {
      uint4 x[EMA_UNROLL], y[EMA_UNROLL];
#pragma unroll
      for (int u = 0; u < EMA_UNROLL; ++u) {
        const int64_t i = i0 + (int64_t)u * EMA_NT;
        if (i < nv) {
          x[u] = sv[i];
          y[u] = tv[i];
        }
      }
#pragma unroll
      for (int u = 0; u < EMA_UNROLL; ++u) {
        const int64_t i = i0 + (int64_t)u * EMA_NT;
        if (i < nv) {
          const S* xs = reinterpret_cast<const S*>(&x[u]);
          S* ys = reinterpret_cast<S*>(&y[u]);
#pragma unroll
          for (int k = 0; k < V; ++k) ys[k] = Ema<T>::f(xs[k], ys[k], a, b);
          tv[i] = y[u];
        }
      }
    }
    begin += nv * V;
  }
  for (int64_t i = begin + threadIdx.x; i < end; i += EMA_NT) t[i] = Ema<T>::f(s[i], t[i], a, b);
}

__global__ void __launch_bounds__(EMA_NT) ema_kernel(const __grid_constant__ EmaTable tab) {
  const int c = (int)blockIdx.x;
  int lo = 0, hi = tab.count;                     // the last entry whose first chunk is <= c (it owns c: chunks > 0)
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (tab.chunk0[mid] <= c) lo = mid; else hi = mid;
  }
  const int dt = tab.dtype[lo];
  const int64_t len = EMA_CHUNK_BYTES / elem_bytes(dt);
  const int64_t begin = (int64_t)(c - tab.chunk0[lo]) * len;
  const int64_t end = min(tab.n[lo], begin + len);
  void* t = tab.t[lo];
  const void* s = tab.s[lo];
  switch (dt) {
    case BXS_EMA_F32: ema_chunk<float>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_F16: ema_chunk<__half>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_BF16: ema_chunk<__nv_bfloat16>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_F64: ema_chunk<double>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_I64: ema_chunk<int64_t>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_I32: ema_chunk<int32_t>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_I16: ema_chunk<int16_t>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_I8: ema_chunk<int8_t>(t, s, begin, end, tab.a, tab.b); break;
    case BXS_EMA_U8: ema_chunk<uint8_t>(t, s, begin, end, tab.a, tab.b); break;
    default: ema_chunk<EmaBool>(t, s, begin, end, tab.a, tab.b); break;
  }
}

struct Span {
  uintptr_t lo, hi;                               // [lo, hi) in bytes
  int64_t k;                                      // table entry
};

// BXS_OK when no two teacher regions overlap and every student region either misses all teacher regions or is exactly
// its own teacher region.
int check_overlaps(void* const* teacher, const void* const* student, const int64_t* count, const int32_t* dtype, int64_t n) {
  std::vector<Span> ts;
  ts.reserve((size_t)n);
  for (int64_t k = 0; k < n; ++k) {
    if (count[k] == 0) continue;
    const uintptr_t lo = reinterpret_cast<uintptr_t>(teacher[k]);
    ts.push_back({lo, lo + (uintptr_t)count[k] * (uintptr_t)elem_bytes(dtype[k]), k});
  }
  std::sort(ts.begin(), ts.end(), [](const Span& x, const Span& y) { return x.lo < y.lo; });
  for (size_t i = 1; i < ts.size(); ++i)
    if (ts[i].lo < ts[i - 1].hi) return BXS_ERR_INVALID_ARG;
  for (int64_t k = 0; k < n; ++k) {
    if (count[k] == 0) continue;
    const uintptr_t lo = reinterpret_cast<uintptr_t>(student[k]);
    const uintptr_t hi = lo + (uintptr_t)count[k] * (uintptr_t)elem_bytes(dtype[k]);
    // teacher regions are disjoint and sorted: the ones that can overlap [lo, hi) start before hi, and only the last of
    // those that start at or before lo can reach into it from the left
    auto it = std::upper_bound(ts.begin(), ts.end(), lo, [](uintptr_t v, const Span& x) { return v < x.lo; });
    if (it != ts.begin()) --it;
    for (; it != ts.end() && it->lo < hi; ++it) {
      if (it->hi <= lo) continue;
      if (it->k != k || it->lo != lo) return BXS_ERR_INVALID_ARG;
    }
  }
  return BXS_OK;
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_momentum_update(void* const* teacher_host, const void* const* student_host, const int64_t* count_host,
                                   const int32_t* dtype_host, int64_t n, const double* ab_host, bxs_stream_t stream) {
  if (n < 0 || !ab_host) return BXS_ERR_INVALID_ARG;
  if (n == 0) return BXS_OK;
  if (!teacher_host || !student_host || !count_host || !dtype_host) return BXS_ERR_INVALID_ARG;
  for (int64_t k = 0; k < n; ++k) {
    if (count_host[k] < 0 || elem_bytes(dtype_host[k]) == 0) return BXS_ERR_INVALID_ARG;
    if (count_host[k] > 0 && (!teacher_host[k] || !student_host[k])) return BXS_ERR_INVALID_ARG;
    if (count_host[k] > INT64_MAX / 8) return BXS_ERR_UNSUPPORTED;
  }
  if (int rc = check_overlaps(teacher_host, student_host, count_host, dtype_host, n)) return rc;
  cudaStream_t st = as_stream(stream);
  EmaTable tab;
  tab.a = ab_host[0];
  tab.b = ab_host[1];
  for (int64_t k0 = 0; k0 < n;) {                 // one launch per EMA_MAX entries, or fewer if the chunks reach INT32_MAX
    int m = 0;
    int64_t chunks = 0;
    for (; k0 + m < n && m < EMA_MAX; ++m) {
      const int64_t k = k0 + m;
      const int64_t c = ceil_div(count_host[k], EMA_CHUNK_BYTES / elem_bytes(dtype_host[k]));
      if (chunks + c > INT32_MAX) {
        if (m == 0) return BXS_ERR_UNSUPPORTED;
        break;
      }
      tab.t[m] = teacher_host[k];
      tab.s[m] = student_host[k];
      tab.n[m] = count_host[k];
      tab.dtype[m] = (uint8_t)dtype_host[k];
      tab.chunk0[m] = (int32_t)chunks;
      chunks += c;
    }
    tab.chunk0[m] = (int32_t)chunks;
    tab.count = m;
    k0 += m;
    if (chunks == 0) continue;
    ema_kernel<<<(unsigned)chunks, EMA_NT, 0, st>>>(tab);
    if (int rc = check_launch()) return rc;
  }
  return BXS_OK;
}
