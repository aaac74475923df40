// a4: Box2Mask's cross-attention mask in one launch -- box2mask_head.py:346-355
//        F.interpolate(mask_pred, size, bilinear, align_corners=False) -> flatten -> repeat over the heads -> sigmoid < 0.5
//     and, optionally, the reset of the forward loop (:397) that clears a row whose bits are all 1.  The reference moves
//     ~270 MB through five kernels and a nonzero (a host synchronisation) per 128x128 layer at B = 1; this reads mask_pred
//     once and writes the bools once.
//
//     Each (b, q) row is split over a thread-block cluster of `cs` CTAs.  A CTA computes its slice of the row into shared
//     memory (one byte per pixel: the bool layout), the "all 1" test is a CTA vote and, across the cluster, an AND of the
//     CTAs' flags read through distributed shared memory, then the slice is stored `heads` times with 16-byte stores.
//     cs is taken from the shape: enough CTAs for ~4 per SM while every CTA keeps at least 2 pixels per thread
//     (BXS_ATTN_CLUSTER = 1, 2, 4 or 8 fixes it for A/B builds, tools/build_variant.py).
#include <cooperative_groups.h>

#include <type_traits>

#include "common.cuh"
#include "half_math.cuh"
#include "resize_core.cuh"

#ifndef BXS_ATTN_CLUSTER
#define BXS_ATTN_CLUSTER 0
#endif

namespace cg = cooperative_groups;

namespace bxs {
namespace {

constexpr int AM_NT = 256;
constexpr int AM_MAX_CLUSTER = 8;                  // portable cluster size
constexpr int64_t AM_SMEM_MAX = 200 * 1024;        // bytes of one CTA's slice of a row

// sigmoid(v) < 0.5 as torch computes it for a tensor of type T: a 16-bit interpolation result is rounded to T, its
// sigmoid is computed in float32 and rounded to T again.  0.5 is exact in every type; NaN compares false.
template <typename T>
__device__ __forceinline__ bool attn_bit(float v) {
  if constexpr (std::is_same_v<T, float>) {
    return sigmoid_exact(v) < 0.5f;
  } else {
    return sigmoid_rounded<T>(Half16Ops<T>::round(v)) < 0.5f;
  }
}

// grid: rows * cs CTAs in clusters of cs (cluster = one (b, q) row); `chunk` (a multiple of 16) pixels per CTA.
// vec: h*w % 16 == 0 and a 16-byte aligned output, so every slice can be stored in 16-byte pieces.
template <typename T>
__global__ void __launch_bounds__(AM_NT) attn_mask_kernel(const T* __restrict__ in, uint8_t* __restrict__ attn, int Q, int H,
                                                          int W, int h, int w, int heads, int64_t chunk, bool reset, bool vec) {
  extern __shared__ __align__(16) uint8_t s_bits[];
  __shared__ int s_full;                                   // this CTA's slice holds no 0
  cg::cluster_group cluster = cg::this_cluster();
  const int cs = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int64_t row = blockIdx.x / cs, N = (int64_t)h * w;
  const int64_t p0 = rank * chunk, p1 = p0 + chunk < N ? p0 + chunk : N;
  const int n = p1 > p0 ? (int)(p1 - p0) : 0;
  const T* plane = in + row * H * W;
  const float sh = rs_scale(H, h, false), sw = rs_scale(W, w, false);

  int zero = 0;
  for (int i = threadIdx.x; i < n; i += AM_NT) {
    const int64_t p = p0 + i;
    const int oy = (int)(p / w), ox = (int)(p - (int64_t)oy * w);
    const bool bit = attn_bit<T>(rs_pixel(plane, H, W, sh, sw, oy, ox, false));
    s_bits[i] = bit;
    zero |= !bit;
  }
  bool clear = false;
  if (reset) {
    const int any_zero = __syncthreads_or(zero);
    if (threadIdx.x == 0) s_full = !any_zero;
    cluster.sync();                                        // every CTA's flag is written (and s_bits complete)
    int full = 1;
    for (int r = 0; r < cs; ++r) full &= *cluster.map_shared_rank(&s_full, r);
    clear = full != 0;
  } else {
    __syncthreads();
  }

  const int64_t b = row / Q, q = row - b * Q, head_stride = (int64_t)Q * N;
  uint8_t* dst = attn + (b * heads * Q + q) * N + p0;      // head k: + k * head_stride
  if (vec) {
    const int n16 = n >> 4;
    const uint4* src = reinterpret_cast<const uint4*>(s_bits);
    for (int i = threadIdx.x; i < heads * n16; i += AM_NT) {
      const int k = i / n16, j = i - k * n16;
      const uint4 v = clear ? make_uint4(0u, 0u, 0u, 0u) : src[j];
      *reinterpret_cast<uint4*>(dst + k * head_stride + 16 * j) = v;
    }
  } else {
    for (int64_t i = threadIdx.x; i < (int64_t)heads * n; i += AM_NT) {
      const int64_t k = i / n, j = i - k * n;
      dst[k * head_stride + j] = clear ? 0 : s_bits[j];
    }
  }
  if (reset) cluster.sync();                               // the other CTAs have read s_full: it may go away
}

int64_t slice_bytes(int64_t N, int cs) { return ceil_div(ceil_div(N, cs), 16) * 16; }

// CTAs per row: from the shape (see the file comment), at least what fits the slice into shared memory
int cluster_size(int64_t rows, int64_t N) {
  int cs = 1;
  while (cs < AM_MAX_CLUSTER && slice_bytes(N, cs) > AM_SMEM_MAX) cs *= 2;
#if BXS_ATTN_CLUSTER > 0
  return std::max(cs, (int)BXS_ATTN_CLUSTER);
#else
  const int64_t target = 4 * (int64_t)sm_count();
  while (cs < AM_MAX_CLUSTER && rows * cs < target && N >= 2 * (int64_t)AM_NT * 2 * cs) cs *= 2;
  return cs;
#endif
}

template <typename T>
int launch(const void* in, uint8_t* attn, int64_t rows, int64_t Q, int64_t H, int64_t W, int64_t h, int64_t w, int64_t heads,
           bool reset, cudaStream_t st) {
  const int64_t N = h * w;
  const int cs = cluster_size(rows, N);
  const int64_t chunk = slice_bytes(N, cs);
  if (rows * cs > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  auto kern = attn_mask_kernel<T>;
  if (const int rc = opt_in_smem(kern, (size_t)chunk)) return rc;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(rows * cs));
  cfg.blockDim = dim3(AM_NT);
  cfg.dynamicSmemBytes = (size_t)chunk;
  cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = (unsigned)cs;
  at[0].val.clusterDim.y = 1;
  at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  const bool vec = N % 16 == 0 && reinterpret_cast<uintptr_t>(attn) % 16 == 0;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kern, static_cast<const T*>(in), attn, (int)Q, (int)H, (int)W, (int)h, (int)w,
                                           (int)heads, chunk, reset, vec);
  if (e != cudaSuccess) {
    cudaGetLastError();
    set_last_error(e);
    return BXS_ERR_LAUNCH;
  }
  return check_launch();
}

bool mul_ok(int64_t a, int64_t b, int64_t& out) { return !__builtin_mul_overflow(a, b, &out); }

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_box2mask_attn_mask(const void* mask_pred, uint8_t* attn, int64_t B, int64_t Q, int64_t H, int64_t W,
                                      int64_t h, int64_t w, int64_t heads, int dtype, int reset_full_rows,
                                      bxs_stream_t stream) {
  if (B < 0 || Q < 0 || H <= 0 || W <= 0 || h <= 0 || w <= 0 || heads < 1) return BXS_ERR_INVALID_ARG;
  if (dtype != BXS_ATTN_F32 && dtype != BXS_ATTN_F16 && dtype != BXS_ATTN_BF16) return BXS_ERR_INVALID_ARG;
  if (B == 0 || Q == 0) return BXS_OK;
  if (!mask_pred || !attn) return BXS_ERR_INVALID_ARG;
  // float source indices (exact below 2^24), int plane offsets, int64 tensor offsets
  if (H >= (1 << 24) || W >= (1 << 24) || h >= (1 << 24) || w >= (1 << 24) || H * W > INT32_MAX || Q > INT32_MAX ||
      heads > INT32_MAX)
    return BXS_ERR_UNSUPPORTED;
  int64_t rows, in_el, out_rows, out_el, copies;
  if (!mul_ok(B, Q, rows) || !mul_ok(rows, H * W, in_el) || !mul_ok(rows, heads, out_rows) || !mul_ok(out_rows, h * w, out_el) ||
      !mul_ok(heads, h * w, copies) || copies > INT32_MAX)
    return BXS_ERR_UNSUPPORTED;
  if (slice_bytes(h * w, AM_MAX_CLUSTER) > AM_SMEM_MAX) return BXS_ERR_UNSUPPORTED;   // the row does not fit 8 CTAs
  const cudaStream_t st = as_stream(stream);
  const bool reset = reset_full_rows != 0;
  switch (dtype) {
    case BXS_ATTN_F16: return launch<__half>(mask_pred, attn, rows, Q, H, W, h, w, heads, reset, st);
    case BXS_ATTN_BF16: return launch<__nv_bfloat16>(mask_pred, attn, rows, Q, H, W, h, w, heads, reset, st);
    default: return launch<float>(mask_pred, attn, rows, Q, H, W, h, w, heads, reset, st);
  }
}
