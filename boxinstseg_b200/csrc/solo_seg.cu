// SOLOv2 inference (get_seg_single of box_solov2_head.py:503-590 and discobox_head.py:1559-1660): per-row mask statistics,
// batched Matrix NMS (mmdet/core/post_processing/matrix_nms.py) and the fused two-stage mask paste.
//
//   stats:  one CTA per distinct candidate row (a (level, image, cell) of the mask predictions): every warp takes 32 pixels
//           at a time, compares them with the threshold and ballots the word of the packed mask; the area is the popcount,
//           and the masked sum is accumulated per lane in float64 and reduced in a fixed order (one float32 rounding).
//   nms:    inter[i, j] = popcount(m_i & m_j) over 32 x 32 tiles of candidate pairs (i < j, same label, both valid), the
//           packed words staged through shared memory in 32-word chunks; a tile without such a pair returns at once.  The
//           IoU goes to the workspace and its column maximum (compensate_iou) is an atomicMax on the bits of a non-negative
//           float: exact and order-independent.  A second launch gives every column its decay coefficient (one warp per
//           column, the minimum over every valid row i, NaN propagating as torch.min does) and the decayed, filtered score.
//   paste:  one thread per output pixel: its four intermediate taps of the (4h, 4w) upsampling, each a lerp of four input
//           pixels (sigmoid on the fly for logits), rounded to the row dtype between and after the stages as ATen rounds a
//           16-bit tensor (or, under autocast, kept in float32: autocast runs upsample_bilinear2d in float32), then the
//           threshold.  The [n, 4h, 4w] intermediate of the reference never exists.
//   maskformer paste: the same per-pixel function (paste_value) on Box2Mask's logit rows, with a first stage of any size
//           and stages that may be skipped, plus each mask's area, masked sum and box folded in the pass that writes it.
//   extents: each mask's set-pixel count and box from bool / uint8 masks (16-byte row loads where W and the base allow),
//           per-CTA partials reduced as the maskformer paste reduces its own.
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "half_math.cuh"
#include "solo_seg_core.cuh"

namespace bxs {
namespace {

constexpr int SS_MAX_SRC = 8;
constexpr int SS_NT = 256;
constexpr int NMS_TILE = 32;

struct RowSources {                    // by value in the kernel parameters
  const void* p[SS_MAX_SRC];
  int64_t start[SS_MAX_SRC + 1];       // first row id of each source; start[n]: the total
  int n;
};

int make_sources(RowSources& s, const void* const* src_host, const int64_t* src_rows_host, int64_t n_src) {
  if (!src_host || !src_rows_host || n_src <= 0) return BXS_ERR_INVALID_ARG;
  if (n_src > SS_MAX_SRC) return BXS_ERR_UNSUPPORTED;
  s = RowSources{};
  s.n = (int)n_src;
  for (int64_t k = 0; k < n_src; ++k) {
    if (src_rows_host[k] < 0 || (src_rows_host[k] && !src_host[k])) return BXS_ERR_INVALID_ARG;
    s.p[k] = src_host[k];
    s.start[k + 1] = s.start[k] + src_rows_host[k];
  }
  return BXS_OK;
}

// the row of id g, or nullptr for an id outside the sources
template <typename T>
__device__ __forceinline__ const T* row_ptr(const RowSources& s, int64_t g, int64_t hw) {
  if (g < 0 || g >= s.start[s.n]) return nullptr;
  int k = 0;
  while (k + 1 < s.n && g >= s.start[k + 1]) ++k;
  return static_cast<const T*>(s.p[k]) + (g - s.start[k]) * hw;
}

// a row element as the probability the reference thresholds and interpolates (widened to float, exact)
__device__ __forceinline__ float prob(float v, bool logits) { return logits ? sigmoid_exact(v) : v; }
__device__ __forceinline__ float prob(__half v, bool logits) { return logits ? sigmoid_rounded(v) : __half2float(v); }

template <typename T>
__device__ __forceinline__ float to_dtype(float v) {
  if constexpr (std::is_same<T, __half>::value) return round_to<__half>(v);
  return v;
}

template <typename T>
__global__ void __launch_bounds__(SS_NT) solo_stats_kernel(RowSources src, const int64_t* __restrict__ rows, int64_t hw,
                                                           int64_t words, int logits, float thr, uint32_t* __restrict__ bits,
                                                           int32_t* __restrict__ area, float* __restrict__ masked_sum) {
  __shared__ double s_sum[SS_NT / kWarp];
  __shared__ int s_cnt[SS_NT / kWarp];
  const int64_t r = blockIdx.x;
  const T* p = row_ptr<T>(src, rows[r], hw);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float t = to_dtype<T>(thr);
  double acc = 0.0;
  int cnt = 0;
#pragma unroll 4
  for (int64_t w = warp; w < words; w += SS_NT / kWarp) {
    const int64_t i = w * kWarp + lane;
    float v = 0.f;
    if (p && i < hw) v = prob(p[i], logits);
    const bool on = v > t;
    const unsigned m = __ballot_sync(kFull, on);
    if (lane == 0) {
      bits[r * words + w] = m;
      cnt += __popc(m);
    }
    if (on) acc += (double)v;
  }
  acc = warp_sum(acc);
  if (lane == 0) {
    s_sum[warp] = acc;
    s_cnt[warp] = cnt;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    int c = 0;
    for (int k = 0; k < SS_NT / kWarp; ++k) {
      s += s_sum[k];
      c += s_cnt[k];
    }
    area[r] = c;
    masked_sum[r] = (float)s;
  }
}

// Candidate pairs of one 32 x 32 tile: rows i0 + ty + 8k (k < 4), column j0 + tx.
__global__ void __launch_bounds__(SS_NT) nms_inter_kernel(const uint32_t* __restrict__ bits, int64_t words,
                                                          const int64_t* __restrict__ row, const int64_t* __restrict__ label,
                                                          const float* __restrict__ area, const int64_t* __restrict__ n_valid,
                                                          int64_t N, int half_inter, float* __restrict__ iou,
                                                          unsigned* __restrict__ comp_bits) {
  __shared__ uint32_t sa[NMS_TILE][NMS_TILE + 1], sb[NMS_TILE][NMS_TILE + 1];
  const int64_t b = blockIdx.z, i0 = (int64_t)blockIdx.y * NMS_TILE, j0 = (int64_t)blockIdx.x * NMS_TILE;
  const int64_t nv = min(n_valid[b], N);
  if (i0 >= j0 + NMS_TILE - 1 || i0 >= nv || j0 >= nv) return;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t base = b * N, j = j0 + tx;
  const int64_t lj = j < nv ? label[base + j] : -1;
  bool need[4];
  int any = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int64_t i = i0 + ty + 8 * k;
    need[k] = j < nv && i < j && label[base + i] == lj;
    any |= need[k];
  }
  if (!__syncthreads_or(any)) return;
  const uint32_t* ra[4];
  const uint32_t* rb[4];
#pragma unroll
  for (int m = 0; m < 4; ++m) {
    const int64_t gi = i0 + ty + 8 * m, gj = j0 + ty + 8 * m;
    ra[m] = gi < nv ? bits + row[base + gi] * words : nullptr;
    rb[m] = gj < nv ? bits + row[base + gj] * words : nullptr;
  }
  int acc[4] = {0, 0, 0, 0};
  for (int64_t w0 = 0; w0 < words; w0 += NMS_TILE) {
    const int64_t w = w0 + tx;
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      sa[ty + 8 * m][tx] = ra[m] && w < words ? __ldg(ra[m] + w) : 0u;
      sb[ty + 8 * m][tx] = rb[m] && w < words ? __ldg(rb[m] + w) : 0u;
    }
    __syncthreads();
#pragma unroll 8
    for (int kw = 0; kw < NMS_TILE; ++kw) {
      const uint32_t bj = sb[tx][kw];
#pragma unroll
      for (int k = 0; k < 4; ++k) acc[k] += __popc(sa[ty + 8 * k][kw] & bj);
    }
    __syncthreads();
  }
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (!need[k]) continue;
    const int64_t i = i0 + ty + 8 * k;
    float inter = (float)acc[k];
    if (half_inter) inter = round_to<__half>(inter);
    const float v = nms_iou(inter, area[base + i], area[base + j]);
    iou[(base + j) * N + i] = v;
    atomicMax(comp_bits + base + j, __float_as_uint(v));
  }
}

__global__ void __launch_bounds__(SS_NT) nms_decay_kernel(const int64_t* __restrict__ label, const float* __restrict__ score,
                                                          const int64_t* __restrict__ n_valid, int64_t B, int64_t N,
                                                          const float* __restrict__ iou, const unsigned* __restrict__ comp_bits,
                                                          int kernel, float nsig, float filter_thr, float* __restrict__ out) {
  const int64_t gw = (int64_t)blockIdx.x * (SS_NT / kWarp) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (gw >= B * N) return;
  const int64_t b = gw / N, j = gw % N, base = b * N;
  const int64_t nv = min(n_valid[b], N);
  if (j >= nv) {
    if (lane == 0) out[base + j] = -INFINITY;
    return;
  }
  const int64_t lj = label[base + j];
  float m = INFINITY;
  for (int64_t i = lane; i < nv; i += kWarp) {
    const float comp = __uint_as_float(comp_bits[base + i]);
    const float v = (i < j && label[base + i] == lj) ? iou[(base + j) * N + i] : 0.f;
    m = nan_min(m, nms_decay_ratio(v, comp, kernel, nsig));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = nan_min(m, __shfl_xor_sync(kFull, m, o));
  if (lane == 0) {
    const float s = BXS_FMUL(score[base + j], m);
    out[base + j] = (filter_thr > 0.f && !(s >= filter_thr)) ? -INFINITY : s;
  }
}

// interp_f32: the probabilities of a 16-bit row are interpolated and thresholded in float32 without rounding (what
// torch.autocast does to upsample_bilinear2d); else each stage is rounded to T.
template <typename T, bool kRound>
__device__ __forceinline__ float stage(float v) {
  return kRound ? to_dtype<T>(v) : v;
}

template <typename T, bool kRound>
__global__ void __launch_bounds__(SS_NT) solo_paste_kernel(RowSources src, const int64_t* __restrict__ rows, int64_t n, int h,
                                                           int w, int H_img, int W_img, int H_ori, int W_ori, int logits,
                                                           float thr, uint8_t* __restrict__ out) {
  const float t = stage<T, kRound>(thr);
  const int64_t npix = (int64_t)H_ori * W_ori;
  for (int64_t k = blockIdx.y; k < n; k += gridDim.y) {
    const T* p = row_ptr<T>(src, rows[k], (int64_t)h * w);
    uint8_t* o = out + k * npix;
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += (int64_t)gridDim.x * blockDim.x) {
      if (!p) {
        o[pix] = 0;
        continue;
      }
      const int y = (int)(pix / W_ori), x = (int)(pix % W_ori);
      const PasteGeom g{h, w, 4 * h, 4 * w, H_img, W_img, H_ori, W_ori, false, false};
      o[pix] = paste_value<false>(
                   g, y, x, [&](int q, int d) { return prob((p + q)[d], logits); },
                   [](float v) { return stage<T, kRound>(v); }) > t;
    }
  }
}

// A CTA's MaskStats -> *out, written by thread 0: lanes by the butterfly, warps in index order, so that the float64 sum is
// the same from run to run.  Every thread of the CTA calls it.
__device__ __forceinline__ void mask_stats_cta_partial(MaskStats st, MaskStats* s_part, MaskStats* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  st.sum = warp_sum(st.sum);
  st.area = __reduce_add_sync(kFull, st.area);
  st.x0 = __reduce_min_sync(kFull, st.x0);
  st.y0 = __reduce_min_sync(kFull, st.y0);
  st.x1 = __reduce_max_sync(kFull, st.x1);
  st.y1 = __reduce_max_sync(kFull, st.y1);
  if (lane == 0) s_part[warp] = st;
  __syncthreads();
  if (threadIdx.x == 0) {
    MaskStats s = s_part[0];
    for (int i = 1; i < SS_NT / kWarp; ++i) mask_stats_merge(s, s_part[i]);
    *out = s;
  }
  __syncthreads();
}

// MaskFormer's instance masks (maskformer_fusion_head.py:112-241 after box2mask_head.py:445-459): the same per-pixel paste
// of logit rows, thresholded at 0, a float16 row rounded after each stage; each CTA also folds its set pixels into a
// MaskStats (sigmoid as torch computes it for T) and writes it to part[k * gridDim.x + blockIdx.x].
template <typename T>
__global__ void __launch_bounds__(SS_NT) maskformer_paste_kernel(RowSources src, const int64_t* __restrict__ rows, int64_t n,
                                                                 PasteGeom g, uint8_t* __restrict__ out,
                                                                 MaskStats* __restrict__ part) {
  constexpr bool kRound = std::is_same<T, __half>::value;
  __shared__ MaskStats s_part[SS_NT / kWarp];
  const int64_t npix = (int64_t)g.H_out * g.W_out;
  for (int64_t k = blockIdx.y; k < n; k += gridDim.y) {
    const T* p = row_ptr<T>(src, rows[k], (int64_t)g.h * g.w);
    uint8_t* o = out + k * npix;
    MaskStats st = mask_stats_empty();
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += (int64_t)gridDim.x * blockDim.x) {
      const int y = (int)(pix / g.W_out), x = (int)(pix % g.W_out);
      const float v = p ? paste_value<true>(
                              g, y, x, [&](int q, int d) { return prob((p + q)[d], false); },
                              [](float u) { return stage<T, kRound>(u); })
                        : 0.f;
      const bool on = v > 0.f;
      o[pix] = on;
      if (on) mask_stats_add(st, y, x, kRound ? prob(__float2half_rn(v), true) : prob(v, true));
    }
    mask_stats_cta_partial(st, s_part, part + k * gridDim.x + blockIdx.x);
  }
}

// the n_part partials of every row, in index order -> area, masked_sum (one float32 rounding; kSum = false: not written),
// box.  The maskformer paste and the mask extents reduce their partials here.
template <bool kSum>
__global__ void __launch_bounds__(SS_NT) mask_stats_reduce_kernel(const MaskStats* __restrict__ part, int64_t n, int n_part,
                                                                  int32_t* __restrict__ area, float* __restrict__ masked_sum,
                                                                  float* __restrict__ box) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  MaskStats s = part[k * n_part];
  for (int i = 1; i < n_part; ++i) mask_stats_merge(s, part[k * n_part + i]);
  area[k] = s.area;
  if constexpr (kSum) masked_sum[k] = (float)s.sum;
  mask_stats_box(s, box + 4 * k);
}

constexpr int MF_MAX_PARTS = 64;       // CTAs per row of the maskformer paste: 256-thread CTAs, one partial each

// The set (non-zero) bytes of the 16 bytes q, the first at column x of row y, folded into s.  W % 16 == 0 keeps the 16
// bytes in one row.  __vcmpne4 gives 0xff per non-zero byte; its low bits, gathered, are a 16-bit mask of the set bytes.
__device__ __forceinline__ void mask_extents_add16(MaskStats& s, const uint4& q, int y, int x) {
  const unsigned w[4] = {q.x, q.y, q.z, q.w};
  unsigned m = 0;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const unsigned b = __vcmpne4(w[j], 0u) & 0x01010101u;
    m |= ((b | (b >> 7) | (b >> 14) | (b >> 21)) & 0xfu) << (4 * j);
  }
  if (!m) return;
  s.area += __popc(m);
  s.x0 = min(s.x0, x + __ffs(m) - 1);
  s.x1 = max(s.x1, x + 31 - __clz(m));
  s.y0 = min(s.y0, y);
  s.y1 = max(s.y1, y);
}

// Each CTA folds the set bytes of its share of mask k (its own run of the mask's 16-byte vectors, kVec, or bytes) into
// a MaskStats and writes it to part[k * gridDim.x + blockIdx.x], as the maskformer paste writes its partials; the sum
// stays 0.  Integer counts and extents only: the result does not depend on the order of the reduction.
template <bool kVec>
__global__ void __launch_bounds__(SS_NT) mask_extents_kernel(const uint8_t* __restrict__ masks, int64_t n, int H, int W,
                                                             MaskStats* __restrict__ part) {
  __shared__ MaskStats s_part[SS_NT / kWarp];
  const int hw = H * W;
  const int items = kVec ? hw / 16 : hw;
  const int stride = gridDim.x * SS_NT;
  for (int64_t k = blockIdx.y; k < n; k += gridDim.y) {
    const uint8_t* m = masks + k * hw;
    MaskStats st = mask_stats_empty();
#pragma unroll 4
    for (int i = blockIdx.x * SS_NT + threadIdx.x; i < items; i += stride) {
      if constexpr (kVec) {
        const int o = 16 * i, y = o / W;
        mask_extents_add16(st, __ldg(reinterpret_cast<const uint4*>(m) + i), y, o - y * W);
      } else if (__ldg(m + i)) {
        const int y = i / W;
        mask_stats_add(st, y, i - y * W, 0.f);
      }
    }
    mask_stats_cta_partial(st, s_part, part + k * gridDim.x + blockIdx.x);
  }
}

// CTAs per mask of mask_extents_kernel: about four vectors (or bytes) per thread, at most MF_MAX_PARTS
int64_t extents_parts(int64_t H, int64_t W, bool vec) {
  const int64_t items = vec ? H * W / 16 : H * W;
  return std::max<int64_t>(1, std::min<int64_t>(ceil_div(items, 4 * SS_NT), MF_MAX_PARTS));
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_solo_mask_stats(const void* const* src_host, const int64_t* src_rows_host, int64_t n_src, int64_t hw,
                                   int dtype, int logits, const int64_t* rows, int64_t n_rows, float mask_thr, uint32_t* bits,
                                   int32_t* area, float* masked_sum, bxs_stream_t stream) {
  RowSources src;
  if (int rc = make_sources(src, src_host, src_rows_host, n_src)) return rc;
  if (hw <= 0 || n_rows < 0 || (dtype != 0 && dtype != 1)) return BXS_ERR_INVALID_ARG;
  if (n_rows > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  if (n_rows == 0) return BXS_OK;
  if (!rows || !bits || !area || !masked_sum) return BXS_ERR_INVALID_ARG;
  const int64_t words = ceil_div(hw, kWarp);
  auto kern = dtype == 0 ? solo_stats_kernel<float> : solo_stats_kernel<__half>;
  kern<<<(unsigned)n_rows, SS_NT, 0, as_stream(stream)>>>(src, rows, hw, words, logits, mask_thr, bits, area, masked_sum);
  return check_launch();
}

extern "C" int64_t bxs_matrix_nms_workspace_bytes(int64_t B, int64_t N) {
  if (B <= 0 || N <= 0) return 0;
  Carver c(nullptr);
  c.take((size_t)(B * N * N) * sizeof(float));
  c.take((size_t)(B * N) * sizeof(unsigned));
  return (int64_t)c.off;
}

extern "C" int bxs_matrix_nms(const uint32_t* bits, int64_t words, const int64_t* row, const int64_t* label, const float* area,
                              const float* score, const int64_t* n_valid, int64_t B, int64_t N, int kernel, float sigma,
                              float filter_thr, int half_inter, void* workspace, float* out_score, bxs_stream_t stream) {
  if (B < 0 || N < 0 || words <= 0 || (kernel != kNmsGaussian && kernel != kNmsLinear)) return BXS_ERR_INVALID_ARG;
  if (B == 0 || N == 0) return BXS_OK;
  if (!bits || !row || !label || !area || !score || !n_valid || !workspace || !out_score) return BXS_ERR_INVALID_ARG;
  if (B > 65535 || ceil_div(N, NMS_TILE) > 65535 || B * N > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  Carver c(workspace);
  float* iou = reinterpret_cast<float*>(c.take((size_t)(B * N * N) * sizeof(float)));
  unsigned* comp = reinterpret_cast<unsigned*>(c.take((size_t)(B * N) * sizeof(unsigned)));
  cudaStream_t s = as_stream(stream);
  if (cudaMemsetAsync(comp, 0, (size_t)(B * N) * sizeof(unsigned), s) != cudaSuccess) return check_launch();
  const unsigned tiles = (unsigned)ceil_div(N, NMS_TILE);
  nms_inter_kernel<<<dim3(tiles, tiles, (unsigned)B), SS_NT, 0, s>>>(bits, words, row, label, area, n_valid, N, half_inter, iou,
                                                                     comp);
  if (int rc = check_launch()) return rc;
  const float nsig = -1.f * sigma;
  nms_decay_kernel<<<(unsigned)ceil_div(B * N, SS_NT / kWarp), SS_NT, 0, s>>>(label, score, n_valid, B, N, iou, comp, kernel,
                                                                              nsig, filter_thr, out_score);
  return check_launch();
}

extern "C" int bxs_solo_paste_masks(const void* const* src_host, const int64_t* src_rows_host, int64_t n_src, int64_t h,
                                    int64_t w, int dtype, int logits, int interp_f32, const int64_t* rows, int64_t n,
                                    int64_t H_img, int64_t W_img, int64_t H_ori, int64_t W_ori, float mask_thr,
                                    uint8_t* out, bxs_stream_t stream) {
  RowSources src;
  if (int rc = make_sources(src, src_host, src_rows_host, n_src)) return rc;
  if (h <= 0 || w <= 0 || n < 0 || H_img <= 0 || W_img <= 0 || H_ori <= 0 || W_ori <= 0 || (dtype != 0 && dtype != 1))
    return BXS_ERR_INVALID_ARG;
  if (H_img > 4 * h || W_img > 4 * w) return BXS_ERR_INVALID_ARG;          // the crop lies inside the (4h, 4w) plane
  if (4 * h > INT32_MAX || 4 * w > INT32_MAX || H_ori * W_ori > INT32_MAX || h * w > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  if (n == 0) return BXS_OK;
  if (!rows || !out) return BXS_ERR_INVALID_ARG;
  const int64_t npix = H_ori * W_ori;
  const unsigned gx = (unsigned)std::min<int64_t>(ceil_div(npix, SS_NT), 1024);
  const unsigned gy = (unsigned)std::min<int64_t>(n, 65535);
  auto kern = dtype == 0 ? solo_paste_kernel<float, false>
                         : (interp_f32 ? solo_paste_kernel<__half, false> : solo_paste_kernel<__half, true>);
  kern<<<dim3(gx, gy), SS_NT, 0, as_stream(stream)>>>(src, rows, n, (int)h, (int)w, (int)H_img, (int)W_img, (int)H_ori,
                                                      (int)W_ori, logits, mask_thr, out);
  return check_launch();
}

extern "C" int64_t bxs_maskformer_paste_workspace_bytes(int64_t n) {
  if (n <= 0) return 0;
  return n * MF_MAX_PARTS * (int64_t)sizeof(MaskStats);
}

extern "C" int bxs_maskformer_paste_masks(const void* const* src_host, const int64_t* src_rows_host, int64_t n_src, int64_t h,
                                          int64_t w, int dtype, const int64_t* rows, int64_t n, int64_t H_pad, int64_t W_pad,
                                          int64_t H_img, int64_t W_img, int rescale, int64_t H_out, int64_t W_out,
                                          void* workspace, uint8_t* out, int32_t* area, float* masked_sum, float* box,
                                          bxs_stream_t stream) {
  RowSources src;
  if (int rc = make_sources(src, src_host, src_rows_host, n_src)) return rc;
  if (h <= 0 || w <= 0 || n < 0 || H_img <= 0 || W_img <= 0 || H_out <= 0 || W_out <= 0 || (dtype != 0 && dtype != 1))
    return BXS_ERR_INVALID_ARG;
  if (h > H_pad || w > W_pad || H_img > H_pad || W_img > W_pad) return BXS_ERR_INVALID_ARG;
  if (!rescale && (H_out != H_img || W_out != W_img)) return BXS_ERR_INVALID_ARG;
  if (H_pad > INT32_MAX || W_pad > INT32_MAX || h * w > INT32_MAX || H_out * W_out > INT32_MAX || n > INT32_MAX)
    return BXS_ERR_UNSUPPORTED;
  if (n == 0) return BXS_OK;
  if (!rows || !workspace || !out || !area || !masked_sum || !box) return BXS_ERR_INVALID_ARG;
  const PasteGeom g{(int)h, (int)w, (int)H_pad, (int)W_pad, (int)H_img, (int)W_img, (int)H_out, (int)W_out,
                    h == H_pad && w == W_pad, !rescale};
  const unsigned gx = (unsigned)std::min<int64_t>(ceil_div(H_out * W_out, SS_NT), MF_MAX_PARTS);
  const unsigned gy = (unsigned)std::min<int64_t>(n, 65535);
  MaskStats* part = static_cast<MaskStats*>(workspace);
  cudaStream_t s = as_stream(stream);
  auto kern = dtype == 0 ? maskformer_paste_kernel<float> : maskformer_paste_kernel<__half>;
  kern<<<dim3(gx, gy), SS_NT, 0, s>>>(src, rows, n, g, out, part);
  if (int rc = check_launch()) return rc;
  mask_stats_reduce_kernel<true><<<(unsigned)ceil_div(n, SS_NT), SS_NT, 0, s>>>(part, n, (int)gx, area, masked_sum, box);
  return check_launch();
}

extern "C" int64_t bxs_mask_extents_workspace_bytes(int64_t n, int64_t H, int64_t W) {
  if (n <= 0 || H < 0 || W < 0) return 0;
  return n * extents_parts(H, W, false) * (int64_t)sizeof(MaskStats);      // the byte path's count bounds the vector path's
}

extern "C" int bxs_mask_extents(const uint8_t* masks, int64_t n, int64_t H, int64_t W, void* workspace, int32_t* area,
                                float* box, bxs_stream_t stream) {
  if (n < 0 || H < 0 || W < 0) return BXS_ERR_INVALID_ARG;
  if (H * W > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  if (n == 0) return BXS_OK;
  if ((!masks && H * W > 0) || !workspace || !area || !box) return BXS_ERR_INVALID_ARG;
  const bool vec = W % 16 == 0 && reinterpret_cast<uintptr_t>(masks) % 16 == 0;
  const int64_t gx = extents_parts(H, W, vec);
  const unsigned gy = (unsigned)std::min<int64_t>(n, 65535);
  MaskStats* part = static_cast<MaskStats*>(workspace);
  cudaStream_t s = as_stream(stream);
  auto kern = vec ? mask_extents_kernel<true> : mask_extents_kernel<false>;
  kern<<<dim3((unsigned)gx, gy), SS_NT, 0, s>>>(masks, n, (int)H, (int)W, part);
  if (int rc = check_launch()) return rc;
  mask_stats_reduce_kernel<false><<<(unsigned)ceil_div(n, SS_NT), SS_NT, 0, s>>>(part, n, (int)gx, area, nullptr, box);
  return check_launch();
}
