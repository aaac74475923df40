// CondInst inference (CondInstBoxHead.get_bboxes / _get_bboxes, condinst_head.py:640-853, nms_with_others :18-83, mmcv's
// batched_nms; CondInstMaskHead.simple_test :1234-1286): the level walk over the raw predictions, the batched per-class NMS
// and the fused mask paste.
//
//   key:     one thread per (image, level, point): max_c sigmoid(cls_c) * sigmoid(ctr), the value the per-level top-k
//            ranks (:781), read in place from every level's [B,C,H,W] tensors through a level table passed by value (any
//            element strides); padded per level with -inf.
//   decode:  one thread per (image, selected slot): the point the top-k chose (or the slot's own point when the level is not
//            cut), its distance2bbox box with the per-image clamp and the optional division by scale_factor, sigmoid(ctr),
//            and per class the candidate flag sigmoid(cls) > score_thr and its score sigmoid(cls) * sigmoid(ctr).
//   gather:  the dynamic-head parameters, the point and the level of chosen slots, again straight from the level tensors.
//   nms:     one thread per candidate row of a (image, class) segment sorted by score: the bits of the later candidates of
//            its segment that it suppresses (mmcv's test on the offset boxes), 64 per word, so the workspace is
//            sum_s n_s * ceil(n_s / 64) words; then one warp per segment resolves the greedy order on the device.
//   paste:   one thread per output pixel: sigmoid -> aligned_bilinear(., f) -> crop -> (bilinear resize to the original
//            size) -> > 0.5, with the taps of resize_core.cuh; the [n, f*h, f*w] plane of the reference never exists.
// No atomics anywhere: every value and every order is the same from run to run.
#include <algorithm>

#include "boxinst_common.cuh"         // sigmoid_exact
#include "box_nms_core.cuh"
#include "common.cuh"

namespace bxs {
namespace {

constexpr int CI_MAX_LEVELS = 8;
constexpr int CI_MAX_IMGS = 32;
constexpr int CI_NT = 256;
constexpr int NMS_WORD = 64;

struct CiLevel {
  const float* cls;      // [B,C,H,W] with element strides cs
  const float* ctr;      // [B,1,H,W]
  const float* bbox;     // [B,4,H,W]
  const float* param;    // [B,P,H,W]
  int64_t cs[4], ts[4], bs[4], ps[4];
  int H, W;
  float stride;
  int topk;              // the level was cut by the top-k: slot r reads the r-th index of `order`
  int64_t slot0;         // first slot of the level
};

struct CiTable {         // by value in the kernel parameters
  CiLevel lv[CI_MAX_LEVELS];
  int n;
  int64_t S;             // slots per image
  float img_h[CI_MAX_IMGS], img_w[CI_MAX_IMGS];
  float sf[CI_MAX_IMGS][4];
  int rescale;
};

__device__ __forceinline__ int level_of(const CiTable& t, int64_t s) {
  int l = 0;
  while (l + 1 < t.n && s >= t.lv[l + 1].slot0) ++l;
  return l;
}

__device__ __forceinline__ float at(const float* p, const int64_t* st, int64_t b, int64_t c, int y, int x) {
  return __ldg(p + b * st[0] + c * st[1] + (int64_t)y * st[2] + (int64_t)x * st[3]);
}

__global__ void __launch_bounds__(CI_NT) ci_key_kernel(CiTable t, int64_t B, int64_t C, int64_t Pmax, float* __restrict__ key) {
  const int64_t total = B * t.n * Pmax;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = g % Pmax, bl = g / Pmax;
    const int l = (int)(bl % t.n);
    const int64_t b = bl / t.n;
    const CiLevel& lv = t.lv[l];
    if (p >= (int64_t)lv.H * lv.W) {
      key[g] = -INFINITY;
      continue;
    }
    const int y = (int)(p / lv.W), x = (int)(p % lv.W);
    const float ctr = sigmoid_exact(at(lv.ctr, lv.ts, b, 0, y, x));
    float m = -INFINITY;
    for (int64_t c = 0; c < C; ++c) {
      const float v = __fmul_rn(sigmoid_exact(at(lv.cls, lv.cs, b, c, y, x)), ctr);
      m = (v > m || v != v) ? v : m;          // torch.max: a NaN wins and stays
    }
    key[g] = m;
  }
}

__global__ void __launch_bounds__(CI_NT) ci_decode_kernel(CiTable t, int64_t B, int64_t C, const int64_t* __restrict__ order,
                                                          int64_t Pmax, float thr, float* __restrict__ box,
                                                          float* __restrict__ ctr_out, int64_t* __restrict__ point,
                                                          uint8_t* __restrict__ cand, float* __restrict__ score,
                                                          float* __restrict__ sig_out) {
  const int64_t total = B * t.S;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = g / t.S, s = g % t.S;
    const int l = level_of(t, s);
    const CiLevel& lv = t.lv[l];
    const int64_t r = s - lv.slot0;
    const int64_t p = lv.topk ? order[(b * t.n + l) * Pmax + r] : r;
    const int y = (int)(p / lv.W), x = (int)(p % lv.W);
    float d[4], o[4];
    for (int k = 0; k < 4; ++k) d[k] = at(lv.bbox, lv.bs, b, k, y, x);
    ci_decode_box(ci_point(x, lv.stride), ci_point(y, lv.stride), d, t.img_h[b], t.img_w[b], t.rescale ? t.sf[b] : nullptr, o);
    for (int k = 0; k < 4; ++k) box[g * 4 + k] = o[k];
    const float ctr = sigmoid_exact(at(lv.ctr, lv.ts, b, 0, y, x));
    ctr_out[g] = ctr;
    point[g] = p;
    for (int64_t c = 0; c < C; ++c) {
      const float sg = sigmoid_exact(at(lv.cls, lv.cs, b, c, y, x));
      cand[g * C + c] = sg > thr;
      score[g * C + c] = __fmul_rn(sg, ctr);
      if (sig_out) sig_out[g * C + c] = sg;
    }
  }
}

__global__ void __launch_bounds__(CI_NT) ci_gather_kernel(CiTable t, int64_t P, const int64_t* __restrict__ point,
                                                          const int64_t* __restrict__ rows, int64_t n, float* __restrict__ params,
                                                          float* __restrict__ coors, int64_t* __restrict__ level) {
  const int64_t total = n * P;
  for (int64_t g = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; g < total; g += (int64_t)gridDim.x * blockDim.x) {
    const int64_t k = g / P, j = g % P, row = rows[k];
    const int64_t b = row / t.S;
    const int l = level_of(t, row % t.S);
    const CiLevel& lv = t.lv[l];
    const int64_t p = point[row];
    const int y = (int)(p / lv.W), x = (int)(p % lv.W);
    params[g] = at(lv.param, lv.ps, b, j, y, x);
    if (j == 0) {
      coors[2 * k] = ci_point(x, lv.stride);
      coors[2 * k + 1] = ci_point(y, lv.stride);
      level[k] = l;
    }
  }
}

// the segment of sorted row i: seg_start[s] <= i < seg_start[s + 1] (empty segments skipped)
__device__ __forceinline__ int64_t segment_of(const int64_t* seg_start, int64_t n_seg, int64_t i) {
  int64_t lo = 0, hi = n_seg;                       // the last s with seg_start[s] <= i
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (seg_start[mid] <= i) lo = mid; else hi = mid - 1;
  }
  return lo;
}

__global__ void __launch_bounds__(CI_NT) nms_mask_kernel(const float* __restrict__ boxes, const int64_t* __restrict__ seg_start,
                                                         const int64_t* __restrict__ mask_off, int64_t n_seg, int64_t N, float thr,
                                                         unsigned long long* __restrict__ mask) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N) return;
  const int64_t s = segment_of(seg_start, n_seg, i);
  const int64_t s0 = seg_start[s], ns = seg_start[s + 1] - s0, words = (ns + NMS_WORD - 1) / NMS_WORD;
  unsigned long long* row = mask + mask_off[s] + (i - s0) * words;
  const float4 av = __ldg(reinterpret_cast<const float4*>(boxes) + i);
  const float a[4] = {av.x, av.y, av.z, av.w};
  for (int64_t w = (i - s0) / NMS_WORD; w < words; ++w) {
    unsigned long long bits = 0;
    const int64_t j0 = s0 + w * NMS_WORD, j1 = min(j0 + NMS_WORD, s0 + ns);
    for (int64_t j = max(j0, i + 1); j < j1; ++j) {
      const float4 bv = __ldg(reinterpret_cast<const float4*>(boxes) + j);
      const float bb[4] = {bv.x, bv.y, bv.z, bv.w};
      if (ci_suppresses(a, bb, thr)) bits |= 1ull << (j - j0);
    }
    row[w] = bits;
  }
}

// one warp per segment: the greedy pass of mmcv's host loop, on the device
__global__ void __launch_bounds__(kWarp) nms_resolve_kernel(const unsigned long long* __restrict__ mask,
                                                            const int64_t* __restrict__ seg_start,
                                                            const int64_t* __restrict__ mask_off, uint8_t* __restrict__ keep) {
  extern __shared__ unsigned long long removed[];
  const int64_t s = blockIdx.x, s0 = seg_start[s], ns = seg_start[s + 1] - s0, words = (ns + NMS_WORD - 1) / NMS_WORD;
  const int lane = threadIdx.x;
  for (int64_t w = lane; w < words; w += kWarp) removed[w] = 0;
  __syncwarp();
  const unsigned long long* m = mask + mask_off[s];
  for (int64_t i = 0; i < ns; ++i) {
    const bool gone = (removed[i / NMS_WORD] >> (i % NMS_WORD)) & 1ull;
    __syncwarp();
    if (lane == 0) keep[s0 + i] = !gone;
    if (!gone)
      for (int64_t w = i / NMS_WORD + lane; w < words; w += kWarp) removed[w] |= m[i * words + w];
    __syncwarp();
  }
}

__device__ __forceinline__ float ci_prob(const float* p, int h, int w, int i, int j) {
  return sigmoid_exact(__ldg(p + (int64_t)min(i, h - 1) * w + min(j, w - 1)));
}

// pixel (Y, X) of aligned_bilinear(sigmoid(p), f)
__device__ __forceinline__ float ci_aligned(const float* p, int h, int w, int f, int Y, int X) {
  const RsTap ty = ci_aligned_tap(Y, h, f), tx = ci_aligned_tap(X, w, f);
  return rs_lerp2(ty, tx, ci_prob(p, h, w, ty.i0, tx.i0), ci_prob(p, h, w, ty.i0, tx.i0 + tx.ip),
                  ci_prob(p, h, w, ty.i0 + ty.ip, tx.i0), ci_prob(p, h, w, ty.i0 + ty.ip, tx.i0 + tx.ip));
}

__global__ void __launch_bounds__(CI_NT) ci_paste_kernel(const float* __restrict__ logits, int64_t n, int h, int w, int f,
                                                         int H_img, int W_img, int H_out, int W_out, int rescale,
                                                         uint8_t* __restrict__ out) {
  const int64_t npix = (int64_t)H_out * W_out;
  const float sh = rs_scale(H_img, H_out, false), sw = rs_scale(W_img, W_out, false);
  for (int64_t k = blockIdx.y; k < n; k += gridDim.y) {
    const float* p = logits + k * h * w;
    uint8_t* o = out + k * npix;
    for (int64_t pix = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; pix < npix; pix += (int64_t)gridDim.x * blockDim.x) {
      const int y = (int)(pix / W_out), x = (int)(pix % W_out);
      float v;
      if (rescale) {
        const RsTap ty = rs_tap(sh, y, H_img, false), tx = rs_tap(sw, x, W_img, false);
        v = rs_lerp2(ty, tx, ci_aligned(p, h, w, f, ty.i0, tx.i0), ci_aligned(p, h, w, f, ty.i0, tx.i0 + tx.ip),
                     ci_aligned(p, h, w, f, ty.i0 + ty.ip, tx.i0), ci_aligned(p, h, w, f, ty.i0 + ty.ip, tx.i0 + tx.ip));
      } else {
        v = ci_aligned(p, h, w, f, y, x);
      }
      o[pix] = v > 0.5f;
    }
  }
}

// The level table from the host arrays.  Checks everything before any device call.
int make_table(CiTable& t, const float* const* cls, const int64_t* cls_st, const float* const* ctr, const int64_t* ctr_st,
               const float* const* bbox, const int64_t* bbox_st, const float* const* param, const int64_t* param_st,
               const int64_t* H, const int64_t* W, const float* stride, const int64_t* k, int64_t n_levels, int64_t B) {
  if (!H || !W || !stride || n_levels <= 0 || B <= 0) return BXS_ERR_INVALID_ARG;
  if (n_levels > CI_MAX_LEVELS || B > CI_MAX_IMGS) return BXS_ERR_UNSUPPORTED;
  t = CiTable{};
  t.n = (int)n_levels;
  for (int64_t l = 0; l < n_levels; ++l) {
    CiLevel& lv = t.lv[l];
    if (H[l] <= 0 || W[l] <= 0) return BXS_ERR_INVALID_ARG;
    if (H[l] * W[l] > INT32_MAX) return BXS_ERR_UNSUPPORTED;
    lv.H = (int)H[l];
    lv.W = (int)W[l];
    lv.stride = stride[l];
    auto take = [&](const float* const* src, const int64_t* st, const float*& p, int64_t* dst) {
      if (!src) return true;
      if (!src[l] || !st) return false;
      p = src[l];
      for (int d = 0; d < 4; ++d) dst[d] = st[4 * l + d];
      return true;
    };
    if (!take(cls, cls_st, lv.cls, lv.cs) || !take(ctr, ctr_st, lv.ctr, lv.ts) || !take(bbox, bbox_st, lv.bbox, lv.bs) ||
        !take(param, param_st, lv.param, lv.ps))
      return BXS_ERR_INVALID_ARG;
    const int64_t hw = H[l] * W[l];
    const int64_t kl = k ? k[l] : hw;
    if (kl < 0 || kl > hw) return BXS_ERR_INVALID_ARG;
    lv.topk = kl < hw;
    lv.slot0 = t.S;
    t.S += kl;
  }
  return BXS_OK;
}

unsigned grid_of(int64_t total) { return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div(total, CI_NT), 4096)); }

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_condinst_point_scores(const float* const* cls_host, const int64_t* cls_strides_host,
                                         const float* const* ctr_host, const int64_t* ctr_strides_host,
                                         const int64_t* height_host, const int64_t* width_host, int64_t n_levels, int64_t B,
                                         int64_t C, int64_t P_max, float* key, bxs_stream_t stream) {
  static const float unit[CI_MAX_LEVELS] = {1, 1, 1, 1, 1, 1, 1, 1};
  CiTable t;
  if (!cls_host || !ctr_host) return BXS_ERR_INVALID_ARG;
  if (int rc = make_table(t, cls_host, cls_strides_host, ctr_host, ctr_strides_host, nullptr, nullptr, nullptr, nullptr,
                          height_host, width_host, unit, nullptr, n_levels, B))
    return rc;
  if (C <= 0 || !key) return BXS_ERR_INVALID_ARG;
  for (int64_t l = 0; l < n_levels; ++l)
    if ((int64_t)t.lv[l].H * t.lv[l].W > P_max) return BXS_ERR_INVALID_ARG;
  ci_key_kernel<<<grid_of(B * n_levels * P_max), CI_NT, 0, as_stream(stream)>>>(t, B, C, P_max, key);
  return check_launch();
}

extern "C" int bxs_condinst_decode(const float* const* cls_host, const int64_t* cls_strides_host, const float* const* ctr_host,
                                   const int64_t* ctr_strides_host, const float* const* bbox_host,
                                   const int64_t* bbox_strides_host, const int64_t* height_host, const int64_t* width_host,
                                   const float* stride_host, const int64_t* k_host, int64_t n_levels, int64_t B, int64_t C,
                                   const int64_t* order, int64_t P_max, const float* img_hw_host, const float* scale_host,
                                   float score_thr, float* box, float* ctr, int64_t* point, uint8_t* cand, float* score,
                                   float* sig, bxs_stream_t stream) {
  CiTable t;
  if (!cls_host || !ctr_host || !bbox_host || !k_host) return BXS_ERR_INVALID_ARG;
  if (int rc = make_table(t, cls_host, cls_strides_host, ctr_host, ctr_strides_host, bbox_host, bbox_strides_host, nullptr,
                          nullptr, height_host, width_host, stride_host, k_host, n_levels, B))
    return rc;
  if (C <= 0 || !img_hw_host || !box || !ctr || !point || !cand || !score) return BXS_ERR_INVALID_ARG;
  bool cut = false;
  for (int64_t l = 0; l < n_levels; ++l) {
    cut |= t.lv[l].topk != 0;
    if ((int64_t)t.lv[l].H * t.lv[l].W > P_max) return BXS_ERR_INVALID_ARG;
  }
  if (cut && !order) return BXS_ERR_INVALID_ARG;
  for (int64_t b = 0; b < B; ++b) {
    t.img_h[b] = img_hw_host[2 * b];
    t.img_w[b] = img_hw_host[2 * b + 1];
    if (scale_host)
      for (int k = 0; k < 4; ++k) t.sf[b][k] = scale_host[4 * b + k];
  }
  t.rescale = scale_host != nullptr;
  if (t.S == 0) return BXS_OK;
  ci_decode_kernel<<<grid_of(B * t.S), CI_NT, 0, as_stream(stream)>>>(t, B, C, order, P_max, score_thr, box, ctr, point, cand,
                                                                     score, sig);
  return check_launch();
}

extern "C" int bxs_condinst_gather(const float* const* param_host, const int64_t* param_strides_host, const int64_t* height_host,
                                   const int64_t* width_host, const float* stride_host, const int64_t* k_host, int64_t n_levels,
                                   int64_t B, int64_t P, const int64_t* point, const int64_t* rows, int64_t n, float* params,
                                   float* coors, int64_t* level, bxs_stream_t stream) {
  CiTable t;
  if (!param_host || !k_host) return BXS_ERR_INVALID_ARG;
  if (int rc = make_table(t, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, param_host, param_strides_host, height_host,
                          width_host, stride_host, k_host, n_levels, B))
    return rc;
  if (P <= 0 || n < 0) return BXS_ERR_INVALID_ARG;
  if (n == 0) return BXS_OK;
  if (!point || !rows || !params || !coors || !level) return BXS_ERR_INVALID_ARG;
  ci_gather_kernel<<<grid_of(n * P), CI_NT, 0, as_stream(stream)>>>(t, P, point, rows, n, params, coors, level);
  return check_launch();
}

extern "C" int64_t bxs_box_nms_workspace_bytes(const int64_t* seg_count_host, int64_t n_seg) {
  if (!seg_count_host || n_seg <= 0) return 0;
  int64_t words = 0;
  for (int64_t s = 0; s < n_seg; ++s) {
    if (seg_count_host[s] < 0) return 0;
    words += seg_count_host[s] * ceil_div(seg_count_host[s], NMS_WORD);
  }
  return words * (int64_t)sizeof(unsigned long long);
}

extern "C" int bxs_box_nms(const float* boxes, const int64_t* seg_start, const int64_t* mask_off, int64_t N, int64_t n_seg,
                           int64_t max_seg, float iou_thr, void* workspace, uint8_t* keep, bxs_stream_t stream) {
  if (N < 0 || n_seg <= 0 || max_seg < 0) return BXS_ERR_INVALID_ARG;
  if (N == 0) return BXS_OK;
  if (!boxes || !seg_start || !mask_off || !workspace || !keep || max_seg == 0) return BXS_ERR_INVALID_ARG;
  if (reinterpret_cast<uintptr_t>(boxes) % 16 || reinterpret_cast<uintptr_t>(workspace) % 8) return BXS_ERR_INVALID_ARG;
  const size_t smem = (size_t)ceil_div(max_seg, NMS_WORD) * sizeof(unsigned long long);
  if (n_seg > INT32_MAX || smem > 48 * 1024) return BXS_ERR_UNSUPPORTED;
  cudaStream_t s = as_stream(stream);
  auto* mask = static_cast<unsigned long long*>(workspace);
  nms_mask_kernel<<<(unsigned)ceil_div(N, CI_NT), CI_NT, 0, s>>>(boxes, seg_start, mask_off, n_seg, N, iou_thr, mask);
  if (int rc = check_launch()) return rc;
  nms_resolve_kernel<<<(unsigned)n_seg, kWarp, smem, s>>>(mask, seg_start, mask_off, keep);
  return check_launch();
}

extern "C" int bxs_condinst_paste_masks(const float* logits, int64_t n, int64_t h, int64_t w, int64_t factor, int64_t H_img,
                                        int64_t W_img, int64_t H_out, int64_t W_out, int rescale, uint8_t* out,
                                        bxs_stream_t stream) {
  if (n < 0 || h <= 0 || w <= 0 || factor <= 0 || H_img <= 0 || W_img <= 0 || H_out <= 0 || W_out <= 0) return BXS_ERR_INVALID_ARG;
  if (H_img > factor * h || W_img > factor * w) return BXS_ERR_INVALID_ARG;     // the crop lies inside the aligned plane
  if (!rescale && (H_out != H_img || W_out != W_img)) return BXS_ERR_INVALID_ARG;
  if (factor * h + 1 > INT32_MAX || factor * w + 1 > INT32_MAX || H_out * W_out > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  if (n == 0) return BXS_OK;
  if (!logits || !out) return BXS_ERR_INVALID_ARG;
  const int64_t npix = H_out * W_out;
  const unsigned gx = (unsigned)std::min<int64_t>(ceil_div(npix, CI_NT), 1024);
  const unsigned gy = (unsigned)std::min<int64_t>(n, 65535);
  ci_paste_kernel<<<dim3(gx, gy), CI_NT, 0, as_stream(stream)>>>(logits, n, (int)h, (int)w, (int)factor, (int)H_img, (int)W_img,
                                                                 (int)H_out, (int)W_out, rescale, out);
  return check_launch();
}
