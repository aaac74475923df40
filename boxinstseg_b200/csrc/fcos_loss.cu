// The regression and centerness losses of CondInstBoxHead.loss over every FCOS level and image at once --
// condinst_head.py:437-469 with GIoULoss and CrossEntropyLoss(use_sigmoid=True), reduction 'mean' (losses/iou_loss.py,
// cross_entropy_loss.py, utils.py: weight_reduce_loss).
//
//     bbox_pred [B,4,H,W] and centerness [B,1,H,W] of each level are read in place (no permute / cat); the labels and
//     regression targets are bxs_fcos_targets' per-level outputs, point b*H*W + y*W + x of a level.  One thread per
//     (level, image, point):
//       stats  the positive count and the sum of the positives' centerness targets, as per-CTA partials;
//       loss   for a positive ct * (1 - GIoU) and BCE(centerness, ct), and their gradients already scaled by
//              loss_weight / (denominator + FLT_EPSILON); a zero gradient for every other point.  The denominators are
//              read on the device.
//     A one-CTA launch sums each kind of partial in a fixed order.  No atomics and no host synchronisation: losses and
//     gradients are bit-identical from run to run, and the positive count never leaves the device.
#include <cfloat>

#include "common.cuh"
#include "fcos_loss_core.cuh"

namespace bxs {
namespace {

constexpr int FC_MAX_LEVELS = 8;
constexpr int FC_NT = 256;
constexpr int FC_RED_NT = 1024;
constexpr int FC_BWD_NT = 256;

struct FcLevel {
  const float* pred;                         // [B,4,H,W]
  const float* ctr;                          // [B,1,H,W]
  const int64_t* labels;                     // [B*H*W]
  const float* targets;                      // [B*H*W,4]
  float* g_pred;                             // [B,4,H,W] or null
  float* g_ctr;                              // [B,1,H,W] or null
  int64_t P;                                 // H*W
  int64_t W;
  float stride;
};

struct FcTable {
  FcLevel lv[FC_MAX_LEVELS];
  int64_t first[FC_MAX_LEVELS + 1];          // first flattened point of each level; first[n_levels] = B * sum H*W
  int n_levels;
};

struct FcPoint {
  int l;
  int64_t i, b, p;                           // point of the level, its image, its cell y*W + x
};

__device__ __forceinline__ FcPoint locate(const FcTable& tab, int64_t g) {
  FcPoint r;
  r.l = 0;
  while (r.l + 1 < tab.n_levels && tab.first[r.l + 1] <= g) ++r.l;
  r.i = g - tab.first[r.l];
  r.b = r.i / tab.lv[r.l].P;
  r.p = r.i - r.b * tab.lv[r.l].P;
  return r;
}

__device__ __forceinline__ void load_target(const float* t, int64_t i, float v[4]) {
#pragma unroll
  for (int k = 0; k < 4; ++k) v[k] = t[i * 4 + k];
}

// partials[2 * cta + {0, 1}] = (positives, sum of their centerness targets)
__global__ void __launch_bounds__(FC_NT) fcos_stats_kernel(const FcTable tab, int64_t C, float* __restrict__ partials) {
  __shared__ double s_red[FC_NT / kWarp];
  const int64_t g = (int64_t)blockIdx.x * FC_NT + threadIdx.x;
  double n = 0.0, ct = 0.0;
  if (g < tab.first[tab.n_levels]) {
    const FcPoint q = locate(tab, g);
    const FcLevel& lv = tab.lv[q.l];
    const int64_t lab = lv.labels[q.i];
    if (lab >= 0 && lab < C) {
      float t[4];
      load_target(lv.targets, q.i, t);
      n = 1.0;
      ct = fcos_centerness_target(t);
    }
  }
  n = block_sum<double>(n, s_red);
  ct = block_sum<double>(ct, s_red);
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = (float)n;
    partials[2 * blockIdx.x + 1] = (float)ct;
  }
}

// den[0] = max(reduce_mean(num_pos), 1), den[1] = max(reduce_mean(sum ct), 1e-6); partials as in fcos_stats_kernel but
// (sum ct * (1 - GIoU), sum BCE)
__global__ void __launch_bounds__(FC_NT) fcos_loss_kernel(const FcTable tab, int64_t C, const float* __restrict__ den,
                                                          float lw_bbox, float lw_ctr, float* __restrict__ partials) {
  __shared__ double s_red[FC_NT / kWarp];
  const int64_t g = (int64_t)blockIdx.x * FC_NT + threadIdx.x;
  float bbox = 0.f, ctr = 0.f;
  if (g < tab.first[tab.n_levels]) {
    const FcPoint q = locate(tab, g);
    const FcLevel& lv = tab.lv[q.l];
    const int64_t P = lv.P, base = q.b * 4 * P + q.p;
    const int64_t lab = lv.labels[q.i];
    float gp[4] = {0.f, 0.f, 0.f, 0.f}, gc = 0.f;
    if (lab >= 0 && lab < C) {
      float t[4], d[4];
      load_target(lv.targets, q.i, t);
#pragma unroll
      for (int k = 0; k < 4; ++k) d[k] = lv.pred[base + k * P];
      const int64_t y = q.p / lv.W, x = q.p - y * lv.W;
      const FcosPointLoss r = fcos_point_loss(fcos_point_coord(x, lv.stride), fcos_point_coord(y, lv.stride), d, t,
                                              lv.ctr[q.b * P + q.p]);
      bbox = r.bbox;
      ctr = r.ctr;
      const float sb = lw_bbox / (den[1] + FLT_EPSILON), sc = lw_ctr / (den[0] + FLT_EPSILON);
#pragma unroll
      for (int k = 0; k < 4; ++k) gp[k] = r.g_pred[k] * sb;
      gc = r.g_ctr * sc;
    }
    if (lv.g_pred) {
#pragma unroll
      for (int k = 0; k < 4; ++k) lv.g_pred[base + k * P] = gp[k];
    }
    if (lv.g_ctr) lv.g_ctr[q.b * P + q.p] = gc;
  }
  const double sb = block_sum<double>(bbox, s_red);
  const double sc = block_sum<double>(ctr, s_red);
  if (threadIdx.x == 0) {
    partials[2 * blockIdx.x] = (float)sb;
    partials[2 * blockIdx.x + 1] = (float)sc;
  }
}

// sums both columns of the [n,2] partials in a fixed order.  den == null: (out0, out1) = the sums (stats); else out0 =
// lw_bbox * sum0 / (den[1] + eps), out1 = lw_ctr * sum1 / (den[0] + eps) (weight_reduce_loss, then loss_weight *)
__global__ void __launch_bounds__(FC_RED_NT) fcos_sum_kernel(const float* __restrict__ partials, int64_t n,
                                                             const float* __restrict__ den, float lw_bbox, float lw_ctr,
                                                             float* __restrict__ out0, float* __restrict__ out1) {
  __shared__ double s_red[FC_RED_NT / kWarp];
  double a0 = 0.0, a1 = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += FC_RED_NT) {
    a0 += partials[2 * i];
    a1 += partials[2 * i + 1];
  }
  a0 = block_sum<double>(a0, s_red);
  a1 = block_sum<double>(a1, s_red);
  if (threadIdx.x == 0) {
    if (den) {
      *out0 = lw_bbox * ((float)a0 / (den[1] + FLT_EPSILON));
      *out1 = lw_ctr * ((float)a1 / (den[0] + FLT_EPSILON));
    } else {
      *out0 = (float)a0;
      *out1 = (float)a1;
    }
  }
}

// g_pred *= *s_pred, g_ctr *= *s_ctr; nothing to do for an upstream gradient of exactly 1
__global__ void __launch_bounds__(FC_BWD_NT) fcos_scale_kernel(float* __restrict__ g_pred, int64_t n_pred,
                                                               const float* __restrict__ s_pred, float* __restrict__ g_ctr,
                                                               int64_t n_ctr, const float* __restrict__ s_ctr) {
  const float a = g_pred ? *s_pred : 1.f, c = g_ctr ? *s_ctr : 1.f;
  if (a == 1.f && c == 1.f) return;
  const int64_t step = (int64_t)gridDim.x * FC_BWD_NT;
  if (a != 1.f)
    for (int64_t i = (int64_t)blockIdx.x * FC_BWD_NT + threadIdx.x; i < n_pred; i += step) g_pred[i] *= a;
  if (c != 1.f)
    for (int64_t i = (int64_t)blockIdx.x * FC_BWD_NT + threadIdx.x; i < n_ctr; i += step) g_ctr[i] *= c;
}

// fills the level table's shapes; BXS_OK or the status of the first argument that is out of range
int plan(FcTable& tab, const int64_t* height_host, const int64_t* width_host, const float* stride_host, int64_t n_levels,
         int64_t B, int64_t C) {
  if (!height_host || !width_host || !stride_host || n_levels <= 0 || B <= 0 || C <= 0) return BXS_ERR_INVALID_ARG;
  if (n_levels > FC_MAX_LEVELS || C > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  tab = FcTable{};
  tab.n_levels = (int)n_levels;
  int64_t total = 0;
  for (int64_t l = 0; l < n_levels; ++l) {
    const int64_t H = height_host[l], W = width_host[l];
    if (H <= 0 || W <= 0 || !(stride_host[l] > 0.f) || !(stride_host[l] < INFINITY)) return BXS_ERR_INVALID_ARG;
    if (H > INT32_MAX || W > INT32_MAX || H * W > INT32_MAX || B * H * W > INT32_MAX) return BXS_ERR_UNSUPPORTED;
    tab.lv[l].P = H * W;
    tab.lv[l].W = W;
    tab.lv[l].stride = stride_host[l];
    tab.first[l] = total;
    total += B * H * W;
    if (total > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  }
  tab.first[n_levels] = total;
  return BXS_OK;
}

int64_t ctas_of(const FcTable& tab) { return ceil_div(tab.first[tab.n_levels], FC_NT); }

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_fcos_loss_workspace_bytes(const int64_t* height_host, const int64_t* width_host, int64_t n_levels,
                                                 int64_t B) {
  FcTable tab;
  float strides[FC_MAX_LEVELS];
  for (int l = 0; l < FC_MAX_LEVELS; ++l) strides[l] = 1.f;
  if (plan(tab, height_host, width_host, strides, n_levels, B, 1) != BXS_OK) return 0;
  return (int64_t)align_up((size_t)ctas_of(tab) * 2 * sizeof(float));
}

extern "C" int bxs_fcos_loss_stats(const int64_t* const* labels_host, const float* const* targets_host,
                                   const int64_t* height_host, const int64_t* width_host, const float* stride_host,
                                   float* stats, void* workspace, int64_t n_levels, int64_t B, int64_t C,
                                   bxs_stream_t stream) {
  FcTable tab;
  if (const int rc = plan(tab, height_host, width_host, stride_host, n_levels, B, C)) return rc;
  if (!labels_host || !targets_host || !stats || !workspace) return BXS_ERR_INVALID_ARG;
  for (int64_t l = 0; l < n_levels; ++l) {
    if (!labels_host[l] || !targets_host[l]) return BXS_ERR_INVALID_ARG;
    tab.lv[l].labels = labels_host[l];
    tab.lv[l].targets = targets_host[l];
  }
  const cudaStream_t st = as_stream(stream);
  float* partials = static_cast<float*>(workspace);
  const int64_t ctas = ctas_of(tab);
  fcos_stats_kernel<<<(unsigned)ctas, FC_NT, 0, st>>>(tab, C, partials);
  if (const int rc = check_launch()) return rc;
  fcos_sum_kernel<<<1, FC_RED_NT, 0, st>>>(partials, ctas, nullptr, 0.f, 0.f, stats, stats + 1);
  return check_launch();
}

extern "C" int bxs_fcos_loss_forward(const float* const* pred_host, const float* const* ctr_host,
                                     const int64_t* const* labels_host, const float* const* targets_host,
                                     float* const* g_pred_host, float* const* g_ctr_host, const int64_t* height_host,
                                     const int64_t* width_host, const float* stride_host, const float* den, float* loss_bbox,
                                     float* loss_ctr, void* workspace, int64_t n_levels, int64_t B, int64_t C, float lw_bbox, float lw_ctr,
                                     bxs_stream_t stream) {
  FcTable tab;
  if (const int rc = plan(tab, height_host, width_host, stride_host, n_levels, B, C)) return rc;
  if (!pred_host || !ctr_host || !labels_host || !targets_host || !den || !loss_bbox || !loss_ctr || !workspace) return BXS_ERR_INVALID_ARG;
  for (int64_t l = 0; l < n_levels; ++l) {
    if (!pred_host[l] || !ctr_host[l] || !labels_host[l] || !targets_host[l] || (g_pred_host && !g_pred_host[l]) ||
        (g_ctr_host && !g_ctr_host[l]))
      return BXS_ERR_INVALID_ARG;
    FcLevel& lv = tab.lv[l];
    lv.pred = pred_host[l];
    lv.ctr = ctr_host[l];
    lv.labels = labels_host[l];
    lv.targets = targets_host[l];
    lv.g_pred = g_pred_host ? g_pred_host[l] : nullptr;
    lv.g_ctr = g_ctr_host ? g_ctr_host[l] : nullptr;
  }
  const cudaStream_t st = as_stream(stream);
  float* partials = static_cast<float*>(workspace);
  const int64_t ctas = ctas_of(tab);
  fcos_loss_kernel<<<(unsigned)ctas, FC_NT, 0, st>>>(tab, C, den, lw_bbox, lw_ctr, partials);
  if (const int rc = check_launch()) return rc;
  fcos_sum_kernel<<<1, FC_RED_NT, 0, st>>>(partials, ctas, den, lw_bbox, lw_ctr, loss_bbox, loss_ctr);
  return check_launch();
}

extern "C" int bxs_fcos_loss_backward(float* g_pred, int64_t n_pred, const float* g_loss_bbox, float* g_ctr, int64_t n_ctr,
                                      const float* g_loss_ctr, bxs_stream_t stream) {
  if (n_pred < 0 || n_ctr < 0 || (g_pred && !g_loss_bbox) || (g_ctr && !g_loss_ctr) || (!g_pred && n_pred) ||
      (!g_ctr && n_ctr))
    return BXS_ERR_INVALID_ARG;
  const int64_t n = std::max(n_pred, n_ctr);
  if (n == 0) return BXS_OK;
  const int64_t ctas = std::min<int64_t>(ceil_div(n, FC_BWD_NT), 4 * (int64_t)sm_count());
  fcos_scale_kernel<<<(unsigned)ctas, FC_BWD_NT, 0, as_stream(stream)>>>(g_pred, n_pred, g_loss_bbox, g_ctr, n_ctr,
                                                                        g_loss_ctr);
  return check_launch();
}
