// Sigmoid focal loss over every FPN level at once -- BoxSOLOv2's category branch (box_solov2_head.py:370-383)
//     self.loss_cate(cat([cate_pred.permute(0,2,3,1).reshape(-1,C) for each level]), cat(labels), avg_factor=num_ins + 1)
//     and CondInstBoxHead's classification branch on the rectangular FCOS levels (condinst_head.py:404-445, avg_factor =
//     num_pos), with mmdet's FocalLoss(use_sigmoid=True) (mmdet/models/losses/focal_loss.py, utils.py: weight_reduce_loss).
//
//     The logits stay in each level's own NCHW layout: a CTA owns FL_TILE cells of one (level, image), loads their labels once,
//     walks the C class planes with reads coalesced along the cells, writes d loss / d logit in the same pass and leaves one
//     FP32 partial.  A second, one-CTA launch sums the partials in a fixed order: loss and gradient are bit-identical from
//     run to run (no atomics).  avg_factor is read on the device, so nothing synchronises with the host.
#include <cfloat>

#include "common.cuh"

namespace bxs {
namespace {

constexpr int FL_MAX_LEVELS = 8;
constexpr int FL_TILE = 64;                  // cells per CTA (one warp pair of a class plane)
constexpr int FL_NT = 256;                   // FL_NT / FL_TILE class planes in flight per CTA
constexpr int FL_GROUPS = FL_NT / FL_TILE;
constexpr int FL_RED_NT = 1024;

struct FocalLevel {
  const float* logits;                       // [B,C,S2]
  const int64_t* labels;                     // [B,S2]
  float* grad;                               // [B,C,S2] or null
  int64_t S2;
  int64_t tiles;                             // CTAs per image
};

struct FocalTable {
  FocalLevel lv[FL_MAX_LEVELS];
  int64_t first[FL_MAX_LEVELS + 1];          // first CTA of each level; first[n_levels] = grid size
  int n_levels;
};

// loss and d loss / dx of one element: the stable form of py_sigmoid_focal_loss (BCE-with-logits as a softplus, times
// (alpha t + (1-alpha)(1-t)) pt^gamma).  log p and log(1-p) share one softplus term (log_sigmoid_pair).
__device__ __forceinline__ float focal_element(float x, bool pos, float gamma, float alpha, float& dx) {
  float lp, lm;
  log_sigmoid_pair(x, lp, lm);
  const float p = expf(lp), q = expf(lm);    // p = sigmoid(x), q = 1 - p, both without cancellation
  if (pos) {
    const float w = alpha * powf(q, gamma);
    dx = -w * (q - gamma * p * lp);          // -alpha (1-p)^g (1 - p - g p log p)
    return -w * lp;                          // alpha (1-p)^g softplus(-x)
  }
  const float w = (1.f - alpha) * powf(p, gamma);
  dx = -w * (gamma * q * lm - p);            // -(1-alpha) p^g (g (1-p) log(1-p) - p)
  return -w * lm;                            // (1-alpha) p^g softplus(x)
}

__global__ void __launch_bounds__(FL_NT) focal_levels_kernel(const FocalTable tab, int C, const float* __restrict__ avg_factor,
                                                              float gamma, float alpha, float loss_weight,
                                                              float* __restrict__ partials) {
  __shared__ int s_lab[FL_TILE];
  __shared__ float s_red[FL_NT / kWarp];
  const int64_t cta = blockIdx.x;
  int l = 0;
  while (l + 1 < tab.n_levels && tab.first[l + 1] <= cta) ++l;
  const FocalLevel lv = tab.lv[l];
  const int64_t local = cta - tab.first[l], b = local / lv.tiles, c0 = (local - b * lv.tiles) * FL_TILE;
  const int n = lv.S2 - c0 < FL_TILE ? (int)(lv.S2 - c0) : FL_TILE;
  if (threadIdx.x < n) {
    const int64_t t = lv.labels[b * lv.S2 + c0 + threadIdx.x];
    s_lab[threadIdx.x] = (t >= 0 && t < C) ? (int)t : -1;     // outside [0, C): background, every class negative
  }
  __syncthreads();
  const float scale = loss_weight / (*avg_factor + FLT_EPSILON);     // weight_reduce_loss: sum / (avg_factor + eps)
  const int cell = threadIdx.x % FL_TILE, grp = threadIdx.x / FL_TILE;
  float acc = 0.f;
  if (cell < n) {
    const int lab = s_lab[cell];
    const int64_t base = b * C * lv.S2 + c0 + cell;
    for (int c = grp; c < C; c += FL_GROUPS) {
      const int64_t i = base + (int64_t)c * lv.S2;
      float dx;
      acc += focal_element(lv.logits[i], c == lab, gamma, alpha, dx);
      if (lv.grad) lv.grad[i] = dx * scale;
    }
  }
  acc = block_sum<float>(acc, s_red);
  if (threadIdx.x == 0) partials[cta] = acc;
}

__global__ void __launch_bounds__(FL_RED_NT) focal_reduce_kernel(const float* __restrict__ partials, int64_t n,
                                                                 const float* __restrict__ avg_factor, float loss_weight,
                                                                 float* __restrict__ loss) {
  __shared__ double s_red[FL_RED_NT / kWarp];
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += FL_RED_NT) acc += partials[i];
  acc = block_sum<double>(acc, s_red);
  if (threadIdx.x == 0) *loss = loss_weight * ((float)acc / (*avg_factor + FLT_EPSILON));
}

// fills the level table from each level's cell count (H_l * W_l); BXS_OK or the status of the first argument that is out of
// range
int plan(FocalTable& tab, const int64_t* cells_host, int64_t n_levels, int64_t B, int64_t C) {
  if (!cells_host || n_levels <= 0 || B <= 0 || C <= 0) return BXS_ERR_INVALID_ARG;
  if (n_levels > FL_MAX_LEVELS) return BXS_ERR_UNSUPPORTED;
  if (C > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  tab = FocalTable{};
  tab.n_levels = (int)n_levels;
  int64_t total = 0;
  for (int64_t l = 0; l < n_levels; ++l) {
    const int64_t n = cells_host[l];
    if (n <= 0) return BXS_ERR_INVALID_ARG;
    if (n > (int64_t(1) << 30)) return BXS_ERR_UNSUPPORTED;          // S2 * B * C stays far inside int64
    tab.lv[l].S2 = n;
    tab.lv[l].tiles = ceil_div(n, FL_TILE);
    tab.first[l] = total;
    total += B * tab.lv[l].tiles;
  }
  tab.first[n_levels] = total;
  return total > INT32_MAX ? BXS_ERR_UNSUPPORTED : BXS_OK;
}

// the square-grid form: S_l <= 0 stays invalid, S_l > 2^15 (more than 2^30 cells) stays unsupported
int plan_grid(FocalTable& tab, const int64_t* grid_host, int64_t n_levels, int64_t B, int64_t C) {
  if (!grid_host || n_levels <= 0 || n_levels > FL_MAX_LEVELS) return plan(tab, grid_host, n_levels, B, C);
  int64_t cells[FL_MAX_LEVELS];
  for (int64_t l = 0; l < n_levels; ++l) {
    const int64_t S = grid_host[l];
    cells[l] = S <= 0 ? S : S > (1 << 15) ? (int64_t(1) << 31) : S * S;
  }
  return plan(tab, cells, n_levels, B, C);
}

// fills the table's pointers and runs both launches
int focal_forward(FocalTable& tab, const float* const* logits_host, const int64_t* const* labels_host,
                  float* const* grad_host, const float* avg_factor, float* loss, void* workspace, int64_t C, float gamma,
                  float alpha, float loss_weight, bxs_stream_t stream) {
  if (!logits_host || !labels_host || !avg_factor || !loss || !workspace || !(gamma >= 0.f)) return BXS_ERR_INVALID_ARG;
  const int64_t n_levels = tab.n_levels;
  for (int64_t l = 0; l < n_levels; ++l) {
    if (!logits_host[l] || !labels_host[l] || (grad_host && !grad_host[l])) return BXS_ERR_INVALID_ARG;
    tab.lv[l].logits = logits_host[l];
    tab.lv[l].labels = labels_host[l];
    tab.lv[l].grad = grad_host ? grad_host[l] : nullptr;
  }
  const cudaStream_t st = as_stream(stream);
  float* partials = static_cast<float*>(workspace);
  const int64_t ctas = tab.first[n_levels];
  focal_levels_kernel<<<(unsigned)ctas, FL_NT, 0, st>>>(tab, (int)C, avg_factor, gamma, alpha, loss_weight, partials);
  if (const int rc = check_launch()) return rc;
  focal_reduce_kernel<<<1, FL_RED_NT, 0, st>>>(partials, ctas, avg_factor, loss_weight, loss);
  return check_launch();
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(const int64_t* grid_host, int64_t n_levels, int64_t B) {
  FocalTable tab;
  if (plan_grid(tab, grid_host, n_levels, B, 1) != BXS_OK) return 0;
  return (int64_t)align_up((size_t)tab.first[n_levels] * sizeof(float));
}

extern "C" int bxs_sigmoid_focal_loss_levels_forward(const float* const* logits_host, const int64_t* const* labels_host,
                                                     const int64_t* grid_host, float* const* grad_host,
                                                     const float* avg_factor, float* loss, void* workspace, int64_t n_levels,
                                                     int64_t B, int64_t C, float gamma, float alpha, float loss_weight,
                                                     bxs_stream_t stream) {
  FocalTable tab;
  if (const int rc = plan_grid(tab, grid_host, n_levels, B, C)) return rc;
  return focal_forward(tab, logits_host, labels_host, grad_host, avg_factor, loss, workspace, C, gamma, alpha, loss_weight,
                       stream);
}

extern "C" int64_t bxs_sigmoid_focal_loss_cells_forward_workspace_bytes(const int64_t* cells_host, int64_t n_levels, int64_t B) {
  FocalTable tab;
  if (plan(tab, cells_host, n_levels, B, 1) != BXS_OK) return 0;
  return (int64_t)align_up((size_t)tab.first[n_levels] * sizeof(float));
}

extern "C" int bxs_sigmoid_focal_loss_cells_forward(const float* const* logits_host, const int64_t* const* labels_host,
                                                    const int64_t* cells_host, float* const* grad_host,
                                                    const float* avg_factor, float* loss, void* workspace, int64_t n_levels,
                                                    int64_t B, int64_t C, float gamma, float alpha, float loss_weight,
                                                    bxs_stream_t stream) {
  FocalTable tab;
  if (const int rc = plan(tab, cells_host, n_levels, B, C)) return rc;
  return focal_forward(tab, logits_host, labels_host, grad_host, avg_factor, loss, workspace, C, gamma, alpha, loss_weight,
                       stream);
}
