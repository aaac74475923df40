// Softmax cross-entropy of Box2Mask's classification branch over every decoder layer at once -- box2mask_head.py:248-258
//     self.loss_cls(cls_scores.flatten(0, 1), labels.flatten(0, 1), label_weights, avg_factor=class_weight[labels].sum())
//     with mmdet's CrossEntropyLoss(use_sigmoid=False, reduction='mean', class_weight=w) (cross_entropy_loss.py, utils.py:
//     weight_reduce_loss), once per decoder layer.
//
//     One warp owns one query row: with m the row maximum, d_k = x_k - m and ls = log sum_k exp(d_k), the row's loss
//     w[y] (ls - d_y) and its gradient w[y] (exp(d_k - ls) - [k == y]) * loss_weight / (avg_factor + FLT_EPSILON), written
//     in the same pass.  Every term stays relative to m, as in F.cross_entropy's log_softmax: adding m back (lse = m + ls)
//     before subtracting would round the loss and the softmax to ulp(m), far coarser than a confident row's loss.  avg_factor
//     = sum_i w[y_i] depends on the labels only: every CTA re-reads its layer's B*Q labels in one fixed order, so it is known
//     on the device before the first gradient is written.  Each CTA leaves one FP32 partial; a second launch (one CTA per
//     layer) sums them in a fixed order.  No atomics: loss and gradient are bit-identical from run to run.
#include <cfloat>

#include "common.cuh"

namespace bxs {
namespace {

constexpr int CE_MAX_LAYERS = 16;
constexpr int CE_NT = 256;
constexpr int CE_WARPS = CE_NT / kWarp;
constexpr int CE_ROWS_PER_WARP = 4;
constexpr int CE_ROWS = CE_WARPS * CE_ROWS_PER_WARP;    // query rows per CTA
constexpr int CE_RED_NT = 256;
constexpr int CE_BWD_NT = 256;

struct CeTable {
  const float* scores[CE_MAX_LAYERS];        // [B,Q,K] of layer l
  float* grad[CE_MAX_LAYERS];                // [B,Q,K] of layer l, or null
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(kFull, v, o));
  return v;
}

// the label's class weight, or 0 for a label outside [0, K) (such a row adds nothing anywhere)
__device__ __forceinline__ float label_weight(int64_t y, int64_t K, const float* __restrict__ cw) {
  return (y >= 0 && y < K) ? (cw ? cw[y] : 1.f) : 0.f;
}

__global__ void __launch_bounds__(CE_NT) ce_layers_kernel(const CeTable tab, const int64_t* __restrict__ labels,
                                                           const float* __restrict__ cw, int64_t N, int64_t K,
                                                           int64_t tiles, float loss_weight, float* __restrict__ partials,
                                                           float* __restrict__ avg_out) {
  __shared__ double s_red[CE_NT / kWarp];
  __shared__ float s_avg;
  __shared__ float s_row[CE_WARPS];
  const int64_t cta = blockIdx.x, l = cta / tiles, r0 = (cta - l * tiles) * CE_ROWS;
  const int64_t* lab = labels + l * N;

  // avg_factor of layer l: the same threads, the same order, the same tree in every CTA of the layer
  double a = 0.0;
  for (int64_t i = threadIdx.x; i < N; i += CE_NT) a += label_weight(lab[i], K, cw);
  a = block_sum<double>(a, s_red);
  if (threadIdx.x == 0) {
    s_avg = (float)a;
    if (r0 == 0) avg_out[l] = (float)a;
  }
  __syncthreads();
  const float scale = loss_weight / (s_avg + FLT_EPSILON);     // weight_reduce_loss: sum / (avg_factor + eps)

  const int lane = threadIdx.x % kWarp, warp = threadIdx.x / kWarp;
  const float* __restrict__ x = tab.scores[l];
  float* __restrict__ g = tab.grad[l];
  float acc = 0.f;                                           // lane 0: this warp's rows, in row order
  for (int j = 0; j < CE_ROWS_PER_WARP; ++j) {
    const int64_t row = r0 + warp * CE_ROWS_PER_WARP + j;
    if (row >= N) break;
    const float* xr = x + row * K;
    float m = -INFINITY;
    for (int64_t k = lane; k < K; k += kWarp) m = fmaxf(m, xr[k]);
    m = warp_max(m);
    float s = 0.f;
    for (int64_t k = lane; k < K; k += kWarp) s += expf(xr[k] - m);
    s = warp_sum(s);
    const float ls = logf(s);                                  // log-sum-exp relative to the row maximum
    const int64_t y = lab[row];
    const float w = label_weight(y, K, cw);
    if (lane == 0 && w != 0.f) acc += w * (ls - (xr[y] - m));
    if (g) {
      float* gr = g + row * K;
      const float ws = w * scale;
      for (int64_t k = lane; k < K; k += kWarp) gr[k] = ws * (expf((xr[k] - m) - ls) - (k == y ? 1.f : 0.f));
    }
  }
  if (lane == 0) s_row[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < CE_WARPS; ++w) t += s_row[w];
    partials[cta] = t;
  }
}

__global__ void __launch_bounds__(CE_RED_NT) ce_reduce_kernel(const float* __restrict__ partials, int64_t tiles,
                                                               const float* __restrict__ avg, float loss_weight,
                                                               float* __restrict__ loss) {
  __shared__ double s_red[CE_RED_NT / kWarp];
  const int64_t l = blockIdx.x;
  double acc = 0.0;
  for (int64_t i = threadIdx.x; i < tiles; i += CE_RED_NT) acc += partials[l * tiles + i];
  acc = block_sum<double>(acc, s_red);
  if (threadIdx.x == 0) loss[l] = loss_weight * ((float)acc / (avg[l] + FLT_EPSILON));
}

// grad *= g_loss[l] for every layer; nothing to do for an upstream gradient of exactly 1
__global__ void __launch_bounds__(CE_BWD_NT) ce_scale_kernel(const CeTable tab, const float* __restrict__ g_loss, int64_t n,
                                                              int64_t ctas_per_layer) {
  const int64_t l = blockIdx.x / ctas_per_layer, c = blockIdx.x - l * ctas_per_layer;
  const float s = g_loss[l];
  if (s == 1.f) return;
  float* __restrict__ g = tab.grad[l];
  for (int64_t i = c * CE_BWD_NT + threadIdx.x; i < n; i += ctas_per_layer * CE_BWD_NT) g[i] *= s;
}

// BXS_OK or the status of the first size argument that is out of range
int check_sizes(int64_t L, int64_t B, int64_t Q, int64_t K) {
  if (L <= 0 || B <= 0 || Q <= 0 || K <= 0) return BXS_ERR_INVALID_ARG;
  if (L > CE_MAX_LAYERS) return BXS_ERR_UNSUPPORTED;
  if (B * Q > INT32_MAX || K > INT32_MAX || B * Q > INT64_MAX / K) return BXS_ERR_UNSUPPORTED;
  if (L * ceil_div(B * Q, CE_ROWS) > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  return BXS_OK;
}

size_t partials_bytes(int64_t L, int64_t N) { return align_up((size_t)(L * ceil_div(N, CE_ROWS)) * sizeof(float)); }

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_softmax_cross_entropy_layers_forward_workspace_bytes(int64_t L, int64_t B, int64_t Q) {
  if (check_sizes(L, B, Q, 1) != BXS_OK) return 0;
  return (int64_t)(partials_bytes(L, B * Q) + align_up((size_t)L * sizeof(float)));
}

extern "C" int bxs_softmax_cross_entropy_layers_forward(const float* const* scores_host, const int64_t* labels,
                                                        const float* class_weight, float* const* grad_host, float* loss,
                                                        void* workspace, int64_t L, int64_t B, int64_t Q, int64_t K,
                                                        float loss_weight, bxs_stream_t stream) {
  if (const int rc = check_sizes(L, B, Q, K)) return rc;
  if (!scores_host || !labels || !loss || !workspace) return BXS_ERR_INVALID_ARG;
  CeTable tab{};
  for (int64_t l = 0; l < L; ++l) {
    if (!scores_host[l] || (grad_host && !grad_host[l])) return BXS_ERR_INVALID_ARG;
    tab.scores[l] = scores_host[l];
    tab.grad[l] = grad_host ? grad_host[l] : nullptr;
  }
  const int64_t N = B * Q, tiles = ceil_div(N, CE_ROWS);
  float* partials = static_cast<float*>(workspace);
  float* avg = reinterpret_cast<float*>(static_cast<char*>(workspace) + partials_bytes(L, N));
  const cudaStream_t st = as_stream(stream);
  ce_layers_kernel<<<(unsigned)(L * tiles), CE_NT, 0, st>>>(tab, labels, class_weight, N, K, tiles, loss_weight, partials,
                                                             avg);
  if (const int rc = check_launch()) return rc;
  ce_reduce_kernel<<<(unsigned)L, CE_RED_NT, 0, st>>>(partials, tiles, avg, loss_weight, loss);
  return check_launch();
}

extern "C" int bxs_softmax_cross_entropy_layers_backward(float* const* grad_host, const float* g_loss, int64_t L, int64_t B,
                                                         int64_t Q, int64_t K, bxs_stream_t stream) {
  if (const int rc = check_sizes(L, B, Q, K)) return rc;
  if (!grad_host || !g_loss) return BXS_ERR_INVALID_ARG;
  CeTable tab{};
  for (int64_t l = 0; l < L; ++l) {
    if (!grad_host[l]) return BXS_ERR_INVALID_ARG;
    tab.grad[l] = grad_host[l];
  }
  const int64_t n = B * Q * K;
  const int64_t per_layer = std::min<int64_t>(ceil_div(n, CE_BWD_NT), std::max<int64_t>(1, 4 * sm_count() / L));
  ce_scale_kernel<<<(unsigned)(L * per_layer), CE_BWD_NT, 0, as_stream(stream)>>>(tab, g_loss, n, per_layer);
  return check_launch();
}
