// CondInst's mask-supervised losses: the dice mask loss of CondInstMaskHead.loss with boxinst_enabled=False
// (condinst_head.py:117-131, 1298-1341) and the semantic targets of CondInstSegmHead (:950-968).
//
//     The ground-truth masks are read in place: each image's uint8 [G_b, H, W] masks, at any strides, travel in a table in
//     the kernel parameters together with the images' ground-truth offsets.  No [N, h, w] target and no [G, H, W]
//     temporary exists.
//
//     dice   target pixel (y, x) of instance i = mask[gt_inds[i]][start + y*s, start + x*s] as a float (the reference's
//            m[:, start::s, start::s].to(float)).  A (chunk, instance) CTA grid writes double partials of
//            I = sum sigmoid(x) * t, S = sum sigmoid(x)^2 and T = sum t^2; one CTA sums them in a fixed order, and writes
//            the sums and mean_i(1 - 2 I_i / (S_i + T_i + 1e-5)).  The backward reads the logits and targets once more.
//     semantic  areas (an int64 sum of the byte values of each mask), then at each sampled pixel the label of the first
//            ground truth of least weight (area where the mask is non-zero, 1e8 elsewhere); num_classes where that
//            weight is 1e8.
//
//     No float atomics and no host synchronisation: every result is bit-identical from run to run.
#include "common.cuh"

namespace bxs {
namespace {

constexpr int CS_MAX_IMAGES = 64;
constexpr int CS_NT = 256;
constexpr int CS_PER_THREAD = 16;                  // pixels per thread of a dice chunk, all loads issued before any use
constexpr int64_t CS_CHUNK = (int64_t)CS_NT * CS_PER_THREAD;
constexpr int CS_RED_NT = 1024;
constexpr int CS_AREA_ROWS = 16;                   // mask rows per CTA of the area sum
constexpr int64_t CS_INF = 100000000;              // condinst_head.py:16, INF = 1e8 assigned into an int64 tensor

struct CsImage {
  const uint8_t* mask;                             // [G_b, H, W] at element strides sg, sh, sw
  const int64_t* labels;                           // [G_b] (semantic targets only)
  int64_t sg, sh, sw;
};

struct CsTable {
  CsImage im[CS_MAX_IMAGES];
  int64_t gt_first[CS_MAX_IMAGES + 1];             // first global ground-truth index of each image; [B] = sum G_b
  int n_images;
};

// the image of global ground truth `gt` (gt_first[n_images] > gt >= 0)
__device__ __forceinline__ int image_of(const CsTable& tab, int64_t gt) {
  int b = 0;
  while (b + 1 < tab.n_images && tab.gt_first[b + 1] <= gt) ++b;
  return b;
}

// ground truth gt's mask, or null when gt is outside [0, sum G_b)
__device__ __forceinline__ const uint8_t* gt_mask(const CsTable& tab, int64_t gt, int64_t& sh, int64_t& sw) {
  if (gt < 0 || gt >= tab.gt_first[tab.n_images]) return nullptr;
  const int b = image_of(tab, gt);
  const CsImage& im = tab.im[b];
  sh = im.sh;
  sw = im.sw;
  return im.mask + (gt - tab.gt_first[b]) * im.sg;
}

// torch's sigmoid: 1 / (1 + exp(-x)), with exp(-|x|) so that the small side keeps its relative precision
__device__ __forceinline__ float sigmoid_acc(float x, float& one_minus) {
  const float e = expf(-fabsf(x));
  const float big = 1.f / (1.f + e), small = e * big;
  one_minus = x >= 0.f ? small : big;
  return x >= 0.f ? big : small;
}

// the CTA's CS_PER_THREAD pixels per thread of instance i: logits v, targets t (0 past the end)
__device__ __forceinline__ void load_chunk(const float* __restrict__ x, const uint8_t* m, int64_t sh, int64_t sw,
                                           uint32_t hw, uint32_t w, int64_t start, int64_t s, float v[CS_PER_THREAD],
                                           float t[CS_PER_THREAD]) {
  const uint32_t p0 = blockIdx.x * (uint32_t)CS_CHUNK + threadIdx.x;
#pragma unroll
  for (int k = 0; k < CS_PER_THREAD; ++k) {
    const uint32_t p = p0 + k * CS_NT;
    v[k] = p < hw ? __ldg(x + p) : 0.f;
    uint32_t byte = 0;
    if (p < hw && m) {
      const uint32_t y = p / w, c = p - y * w;
      byte = __ldg(m + (start + (int64_t)y * s) * sh + (start + (int64_t)c * s) * sw);
    }
    t[k] = (float)byte;
  }
}

// partials[(i * chunks + chunk) * 3 + {0, 1, 2}] = this CTA's (I, S, T) of instance i = blockIdx.y; T is NaN for a
// ground-truth index outside the table
__global__ void __launch_bounds__(CS_NT) dice_partials_kernel(const float* __restrict__ logits,
                                                              const int32_t* __restrict__ gt_inds, const CsTable tab,
                                                              uint32_t hw, uint32_t w, int64_t start, int64_t s,
                                                              double* __restrict__ partials) {
  __shared__ double s_red[CS_NT / kWarp];
  const int64_t i = blockIdx.y;
  int64_t sh = 0, sw = 0;
  const uint8_t* m = gt_mask(tab, gt_inds[i], sh, sw);
  float v[CS_PER_THREAD], t[CS_PER_THREAD];
  load_chunk(logits + i * hw, m, sh, sw, hw, w, start, s, v, t);
  const uint32_t p0 = blockIdx.x * (uint32_t)CS_CHUNK + threadIdx.x;
  float I = 0.f, S = 0.f, T = 0.f;
#pragma unroll
  for (int k = 0; k < CS_PER_THREAD; ++k) {
    if (p0 + k * CS_NT < hw) {
      float om;
      const float sg = sigmoid_acc(v[k], om);
      I += sg * t[k];
      S += sg * sg;
      T += t[k] * t[k];
    }
  }
  const double dI = block_sum<double>(I, s_red);
  const double dS = block_sum<double>(S, s_red);
  const double dT = block_sum<double>(T, s_red);
  if (threadIdx.x == 0) {
    double* out = partials + (i * gridDim.x + blockIdx.x) * 3;
    out[0] = dI;
    out[1] = dS;
    out[2] = m ? dT : __longlong_as_double(0x7ff8000000000000ll);
  }
}

// one CTA: warp k sums the partials of instances k, k + 32, ... in chunk order -> sums [N,3] (float), and
// loss = mean_i(1 - 2 I / (S + T + 1e-5)) with each instance's term in the reference's float32 operation order
__global__ void __launch_bounds__(CS_RED_NT) dice_finalize_kernel(const double* __restrict__ partials, int64_t N,
                                                                  int64_t chunks, float* __restrict__ sums,
                                                                  float* __restrict__ loss) {
  __shared__ double s_red[CS_RED_NT / kWarp];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  double acc = 0.0;
  for (int64_t i = wid; i < N; i += CS_RED_NT / kWarp) {
    double a[3] = {0.0, 0.0, 0.0};
    for (int64_t c = lane; c < chunks; c += kWarp)
#pragma unroll
      for (int q = 0; q < 3; ++q) a[q] += partials[(i * chunks + c) * 3 + q];
#pragma unroll
    for (int q = 0; q < 3; ++q) a[q] = warp_sum(a[q]);
    if (lane == 0) {
      const float I = (float)a[0], S = (float)a[1], T = (float)a[2];
      sums[3 * i] = I;
      sums[3 * i + 1] = S;
      sums[3 * i + 2] = T;
      acc += (double)(1.f - (2.f * I) / ((S + T) + 1e-5f));
    }
  }
  acc = block_sum<double>(acc, s_red);
  if (threadIdx.x == 0) *loss = (float)(acc / (double)N);
}

// g_logits[i, p] = g * (2 / N) * (2 I sigma / U^2 - t / U) * sigma * (1 - sigma), U = S + T + 1e-5 (NaN throughout for a
// ground-truth index outside the table: its T is NaN)
__global__ void __launch_bounds__(CS_NT) dice_backward_kernel(const float* __restrict__ logits,
                                                              const int32_t* __restrict__ gt_inds, const CsTable tab,
                                                              uint32_t hw, uint32_t w, int64_t start, int64_t s,
                                                              int64_t N, const float* __restrict__ sums,
                                                              const float* __restrict__ g_loss,
                                                              float* __restrict__ g_logits) {
  const int64_t i = blockIdx.y;
  int64_t sh = 0, sw = 0;
  const uint8_t* m = gt_mask(tab, gt_inds[i], sh, sw);
  float v[CS_PER_THREAD], t[CS_PER_THREAD];
  load_chunk(logits + i * hw, m, sh, sw, hw, w, start, s, v, t);
  const double U = (double)((sums[3 * i + 1] + sums[3 * i + 2]) + 1e-5f);
  const double b = (double)*g_loss * 2.0 / ((double)N * U);
  const float cb = (float)b, ca = (float)(b * 2.0 * (double)sums[3 * i] / U);
  float* out = g_logits + i * hw;
  const uint32_t p0 = blockIdx.x * (uint32_t)CS_CHUNK + threadIdx.x;
#pragma unroll
  for (int k = 0; k < CS_PER_THREAD; ++k) {
    const uint32_t p = p0 + k * CS_NT;
    if (p < hw) {
      float om;
      const float sg = sigmoid_acc(v[k], om);
      out[p] = (ca * sg - cb * t[k]) * (sg * om);
    }
  }
}

// areas[gt] += the byte values of CS_AREA_ROWS rows of ground truth gt = blockIdx.y (areas zeroed before); integer
// atomics, so the sum does not depend on their order
__global__ void __launch_bounds__(CS_NT) semantic_areas_kernel(const CsTable tab, int64_t H, int64_t W,
                                                               unsigned long long* __restrict__ areas) {
  __shared__ unsigned long long s_red[CS_NT / kWarp];
  const int64_t gt = blockIdx.y;
  const int b = image_of(tab, gt);
  const CsImage& im = tab.im[b];
  const uint8_t* m = im.mask + (gt - tab.gt_first[b]) * im.sg;
  const int64_t r0 = (int64_t)blockIdx.x * CS_AREA_ROWS, rows = min((int64_t)CS_AREA_ROWS, H - r0);
  unsigned long long acc = 0;
  const bool vec = im.sw == 1 && W % 16 == 0 && im.sh % 16 == 0 && ((uintptr_t)m % 16) == 0;
  if (vec) {
    const int64_t per_row = W / 16, n = rows * per_row;
    for (int64_t k = threadIdx.x; k < n; k += CS_NT) {
      const int64_t r = k / per_row, c = k - r * per_row;
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(m + (r0 + r) * im.sh) + c);
      acc += __dp4a(q.x, 0x01010101u, 0u) + __dp4a(q.y, 0x01010101u, 0u) + __dp4a(q.z, 0x01010101u, 0u) +
             __dp4a(q.w, 0x01010101u, 0u);
    }
  } else {
    const int64_t n = rows * W;
    for (int64_t k = threadIdx.x; k < n; k += CS_NT) {
      const int64_t r = k / W, c = k - r * W;
      acc += __ldg(m + (r0 + r) * im.sh + c * im.sw);
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) s_red[wid] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long sum = 0;
    for (int k = 0; k < CS_NT / kWarp; ++k) sum += s_red[k];
    if (sum) atomicAdd(areas + gt, sum);
  }
}

// targets[b, i, j] for every image b and sampled pixel (start + s*i, start + s*j)
__global__ void __launch_bounds__(CS_NT) semantic_labels_kernel(const CsTable tab, int64_t oh, int64_t ow, int64_t start,
                                                                int64_t s, int64_t num_classes,
                                                                const int64_t* __restrict__ areas,
                                                                int64_t* __restrict__ targets) {
  const int64_t per_img = oh * ow;
  const int64_t idx = (int64_t)blockIdx.x * CS_NT + threadIdx.x;
  if (idx >= (int64_t)tab.n_images * per_img) return;
  const int b = (int)(idx / per_img);
  const int64_t p = idx - b * per_img, i = p / ow, j = p - i * ow;
  const CsImage& im = tab.im[b];
  const int64_t G = tab.gt_first[b + 1] - tab.gt_first[b];
  const uint8_t* px = im.mask + (start + i * s) * im.sh + (start + j * s) * im.sw;
  int64_t best = 0, arg = -1;
  for (int64_t g = 0; g < G; ++g) {
    const int64_t wgt = __ldg(px + g * im.sg) ? areas[tab.gt_first[b] + g] : CS_INF;
    if (arg < 0 || wgt < best) {                   // strict: the first index on ties, as torch.min(dim)
      best = wgt;
      arg = g;
    }
  }
  targets[idx] = (arg < 0 || best == CS_INF) ? num_classes : im.labels[arg];
}

// fills the table from the host arrays; BXS_OK or the status of the first argument out of range
int fill_table(CsTable& tab, const uint8_t* const* mask_host, const int64_t* strides_host, const int64_t* gt_off_host,
               const int64_t* const* labels_host, int64_t B, int64_t H, int64_t W) {
  if (!mask_host || !strides_host || !gt_off_host || B <= 0 || H <= 0 || W <= 0) return BXS_ERR_INVALID_ARG;
  if (B > CS_MAX_IMAGES) return BXS_ERR_UNSUPPORTED;
  tab = CsTable{};
  tab.n_images = (int)B;
  if (gt_off_host[0] != 0) return BXS_ERR_INVALID_ARG;
  for (int64_t b = 0; b < B; ++b) {
    const int64_t G = gt_off_host[b + 1] - gt_off_host[b];
    const int64_t* st = strides_host + 3 * b;
    if (G < 0 || st[0] < 0 || st[1] < 0 || st[2] < 0) return BXS_ERR_INVALID_ARG;
    if (G > 0 && (!mask_host[b] || (labels_host && !labels_host[b]))) return BXS_ERR_INVALID_ARG;
    tab.im[b] = CsImage{mask_host[b], labels_host ? labels_host[b] : nullptr, st[0], st[1], st[2]};
    tab.gt_first[b] = gt_off_host[b];
  }
  tab.gt_first[B] = gt_off_host[B];
  if (tab.gt_first[B] > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  return BXS_OK;
}

// the dice call's shape checks: every sampled pixel inside [H, W], one chunk grid row per instance
int dice_check(int64_t N, int64_t h, int64_t w, int64_t H, int64_t W, int64_t start, int64_t stride) {
  if (N < 0 || h <= 0 || w <= 0 || start < 0 || stride <= 0) return BXS_ERR_INVALID_ARG;
  if (start + (h - 1) * stride >= H || start + (w - 1) * stride >= W) return BXS_ERR_INVALID_ARG;
  if (h * w > INT32_MAX - CS_CHUNK || N > 65535) return BXS_ERR_UNSUPPORTED;
  return BXS_OK;
}

int64_t dice_chunks(int64_t h, int64_t w) { return ceil_div(h * w, CS_CHUNK); }

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_condinst_dice_workspace_bytes(int64_t N, int64_t h, int64_t w) {
  if (N < 0 || h <= 0 || w <= 0) return 0;
  return (int64_t)align_up((size_t)(N * dice_chunks(h, w) * 3) * sizeof(double));
}

extern "C" int bxs_condinst_dice_forward(const float* logits, const int32_t* gt_inds, int64_t N, int64_t h, int64_t w,
                                         const uint8_t* const* mask_host, const int64_t* mask_strides_host,
                                         const int64_t* gt_off_host, int64_t B, int64_t H, int64_t W, int64_t start,
                                         int64_t stride, float* sums, float* loss, void* workspace,
                                         bxs_stream_t stream) {
  CsTable tab;
  if (const int rc = fill_table(tab, mask_host, mask_strides_host, gt_off_host, nullptr, B, H, W)) return rc;
  if (const int rc = dice_check(N, h, w, H, W, start, stride)) return rc;
  if (N == 0) return BXS_OK;
  if (!logits || !gt_inds || !sums || !loss || !workspace) return BXS_ERR_INVALID_ARG;
  const cudaStream_t st = as_stream(stream);
  const int64_t chunks = dice_chunks(h, w);
  double* partials = static_cast<double*>(workspace);
  dice_partials_kernel<<<dim3((unsigned)chunks, (unsigned)N), CS_NT, 0, st>>>(logits, gt_inds, tab, (uint32_t)(h * w),
                                                                               (uint32_t)w, start, stride, partials);
  if (const int rc = check_launch()) return rc;
  dice_finalize_kernel<<<1, CS_RED_NT, 0, st>>>(partials, N, chunks, sums, loss);
  return check_launch();
}

extern "C" int bxs_condinst_dice_backward(const float* logits, const int32_t* gt_inds, int64_t N, int64_t h, int64_t w,
                                          const uint8_t* const* mask_host, const int64_t* mask_strides_host,
                                          const int64_t* gt_off_host, int64_t B, int64_t H, int64_t W, int64_t start,
                                          int64_t stride, const float* sums, const float* g_loss, float* g_logits,
                                          bxs_stream_t stream) {
  CsTable tab;
  if (const int rc = fill_table(tab, mask_host, mask_strides_host, gt_off_host, nullptr, B, H, W)) return rc;
  if (const int rc = dice_check(N, h, w, H, W, start, stride)) return rc;
  if (N == 0) return BXS_OK;
  if (!logits || !gt_inds || !sums || !g_loss || !g_logits) return BXS_ERR_INVALID_ARG;
  dice_backward_kernel<<<dim3((unsigned)dice_chunks(h, w), (unsigned)N), CS_NT, 0, as_stream(stream)>>>(
      logits, gt_inds, tab, (uint32_t)(h * w), (uint32_t)w, start, stride, N, sums, g_loss, g_logits);
  return check_launch();
}

extern "C" int bxs_condinst_semantic_targets(const uint8_t* const* mask_host, const int64_t* mask_strides_host,
                                             const int64_t* const* labels_host, const int64_t* gt_off_host, int64_t B,
                                             int64_t H, int64_t W, int64_t stride, int64_t num_classes, int64_t* areas,
                                             int64_t* targets, bxs_stream_t stream) {
  if (!labels_host) return BXS_ERR_INVALID_ARG;
  CsTable tab;
  if (const int rc = fill_table(tab, mask_host, mask_strides_host, gt_off_host, labels_host, B, H, W)) return rc;
  if (stride <= 0 || num_classes < 0) return BXS_ERR_INVALID_ARG;
  const int64_t start = stride / 2;
  const int64_t oh = start < H ? (H - start + stride - 1) / stride : 0, ow = start < W ? (W - start + stride - 1) / stride : 0;
  const int64_t n_out = B * oh * ow, G = tab.gt_first[B];
  if ((n_out > 0 && !targets) || (G > 0 && !areas)) return BXS_ERR_INVALID_ARG;
  if (ceil_div(H, CS_AREA_ROWS) > INT32_MAX || G > 65535 || ceil_div(n_out, CS_NT) > INT32_MAX)
    return BXS_ERR_UNSUPPORTED;
  const cudaStream_t st = as_stream(stream);
  if (G > 0) {
    if (const cudaError_t e = cudaMemsetAsync(areas, 0, (size_t)G * sizeof(int64_t), st)) {
      set_last_error(e);
      return BXS_ERR_LAUNCH;
    }
    semantic_areas_kernel<<<dim3((unsigned)ceil_div(H, CS_AREA_ROWS), (unsigned)G), CS_NT, 0, st>>>(
        tab, H, W, reinterpret_cast<unsigned long long*>(areas));
    if (const int rc = check_launch()) return rc;
  }
  if (n_out == 0) return BXS_OK;
  semantic_labels_kernel<<<(unsigned)ceil_div(n_out, CS_NT), CS_NT, 0, st>>>(tab, oh, ow, start, stride, num_classes,
                                                                             areas, targets);
  return check_launch();
}
