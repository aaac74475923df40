// a6 (dense form), a10: box-projection dice loss on arbitrary score/target maps and the (unused by the
// heads) length regulariser -- forward + backward.  (The a9 region level-set energy is fused_assembly.cu.)
// Replaces BoxProjectionLoss (mmdet/models/losses/box_projection_loss.py:11-42), mil_loss+dice_loss
// (mmdet/models/dense_heads/discobox_head.py:542-562), length_regularization
// (mmdet/models/losses/levelset_loss.py:47-60).
//
// These run on a few dozen instance maps (<= 20 MB, L2 resident): the design goal is ONE pass
// per reduction with deterministic two-stage sums (per-CTA partials -> fixed-order finalize)
// instead of the reference's ~8 elementwise launches with [n,C,h,w] temporaries each.
#include <algorithm>

#include "boxinst_common.cuh"         // fkey / fkey_inv / pack_key: one tie rule with the BoxInst loss kernels

namespace bxs {
namespace {

constexpr int NT = 256;

// ---------------------------------------------------------------------------------------
// projection: row / column maxima of scores (with first arg-max) and of targets
// ---------------------------------------------------------------------------------------
struct PrjWs {
  unsigned long long* col_s;   // [n*w] zeroed      (key << 32 | ~y)
  unsigned* col_t;             // [n*w] zeroed      key of the target column max
  size_t zero_bytes;
  unsigned long long* row_s;   // [n*h]
  float* row_t;                // [n*h]
  float* coef_row;             // [n*h] d loss / d (row max score)
  float* coef_col;             // [n*w]
  int* arg_row;                // [n*h]
  int* arg_col;                // [n*w]
  size_t total_bytes;
};

inline PrjWs carve_prj(void* base, int64_t n, int64_t h, int64_t w) {
  PrjWs p{};
  Carver c(base);
  p.col_s = (unsigned long long*)c.take(8 * n * w);
  p.col_t = (unsigned*)c.take(4 * n * w);
  p.zero_bytes = c.off;
  p.row_s = (unsigned long long*)c.take(8 * n * h);
  p.row_t = (float*)c.take(4 * n * h);
  p.coef_row = (float*)c.take(4 * n * h);
  p.coef_col = (float*)c.take(4 * n * w);
  p.arg_row = (int*)c.take(4 * n * h);
  p.arg_col = (int*)c.take(4 * n * w);
  p.total_bytes = c.off;
  return p;
}

// one warp per row: coalesced lane-strided loads, integer redux for max / first arg-max
__global__ void __launch_bounds__(NT) prj_rows_kernel(const float* __restrict__ scores, const float* __restrict__ targets,
                                                      int64_t rows_total, int w, PrjWs ws) {
  const int lane = threadIdx.x & 31;
  const int64_t row = blockIdx.x * (int64_t)(NT / 32) + (threadIdx.x >> 5);
  if (row >= rows_total) return;
  const float* s = scores + row * w;
  const float* t = targets + row * w;
  float ms = -INFINITY, mt = -INFINITY;
  for (int x = lane; x < w; x += 32) { ms = fmaxf(ms, __ldg(s + x)); mt = fmaxf(mt, __ldg(t + x)); }
  const unsigned ks = __reduce_max_sync(kFull, fkey(ms));
  const unsigned kt = __reduce_max_sync(kFull, fkey(mt));
  const float vs = fkey_inv(ks);
  int cand = 0x7fffffff;
  for (int x = lane; x < w; x += 32)
    if (__ldg(s + x) == vs) { cand = x; break; }           // ascending: first match of this lane
  const int arg = __reduce_min_sync(kFull, cand);
  if (lane == 0) {
    ws.row_s[row] = pack_key(ks, arg == 0x7fffffff ? 0 : arg);
    ws.row_t[row] = fkey_inv(kt);
  }
}

// one thread per column and row segment; segments combined with order-independent integer atomics
__global__ void __launch_bounds__(NT) prj_cols_kernel(const float* __restrict__ scores, const float* __restrict__ targets,
                                                      int h, int w, int rows_per_seg, PrjWs ws) {
  const int x = blockIdx.x * NT + threadIdx.x;
  const int n = blockIdx.z, y0 = blockIdx.y * rows_per_seg, y1 = min(y0 + rows_per_seg, h);
  if (x >= w) return;
  const float* s = scores + (int64_t)n * h * w + x;
  const float* t = targets + (int64_t)n * h * w + x;
  float ms = -INFINITY, mt = -INFINITY;
  int ay = -1;
  for (int y = y0; y < y1; ++y) {
    const float v = __ldg(s + (int64_t)y * w);
    if (v > ms || ay < 0) { ms = v; ay = y; }
    mt = fmaxf(mt, __ldg(t + (int64_t)y * w));
  }
  if (ay >= 0) {
    atomicMax(ws.col_s + (int64_t)n * w + x, pack_key(fkey(ms), ay));
    atomicMax(ws.col_t + (int64_t)n * w + x, fkey(mt));
  }
}

// dice over both profiles + gradient coefficients; one CTA per instance
__global__ void __launch_bounds__(NT) prj_finalize_kernel(int h, int w, PrjWs ws, float eps, float loss_weight,
                                                          float* __restrict__ loss) {
  __shared__ float s_red[NT / 32];
  __shared__ float s_bc[2];
  const int n = blockIdx.x;
  float total = 0.f;
  for (int axis = 0; axis < 2; ++axis) {
    const int L = axis == 0 ? h : w;
    float inter = 0.f, x2 = 0.f, t2 = 0.f;
    for (int i = threadIdx.x; i < L; i += NT) {
      float s, t;
      if (axis == 0) { s = fkey_inv((unsigned)(ws.row_s[(int64_t)n * h + i] >> 32)); t = ws.row_t[(int64_t)n * h + i]; }
      else { s = fkey_inv((unsigned)(ws.col_s[(int64_t)n * w + i] >> 32)); t = fkey_inv(ws.col_t[(int64_t)n * w + i]); }
      inter = fmaf(s, t, inter); x2 = fmaf(s, s, x2); t2 = fmaf(t, t, t2);
    }
    inter = block_sum<float>(inter, s_red);
    x2 = block_sum<float>(x2, s_red);
    t2 = block_sum<float>(t2, s_red);
    if (threadIdx.x == 0) {
      const float u = x2 + t2 + eps;
      s_bc[0] = inter; s_bc[1] = u;
      total += 1.f - 2.f * inter / u;
    }
    __syncthreads();
    const float I = s_bc[0], U = s_bc[1];
    for (int i = threadIdx.x; i < L; i += NT) {
      unsigned long long p;
      float t;
      if (axis == 0) { p = ws.row_s[(int64_t)n * h + i]; t = ws.row_t[(int64_t)n * h + i]; }
      else { p = ws.col_s[(int64_t)n * w + i]; t = fkey_inv(ws.col_t[(int64_t)n * w + i]); }
      const float s = fkey_inv((unsigned)(p >> 32));
      const float c = loss_weight * (-2.f * t / U + 4.f * I * s / (U * U));
      const int a = (int)(0xffffffffu - (unsigned)(p & 0xffffffffull));
      if (axis == 0) { ws.coef_row[(int64_t)n * h + i] = c; ws.arg_row[(int64_t)n * h + i] = a; }
      else { ws.coef_col[(int64_t)n * w + i] = c; ws.arg_col[(int64_t)n * w + i] = a; }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) loss[n] = loss_weight * total;
}

__global__ void __launch_bounds__(NT) prj_bwd_kernel(int64_t total, int h, int w, PrjWs ws, const float* __restrict__ g_loss,
                                                     float* __restrict__ g_scores) {
  for (int64_t i = blockIdx.x * (int64_t)NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    const int x = i % w, y = (i / w) % h;
    const int64_t n = i / ((int64_t)w * h);
    float v = 0.f;
    if (ws.arg_row[n * h + y] == x) v += ws.coef_row[n * h + y];
    if (ws.arg_col[n * w + x] == y) v += ws.coef_col[n * w + x];
    g_scores[i] = v * g_loss[n];
  }
}

// length regulariser: sum |dy| + sum |dx| per instance (all channels)
__global__ void __launch_bounds__(NT) length_fwd_kernel(const float* __restrict__ s, int C, int h, int w, int chunks,
                                                        float* __restrict__ partial) {
  __shared__ float s_red[NT / 32];
  const int n = blockIdx.y, chunk = blockIdx.x;
  const int64_t total = (int64_t)C * h * w;
  const float* base = s + (int64_t)n * total;
  float acc = 0.f;
  for (int64_t i = chunk * (int64_t)NT + threadIdx.x; i < total; i += (int64_t)chunks * NT) {
    const int x = i % w, y = (i / w) % h;
    const float v = base[i];
    if (y + 1 < h) acc += fabsf(base[i + w] - v);
    if (x + 1 < w) acc += fabsf(base[i + 1] - v);
  }
  acc = block_sum<float>(acc, s_red);
  if (threadIdx.x == 0) partial[(int64_t)n * chunks + chunk] = acc;
}

__global__ void sum_chunks_kernel(const float* __restrict__ partial, int chunks, float* __restrict__ out) {
  const int n = blockIdx.x;
  if (threadIdx.x != 0) return;
  float acc = 0.f;
  for (int k = 0; k < chunks; ++k) acc += partial[(int64_t)n * chunks + k];
  out[n] = acc;
}

__device__ __forceinline__ float sgn(float v) { return (v > 0.f) - (v < 0.f); }

__global__ void __launch_bounds__(NT) length_bwd_kernel(const float* __restrict__ s, const float* __restrict__ g_loss,
                                                        int C, int h, int w, int64_t total_all, float* __restrict__ g) {
  const int64_t per = (int64_t)C * h * w;
  for (int64_t i = blockIdx.x * (int64_t)NT + threadIdx.x; i < total_all; i += (int64_t)gridDim.x * NT) {
    const int x = i % w, y = (i / w) % h;
    const int64_t n = i / per;
    const float v = s[i];
    float acc = 0.f;
    if (y + 1 < h) acc -= sgn(s[i + w] - v);
    if (y > 0) acc += sgn(v - s[i - w]);
    if (x + 1 < w) acc -= sgn(s[i + 1] - v);
    if (x > 0) acc += sgn(v - s[i - 1]);
    g[i] = acc * g_loss[n];
  }
}

inline int pick_chunks(int64_t n, int64_t work_items) {
  int64_t want = ceil_div((int64_t)sm_count() * 4, n > 0 ? n : 1);
  int64_t maxc = ceil_div(work_items, NT);
  int64_t c = want < maxc ? want : maxc;
  return (int)(c < 1 ? 1 : (c > 64 ? 64 : c));
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_projection_workspace_bytes(int64_t n, int64_t h, int64_t w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return (int64_t)carve_prj(nullptr, n, h, w).total_bytes;
}

extern "C" int bxs_projection_loss_forward(const float* scores, const float* targets, float* loss, void* workspace,
                                           int64_t n, int64_t h, int64_t w, float eps, float loss_weight,
                                           bxs_stream_t stream) {
  if (!scores || !targets || !loss || !workspace || n <= 0 || h <= 0 || w <= 0 || n >= 65536 ||
      h * w >= (int64_t(1) << 31))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  PrjWs ws = carve_prj(workspace, n, h, w);
  cudaMemsetAsync(workspace, 0, ws.zero_bytes, st);
  prj_rows_kernel<<<(unsigned)ceil_div(n * h, NT / 32), NT, 0, st>>>(scores, targets, n * h, (int)w, ws);
  int segs = (int)std::min<int64_t>(ceil_div(h, 8), std::max<int64_t>(1, ceil_div((int64_t)sm_count() * 8 * NT, n * w)));
  const int rows_per_seg = (int)ceil_div(h, segs);
  segs = (int)ceil_div(h, rows_per_seg);
  prj_cols_kernel<<<dim3((unsigned)ceil_div(w, NT), segs, (unsigned)n), NT, 0, st>>>(scores, targets, (int)h, (int)w,
                                                                                      rows_per_seg, ws);
  prj_finalize_kernel<<<(unsigned)n, NT, 0, st>>>((int)h, (int)w, ws, eps, loss_weight, loss);
  return check_launch();
}

extern "C" int bxs_projection_loss_backward(const void* workspace, const float* g_loss, float* g_scores, int64_t n,
                                            int64_t h, int64_t w, bxs_stream_t stream) {
  if (!workspace || !g_loss || !g_scores || n <= 0 || h <= 0 || w <= 0) return BXS_ERR_INVALID_ARG;
  PrjWs ws = carve_prj(const_cast<void*>(workspace), n, h, w);
  const int64_t total = n * h * w;
  const int blocks = (int)std::min<int64_t>(ceil_div(total, NT), (int64_t)sm_count() * 16);
  prj_bwd_kernel<<<blocks, NT, 0, as_stream(stream)>>>(total, (int)h, (int)w, ws, g_loss, g_scores);
  return check_launch();
}

extern "C" int bxs_length_reg_forward(const float* scores, float* out, void* workspace, int64_t n, int64_t C, int64_t h,
                                      int64_t w, bxs_stream_t stream) {
  if (!scores || !out || !workspace || n <= 0 || n >= 65536 || C <= 0 || h <= 0 || w <= 0) return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  const int chunks = pick_chunks(n, C * h * w);
  length_fwd_kernel<<<dim3(chunks, (unsigned)n), NT, 0, st>>>(scores, (int)C, (int)h, (int)w, chunks, (float*)workspace);
  sum_chunks_kernel<<<(unsigned)n, 32, 0, st>>>((const float*)workspace, chunks, out);
  return check_launch();
}

extern "C" int bxs_length_reg_backward(const float* scores, const float* g_out, float* g_scores, int64_t n, int64_t C,
                                       int64_t h, int64_t w, bxs_stream_t stream) {
  if (!scores || !g_out || !g_scores || n <= 0 || C <= 0 || h <= 0 || w <= 0) return BXS_ERR_INVALID_ARG;
  const int64_t total = n * C * h * w;
  const int blocks = (int)std::min<int64_t>(ceil_div(total, NT), (int64_t)sm_count() * 16);
  length_bwd_kernel<<<blocks, NT, 0, as_stream(stream)>>>(scores, g_out, (int)C, (int)h, (int)w, total, g_scores);
  return check_launch();
}

// ---------------------------------------------------------------------------------------
// SURVEY 8f rank 1: projection profiles of a bilinearly UPSAMPLED map without materialising it.
// BoxMatchingCost (mmdet/core/bbox/match_costs/match_cost.py:400-425) takes row / column maxima of the mask
// predictions after Box2MaskHead._get_target_single upsampled them to the GT resolution
// (box2mask_head.py:157-161: [100,1,1024,1024] = 420 MB per image per decoder layer).  Here every output pixel is
// evaluated on the fly (PyTorch bilinear, align_corners=False) and reduced immediately.
// ---------------------------------------------------------------------------------------
namespace bxs {
namespace {

__device__ __forceinline__ void bilinear_src(int dst, float scale, int in_size, int& i0, int& i1, float& l1) {
  float src = scale * ((float)dst + 0.5f) - 0.5f;        // area_pixel_compute_source_index, align_corners=False
  src = src < 0.f ? 0.f : src;
  i0 = min((int)src, in_size - 1);
  i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
  l1 = src - (float)i0;
}

constexpr int UPK = 32;                                   // output columns per lane and panel -> panel = 1024 columns

// grid (row groups, n), 256 threads; warp w handles output rows Y = group*rows_per_block + w, +8, ...
__global__ void __launch_bounds__(NT) upsampled_rowcol_max_kernel(const float* __restrict__ x, int h, int w, int H, int W,
                                                                  int rows_per_block, float sy, float sx,
                                                                  unsigned* __restrict__ row_key,
                                                                  unsigned* __restrict__ col_key) {
  extern __shared__ float s_b[];                          // [8 warps][w] vertically blended low-res rows
  const int n = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const float* in = x + (int64_t)n * h * w;
  float* b = s_b + warp * w;
  const int y_begin = blockIdx.x * rows_per_block, y_end = min(y_begin + rows_per_block, H);
  for (int panel0 = 0; panel0 < W; panel0 += 32 * UPK) {
    float cmax[UPK];
#pragma unroll
    for (int k = 0; k < UPK; ++k) cmax[k] = -INFINITY;
    for (int Y = y_begin + warp; Y < y_end; Y += NT / 32) {
      int y0, y1;
      float fy;
      bilinear_src(Y, sy, h, y0, y1, fy);
      for (int i = lane; i < w; i += 32)
        b[i] = (1.f - fy) * __ldg(in + (int64_t)y0 * w + i) + fy * __ldg(in + (int64_t)y1 * w + i);
      __syncwarp();
      float rmax = -INFINITY;
#pragma unroll
      for (int k = 0; k < UPK; ++k) {
        const int X = panel0 + k * 32 + lane;
        if (X < W) {
          int x0, x1;
          float fx;
          bilinear_src(X, sx, w, x0, x1, fx);
          const float v = (1.f - fx) * b[x0] + fx * b[x1];
          rmax = fmaxf(rmax, v);
          cmax[k] = fmaxf(cmax[k], v);
        }
      }
      const unsigned rk = __reduce_max_sync(kFull, fkey(rmax));
      if (lane == 0) atomicMax(row_key + (int64_t)n * H + Y, rk);      // several panels may contribute
      __syncwarp();
    }
#pragma unroll
    for (int k = 0; k < UPK; ++k) {
      const int X = panel0 + k * 32 + lane;
      if (X < W && cmax[k] > -INFINITY) atomicMax(col_key + (int64_t)n * W + X, fkey(cmax[k]));
    }
  }
}

__global__ void decode_keys_kernel(const unsigned* __restrict__ keys, float* __restrict__ out, int64_t total, int act) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float v = fkey_inv(keys[i]);
    out[i] = act ? 1.f / (1.f + expf(-v)) : v;
  }
}

}  // namespace
}  // namespace bxs

// x [n,h,w] -> row_prof [n,H], col_prof [n,W]: maxima over the (virtual) bilinear resize of x to H x W, optionally
// followed by a sigmoid (monotone, so applied to the profiles).  H == h and W == w gives plain row/column maxima.
// workspace: (n*H + n*W) * 4 bytes.
extern "C" int bxs_upsampled_rowcol_max(const float* x, float* row_prof, float* col_prof, void* workspace, int64_t n,
                                        int64_t h, int64_t w, int64_t H, int64_t W, int sigmoid_act, bxs_stream_t stream) {
  if (!x || !row_prof || !col_prof || !workspace || n <= 0 || n >= 65536 || h <= 0 || w <= 0 || H <= 0 || W <= 0)
    return BXS_ERR_INVALID_ARG;
  if (w > 8192) return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  unsigned* row_key = (unsigned*)workspace;
  unsigned* col_key = row_key + n * H;
  cudaMemsetAsync(workspace, 0, sizeof(unsigned) * n * (H + W), st);
  int groups = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(H, 8), ceil_div((int64_t)sm_count() * 4, n)));
  const int rows = (int)ceil_div(H, groups);
  groups = (int)ceil_div(H, rows);
  const size_t sm = (size_t)(NT / 32) * w * sizeof(float);
  if (sm > 48 * 1024 && opt_in_smem(upsampled_rowcol_max_kernel, sm) != BXS_OK) return BXS_ERR_LAUNCH;
  upsampled_rowcol_max_kernel<<<dim3(groups, (unsigned)n), NT, sm, st>>>(x, (int)h, (int)w, (int)H, (int)W, rows,
                                                                         (float)h / (float)H, (float)w / (float)W, row_key,
                                                                         col_key);
  const int64_t tr = n * H, tc = n * W;
  decode_keys_kernel<<<(unsigned)std::min<int64_t>(ceil_div(tr, 256), 1024), 256, 0, st>>>(row_key, row_prof, tr, sigmoid_act);
  decode_keys_kernel<<<(unsigned)std::min<int64_t>(ceil_div(tc, 256), 1024), 256, 0, st>>>(col_key, col_prof, tc, sigmoid_act);
  return check_launch();
}
