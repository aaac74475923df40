// The dynamic kernels of some grid cells of every level, packed for ONE dense dynamic convolution per operand
//     replaces the gather kernel_preds[l][b].view(C, -1)[:, grid_order] of discobox_head.py:1180-1189 for every (level, image),
//     whose per-(level, image) F.conv2d (:1214-1227) all read the same operand s_ins_pred[b], and the positive cells of
//     BoxSOLOv2's levels of one size (box_solov2_head.py:204-216 indexed as :317-320).
//
//     pack:   packed[b, r, c] = grid_l[b, c, cell] for the r-th row of image b (levels in order, each level's cells in the
//             order given: the reference's loop order, repeats included); rows past an image's total are zero.  A pure gather
//             of 4- or 2-byte elements, one thread per packed element, writes coalesced along c.
//     unpack: d/d grid_l[b, c, cell] = sum, in row order, of d/d packed[b, r, c] over the rows r of segment (l, b) that name
//             the cell, accumulated in FP32 and rounded once; 0 for every other cell.  One CTA per (level, image, channel
//             chunk) threads the segment's rows of each cell into a list in shared memory (first row first), then every
//             thread walks the list of its (cell, channel): a gather, no atomics, bit-identical from run to run.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "common.cuh"
#include "half_math.cuh"

namespace bxs {
namespace {

constexpr int DC_MAX_LEVELS = 8;
constexpr int DC_MAX_IMAGES = 16;
constexpr int DC_MAX_GRID = 64;              // S_l: the unpack keeps one list head per cell in shared memory
constexpr int DC_MAX_ROWS = 2048;            // I_pad: ... and one link per row
constexpr int DC_NT = 256;
constexpr int DC_CCH = 16;                   // channels per unpack CTA

struct DiscoCellsPlan {
  const void* grids[DC_MAX_LEVELS];          // [B,C,S_l,S_l] (pack)
  void* g_grids[DC_MAX_LEVELS];              // [B,C,S_l,S_l] (unpack)
  int32_t S[DC_MAX_LEVELS];
  int32_t row0[DC_MAX_IMAGES][DC_MAX_LEVELS + 1];   // first packed row of (image, level); [b][n_levels]: the image's total
  int32_t flat0[DC_MAX_LEVELS][DC_MAX_IMAGES];      // first entry of segment (level, image) in the flat cell list
  int n_levels, B, C, I_pad;
};

// BXS_OK, or the status of the first argument out of range.  All checks are on the host.
int plan(DiscoCellsPlan& p, const int64_t* grid_host, const int64_t* counts_host, const int32_t* cells, int64_t n_cells,
         int64_t n_levels, int64_t B, int64_t C, int64_t I_pad, int dtype) {
  if (!grid_host || !counts_host || n_levels <= 0 || B <= 0 || C <= 0 || I_pad < 0 || n_cells < 0) return BXS_ERR_INVALID_ARG;
  if (dtype < 0 || dtype > 2) return BXS_ERR_INVALID_ARG;
  if (n_levels > DC_MAX_LEVELS || B > DC_MAX_IMAGES || C > INT32_MAX / DC_MAX_ROWS || I_pad > DC_MAX_ROWS)
    return BXS_ERR_UNSUPPORTED;
  if (n_cells && !cells) return BXS_ERR_INVALID_ARG;
  p = DiscoCellsPlan{};
  p.n_levels = (int)n_levels;
  p.B = (int)B;
  p.C = (int)C;
  p.I_pad = (int)I_pad;
  for (int64_t l = 0; l < n_levels; ++l) {
    if (grid_host[l] <= 0) return BXS_ERR_INVALID_ARG;
    if (grid_host[l] > DC_MAX_GRID) return BXS_ERR_UNSUPPORTED;
    p.S[l] = (int32_t)grid_host[l];
  }
  int64_t flat = 0;
  for (int64_t l = 0; l < n_levels; ++l)
    for (int64_t b = 0; b < B; ++b) {
      const int64_t n = counts_host[l * B + b];
      if (n < 0 || n > DC_MAX_ROWS) return BXS_ERR_INVALID_ARG;
      p.flat0[l][b] = (int32_t)flat;
      flat += n;
    }
  if (flat != n_cells) return BXS_ERR_INVALID_ARG;                   // the counts must cover the cell list exactly
  for (int64_t b = 0; b < B; ++b) {
    int64_t row = 0;
    for (int64_t l = 0; l < n_levels; ++l) {
      p.row0[b][l] = (int32_t)row;
      row += counts_host[l * B + b];
    }
    if (row > I_pad) return BXS_ERR_INVALID_ARG;                     // an image's rows must fit the packed operand
    p.row0[b][n_levels] = (int32_t)row;
  }
  return BXS_OK;
}

// T: the element as raw bits (float32: uint32_t, float16 / bfloat16: uint16_t); a zero bit pattern is +0.
template <typename T>
__global__ void __launch_bounds__(DC_NT) disco_cells_pack_kernel(const DiscoCellsPlan p, const int32_t* __restrict__ cells,
                                                                   T* __restrict__ packed, int32_t* __restrict__ status) {
  const int64_t total = (int64_t)p.B * p.I_pad * p.C;
  for (int64_t i = (int64_t)blockIdx.x * DC_NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * DC_NT) {
    const int c = (int)(i % p.C);
    const int64_t br = i / p.C;
    const int r = (int)(br % p.I_pad), b = (int)(br / p.I_pad);
    T v = T(0);
    if (r < p.row0[b][p.n_levels]) {
      int l = 0;
      while (r >= p.row0[b][l + 1]) ++l;
      const int cell = cells[p.flat0[l][b] + (r - p.row0[b][l])];
      const int S2 = p.S[l] * p.S[l];
      if (cell >= 0 && cell < S2)
        v = static_cast<const T*>(p.grids[l])[((int64_t)b * p.C + c) * S2 + cell];
      else if (status)
        *status = BXS_ERR_INVALID_ARG;                               // the row stays zero
    }
    packed[i] = v;
  }
}

template <typename T>
struct Widen {
  static __device__ __forceinline__ float widen(T x) { return Half16Ops<T>::widen(x); }
  static __device__ __forceinline__ T round(float x) { return Half16Ops<T>::round(x); }
};
template <>
struct Widen<float> {
  static __device__ __forceinline__ float widen(float x) { return x; }
  static __device__ __forceinline__ float round(float x) { return x; }
};

template <typename T>
__global__ void __launch_bounds__(DC_NT) disco_cells_unpack_kernel(const DiscoCellsPlan p, const int32_t* __restrict__ cells,
                                                                     const T* __restrict__ g_packed) {
  __shared__ int s_head[DC_MAX_GRID * DC_MAX_GRID];
  __shared__ int s_next[DC_MAX_ROWS];
  const int l = blockIdx.z, b = blockIdx.y, c0 = blockIdx.x * DC_CCH;
  const int S2 = p.S[l] * p.S[l];
  const int r0 = p.row0[b][l], n = p.row0[b][l + 1] - r0;
  const int32_t* seg = cells + p.flat0[l][b];
  for (int s = threadIdx.x; s < S2; s += DC_NT) s_head[s] = -1;
  for (int k = threadIdx.x; k < n; k += DC_NT) s_next[k] = seg[k];
  __syncthreads();
  if (threadIdx.x == 0) {                    // rows last to first: each cell's list ends up in row order
    for (int k = n - 1; k >= 0; --k) {
      const int cell = s_next[k];
      if (cell >= 0 && cell < S2) {
        s_next[k] = s_head[cell];
        s_head[cell] = k;
      } else {
        s_next[k] = -1;                      // packed as a zero row: no gradient to any cell
      }
    }
  }
  __syncthreads();
  const int nc = min(DC_CCH, p.C - c0);
  T* out = static_cast<T*>(p.g_grids[l]) + ((int64_t)b * p.C + c0) * S2;
  const T* g = g_packed + ((int64_t)b * p.I_pad + r0) * p.C + c0;
  for (int idx = threadIdx.x; idx < nc * S2; idx += DC_NT) {
    const int c = idx / S2, s = idx - c * S2;
    float acc = 0.f;
    for (int k = s_head[s]; k >= 0; k = s_next[k]) acc += Widen<T>::widen(g[(int64_t)k * p.C + c]);
    out[(int64_t)c * S2 + s] = Widen<T>::round(acc);
  }
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_disco_cells_pack(const void* const* grids_host, const int64_t* grid_host, const int64_t* counts_host,
                                    const int32_t* cells, int64_t n_cells, void* packed, int32_t* status, int64_t n_levels,
                                    int64_t B, int64_t C, int64_t I_pad, int dtype, bxs_stream_t stream) {
  DiscoCellsPlan p;
  if (const int rc = plan(p, grid_host, counts_host, cells, n_cells, n_levels, B, C, I_pad, dtype)) return rc;
  if (!grids_host || (I_pad && !packed)) return BXS_ERR_INVALID_ARG;
  for (int64_t l = 0; l < n_levels; ++l) {
    if (!grids_host[l]) return BXS_ERR_INVALID_ARG;
    p.grids[l] = grids_host[l];
  }
  const int64_t total = B * I_pad * C;
  if (!total) return BXS_OK;
  const cudaStream_t st = as_stream(stream);
  const int ctas = grid_for(total, DC_NT);
  if (dtype == 0)
    disco_cells_pack_kernel<uint32_t><<<ctas, DC_NT, 0, st>>>(p, cells, static_cast<uint32_t*>(packed), status);
  else
    disco_cells_pack_kernel<uint16_t><<<ctas, DC_NT, 0, st>>>(p, cells, static_cast<uint16_t*>(packed), status);
  return check_launch();
}

extern "C" int bxs_disco_cells_unpack_grad(const void* g_packed, const int64_t* grid_host, const int64_t* counts_host,
                                           const int32_t* cells, int64_t n_cells, void* const* g_grids_host, int64_t n_levels,
                                           int64_t B, int64_t C, int64_t I_pad, int dtype, bxs_stream_t stream) {
  DiscoCellsPlan p;
  if (const int rc = plan(p, grid_host, counts_host, cells, n_cells, n_levels, B, C, I_pad, dtype)) return rc;
  if (!g_grids_host || (n_cells && !g_packed)) return BXS_ERR_INVALID_ARG;
  for (int64_t l = 0; l < n_levels; ++l) {
    if (!g_grids_host[l]) return BXS_ERR_INVALID_ARG;
    p.g_grids[l] = g_grids_host[l];
  }
  const cudaStream_t st = as_stream(stream);
  const dim3 grid((unsigned)ceil_div(C, DC_CCH), (unsigned)B, (unsigned)n_levels);
  if (dtype == 0)
    disco_cells_unpack_kernel<float><<<grid, DC_NT, 0, st>>>(p, cells, static_cast<const float*>(g_packed));
  else if (dtype == 1)
    disco_cells_unpack_kernel<__half><<<grid, DC_NT, 0, st>>>(p, cells, static_cast<const __half*>(g_packed));
  else
    disco_cells_unpack_kernel<__nv_bfloat16><<<grid, DC_NT, 0, st>>>(p, cells, static_cast<const __nv_bfloat16*>(g_packed));
  return check_launch();
}
