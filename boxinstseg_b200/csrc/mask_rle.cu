// COCO run-length encoding of instance masks, bit-exact with pycocotools' mask.encode (maskApi.c rleEncode + rleToString),
// which mmdet's encode_mask_results (mmdet/core/mask/utils.py:38-65) calls once per mask on the host.
//
// Runs.  In column-major order j = x * H + y a run closes at every j whose byte differs from byte j - 1 (byte -1 counts
// as 0): a "boundary".  The counts of a mask are the differences of its boundary positions, starting from 0, and then
// H * W minus the last one.  A thread owns 4 adjacent columns of one band of RLE_ROWS rows and reads one 4-byte word per
// row, so a warp reads 128 contiguous bytes of a row; each byte is compared with the byte above it, the band's first row
// with the row above the band, and row 0 with the last byte of the previous column.  Each (mask, column, band) is a
// segment of the column-major order:
//   runs:   boundary kernel (count and last position of every segment) -> segment scan (per mask, exclusive, in place)
//           -> mask scan (run offsets of the masks, int64 [n + 1]).
//   counts: the boundary walk again, now writing each boundary's count at its scanned place; the mask's last segment also
//           writes the closing count.
// Strings.  Each count's delta (rle_delta) and its character count (mask_rle_core.cuh) -> per-tile sums -> a scan of the
// tiles -> the same walk writing the characters at their scanned place, and each mask's byte offset.
// No atomics: the output is the same from run to run.
#include <cuda_runtime.h>

#include "common.cuh"
#include "mask_rle_core.cuh"

namespace bxs {
namespace {

constexpr int RLE_NT = 256;                       // threads per CTA of every kernel here but the single-CTA scan
constexpr int RLE_ROWS = 64;                      // rows per band of the boundary walk
constexpr int RLE_SCAN_NT = 1024;                 // threads of the single-CTA scan
constexpr int RLE_SCAN_IT = 4;                    // items per thread and chunk of the segment and single-CTA scans
constexpr int RLE_STR_IT = 16;                    // counts per thread of the string kernels
constexpr int RLE_TILE = RLE_NT * RLE_STR_IT;     // counts per CTA of the string kernels
constexpr int64_t RLE_MAX_PIXELS = int64_t(1) << 29;

// A segment: its boundaries' count and the position of the last one (-1: none).  After the segment scan: the boundaries
// of the mask before the segment, and the position of the last of them (0 when there is none: the first count starts
// at 0).  Positions grow along the scan order, so "last" combines by max.
struct RleSeg {
  int32_t cnt, last;
};

__device__ __forceinline__ RleSeg seg_combine(RleSeg a, RleSeg b) { return {a.cnt + b.cnt, max(a.last, b.last)}; }

__device__ __forceinline__ RleSeg shfl_up(RleSeg v, int d) {
  return {__shfl_up_sync(kFull, v.cnt, d), __shfl_up_sync(kFull, v.last, d)};
}
__device__ __forceinline__ int64_t shfl_up(int64_t v, int d) { return __shfl_up_sync(kFull, v, d); }

__device__ __forceinline__ RleSeg combine(RleSeg a, RleSeg b) { return seg_combine(a, b); }
__device__ __forceinline__ int64_t combine(int64_t a, int64_t b) { return a + b; }

// Exclusive scan of one value per thread across the CTA, in thread order, starting from `carry`; *total gets carry
// combined with every value.  s_warp holds 32 values.  Every thread calls it; it ends with the CTA synchronised.
template <typename T>
__device__ __forceinline__ T block_exclusive_scan(T v, T carry, T* s_warp, T* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarp = blockDim.x >> 5;
  T inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const T o = shfl_up(inc, d);
    if (lane >= d) inc = combine(o, inc);
  }
  if (lane == 31) s_warp[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    T w = lane < nwarp ? s_warp[lane] : T{};
    T winc = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const T o = shfl_up(winc, d);
      if (lane >= d) winc = combine(o, winc);
    }
    if (lane < nwarp) s_warp[lane] = winc;           // inclusive over warps
  }
  __syncthreads();
  T before = warp ? combine(carry, s_warp[warp - 1]) : carry;
  const T excl_in_warp = shfl_up(inc, 1);
  if (lane) before = combine(before, excl_in_warp);
  *total = combine(carry, s_warp[nwarp - 1]);
  __syncthreads();
  return before;
}

// The 4 bytes of row y at columns x0 .. x0 + 3 as one little-endian word (byte c = column x0 + c; 0 past W).  kVec: the
// row is read as one aligned word (W % 4 == 0 and a 4-byte aligned base).
template <bool kVec>
__device__ __forceinline__ uint32_t rle_word(const uint8_t* m, int y, int x0, int W) {
  const uint8_t* p = m + (int64_t)y * W + x0;
  if constexpr (kVec) return __ldg(reinterpret_cast<const uint32_t*>(p));
  uint32_t w = 0;
#pragma unroll
  for (int c = 0; c < 4; ++c)
    if (x0 + c < W) w |= (uint32_t)__ldg(p + c) << (8 * c);
  return w;
}

// The boundary walk of one segment group: mask k, band b, columns 4g .. 4g + 3.  kWrite = false: each column's segment
// (boundary count, last position) -> seg.  kWrite = true: seg holds the scanned states; each boundary's count goes to
// counts[offsets[k] + its index in the mask], and the mask's last column of its last band closes the mask.
template <bool kVec, bool kWrite>
__global__ void __launch_bounds__(RLE_NT) rle_boundary_kernel(const uint8_t* __restrict__ masks, int64_t n, int H, int W,
                                                              int NB, int G, RleSeg* __restrict__ seg,
                                                              const int64_t* __restrict__ offsets,
                                                              uint32_t* __restrict__ counts) {
  const int64_t per_mask = (int64_t)NB * G, total = n * per_mask;
  const int hw = H * W;
  for (int64_t id = (int64_t)blockIdx.x * RLE_NT + threadIdx.x; id < total; id += (int64_t)gridDim.x * RLE_NT) {
    const int64_t k = id / per_mask;
    const int r = (int)(id - k * per_mask), b = r / G, x0 = 4 * (r - b * G);
    const int y0 = b * RLE_ROWS, y1 = min(y0 + RLE_ROWS, H);
    const uint8_t* m = masks + k * hw;
    // the bytes of the columns below W: past W both words hold 0, except the shifted word of row 0, whose first byte
    // past W is the byte of column W - 1
    const uint32_t valid = W - x0 >= 4 ? 0xffffffffu : (1u << (8 * (W - x0))) - 1u;
    uint32_t p;
    if (y0 > 0) {
      p = rle_word<kVec>(m, y0 - 1, x0, W);
    } else {                                           // row 0 follows the last byte of the previous column
      p = rle_word<kVec>(m, H - 1, x0, W) << 8;
      if (x0 > 0) p |= __ldg(m + (int64_t)(H - 1) * W + x0 - 1);
    }
    int cnt[4] = {0, 0, 0, 0}, last[4] = {-1, -1, -1, -1};
    int64_t idx[4];
    if constexpr (kWrite) {
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if (x0 + c < W) {
          const RleSeg s = seg[(k * W + x0 + c) * NB + b];
          idx[c] = offsets[k] + s.cnt;
          last[c] = s.last;
        }
      }
    }
#pragma unroll 8
    for (int y = y0; y < y1; ++y) {
      const uint32_t w = rle_word<kVec>(m, y, x0, W);
      const uint32_t d = __vcmpne4(w, p) & valid;
      p = w;
      if (!d) continue;
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        if ((d >> (8 * c)) & 1u) {
          const int j = (x0 + c) * H + y;
          if constexpr (kWrite) {
            counts[idx[c]++] = (uint32_t)(j - last[c]);
          } else {
            ++cnt[c];
          }
          last[c] = j;
        }
      }
    }
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int x = x0 + c;
      if (x >= W) continue;
      if constexpr (kWrite) {
        if (x == W - 1 && b == NB - 1) counts[idx[c]] = (uint32_t)(hw - last[c]);
      } else {
        seg[(k * W + x) * NB + b] = RleSeg{cnt[c], last[c]};
      }
    }
  }
}

// Per mask (CTAs stride over the masks): the S segments of the mask scanned in place into their exclusive states, and
// the mask's boundary count -> nb[k].
__global__ void __launch_bounds__(RLE_NT) rle_segment_scan_kernel(RleSeg* __restrict__ seg, int64_t n, int64_t S,
                                                                  int32_t* __restrict__ nb) {
  __shared__ RleSeg s_warp[32];
  for (int64_t k = blockIdx.x; k < n; k += gridDim.x) {
    RleSeg* s = seg + k * S;
    RleSeg carry{0, 0};
    for (int64_t base = 0; base < S; base += (int64_t)RLE_NT * RLE_SCAN_IT) {
      const int64_t i0 = base + (int64_t)threadIdx.x * RLE_SCAN_IT;
      RleSeg v[RLE_SCAN_IT], t{0, -1};
#pragma unroll
      for (int i = 0; i < RLE_SCAN_IT; ++i) {
        v[i] = i0 + i < S ? s[i0 + i] : RleSeg{0, -1};
        t = seg_combine(t, v[i]);
      }
      RleSeg next;
      RleSeg e = block_exclusive_scan(t, carry, s_warp, &next);
#pragma unroll
      for (int i = 0; i < RLE_SCAN_IT; ++i) {
        if (i0 + i < S) s[i0 + i] = e;
        e = seg_combine(e, v[i]);
      }
      carry = next;
    }
    if (threadIdx.x == 0) nb[k] = carry.cnt;
  }
}

// One CTA: out[i] = sum_{i' < i} (in[i'] + add) for i < n, out[n] = the whole sum.
template <typename T>
__global__ void __launch_bounds__(RLE_SCAN_NT) rle_offsets_scan_kernel(const T* __restrict__ in, int64_t n, int add,
                                                                       int64_t* __restrict__ out) {
  __shared__ int64_t s_warp[32];
  int64_t carry = 0;
  for (int64_t base = 0; base < n; base += (int64_t)RLE_SCAN_NT * RLE_SCAN_IT) {
    const int64_t i0 = base + (int64_t)threadIdx.x * RLE_SCAN_IT;
    int64_t v[RLE_SCAN_IT], t = 0;
#pragma unroll
    for (int i = 0; i < RLE_SCAN_IT; ++i) {
      v[i] = i0 + i < n ? (int64_t)in[i0 + i] + add : 0;
      t += v[i];
    }
    int64_t next;
    int64_t e = block_exclusive_scan(t, carry, s_warp, &next);
#pragma unroll
    for (int i = 0; i < RLE_SCAN_IT; ++i) {
      if (i0 + i < n) out[i0 + i] = e;
      e += v[i];
    }
    carry = next;
  }
  if (threadIdx.x == 0) out[n] = carry;
}

// The RLE_STR_IT counts of this thread, from i0 on: for each, its mask k (offsets[k] <= i < offsets[k + 1]), its
// mask-local index li and its delta, handed to f(i, k, li, x).
template <typename F>
__device__ __forceinline__ void rle_for_counts(const uint32_t* __restrict__ counts, const int64_t* __restrict__ offsets,
                                               int64_t n, int64_t R, int64_t i0, F f) {
  if (i0 >= R) return;
  int64_t lo = 0, hi = n - 1;                          // the last k with offsets[k] <= i0
  while (lo < hi) {
    const int64_t mid = (lo + hi + 1) >> 1;
    if (offsets[mid] <= i0) lo = mid;
    else hi = mid - 1;
  }
  int64_t k = lo, start = offsets[k], end = offsets[k + 1];
  uint32_t c2 = i0 - start >= 2 ? counts[i0 - 2] : 0u, c1 = i0 - start >= 1 ? counts[i0 - 1] : 0u;
  const int64_t i1 = min(i0 + RLE_STR_IT, R);
  for (int64_t i = i0; i < i1; ++i) {
    while (i >= end) {                                 // every mask has at least one count
      ++k;
      start = end;
      end = offsets[k + 1];
    }
    const uint32_t c = counts[i];
    const int64_t li = i - start;
    f(i, k, li, li > 2 ? (int64_t)c - (int64_t)c2 : (int64_t)c);   // rle_delta on the sliding window
    c2 = c1;
    c1 = c;
  }
}

// Characters of each CTA's RLE_TILE counts -> tile_sum[blockIdx.x].
__global__ void __launch_bounds__(RLE_NT) rle_tile_chars_kernel(const uint32_t* __restrict__ counts,
                                                                const int64_t* __restrict__ offsets, int64_t n, int64_t R,
                                                                int64_t* __restrict__ tile_sum) {
  __shared__ int64_t s_warp[32];
  int64_t len = 0;
  rle_for_counts(counts, offsets, n, R, (int64_t)blockIdx.x * RLE_TILE + (int64_t)threadIdx.x * RLE_STR_IT,
                 [&](int64_t, int64_t, int64_t, int64_t x) { len += rle_char_len(x); });
  int64_t total;
  block_exclusive_scan(len, int64_t(0), s_warp, &total);
  if (threadIdx.x == 0) tile_sum[blockIdx.x] = total;
}

// The characters of each count at tile_off[tile] + the characters before it in the tile; the first count of mask k also
// gives char_off[k].  char_off[n] = the total.
__global__ void __launch_bounds__(RLE_NT) rle_emit_kernel(const uint32_t* __restrict__ counts,
                                                          const int64_t* __restrict__ offsets, int64_t n, int64_t R,
                                                          const int64_t* __restrict__ tile_off, int64_t n_tiles,
                                                          uint8_t* __restrict__ chars, int64_t* __restrict__ char_off) {
  __shared__ int64_t s_warp[32];
  const int64_t i0 = (int64_t)blockIdx.x * RLE_TILE + (int64_t)threadIdx.x * RLE_STR_IT;
  int64_t len = 0;
  rle_for_counts(counts, offsets, n, R, i0, [&](int64_t, int64_t, int64_t, int64_t x) { len += rle_char_len(x); });
  int64_t total;
  int64_t pos = block_exclusive_scan(len, tile_off[blockIdx.x], s_warp, &total);
  rle_for_counts(counts, offsets, n, R, i0, [&](int64_t, int64_t k, int64_t li, int64_t x) {
    if (li == 0) char_off[k] = pos;
    pos += rle_emit(x, chars + pos);
  });
  if (blockIdx.x == 0 && threadIdx.x == 0) char_off[n] = tile_off[n_tiles];
}

int64_t rle_bands(int64_t H) { return ceil_div(H, RLE_ROWS); }

// The runs workspace: the segment states, then the boundary count of every mask.
size_t rle_runs_layout(int64_t n, int64_t H, int64_t W, void* base, RleSeg** seg, int32_t** nb) {
  Carver c(base);
  RleSeg* s = reinterpret_cast<RleSeg*>(c.take((size_t)(n * W * rle_bands(H)) * sizeof(RleSeg)));
  int32_t* b = reinterpret_cast<int32_t*>(c.take((size_t)n * sizeof(int32_t)));
  if (seg) *seg = s;
  if (nb) *nb = b;
  return c.off;
}

bool rle_vec(const uint8_t* masks, int64_t W) { return W % 4 == 0 && reinterpret_cast<uintptr_t>(masks) % 4 == 0; }

template <bool kWrite>
int rle_walk(const uint8_t* masks, int64_t n, int64_t H, int64_t W, RleSeg* seg, const int64_t* offsets, uint32_t* counts,
             cudaStream_t s) {
  const int64_t NB = rle_bands(H), G = ceil_div(W, 4);
  const int grid = grid_for(n * NB * G, RLE_NT);
  auto kern = rle_vec(masks, W) ? rle_boundary_kernel<true, kWrite> : rle_boundary_kernel<false, kWrite>;
  kern<<<grid, RLE_NT, 0, s>>>(masks, n, (int)H, (int)W, (int)NB, (int)G, seg, offsets, counts);
  return check_launch();
}

int rle_check_masks(const uint8_t* masks, int64_t n, int64_t H, int64_t W, const void* workspace, const void* out) {
  if (n < 0 || H < 0 || W < 0) return BXS_ERR_INVALID_ARG;
  if (H * W >= RLE_MAX_PIXELS) return BXS_ERR_UNSUPPORTED;
  if (n == 0) return BXS_OK;
  if ((!masks && H * W > 0) || !workspace || !out) return BXS_ERR_INVALID_ARG;
  return BXS_OK;
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_mask_rle_counts_workspace_bytes(int64_t n, int64_t H, int64_t W) {
  if (n <= 0 || H < 0 || W < 0 || H >= RLE_MAX_PIXELS || W >= RLE_MAX_PIXELS) return 0;
  return (int64_t)rle_runs_layout(n, H, W, nullptr, nullptr, nullptr);
}

extern "C" int bxs_mask_rle_runs(const uint8_t* masks, int64_t n, int64_t H, int64_t W, void* workspace, int64_t* offsets,
                                 bxs_stream_t stream) {
  if (int rc = rle_check_masks(masks, n, H, W, workspace, offsets)) return rc;
  if (n == 0) return BXS_OK;
  RleSeg* seg;
  int32_t* nb;
  rle_runs_layout(n, H, W, workspace, &seg, &nb);
  cudaStream_t s = as_stream(stream);
  const int64_t S = W * rle_bands(H);
  if (S > 0) {
    if (int rc = rle_walk<false>(masks, n, H, W, seg, nullptr, nullptr, s)) return rc;
  }
  rle_segment_scan_kernel<<<(unsigned)std::min<int64_t>(n, (int64_t)sm_count() * 8), RLE_NT, 0, s>>>(seg, n, S, nb);
  if (int rc = check_launch()) return rc;
  rle_offsets_scan_kernel<int32_t><<<1, RLE_SCAN_NT, 0, s>>>(nb, n, 1, offsets);
  return check_launch();
}

extern "C" int bxs_mask_rle_counts(const uint8_t* masks, int64_t n, int64_t H, int64_t W, const void* workspace,
                                   const int64_t* offsets, uint32_t* counts, bxs_stream_t stream) {
  if (int rc = rle_check_masks(masks, n, H, W, workspace, counts)) return rc;
  if (n == 0) return BXS_OK;
  if (!offsets) return BXS_ERR_INVALID_ARG;
  cudaStream_t s = as_stream(stream);
  if (H * W == 0) {                                    // one count of 0 per mask
    if (cudaError_t e = cudaMemsetAsync(counts, 0, (size_t)n * sizeof(uint32_t), s)) {
      set_last_error(e);
      return BXS_ERR_LAUNCH;
    }
    return BXS_OK;
  }
  RleSeg* seg;
  rle_runs_layout(n, H, W, const_cast<void*>(workspace), &seg, nullptr);
  return rle_walk<true>(masks, n, H, W, seg, offsets, counts, s);
}

extern "C" int64_t bxs_mask_rle_strings_workspace_bytes(int64_t n, int64_t R) {
  if (n <= 0 || R < n) return 0;
  const int64_t tiles = ceil_div(R, RLE_TILE);
  Carver c(nullptr);
  c.take((size_t)tiles * sizeof(int64_t));
  c.take((size_t)(tiles + 1) * sizeof(int64_t));
  return (int64_t)c.off;
}

extern "C" int bxs_mask_rle_strings(const uint32_t* counts, const int64_t* offsets, int64_t n, int64_t R, void* workspace,
                                    uint8_t* chars, int64_t* char_offsets, bxs_stream_t stream) {
  if (n < 0 || R < n) return BXS_ERR_INVALID_ARG;
  if (n == 0) return BXS_OK;
  if (!counts || !offsets || !workspace || !chars || !char_offsets) return BXS_ERR_INVALID_ARG;
  const int64_t tiles = ceil_div(R, RLE_TILE);
  if (tiles > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  Carver c(workspace);
  int64_t* tile_sum = reinterpret_cast<int64_t*>(c.take((size_t)tiles * sizeof(int64_t)));
  int64_t* tile_off = reinterpret_cast<int64_t*>(c.take((size_t)(tiles + 1) * sizeof(int64_t)));
  cudaStream_t s = as_stream(stream);
  rle_tile_chars_kernel<<<(unsigned)tiles, RLE_NT, 0, s>>>(counts, offsets, n, R, tile_sum);
  if (int rc = check_launch()) return rc;
  rle_offsets_scan_kernel<int64_t><<<1, RLE_SCAN_NT, 0, s>>>(tile_sum, tiles, 0, tile_off);
  if (int rc = check_launch()) return rc;
  rle_emit_kernel<<<(unsigned)tiles, RLE_NT, 0, s>>>(counts, offsets, n, R, tile_off, tiles, chars, char_offsets);
  return check_launch();
}
