// Dense masks of axis-aligned rectangles: out[g, y, x] = (y0_g <= y < y1_g) && (x0_g <= x < x1_g) for a batch of images,
// the bytes of mmdet's GenerateBoxMask (mmdet/datasets/pipelines/loading.py:647-668) written on the device from G x 4
// integers instead of copied from a host array.
//
//     The per-image sizes, output pointers and int32 rectangles travel by value in the kernel parameters: no
//     host-to-device copy and no host synchronisation, so a call can be captured in a CUDA graph.  One launch per
//     RZ_MAX_SEGS images or RZ_MAX_RECTS rectangles; an image with more rectangles spans several launches.
//
//     CTA (band, m) writes RZ_ROWS rows of the launch's mask m, one warp per row.  A row decides its span once: [x0, x1)
//     inside [y0, y1), empty elsewhere.  Each row is a scalar head up to the first 16-byte boundary, 16-byte vector stores
//     and a scalar tail, so any W and any element-aligned base work.  Purely write-bound: no reads of global memory, no
//     atomics, every output element written exactly once.
#include "common.cuh"

namespace bxs {
namespace {

constexpr int RZ_NT = 256;                         // threads per CTA: 8 warps
constexpr int RZ_ROWS = 32;                        // rows per CTA, RZ_ROWS / 8 per warp
constexpr int RZ_MAX_SEGS = 64;                    // image segments per launch
constexpr int RZ_MAX_RECTS = 1792;                 // rectangles (= masks) per launch
constexpr int64_t RZ_MAX_HW = INT32_MAX;           // H * W of one image

struct RzSeg {
  char* out;                                       // the segment's first mask, [n, H, W] dense
  int32_t H, W;
  int32_t r0, n;                                   // its rectangles rect[r0 .. r0 + n - 1]
};

struct RzTable {                                   // by value in the kernel parameters
  int4 rect[RZ_MAX_RECTS];                         // (y0, x0, y1, x1), 0 <= y0 <= y1 <= H, 0 <= x0 <= x1 <= W
  RzSeg seg[RZ_MAX_SEGS];
  int32_t n_segs;
  uint32_t one;                                    // the bit pattern of 1 in the output type
};
static_assert(sizeof(RzTable) <= 32764, "the table must fit the 32 KB kernel-parameter limit");

template <int ES> struct Elem;
template <> struct Elem<1> { using T = uint8_t; };
template <> struct Elem<2> { using T = uint16_t; };
template <> struct Elem<4> { using T = uint32_t; };

// one row of W elements at `row`: elements [xs, xe) are `one`, the rest 0
template <int ES>
__device__ __forceinline__ void write_row(char* row, int32_t W, int32_t xs, int32_t xe, uint32_t one, int lane) {
  using T = typename Elem<ES>::T;
  constexpr int V = 16 / ES;                       // elements per vector
  T* e = reinterpret_cast<T*>(row);
  const int32_t head = min(W, (int32_t)(((16 - (reinterpret_cast<uintptr_t>(row) & 15)) & 15) / ES));
  if (lane < head) e[lane] = (lane >= xs && lane < xe) ? (T)one : (T)0;
  const int32_t nv = (W - head) / V;
  uint4* vec = reinterpret_cast<uint4*>(e + head);
  for (int32_t v = lane; v < nv; v += kWarp) {
    const int32_t e0 = head + v * V;
    union { uint4 q; T t[V]; } u;
#pragma unroll
    for (int k = 0; k < V; ++k) u.t[k] = (e0 + k >= xs && e0 + k < xe) ? (T)one : (T)0;
    vec[v] = u.q;
  }
  const int32_t t0 = head + nv * V;
  if (t0 + lane < W) e[t0 + lane] = (t0 + lane >= xs && t0 + lane < xe) ? (T)one : (T)0;
}

template <int ES>
__global__ void __launch_bounds__(RZ_NT) box_masks_kernel(const RzTable tab) {
  const int32_t m = blockIdx.y;                    // the launch's mask = its rectangle
  int s = 0;
  while (s + 1 < tab.n_segs && tab.seg[s + 1].r0 <= m) ++s;
  const RzSeg& seg = tab.seg[s];
  const int32_t y_first = blockIdx.x * RZ_ROWS;
  if (y_first >= seg.H) return;
  const int4 r = tab.rect[m];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  char* mask = seg.out + (int64_t)(m - seg.r0) * seg.H * seg.W * ES;
  const int32_t y_end = min(seg.H, y_first + RZ_ROWS);
  for (int32_t y = y_first + wid; y < y_end; y += RZ_NT / kWarp) {
    const bool in = y >= r.x && y < r.z;
    write_row<ES>(mask + (int64_t)y * seg.W * ES, seg.W, in ? r.y : 0, in ? r.w : 0, tab.one, lane);
  }
}

int launch(const RzTable& tab, int32_t n_rects, int32_t max_h, int elem_bytes, cudaStream_t st) {
  const dim3 grid((unsigned)ceil_div(max_h, RZ_ROWS), (unsigned)n_rects);
  switch (elem_bytes) {
    case 1: box_masks_kernel<1><<<grid, RZ_NT, 0, st>>>(tab); break;
    case 2: box_masks_kernel<2><<<grid, RZ_NT, 0, st>>>(tab); break;
    default: box_masks_kernel<4><<<grid, RZ_NT, 0, st>>>(tab); break;
  }
  return check_launch();
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_box_masks_rasterize(void* const* out_host, const int32_t* rects_host, const int64_t* sizes_host,
                                       int64_t B, int elem_bytes, int64_t one_bits, bxs_stream_t stream) {
  if (B < 0 || (B > 0 && (!out_host || !sizes_host))) return BXS_ERR_INVALID_ARG;
  if (elem_bytes != 1 && elem_bytes != 2 && elem_bytes != 4) return BXS_ERR_INVALID_ARG;
  if (one_bits < 0 || (elem_bytes < 4 && one_bits >= ((int64_t)1 << (8 * elem_bytes))) || one_bits > UINT32_MAX)
    return BXS_ERR_INVALID_ARG;
  // every check before any device call
  int64_t total = 0, unsupported = 0;
  for (int64_t b = 0; b < B; ++b) {
    const int64_t G = sizes_host[3 * b], H = sizes_host[3 * b + 1], W = sizes_host[3 * b + 2];
    if (G < 0 || H < 0 || W < 0) return BXS_ERR_INVALID_ARG;
    if (G > 0 && H > 0 && W > 0 && (!out_host[b] || reinterpret_cast<uintptr_t>(out_host[b]) % elem_bytes))
      return BXS_ERR_INVALID_ARG;
    if (G > 0 && !rects_host) return BXS_ERR_INVALID_ARG;
    for (int64_t g = 0; g < G; ++g) {
      const int32_t* r = rects_host + 4 * (total + g);
      if (r[0] < 0 || r[0] > r[2] || r[2] > H || r[1] < 0 || r[1] > r[3] || r[3] > W) return BXS_ERR_INVALID_ARG;
    }
    if (H > 0 && W > RZ_MAX_HW / H) unsupported = 1;
    total += G;
  }
  if (unsupported) return BXS_ERR_UNSUPPORTED;
  const cudaStream_t st = as_stream(stream);
  RzTable tab;
  tab.n_segs = 0;
  tab.one = (uint32_t)one_bits;
  int32_t n_rects = 0, max_h = 0;
  int64_t first = 0;                               // the image's first rectangle in rects_host
  for (int64_t b = 0; b < B; first += sizes_host[3 * b], ++b) {
    const int64_t G = sizes_host[3 * b], H = sizes_host[3 * b + 1], W = sizes_host[3 * b + 2];
    if (G == 0 || H == 0 || W == 0) continue;
    for (int64_t g = 0; g < G;) {
      if (tab.n_segs == RZ_MAX_SEGS || n_rects == RZ_MAX_RECTS) {
        if (const int rc = launch(tab, n_rects, max_h, elem_bytes, st)) return rc;
        tab.n_segs = n_rects = max_h = 0;
      }
      const int32_t n = (int32_t)std::min<int64_t>(G - g, RZ_MAX_RECTS - n_rects);
      tab.seg[tab.n_segs++] = RzSeg{static_cast<char*>(out_host[b]) + g * H * W * elem_bytes, (int32_t)H, (int32_t)W,
                                    n_rects, n};
      for (int32_t k = 0; k < n; ++k) {
        const int32_t* r = rects_host + 4 * (first + g + k);
        tab.rect[n_rects + k] = make_int4(r[0], r[1], r[2], r[3]);
      }
      n_rects += n;
      max_h = std::max(max_h, (int32_t)H);
      g += n;
    }
  }
  if (n_rects > 0) return launch(tab, n_rects, max_h, elem_bytes, st);
  return BXS_OK;
}
