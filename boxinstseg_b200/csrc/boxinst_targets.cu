// a5: BoxInst target building on the GPU -- de-normalise -> uint8 -> stride x stride mean ->
// uint8 -> CIE-LAB -> 8-neighbour colour similarity -> threshold bits; box -> grid rectangle.
// Replaces CondInstMaskHead.get_targets / get_bitmasks_from_boxes / get_original_image /
// get_image_color_similarity (condinst_head.py:170-246, 1345-1448), which round-trip every image
// through the host (mmcv.tensor2imgs, skimage.color.rgb2lab) and loop over GT boxes in Python.
//
// Exactness: everything up to the uint8 downsampled image is integer work and is bit-exact
// (two separately rounded fp32 ops reproduce OpenCV's multiply/add; sums of <=255*s*s are exact).
// LAB is evaluated in float64 exactly as scikit-image does and only then cast to float32.
#include "common.cuh"

namespace bxs {
namespace {

struct Norm { float mean[3]; float std[3]; };

// scikit-image rgb2lab constants: sRGB D65 matrix, D65 2-degree white point
__device__ __forceinline__ void rgb_u8_to_lab(int r, int g, int b, float* lab) {
  double c[3] = {r / 255.0, g / 255.0, b / 255.0};
#pragma unroll
  for (int k = 0; k < 3; ++k) c[k] = c[k] > 0.04045 ? pow((c[k] + 0.055) / 1.055, 2.4) : c[k] / 12.92;
  double x = (0.412453 * c[0] + 0.357580 * c[1] + 0.180423 * c[2]) / 0.95047;
  double y = (0.212671 * c[0] + 0.715160 * c[1] + 0.072169 * c[2]) / 1.0;
  double z = (0.019334 * c[0] + 0.119193 * c[1] + 0.950227 * c[2]) / 1.08883;
  double f[3] = {x, y, z};
#pragma unroll
  for (int k = 0; k < 3; ++k) f[k] = f[k] > 0.008856 ? cbrt(f[k]) : 7.787 * f[k] + 16.0 / 116.0;
  lab[0] = (float)(116.0 * f[1] - 16.0);
  lab[1] = (float)(500.0 * (f[0] - f[1]));
  lab[2] = (float)(200.0 * (f[1] - f[2]));
}

// Python slice semantics of `full[int(y1):int(y2)+1, int(x1):int(x2)+1] = 1` followed by
// `[s//2::s, s//2::s]`  (condinst_head.py:1429-1432)
__device__ __forceinline__ void slice_range(float lo_f, float hi_f, int len, int s, int& g0, int& g1) {
  int start = (int)lo_f, stop = (int)hi_f + 1;       // int(): truncation toward zero
  if (start < 0) start += len;
  if (stop < 0) stop += len;
  start = min(max(start, 0), len);
  stop = min(max(stop, 0), len);
  // sampled positions s/2 + k*s inside [start, stop)
  const int h = s / 2;
  g0 = start <= h ? 0 : (start - h + s - 1) / s;
  g1 = stop - 1 >= h ? (stop - 1 - h) / s : -1;
  const int glen = (len - h + s - 1) / s;
  g1 = min(g1, glen - 1);
}

// one output pixel (b, j, i) of the stride-s LAB image and its validity
__device__ __forceinline__ void lab_pixel(const float* __restrict__ img, const Norm& nm, int ih, int iw, int removed,
                                          float* __restrict__ lab, uint8_t* __restrict__ valid, int b, int j, int i, int H,
                                          int W, int Hp, int Wp, int s) {
  int u8[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* plane = img + ((int64_t)b * 3 + c) * Hp * Wp;
    int sum = 0;
    for (int dy = 0; dy < s; ++dy) {
      const int y = j * s + dy;
      if (y >= ih) break;                                       // zero padding below the image
      for (int dx = 0; dx < s; ++dx) {
        const int x = i * s + dx;
        if (x >= iw) break;
        // tensor2imgs: float32 multiply, float32 add (separately rounded), astype(uint8)
        float f = __fadd_rn(__fmul_rn(__ldg(plane + (int64_t)y * Wp + x), nm.std[c]), nm.mean[c]);
        sum += (int)fminf(fmaxf(truncf(f), 0.f), 255.f);
      }
    }
    // avg_pool2d in fp32 (exact integer sum), then .byte() truncation
    u8[c] = (int)truncf(__fdiv_rn((float)sum, (float)(s * s)));
  }
  float l3[3];
  rgb_u8_to_lab(u8[0], u8[1], u8[2], l3);
  const int64_t plane_sz = (int64_t)H * W, o = (int64_t)j * W + i;
  lab[((int64_t)b * 3 + 0) * plane_sz + o] = l3[0];
  lab[((int64_t)b * 3 + 1) * plane_sz + o] = l3[1];
  lab[((int64_t)b * 3 + 2) * plane_sz + o] = l3[2];
  const int sy = j * s + s / 2, sx = i * s + s / 2;
  valid[(int64_t)b * plane_sz + o] = (sy < ih - removed && sx < iw) ? 1 : 0;
}

// The per-image metadata of up to kMaxMetaImages images travels BY VALUE in the kernel parameters (no host-to-device
// copy, nothing to keep alive, capturable in a CUDA graph): image sizes, removed bottom rows, and the running GT count
// (gt_end[b] = number of GT boxes of images 0..b).  Larger batches take one launch per chunk of that many images.
constexpr int kMaxMetaImages = 64;
struct TargetsMeta {
  int ih[kMaxMetaImages], iw[kMaxMetaImages], removed[kMaxMetaImages], gt_end[kMaxMetaImages];
  Norm nm;
};

// lab + validity of every stride-s pixel; the tail of the grid also turns the GT boxes into grid rectangles and writes
// the image index of every GT (get_bitmasks_from_boxes' per-image loop, condinst_head.py:1417-1448).  All pointers and
// counts are those of one chunk of images; b0, the chunk's first image, makes gt_img a batch-wide image index.
__global__ void lab_rects_kernel(const float* __restrict__ img, const float* __restrict__ boxes,
                                 const __grid_constant__ TargetsMeta meta, float* __restrict__ lab, uint8_t* __restrict__ valid,
                                 int32_t* __restrict__ rects, int32_t* __restrict__ gt_img, int B, int b0, int G, int Hp, int Wp,
                                 int s) {
  const int H = Hp / s, W = Wp / s;
  const int64_t total = (int64_t)B * H * W;
  const int64_t tid0 = blockIdx.x * (int64_t)blockDim.x + threadIdx.x, nth = (int64_t)gridDim.x * blockDim.x;
  for (int64_t idx = tid0; idx < total; idx += nth) {
    const int i = idx % W, j = (idx / W) % H, b = idx / ((int64_t)W * H);
    lab_pixel(img, meta.nm, meta.ih[b], meta.iw[b], meta.removed[b], lab, valid, b, j, i, H, W, Hp, Wp, s);
  }
  for (int64_t g = nth - 1 - tid0; g < G; g += nth) {            // the last threads of the grid: least pixel work
    const float x1 = boxes[4 * g], y1 = boxes[4 * g + 1], x2 = boxes[4 * g + 2], y2 = boxes[4 * g + 3];
    int j0, j1, i0, i1;
    slice_range(y1, y2, Hp, s, j0, j1);
    slice_range(x1, x2, Wp, s, i0, i1);
    *reinterpret_cast<int4*>(rects + 4 * g) = make_int4(j0, j1, i0, i1);
    int b = 0;
    while (b < B - 1 && g >= meta.gt_end[b]) ++b;
    gt_img[g] = b0 + b;
  }
}

__global__ void similarity_kernel(const float* __restrict__ lab, const uint8_t* __restrict__ valid,
                                  float* __restrict__ sim, uint8_t* __restrict__ edge_bits, int B, int H, int W,
                                  int size, int dil, float thresh) {
  const int R = (size / 2) * dil, K = size * size - 1;
  const int64_t plane = (int64_t)H * W, total = (int64_t)B * plane;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int x = idx % W, y = (idx / W) % H, b = idx / plane;
    const float* L = lab + (int64_t)b * 3 * plane;
    const float p0 = L[(int64_t)y * W + x], p1 = L[plane + (int64_t)y * W + x], p2 = L[2 * plane + (int64_t)y * W + x];
    unsigned bits = 0;
    int c = 0;
    for (int dy = -R; dy <= R; dy += dil)
      for (int dx = -R; dx <= R; dx += dil) {
        if (dy == 0 && dx == 0) continue;
        const int qy = y + dy, qx = x + dx;
        float s = 0.f;      // out-of-image neighbour: the unfolded mask is zero padded
        if (qy >= 0 && qy < H && qx >= 0 && qx < W && valid[(int64_t)b * plane + (int64_t)qy * W + qx]) {
          const int64_t q = (int64_t)qy * W + qx;
          const float d0 = p0 - L[q], d1 = p1 - L[plane + q], d2 = p2 - L[2 * plane + q];
          const float n2 = __fadd_rn(__fadd_rn(__fmul_rn(d0, d0), __fmul_rn(d1, d1)), __fmul_rn(d2, d2));
          s = expf(-__fmul_rn(__fsqrt_rn(n2), 0.5f));
        }
        if (sim) sim[(((int64_t)b * K + c) * H + y) * W + x] = s;
        if (s >= thresh && c < 8) bits |= 1u << c;
        ++c;
      }
    if (edge_bits) edge_bits[idx] = (uint8_t)bits;
  }
}

__global__ void bitmask_kernel(const int32_t* __restrict__ rects, float* __restrict__ out, int64_t G, int H, int W) {
  const int64_t total = G * H * W;
  for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < total;
       idx += (int64_t)gridDim.x * blockDim.x) {
    const int x = idx % W, y = (idx / W) % H;
    const int64_t g = idx / ((int64_t)W * H);
    const int4 r = *reinterpret_cast<const int4*>(rects + 4 * g);
    out[idx] = (y >= r.x && y <= r.y && x >= r.z && x <= r.w) ? 1.f : 0.f;
  }
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_boxinst_bitmasks(const int32_t* rects, float* bitmasks, int64_t G, int64_t H, int64_t W,
                                    bxs_stream_t stream) {
  if (G == 0) return BXS_OK;
  if (!rects || !bitmasks || G < 0 || H <= 0 || W <= 0) return BXS_ERR_INVALID_ARG;
  bitmask_kernel<<<grid_for(G * H * W, 256), 256, 0, as_stream(stream)>>>(rects, bitmasks, G, (int)H, (int)W);
  return check_launch();
}


// ---------------------------------------------------------------------------------------
// Whole target build of a batch: LAB + validity + grid rectangles + GT image index, one launch per kMaxMetaImages
// images with the metadata by value, then the colour similarity / edge bits in one launch.  No host-to-device copies,
// capturable in a CUDA graph.
// ---------------------------------------------------------------------------------------
extern "C" int bxs_boxinst_targets_forward(const float* img, const float* boxes, const int32_t* img_hw_host,
                                           const int32_t* removed_rows_host, const int32_t* num_gts_host,
                                           const float* mean3_host, const float* std3_host, float* lab, uint8_t* valid,
                                           float* sim, uint8_t* edge_bits, int32_t* rects, int32_t* gt_img, int64_t B,
                                           int64_t Hp, int64_t Wp, int stride, int size, int dilation, float thresh,
                                           bxs_stream_t stream) {
  if (!img || !img_hw_host || !removed_rows_host || !num_gts_host || !mean3_host || !std3_host || !lab || !valid ||
      (!sim && !edge_bits) || B <= 0 || Hp <= 0 || Wp <= 0 || stride <= 0 || stride > 256 || Hp % stride || Wp % stride ||
      size < 3 || !(size & 1) || dilation < 1 || (edge_bits && size != 3))
    return BXS_ERR_INVALID_ARG;
  int64_t G = 0;
  for (int64_t b = 0; b < B; ++b) {
    if (num_gts_host[b] < 0) return BXS_ERR_INVALID_ARG;
    G += num_gts_host[b];
  }
  if (G > 0 && (!boxes || !rects || !gt_img)) return BXS_ERR_INVALID_ARG;
  TargetsMeta meta;
  for (int c = 0; c < 3; ++c) { meta.nm.mean[c] = mean3_host[c]; meta.nm.std[c] = std3_host[c]; }
  const int64_t H = Hp / stride, W = Wp / stride;
  cudaStream_t st = as_stream(stream);
  for (int64_t b0 = 0, g0 = 0; b0 < B; b0 += kMaxMetaImages) {
    const int64_t nb = std::min<int64_t>(B - b0, kMaxMetaImages), total = nb * H * W;
    int64_t gc = 0;
    for (int b = 0; b < kMaxMetaImages; ++b) {
      const bool in = b < nb;
      if (in) gc += num_gts_host[b0 + b];
      meta.ih[b] = in ? img_hw_host[2 * (b0 + b)] : 0;
      meta.iw[b] = in ? img_hw_host[2 * (b0 + b) + 1] : 0;
      meta.removed[b] = in ? removed_rows_host[b0 + b] : 0;
      meta.gt_end[b] = (int)gc;
    }
    lab_rects_kernel<<<(unsigned)std::max<int64_t>(ceil_div(total, 128), ceil_div(std::min<int64_t>(gc, total), 128)), 128, 0,
                       st>>>(img + b0 * 3 * Hp * Wp, boxes + 4 * g0, meta, lab + b0 * 3 * H * W, valid + b0 * H * W,
                             rects + 4 * g0, gt_img + g0, (int)nb, (int)b0, (int)gc, (int)Hp, (int)Wp, stride);
    const int rc = check_launch();
    if (rc != BXS_OK) return rc;
    g0 += gc;
  }
  similarity_kernel<<<grid_for(B * H * W, 128), 128, 0, st>>>(lab, valid, sim, edge_bits, (int)B, (int)H, (int)W, size,
                                                               dilation, thresh);
  return check_launch();
}

// CIE-LAB of packed uint8 RGB triplets (test hook for the colour conversion: all 2^24 colours against the oracle)
namespace bxs { namespace {
__global__ void lab_of_u8_kernel(const uint8_t* __restrict__ rgb, float* __restrict__ lab, int64_t n) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    rgb_u8_to_lab(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], lab + 3 * i);
}
} }
extern "C" int bxs_rgb_u8_to_lab(const uint8_t* rgb, float* lab, int64_t n, bxs_stream_t stream) {
  if (n == 0) return BXS_OK;
  if (!rgb || !lab || n < 0) return BXS_ERR_INVALID_ARG;
  lab_of_u8_kernel<<<grid_for(n, 256), 256, 0, as_stream(stream)>>>(rgb, lab, n);
  return check_launch();
}
