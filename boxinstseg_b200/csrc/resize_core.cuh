// a18: the per-pixel arithmetic of the bilinear resize (ATen UpSample.cuh semantics: source index, lambdas, the order of the
// four products), shared by bxs_bilinear_resize_forward (fused_assembly.cu) and bxs_corr_paste (corr.cu) so that both give
// the same bits for the same input.
#pragma once

namespace bxs {

__device__ __forceinline__ float rs_scale(int in, int out, bool align) {
  if (align) return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  return (float)in / (float)out;
}
__device__ __forceinline__ float rs_src(float scale, int dst, bool align) {
  if (align) return scale * (float)dst;
  const float s = scale * ((float)dst + 0.5f) - 0.5f;
  return s < 0.f ? 0.f : s;
}
struct RsTap { int i0, ip; float l0, l1; };      // first tap, 0/1 offset of the second, weights
__device__ __forceinline__ RsTap rs_tap(float scale, int dst, int in, bool align) {
  RsTap t;
  const float r = rs_src(scale, dst, align);
  t.i0 = (int)r;
  t.ip = t.i0 < in - 1 ? 1 : 0;
  t.l1 = r - (float)t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}

// output pixel (oy, ox) of one h x w plane `in` resized with the scales sh, sw
__device__ __forceinline__ float rs_pixel(const float* __restrict__ in, int h, int w, float sh, float sw, int oy, int ox,
                                          bool align) {
  const RsTap ty = rs_tap(sh, oy, h, align), tx = rs_tap(sw, ox, w, align);
  const float* p = in + ty.i0 * w + tx.i0;
  const float v00 = __ldg(p), v01 = __ldg(p + tx.ip), v10 = __ldg(p + ty.ip * w), v11 = __ldg(p + ty.ip * w + tx.ip);
  return ty.l0 * (tx.l0 * v00 + tx.l1 * v01) + ty.l1 * (tx.l0 * v10 + tx.l1 * v11);
}

}  // namespace bxs
