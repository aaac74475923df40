// a18: the per-pixel arithmetic of the bilinear resize (ATen UpSample.cuh semantics: source index, lambdas, the order of the
// four products), shared by bxs_bilinear_resize_forward (fused_assembly.cu), bxs_corr_paste (corr.cu),
// bxs_box2mask_attn_mask (box2mask_attn.cu) and bxs_solo_paste_masks (solo_seg.cu) so that all give the same bits for the
// same input.  The tap arithmetic (rs_scale, rs_src, rs_tap, rs_lerp2) is host-compilable too, for the host twin of the
// mask paste (tests/host_harness/matrix_nms_host.cpp).
#pragma once
#if defined(__CUDACC__)
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#define BXS_RS_HD __host__ __device__ __forceinline__
#else
#define BXS_RS_HD inline
#endif

namespace bxs {

BXS_RS_HD float rs_scale(int in, int out, bool align) {
  if (align) return out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f;
  return (float)in / (float)out;
}
BXS_RS_HD float rs_src(float scale, int dst, bool align) {
  if (align) return scale * (float)dst;
  const float s = scale * ((float)dst + 0.5f) - 0.5f;
  return s < 0.f ? 0.f : s;
}
struct RsTap { int i0, ip; float l0, l1; };      // first tap, 0/1 offset of the second, weights
BXS_RS_HD RsTap rs_tap(float scale, int dst, int in, bool align) {
  RsTap t;
  const float r = rs_src(scale, dst, align);
  t.i0 = (int)r;
  t.ip = t.i0 < in - 1 ? 1 : 0;
  t.l1 = r - (float)t.i0;
  t.l0 = 1.f - t.l1;
  return t;
}
// the four taps v_yx weighted as ATen weighs them
BXS_RS_HD float rs_lerp2(const RsTap& ty, const RsTap& tx, float v00, float v01, float v10, float v11) {
  return ty.l0 * (tx.l0 * v00 + tx.l1 * v01) + ty.l1 * (tx.l0 * v10 + tx.l1 * v11);
}

#if defined(__CUDACC__)
// a tap widened to float: a 16-bit plane is interpolated in float32, as ATen does (accscalar_t)
__device__ __forceinline__ float rs_load(const float* p) { return __ldg(p); }
__device__ __forceinline__ float rs_load(const __half* p) { return __half2float(__ldg(p)); }
__device__ __forceinline__ float rs_load(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }

// output pixel (oy, ox) of one h x w plane `in` resized with the scales sh, sw
template <typename T>
__device__ __forceinline__ float rs_pixel(const T* __restrict__ in, int h, int w, float sh, float sw, int oy, int ox,
                                          bool align) {
  const RsTap ty = rs_tap(sh, oy, h, align), tx = rs_tap(sw, ox, w, align);
  const T* p = in + ty.i0 * w + tx.i0;
  return rs_lerp2(ty, tx, rs_load(p), rs_load(p + tx.ip), rs_load(p + ty.ip * w), rs_load(p + ty.ip * w + tx.ip));
}
#endif

}  // namespace bxs
