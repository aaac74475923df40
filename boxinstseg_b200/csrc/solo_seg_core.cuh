// SOLOv2 inference: the per-element arithmetic of mask_matrix_nms (mmdet/core/post_processing/matrix_nms.py:63-101) and of
// the two-stage mask paste of get_seg_single (box_solov2_head.py:576-585, discobox_head.py:1645-1653), shared by the kernels
// of solo_seg.cu and, compiled for the host, by tests/host_harness/matrix_nms_host.cpp; the paste and the per-mask
// statistics are also those of MaskFormerFusionHead's instance masks (tests/host_harness/box2mask_infer_host.cpp).
//
// Every floating-point value is one correctly rounded fp32 operation of the reference in the reference's order (the BXS_F*
// macros keep the compiler from contracting a product into a following sum); exp is the C library's expf, which is what
// torch's CUDA exp calls for a float tensor.
#pragma once
#include <math.h>
#include <stdint.h>

#include "assign_core.cuh"            // BXS_HD, BXS_FADD / FSUB / FMUL / FDIV
#include "resize_core.cuh"            // rs_scale, rs_tap, rs_lerp2

namespace bxs {

enum { kNmsGaussian = 0, kNmsLinear = 1 };

// iou_matrix[i, j] = inter / (area[j] + area[i] - inter)   (:77-80: expanded_mask_area + its transpose - inter_matrix)
BXS_HD float nms_iou(float inter, float area_i, float area_j) {
  return BXS_FDIV(inter, BXS_FSUB(BXS_FADD(area_j, area_i), inter));
}

// decay_matrix[i, j] / compensate_matrix[i, j] (gaussian, :91-94; nsig = -1 * sigma) or (1 - iou) / (1 - comp) (linear,
// :96-97), for decay_iou[i, j] = iou (0 off the upper triangle or across labels) and compensate_iou[i] = comp.  The
// decay coefficient of column j is the minimum of this over every row i.
BXS_HD float nms_decay_ratio(float iou, float comp, int kernel, float nsig) {
  if (kernel == kNmsGaussian)
    return BXS_FDIV(expf(BXS_FMUL(nsig, BXS_FMUL(iou, iou))), expf(BXS_FMUL(nsig, BXS_FMUL(comp, comp))));
  return BXS_FDIV(BXS_FSUB(1.f, iou), BXS_FSUB(1.f, comp));
}

// torch.min's order: a NaN wins and stays
BXS_HD float nan_min(float m, float v) { return (v < m || v != v) ? v : m; }

// The taps of output pixel (y, x) of interpolate(interpolate(p, (4h, 4w))[:H_img, :W_img], (H_ori, W_ori)), both bilinear
// with align_corners=False: the second stage reads the four intermediate pixels (y1[a], x1[c]) with weights ty2 / tx2; each
// of those is the first stage's lerp of four input pixels.  The crop only bounds the second stage's source size.
struct PasteTaps {
  RsTap ty2, tx2;
  int y1[2], x1[2];
};
BXS_HD PasteTaps paste_taps(int y, int x, int H_img, int W_img, int H_ori, int W_ori) {
  PasteTaps t;
  t.ty2 = rs_tap(rs_scale(H_img, H_ori, false), y, H_img, false);
  t.tx2 = rs_tap(rs_scale(W_img, W_ori, false), x, W_img, false);
  t.y1[0] = t.ty2.i0;
  t.y1[1] = t.ty2.i0 + t.ty2.ip;
  t.x1[0] = t.tx2.i0;
  t.x1[1] = t.tx2.i0 + t.tx2.ip;
  return t;
}
// first-stage taps of intermediate pixel d1 of the resize of `in` input pixels to `out`
BXS_HD RsTap paste_stage1_tap(int d1, int in, int out) { return rs_tap(rs_scale(in, out, false), d1, in, false); }
// ... of the (4h, 4w) upsampling of SOLOv2's paste
BXS_HD RsTap paste_stage1_tap(int d1, int in) { return paste_stage1_tap(d1, in, 4 * in); }

// interpolate(interpolate(x, (H1, W1))[:H_img, :W_img], (H_out, W_out)) of an h x w plane.  A stage whose input and output
// sizes are equal is skipped (skip1: (h, w) == (H1, W1); skip2: (H_out, W_out) == (H_img, W_img)): its value is read, not
// lerped.  ATen copies there too, and 1 * v + 0 * v' is not v when a neighbour v' is +-inf or NaN.
struct PasteGeom {
  int h, w, H1, W1, H_img, W_img, H_out, W_out;
  bool skip1, skip2;
};

// Output pixel (y, x) before the threshold.  at(o, d) is input element o + d widened to float (the probability for a
// SOLOv2 logit row); rnd(v) rounds a stage's lerp to the row dtype.  kSkip = false: no stage is skipped (SOLOv2's paste),
// and the skip flags are not read.
template <bool kSkip, typename At, typename Rnd>
BXS_HD float paste_value(const PasteGeom& g, int y, int x, At at, Rnd rnd) {
  const bool skip1 = kSkip && g.skip1;
  const auto stage1 = [&](const RsTap& ty, int y1, int x1) {
    if (skip1) return at(y1 * g.w + x1, 0);
    const RsTap tx = paste_stage1_tap(x1, g.w, g.W1);
    const int o = ty.i0 * g.w + tx.i0;
    return rnd(rs_lerp2(ty, tx, at(o, 0), at(o, tx.ip), at(o, ty.ip * g.w), at(o, ty.ip * g.w + tx.ip)));
  };
  if (kSkip && g.skip2) return stage1(skip1 ? RsTap{} : paste_stage1_tap(y, g.h, g.H1), y, x);
  const PasteTaps pt = paste_taps(y, x, g.H_img, g.W_img, g.H_out, g.W_out);
  float v[2][2];
#if defined(__CUDACC__)
#pragma unroll
#endif
  for (int a = 0; a < 2; ++a) {
    const RsTap ty = skip1 ? RsTap{} : paste_stage1_tap(pt.y1[a], g.h, g.H1);
#if defined(__CUDACC__)
#pragma unroll
#endif
    for (int c = 0; c < 2; ++c) v[a][c] = stage1(ty, pt.y1[a], pt.x1[c]);
  }
  return rnd(rs_lerp2(pt.ty2, pt.tx2, v[0][0], v[0][1], v[1][0], v[1][1]));
}

// The statistics of one mask at its output resolution that MaskFormerFusionHead.instance_postprocess (:146-152) and
// mask2bbox (mmdet/core/mask/utils.py:68-89) compute: the set pixels' count, the sum of their sigmoid (float64, summed in
// a fixed order by the callers and rounded once) and their extents.  An empty mask's box is zeros.
struct MaskStats {
  double sum;
  int area, x0, y0, x1, y1;
};
BXS_HD MaskStats mask_stats_empty() { return MaskStats{0.0, 0, INT32_MAX, INT32_MAX, -1, -1}; }
BXS_HD void mask_stats_add(MaskStats& s, int y, int x, float sig) {
  s.sum += (double)sig;
  ++s.area;
  s.x0 = x < s.x0 ? x : s.x0;
  s.y0 = y < s.y0 ? y : s.y0;
  s.x1 = x > s.x1 ? x : s.x1;
  s.y1 = y > s.y1 ? y : s.y1;
}
BXS_HD void mask_stats_merge(MaskStats& s, const MaskStats& o) {
  s.sum += o.sum;
  s.area += o.area;
  s.x0 = o.x0 < s.x0 ? o.x0 : s.x0;
  s.y0 = o.y0 < s.y0 ? o.y0 : s.y0;
  s.x1 = o.x1 > s.x1 ? o.x1 : s.x1;
  s.y1 = o.y1 > s.y1 ? o.y1 : s.y1;
}
// [x_min, y_min, x_max + 1, y_max + 1], or zeros
BXS_HD void mask_stats_box(const MaskStats& s, float* box) {
  const bool any = s.area > 0;
  box[0] = any ? (float)s.x0 : 0.f;
  box[1] = any ? (float)s.y0 : 0.f;
  box[2] = any ? (float)(s.x1 + 1) : 0.f;
  box[3] = any ? (float)(s.y1 + 1) : 0.f;
}

}  // namespace bxs
