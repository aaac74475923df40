// SOLOv2 inference: the per-element arithmetic of mask_matrix_nms (mmdet/core/post_processing/matrix_nms.py:63-101) and of
// the two-stage mask paste of get_seg_single (box_solov2_head.py:576-585, discobox_head.py:1645-1653), shared by the kernels
// of solo_seg.cu and, compiled for the host, by tests/host_harness/matrix_nms_host.cpp.
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
// first-stage taps of intermediate pixel (y1, x1) of the (4h, 4w) upsampling of an h x w plane
BXS_HD RsTap paste_stage1_tap(int d1, int in) { return rs_tap(rs_scale(in, 4 * in, false), d1, in, false); }

}  // namespace bxs
