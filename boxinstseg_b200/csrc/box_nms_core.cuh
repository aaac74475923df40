// CondInst inference: the per-element arithmetic of CondInstBoxHead._get_bboxes (condinst_head.py:762-810: distance2bbox
// with the per-image clamp of mmdet/core/bbox/transforms.py:153-184 and the division by scale_factor), of mmcv's CUDA NMS
// suppression test (devIoU of mmcv/ops/csrc/common/cuda/nms_cuda_kernel.cuh with offset 0) and of aligned_bilinear
// (condinst_head.py:146-167), shared by the kernels of condinst_infer.cu and, compiled for the host, by
// tests/host_harness/box_nms_host.cpp.
//
// Every floating-point value is one correctly rounded fp32 operation in the reference's order (the BXS_F* macros keep the
// compiler from contracting a product into a following sum).
#pragma once
#include <math.h>
#include <stdint.h>

#include "assign_core.cuh"            // BXS_HD, BXS_FADD / FSUB / FMUL / FDIV
#include "resize_core.cuh"            // rs_scale, rs_tap

namespace bxs {

// MlvlPointGenerator(offset=0.5): (x + 0.5) * stride, exact in fp32 for every feature map a detector sees
BXS_HD float ci_point(int x, float stride) { return BXS_FMUL(BXS_FADD((float)x, 0.5f), stride); }

// torch.where(v < 0, 0, v) then torch.where(v > hi, hi, v): a NaN passes through both
BXS_HD float ci_clip(float v, float hi) {
  v = v < 0.f ? 0.f : v;
  return v > hi ? hi : v;
}

// distance2bbox(points, distance, max_shape) of one point: d = (left, top, right, bottom); (img_h, img_w) = max_shape[:2];
// sf = scale_factor (w, h, w, h) or nullptr when not rescaling.  out = (x1, y1, x2, y2).
BXS_HD void ci_decode_box(float px, float py, const float d[4], float img_h, float img_w, const float* sf, float out[4]) {
  out[0] = ci_clip(BXS_FSUB(px, d[0]), img_w);
  out[1] = ci_clip(BXS_FSUB(py, d[1]), img_h);
  out[2] = ci_clip(BXS_FADD(px, d[2]), img_w);
  out[3] = ci_clip(BXS_FADD(py, d[3]), img_h);
  if (sf)
    for (int k = 0; k < 4; ++k) out[k] = BXS_FDIV(out[k], sf[k]);
}

// mmcv's suppression test of box b by the higher-scored box a (offset 0): interS > thr * (Sa + Sb - interS), with
// fmaxf / fminf (a NaN coordinate loses to the other box's).  The boxes are batched_nms's offset boxes.
BXS_HD bool ci_suppresses(const float a[4], const float b[4], float thr) {
  const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
  const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
  const float width = fmaxf(BXS_FSUB(right, left), 0.f), height = fmaxf(BXS_FSUB(bottom, top), 0.f);
  const float inter = BXS_FMUL(width, height);
  const float sa = BXS_FMUL(BXS_FSUB(a[2], a[0]), BXS_FSUB(a[3], a[1]));
  const float sb = BXS_FMUL(BXS_FSUB(b[2], b[0]), BXS_FSUB(b[3], b[1]));
  return inter > BXS_FMUL(thr, BXS_FSUB(BXS_FADD(sa, sb), inter));
}

// aligned_bilinear(t, f) of an h x w plane, pixel (Y, X) of its [f*h, f*w] result: pixel (max(Y - f/2, 0), max(X - f/2, 0))
// of the align_corners=True resize to (f*h + 1, f*w + 1) of t padded by one replicated row and column.  The two taps of
// one axis of that resize; their source indices lie in the padded plane (clamp them to h - 1 / w - 1 to read t).
BXS_HD RsTap ci_aligned_tap(int Y, int in, int f) {
  const int d = Y - f / 2;
  return rs_tap(rs_scale(in + 1, f * in + 1, true), d < 0 ? 0 : d, in + 1, true);
}

}  // namespace bxs
