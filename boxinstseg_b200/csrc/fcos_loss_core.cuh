// Per-point core of CondInstBoxHead.loss's regression and centerness branch (mmdet/models/dense_heads/condinst_head.py:
// 396-469): the location of a point (MlvlPointGenerator.grid_priors, core/anchor/point_generator.py:150-165), its
// centerness target (:855-874), distance2bbox of the prediction and of the target, 1 - GIoU of the two boxes
// (bbox_overlaps(mode='giou', is_aligned=True), core/bbox/iou_calculators/iou2d_calculator.py:204-261, through
// losses/iou_loss.py giou_loss), F.binary_cross_entropy_with_logits, and their gradients.
//
// Every value is ONE correctly rounded fp32 operation of the reference, in the reference's order (the BXS_F* macros of
// assign_core.cuh keep the compiler from contracting a product into a following sum), so the point and the centerness
// target are bit-exact.  At ties the gradients follow autograd's conventions for the reference's lines: the elementwise
// torch.max / torch.min of two tensors hands half the gradient to each side when they are equal, clamp(min=0) passes the
// gradient at 0, and torch.max(union, eps) is a torch.max of two tensors.
//
// The body is BXS_HD so that tests/host_harness/fcos_loss_host.cpp can compile the very same lines for the host and check
// them against the float64 oracle without a GPU.
#pragma once
#include <math.h>
#include <stdint.h>

#include "assign_core.cuh"

namespace bxs {

#if defined(__CUDA_ARCH__)
#define BXS_FSQRT(a) __fsqrt_rn(a)
#else
#define BXS_FSQRT(a) sqrtf(a)
#endif

// ((i + 0.5) * stride): shift_x / shift_y of single_level_grid_priors, exact in fp32
BXS_HD float fcos_point_coord(int64_t i, float stride) { return BXS_FMUL(BXS_FADD((float)i, 0.5f), stride); }

// sqrt((min(l, r) / max(l, r)) * (min(t, b) / max(t, b))) of one positive's regression target
BXS_HD float fcos_centerness_target(const float t[4]) {
  const float lr = BXS_FDIV(fminf(t[0], t[2]), fmaxf(t[0], t[2]));
  const float tb = BXS_FDIV(fminf(t[1], t[3]), fmaxf(t[1], t[3]));
  return BXS_FSQRT(BXS_FMUL(lr, tb));
}

// distance2bbox: (x - l, y - t, x + r, y + b)
BXS_HD void fcos_decode(float x, float y, const float d[4], float box[4]) {
  box[0] = BXS_FSUB(x, d[0]);
  box[1] = BXS_FSUB(y, d[1]);
  box[2] = BXS_FADD(x, d[2]);
  box[3] = BXS_FADD(y, d[3]);
}

// d max(a, b) / d a and d min(a, b) / d a of torch.max / torch.min of two tensors: 1, 1/2 at a tie, 0
BXS_HD float dmax_first(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }
BXS_HD float dmin_first(float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); }
// clamp(min=0) and its gradient mask (passes at 0); a NaN stays NaN
BXS_HD float clamp0(float v) { return v < 0.f ? 0.f : v; }
BXS_HD float dclamp0(float v) { return v >= 0.f ? 1.f : 0.f; }
// torch.max(v, eps) with eps a tensor: a NaN stays NaN
BXS_HD float max_eps(float v, float eps) { return v < eps ? eps : v; }

// 1 - GIoU of the prediction box p and the target box q (x1, y1, x2, y2), and d (1 - GIoU) / d p
BXS_HD float giou_loss_grad(const float p[4], const float q[4], float eps, float gp[4]) {
  const float pw = BXS_FSUB(p[2], p[0]), ph = BXS_FSUB(p[3], p[1]);
  const float area1 = BXS_FMUL(pw, ph);
  const float area2 = BXS_FMUL(BXS_FSUB(q[2], q[0]), BXS_FSUB(q[3], q[1]));
  const float ltx = fmaxf(p[0], q[0]), lty = fmaxf(p[1], q[1]);
  const float rbx = fminf(p[2], q[2]), rby = fminf(p[3], q[3]);
  const float dx = BXS_FSUB(rbx, ltx), dy = BXS_FSUB(rby, lty);
  const float wx = clamp0(dx), wy = clamp0(dy);
  const float overlap = BXS_FMUL(wx, wy);
  const float union_raw = BXS_FSUB(BXS_FADD(area1, area2), overlap);
  const float elx = fminf(p[0], q[0]), ely = fminf(p[1], q[1]);
  const float erx = fmaxf(p[2], q[2]), ery = fmaxf(p[3], q[3]);
  const float uni = max_eps(union_raw, eps);
  const float ious = BXS_FDIV(overlap, uni);
  const float ex = BXS_FSUB(erx, elx), ey = BXS_FSUB(ery, ely);
  const float ewx = clamp0(ex), ewy = clamp0(ey);
  const float earea_raw = BXS_FMUL(ewx, ewy);
  const float earea = max_eps(earea_raw, eps);
  const float frac = BXS_FDIV(BXS_FSUB(earea, uni), earea);
  const float giou = BXS_FSUB(ious, frac);

  // loss = 1 - ious + frac, frac = (earea - uni) / earea, ious = overlap / uni
  const float g_earea = BXS_FSUB(BXS_FDIV(1.f, earea), BXS_FDIV(BXS_FSUB(earea, uni), BXS_FMUL(earea, earea)));
  const float g_uni = BXS_FSUB(BXS_FDIV(overlap, BXS_FMUL(uni, uni)), BXS_FDIV(1.f, earea));
  const float g_earea_raw = BXS_FMUL(g_earea, dmax_first(earea_raw, eps));
  const float g_ex = BXS_FMUL(BXS_FMUL(g_earea_raw, ewy), dclamp0(ex));
  const float g_ey = BXS_FMUL(BXS_FMUL(g_earea_raw, ewx), dclamp0(ey));
  const float g_area1 = BXS_FMUL(g_uni, dmax_first(union_raw, eps));
  const float g_overlap = BXS_FSUB(-BXS_FDIV(1.f, uni), g_area1);
  const float g_dx = BXS_FMUL(BXS_FMUL(g_overlap, wy), dclamp0(dx));
  const float g_dy = BXS_FMUL(BXS_FMUL(g_overlap, wx), dclamp0(dy));
  gp[0] = BXS_FSUB(BXS_FSUB(-BXS_FMUL(g_area1, ph), BXS_FMUL(g_ex, dmin_first(p[0], q[0]))),
                   BXS_FMUL(g_dx, dmax_first(p[0], q[0])));
  gp[1] = BXS_FSUB(BXS_FSUB(-BXS_FMUL(g_area1, pw), BXS_FMUL(g_ey, dmin_first(p[1], q[1]))),
                   BXS_FMUL(g_dy, dmax_first(p[1], q[1])));
  gp[2] = BXS_FADD(BXS_FADD(BXS_FMUL(g_area1, ph), BXS_FMUL(g_ex, dmax_first(p[2], q[2]))),
                   BXS_FMUL(g_dx, dmin_first(p[2], q[2])));
  gp[3] = BXS_FADD(BXS_FADD(BXS_FMUL(g_area1, pw), BXS_FMUL(g_ey, dmax_first(p[3], q[3]))),
                   BXS_FMUL(g_dy, dmin_first(p[3], q[3])));
  return BXS_FSUB(1.f, giou);
}

// F.binary_cross_entropy_with_logits(x, t) = (1 - t) x - log_sigmoid(x), and its d / dx = sigmoid(x) - t
BXS_HD float bce_logits(float x, float t, float& dx) {
  const float e = expf(-fabsf(x));
  const float log_sig = -BXS_FADD(x < 0.f ? -x : 0.f, log1pf(e));
  dx = BXS_FSUB(x >= 0.f ? BXS_FDIV(1.f, BXS_FADD(1.f, e)) : BXS_FDIV(e, BXS_FADD(1.f, e)), t);
  return BXS_FSUB(BXS_FMUL(BXS_FSUB(1.f, t), x), log_sig);
}

struct FcosPointLoss {
  float ct;            // centerness target
  float bbox;          // ct * (1 - GIoU)
  float ctr;           // BCE of the centerness logit against ct
  float g_pred[4];     // d bbox / d (l, t, r, b) of the prediction
  float g_ctr;         // d ctr / d centerness logit
};

// one positive point at (x, y): pred / target are (l, t, r, b) distances, ctr_logit the centerness prediction
BXS_HD FcosPointLoss fcos_point_loss(float x, float y, const float pred[4], const float target[4], float ctr_logit) {
  FcosPointLoss r;
  r.ct = fcos_centerness_target(target);
  float pb[4], tb[4], gb[4];
  fcos_decode(x, y, pred, pb);
  fcos_decode(x, y, target, tb);
  const float l = giou_loss_grad(pb, tb, 1e-6f, gb);
  r.bbox = BXS_FMUL(l, r.ct);
  r.g_pred[0] = -BXS_FMUL(gb[0], r.ct);
  r.g_pred[1] = -BXS_FMUL(gb[1], r.ct);
  r.g_pred[2] = BXS_FMUL(gb[2], r.ct);
  r.g_pred[3] = BXS_FMUL(gb[3], r.ct);
  r.ctr = bce_logits(ctr_logit, r.ct, r.g_ctr);
  return r;
}

}  // namespace bxs
