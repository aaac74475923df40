"""TEST INFRASTRUCTURE (oracle): restatement of ``CondInstBoxHead.loss`` (mmdet/models/dense_heads/condinst_head.py:364-476)
with the losses every BoxInst config uses -- ``FocalLoss(use_sigmoid=True)`` in its CPU form ``py_sigmoid_focal_loss``,
``GIoULoss`` (bbox_overlaps mode 'giou', is_aligned, eps 1e-6) weighted by the centerness targets, and
``CrossEntropyLoss(use_sigmoid=True)`` -- all with reduction 'mean' (``weight_reduce_loss``: sum / (avg_factor + eps)).

The points and the FCOS targets are computed in float32, as the reference does under ``@force_fp32``
(``oracle.fcos_targets``); the loss arithmetic then runs in the dtype of the predictions, float64 for the arbiter, with
the reference's lines in the reference's order so that autograd applies the reference's conventions at ties.  Pinned on
the reference's own code through ``tests/golden/fcos_loss.npz`` (``oracle/make_golden_fcos_loss.py``).
"""
import torch
import torch.nn.functional as F

from oracle import fcos_targets as oft

FLT_EPS = torch.finfo(torch.float32).eps


def centerness_target(t):
    """:855-874 -- sqrt(min(l,r)/max(l,r) * min(t,b)/max(t,b)) of [N,4] targets."""
    lr, tb = t[:, [0, 2]], t[:, [1, 3]]
    if len(lr) == 0:
        return torch.sqrt(lr[..., 0])
    return torch.sqrt((lr.min(dim=-1)[0] / lr.max(dim=-1)[0]) * (tb.min(dim=-1)[0] / tb.max(dim=-1)[0]))


def centerness_target_rn(t):
    """``centerness_target`` of float32 targets with a correctly rounded square root -- what the reference computes on
    CUDA.  torch's vectorised CPU float32 sqrt can land one ulp off the correctly rounded value; the square root of a
    float32 taken in float64 and rounded once is correctly rounded."""
    lr, tb = t[:, [0, 2]], t[:, [1, 3]]
    return torch.sqrt(((lr.min(dim=-1)[0] / lr.max(dim=-1)[0]) * (tb.min(dim=-1)[0] / tb.max(dim=-1)[0])).double()).float()


def distance2bbox(points, d):
    return torch.stack([points[..., 0] - d[..., 0], points[..., 1] - d[..., 1], points[..., 0] + d[..., 2],
                        points[..., 1] + d[..., 3]], -1)


def giou(b1, b2, eps=1e-6):
    """bbox_overlaps(b1, b2, mode='giou', is_aligned=True, eps=eps), iou2d_calculator.py:213-261."""
    area1 = (b1[..., 2] - b1[..., 0]) * (b1[..., 3] - b1[..., 1])
    area2 = (b2[..., 2] - b2[..., 0]) * (b2[..., 3] - b2[..., 1])
    lt = torch.max(b1[..., :2], b2[..., :2])
    rb = torch.min(b1[..., 2:], b2[..., 2:])
    wh = (rb - lt).clamp(min=0)
    overlap = wh[..., 0] * wh[..., 1]
    union = area1 + area2 - overlap
    e_lt = torch.min(b1[..., :2], b2[..., :2])
    e_rb = torch.max(b1[..., 2:], b2[..., 2:])
    eps = union.new_tensor([eps])
    union = torch.max(union, eps)
    ious = overlap / union
    e_wh = (e_rb - e_lt).clamp(min=0)
    e_area = torch.max(e_wh[..., 0] * e_wh[..., 1], eps)
    return ious - (e_area - union) / e_area


def focal_elementwise(pred, onehot, gamma=2.0, alpha=0.25):
    """py_sigmoid_focal_loss before the reduction (focal_loss.py:12-55)."""
    p = pred.sigmoid()
    t = onehot.type_as(pred)
    pt = (1 - p) * t + p * (1 - t)
    w = (alpha * t + (1 - alpha) * (1 - t)) * pt.pow(gamma)
    return F.binary_cross_entropy_with_logits(pred, t, reduction='none') * w


def loss(cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels, strides, num_classes,
         regress_ranges=((-1, 64), (64, 128), (128, 256), (256, 512), (512, oft.INF)), center_sampling=True, radius=1.5,
         norm_on_bbox=True, focal=(2.0, 0.25, 1.0), lw_bbox=1.0, lw_ctr=1.0):
    """The reference's 5-tuple: ({loss_cls, loss_bbox, loss_centerness}, flatten_points, flatten_level_inds,
    flatten_img_inds, flatten_gt_inds), differentiable with respect to the three prediction lists (on their device)."""
    sizes = [tuple(c.shape[-2:]) for c in cls_scores]
    dt, dev = bbox_preds[0].dtype, bbox_preds[0].device
    pts32 = [p.to(dev) for p in oft.grid_points(sizes, strides)]
    labels, targets, inds = oft.get_targets(pts32, [b.float() for b in gt_bboxes], gt_labels, regress_ranges, strides,
                                            num_classes, center_sampling, radius, norm_on_bbox)
    points = [p.to(dt) for p in pts32]
    B, C = cls_scores[0].shape[:2]
    f_cls = torch.cat([c.permute(0, 2, 3, 1).reshape(-1, C) for c in cls_scores])
    f_bbox = torch.cat([b.permute(0, 2, 3, 1).reshape(-1, 4) for b in bbox_preds])
    f_ctr = torch.cat([c.permute(0, 2, 3, 1).reshape(-1) for c in centernesses])
    f_labels = torch.cat(labels)
    f_targets = torch.cat(targets).to(dt)
    f_points = torch.cat([p.repeat(B, 1) for p in points])
    f_gt_inds = torch.cat(inds)
    f_img = torch.cat([torch.arange(B, device=dev).repeat_interleave(h * w) for h, w in sizes])
    f_lvl = torch.cat([torch.full((B * h * w,), i, device=dev).long() for i, (h, w) in enumerate(sizes)])

    pos = ((f_labels >= 0) & (f_labels < num_classes)).nonzero().reshape(-1)
    num_pos = max(torch.tensor(len(pos), dtype=torch.float, device=dev), 1.0)          # reduce_mean at world size 1
    gamma, alpha, lw_cls = focal
    onehot = F.one_hot(f_labels, num_classes=num_classes + 1)[:, :num_classes]
    loss_cls = lw_cls * (focal_elementwise(f_cls, onehot, gamma, alpha).sum() / (num_pos + FLT_EPS))

    p_bbox, p_ctr, p_tgt = f_bbox[pos], f_ctr[pos], f_targets[pos]
    ct = centerness_target(p_tgt)
    denorm = max(ct.sum().detach(), 1e-6)
    if len(pos) > 0:
        p_pts = f_points[pos]
        l_giou = (1 - giou(distance2bbox(p_pts, p_bbox), distance2bbox(p_pts, p_tgt))) * ct
        loss_bbox = lw_bbox * (l_giou.sum() / (denorm + FLT_EPS))
        # binary_cross_entropy hands the label over as .float() and weighs by the float32 valid mask
        bce = F.binary_cross_entropy_with_logits(p_ctr, ct.float(), reduction='none') * ((ct >= 0) & (ct != -100)).float()
        loss_ctr = lw_ctr * (bce.sum() / (num_pos + FLT_EPS))
    else:
        loss_bbox = p_bbox.sum()
        loss_ctr = p_ctr.sum()
    return (dict(loss_cls=loss_cls, loss_bbox=loss_bbox, loss_centerness=loss_ctr), f_points, f_lvl, f_img, f_gt_inds)


def element_terms(points, pred, target, ctr):
    """Per positive, in the dtype of ``pred``: (centerness target, ct * (1 - GIoU), BCE, d(ct * (1 - GIoU))/d pred,
    d BCE / d ctr) by autograd of the lines above -- what the kernel core computes for one point."""
    pred = pred.detach().clone().requires_grad_(True)
    ctr = ctr.detach().clone().requires_grad_(True)
    ct = centerness_target(target)
    bbox = (1 - giou(distance2bbox(points, pred), distance2bbox(points, target))) * ct
    bce = F.binary_cross_entropy_with_logits(ctr, ct, reduction='none')
    g_pred, = torch.autograd.grad(bbox.sum(), pred)
    g_ctr, = torch.autograd.grad(bce.sum(), ctr)
    return ct.detach(), bbox.detach(), bce.detach(), g_pred, g_ctr
