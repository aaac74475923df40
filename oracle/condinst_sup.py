"""TEST INFRASTRUCTURE (oracle): restatement of CondInst's mask-supervised losses
(mmdet/models/dense_heads/condinst_head.py):

* ``dice_coefficient`` (:117-131) with the ``boxinst_enabled=False`` branch of ``CondInstMaskHead.loss`` (:1298-1341): the
  targets ``m[:, s//2::s, s//2::s]`` of the uint8 masks, indexed by ``gt_inds`` and cast to the logits' dtype, then
  ``1 - 2 I / (S + T + 1e-5)`` averaged over the instances.
* ``CondInstSegmHead.get_targets`` (:950-968) and ``loss`` (:935-948), the focal loss in its CPU form
  ``py_sigmoid_focal_loss`` with reduction 'mean' (sum / (avg_factor + eps)).

The arithmetic runs in the dtype it is handed (float64 for the arbiter, float32 for the reference's own lines) and in the
reference's order.  Pinned on the reference's own code through ``tests/golden/condinst_sup.npz``
(``oracle/make_golden_condinst_sup.py``).
"""
import torch

from oracle.fcos_loss import focal_elementwise

INF = 1e8                       # condinst_head.py:16
FLT_EPS = 1.1920928955078125e-07


def dice_coefficient(x, target):
    eps = 1e-5
    n_inst = x.size(0)
    x = x.reshape(n_inst, -1)
    target = target.reshape(n_inst, -1)
    intersection = (x * target).sum(dim=1)
    union = (x ** 2.0).sum(dim=1) + (target ** 2.0).sum(dim=1) + eps
    return 1. - (2 * intersection / union)


def mask_loss(mask_logits, gt_masks, gt_inds, out_stride):
    """``{'loss_mask': ...}`` of CondInstMaskHead.loss with boxinst_enabled=False; mask_logits [N,1,h,w]."""
    start = int(out_stride // 2)
    bitmasks = [m[:, start::out_stride, start::out_stride] for m in gt_masks]
    mask_scores = mask_logits.sigmoid()
    gt_bitmasks = torch.cat(bitmasks, dim=0)[gt_inds].unsqueeze(1).to(mask_scores.dtype)
    if len(mask_scores) == 0:
        return {'loss_mask': 0 * mask_scores.sum()}
    return {'loss_mask': dice_coefficient(mask_scores, gt_bitmasks).mean()}


def semantic_targets(gt_masks, gt_labels, in_stride, num_classes):
    """CondInstSegmHead.get_targets; an image without ground truth gives all ``num_classes`` (the reference raises)."""
    out = []
    for cur_gt_masks, cur_gt_labels in zip(gt_masks, gt_labels):
        h, w = cur_gt_masks.size()[-2:]
        if cur_gt_masks.shape[0] == 0:
            out.append(torch.full((1, h, w), num_classes, dtype=torch.int64))
            continue
        areas = torch.sum(cur_gt_masks, dim=(1, 2), keepdim=True)
        areas = areas.repeat(1, h, w)
        areas[cur_gt_masks == 0] = INF
        min_areas, inds = torch.min(areas, dim=0, keepdim=True)
        labels = cur_gt_labels[:, None, None].repeat(1, h, w)
        per_img = torch.gather(labels, 0, inds)
        per_img[min_areas == INF] = num_classes
        out.append(per_img)
    s = in_stride
    return torch.cat(out, dim=0)[:, s // 2::s, s // 2::s]


def first_min_targets(gt_masks, gt_labels, in_stride, num_classes):
    """The same labels by an explicit first-index scan of the ground truths at every sampled pixel: torch.min(dim)'s
    tie rule stated without relying on torch."""
    s = in_stride
    out = []
    for m, lab in zip(gt_masks, gt_labels):
        sub = m[:, s // 2::s, s // 2::s].long()
        areas = m.long().sum(dim=(1, 2))
        best = torch.full(sub.shape[1:], int(INF), dtype=torch.int64)
        res = torch.full(sub.shape[1:], num_classes, dtype=torch.int64)
        first = torch.ones(sub.shape[1:], dtype=torch.bool)
        for g in range(m.shape[0]):
            wgt = torch.where(sub[g] != 0, areas[g], torch.tensor(int(INF)))
            take = first | (wgt < best)
            best = torch.where(take, wgt, best)
            res = torch.where(take, lab[g].expand_as(res), res)
            first[:] = False
        res[best == int(INF)] = num_classes
        out.append(res)
    return torch.stack(out)


def segm_loss(segm_pred, gt_masks, gt_labels, in_stride, num_classes, gamma=2.0, alpha=0.25, loss_weight=1.0):
    """``{'loss_segm': ...}`` of CondInstSegmHead.loss with FocalLoss(use_sigmoid=True), reduction 'mean'."""
    targets = semantic_targets(gt_masks, gt_labels, in_stride, num_classes).flatten()
    num_pos = (targets != num_classes).sum().float().clamp(min=1.)
    pred = segm_pred.permute(0, 2, 3, 1).flatten(end_dim=2)
    onehot = torch.nn.functional.one_hot(targets, num_classes=num_classes + 1)[:, :num_classes]
    loss = focal_elementwise(pred, onehot, gamma, alpha).sum() / (num_pos + FLT_EPS)      # float32 denominator
    return {'loss_segm': loss_weight * loss}
