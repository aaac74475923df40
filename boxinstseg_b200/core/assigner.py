"""``MaskHungarianAssigner`` -- drop-in for mmdet/core/bbox/assigners/mask_hungarian_assigner.py:14-132 (SURVEY 8f rank 1)
with the cost-matrix assembly of its steps 1-2 on the GPU, and ``ClassificationCost`` (match_cost.py:153-193).

Box2MaskHead._get_target_single (box2mask_head.py:152-169) first upsamples every query's mask prediction to the ground-truth
resolution ([100,1,1024,1024] per image per decoder layer, 420 MB x 10) only so that BoxMatchingCost can take row / column
maxima of it.  ``assign(..., lowres=True)`` hands the LOW-resolution prediction to BoxMatchingCost.cost_from_lowres instead:
the fused bilinear-upsample -> sigmoid -> projection kernel (bxs_upsampled_rowcol_max) never builds that tensor.

Step 3, the Hungarian matching (the reference's scipy.optimize.linear_sum_assignment on the host, :113-123), is the LSAP
kernel of ops.lsap: scipy's algorithm and tie rules in float64, so the matching is scipy's bit for bit, and the cost matrix
stays on the device.  ``assign`` reads one 4-byte status to raise scipy's errors; Box2MaskHead.get_targets matches a whole
decoder layer in one launch without reading anything back.
"""
from collections import namedtuple

import torch

from ..models.builder import MATCH_COST, register
from ..ops.lsap import raise_for_status, solve_batched
from .match_cost import BoxMatchingCost

AssignResult = namedtuple('AssignResult', ['num_gts', 'gt_inds', 'max_overlaps', 'labels'])   # assign_result.py fields


@register(MATCH_COST)
class ClassificationCost:
    """-softmax(cls_pred)[:, gt_labels] * weight (match_cost.py:174-193)."""

    def __init__(self, weight=1.):
        self.weight = weight

    def __call__(self, cls_pred, gt_labels):
        return -cls_pred.softmax(-1)[:, gt_labels] * self.weight


def build_match_cost(cfg):
    if cfg is None or not isinstance(cfg, dict):
        return cfg
    return MATCH_COST.build(cfg)


class _ZeroCost:
    weight = 0.0


class MaskHungarianAssigner:
    """Same constructor and ``assign`` signature as the reference class.  ``mask_cost`` / ``dice_cost`` may be any
    registered match cost; the Box2Mask config uses BoxMatchingCost for the dice slot and weight 0 for the mask slot."""

    def __init__(self, cls_cost=dict(type='ClassificationCost', weight=1.0), mask_cost=None,
                 dice_cost=dict(type='BoxMatchingCost', weight=1.0, pred_act=True, eps=1.0)):
        self.cls_cost = build_match_cost(cls_cost)
        self.mask_cost = build_match_cost(mask_cost) if mask_cost is not None else _ZeroCost()
        self.dice_cost = build_match_cost(dice_cost)

    @torch.no_grad()
    def cost_matrix(self, cls_pred, mask_pred, gt_labels, gt_mask, lowres=False):
        """steps 1-2 of mask_hungarian_assigner.py:92-111: [num_query, num_gt] on the device.
        mask_pred [Q,h,w] (or [Q,1,h,w]); gt_mask [G,H,W] (or [G,1,H,W]).  lowres: mask_pred is still at the head's
        resolution and must be (virtually) resized to gt_mask's (box2mask_head.py:157-161)."""
        cost = 0
        if self.cls_cost.weight != 0 and cls_pred is not None:
            cost = cost + self.cls_cost(cls_pred, gt_labels)
        if self.mask_cost.weight != 0:
            cost = cost + self.mask_cost(mask_pred, gt_mask)
        if self.dice_cost.weight != 0:
            if lowres and isinstance(self.dice_cost, BoxMatchingCost):
                q = mask_pred.reshape(mask_pred.shape[0], *mask_pred.shape[-2:])
                cost = cost + self.dice_cost.cost_from_lowres(q, gt_mask)
            else:
                cost = cost + self.dice_cost(mask_pred, gt_mask)
        return cost

    @torch.no_grad()
    def assign(self, cls_pred, mask_pred, gt_labels, gt_mask, img_meta=None, gt_bboxes_ignore=None, eps=1e-7, lowres=False):
        assert gt_bboxes_ignore is None, 'Only case when gt_bboxes_ignore is None is supported.'
        num_gt, num_query = gt_labels.shape[0], mask_pred.shape[0]
        assigned_gt_inds = mask_pred.new_full((num_query,), -1, dtype=torch.long)
        assigned_labels = mask_pred.new_full((num_query,), -1, dtype=torch.long)
        if num_gt == 0 or num_query == 0:
            if num_gt == 0:
                assigned_gt_inds[:] = 0
            return AssignResult(num_gt, assigned_gt_inds, None, assigned_labels)
        cost = self.cost_matrix(cls_pred, mask_pred, gt_labels, gt_mask, lowres)
        (match,), status = solve_batched([cost])
        raise_for_status(int(status[0]))
        m = match.long()                     # matched ground truth per query or -1 -> gt_inds 0 = background (:125-132)
        labels = torch.where(m >= 0, gt_labels[m.clamp(min=0)].long(), -1)
        return AssignResult(num_gt, m + 1, None, labels)
