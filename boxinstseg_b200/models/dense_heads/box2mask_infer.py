"""Box2Mask inference for the whole batch: MaskFormerFusionHead.simple_test / instance_postprocess
(maskformer_fusion_head.py:112-241, with mask2bbox of mmdet/core/mask/utils.py:68-89) on the mask predictions that
Box2MaskHead.simple_test returns at the mask-feature resolution (or, from the reference's head, at batch_input_shape).

  1. ``F.softmax(mask_cls, -1)[..., :-1]``, the reference's own op, then ONE stable descending sort of every image's
     flattened [Q*K] scores: the top max_per_image (query, class) pairs, equal scores with the lower q*K + c first;
  2. with stuff classes, the thing pairs moved to the front of each image in order (one host read: their counts);
  3. per image, ``bxs_maskformer_paste_masks`` on the chosen query rows, read in place: upsample to batch_input_shape, crop
     to img_shape, resize to ori_shape (rescale), threshold at 0, and in the same pass each mask's area, the sum of its
     sigmoid over the set pixels and its box; the reference's float planes at both resolutions never exist;
  4. det_score = score * masked_sum / (area + 1e-6) in float32 in the reference's operation order.
No host read when num_stuff_classes == 0 (every Box2Mask config): all sizes follow from the shapes."""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ...ops.solo_seg import RowSources, maskformer_paste_rows
from ..builder import HEADS, register


def instance_results(mask_cls, mask_pred, img_metas, num_things, max_per_image, rescale):
    """Per image (labels int64 [n], query int64 [n], bboxes float32 [n, 5], masks bool [n, H, W]) for mask_cls [B,Q,K+1]
    and mask_pred [B,Q,h,w] logits (float32 or float16), upsampled to img_metas[0]['batch_input_shape'] (or read as they
    are when they have that size, or when no image carries the key)."""
    B, Q, K = mask_cls.shape[0], mask_cls.shape[1], mask_cls.shape[2] - 1
    if not 0 <= max_per_image <= Q * K:
        raise RuntimeError('selected index k out of range')            # what torch.topk raises
    scores = F.softmax(mask_cls, dim=-1)[..., :-1]
    top_scores, top = torch.sort(scores.flatten(1), dim=1, descending=True, stable=True)
    top_scores, top = top_scores[:, :max_per_image], top[:, :max_per_image]
    labels, query = top % K, top // K
    if num_things < K:
        thing = labels < num_things
        order = torch.sort((~thing).to(torch.uint8), dim=1, stable=True)[1]
        top_scores, labels, query = [t.gather(1, order) for t in (top_scores, labels, query)]
        counts = thing.sum(1).tolist()                                   # the one host read
    else:
        counts = [max_per_image] * B
    h, w = mask_pred.shape[-2:]
    pad = tuple(img_metas[0].get('batch_input_shape', (h, w)))[:2]
    src = RowSources([mask_pred.flatten(0, 1)])
    out = []
    for b, (meta, n) in enumerate(zip(img_metas, counts)):
        q = query[b, :n]
        masks, area, msum, box = maskformer_paste_rows(src, q + b * Q, pad, meta['img_shape'],
                                                       meta['ori_shape'] if rescale else None)
        det_scores = top_scores[b, :n] * (msum / (area.float() + 1e-6))
        out.append((labels[b, :n], q, torch.cat([box, det_scores[:, None]], dim=-1), masks))
    return out


@register(HEADS, partial=True)
class MaskFormerFusionHead(nn.Module):
    """MaskFormerFusionHead's test path with the reference's signatures, for instance output (every Box2Mask config:
    panoptic_on=False, instance_on=True).  Panoptic and semantic output raise NotImplementedError."""

    def __init__(self, num_things_classes=80, num_stuff_classes=53, test_cfg=None, loss_panoptic=None, init_cfg=None,
                 **kwargs):
        super().__init__()
        self.num_things_classes = num_things_classes
        self.num_stuff_classes = num_stuff_classes
        self.num_classes = num_things_classes + num_stuff_classes
        self.test_cfg = test_cfg

    def forward_train(self, **kwargs):
        """MaskFormerFusionHead has no training loss."""
        return dict()

    def _check_outputs(self):
        cfg = self.test_cfg or {}
        for key, default in (('panoptic_on', True), ('semantic_on', False)):
            if cfg.get(key, default):
                raise NotImplementedError(f'MaskFormerFusionHead: {key}=True is not supported, only instance output')
        return cfg

    def instance_postprocess(self, mask_cls, mask_pred):
        """(labels [n], bboxes [n, 5], masks bool [n, h, w]) of one image: mask_cls [Q, K+1], mask_pred [Q, h, w] logits
        already at their final size (both resize stages are skipped)."""
        cfg = self.test_cfg or {}
        h, w = mask_pred.shape[-2:]
        meta = dict(img_shape=(h, w), batch_input_shape=(h, w))
        labels, _, bboxes, masks = instance_results(mask_cls[None], mask_pred[None], [meta], self.num_things_classes,
                                                    cfg.get('max_per_image', 100), False)[0]
        return labels, bboxes, masks

    def simple_test(self, mask_cls_results, mask_pred_results, img_metas, rescale=False, **kwargs):
        """One dict(ins_results=(labels, bboxes [n, 5], masks bool [n, H, W])) per image, as the reference returns.
        mask_pred_results: [B,Q,h,w] from Box2MaskHead.simple_test, or [B,Q,H_pad,W_pad] already upsampled."""
        cfg = self._check_outputs()
        if not cfg.get('instance_on', False):
            return [dict() for _ in img_metas]
        res = instance_results(mask_cls_results, mask_pred_results, img_metas, self.num_things_classes,
                               cfg.get('max_per_image', 100), rescale)
        return [dict(ins_results=(labels, bboxes, masks)) for labels, _, bboxes, masks in res]
