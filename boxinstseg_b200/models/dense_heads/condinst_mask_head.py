"""``CondInstMaskHead`` -- registry drop-in for mmdet/models/dense_heads/condinst_head.py:1041-1448.

Same constructor kwargs, buffers (``sizes_of_interest``, ``_iter``), ``param_conv`` attribute and
``forward`` / ``loss`` / ``get_targets`` methods as the reference, so
``configs/boxinst/boxinst_r50_fpn_1x_coco.py`` builds it unchanged; the arithmetic runs in the
sm_90a kernels of libboxseg_b200:
  forward      -> ops.condinst.dynamic_mask_head   (a1: rel-coords + 3 dynamic 1x1 convs + aligned x2)
  get_targets  -> ops.boxinst.boxinst_targets      (a5: no host round trip, no per-GT Python loop)
  loss         -> ops.boxinst.boxinst_mask_loss    (a6+a7+a8 fused; no [N,8,H,W] tensors)
                  ops.condinst.dice_mask_loss      (boxinst_enabled=False: the masks sampled in place, no [N,h,w] target)
There is no CPU fallback: a missing extension raises.
"""
import torch
import torch.nn as nn

from ...ops import boxinst as boxinst_ops
from ..builder import HEADS, register


@register(HEADS, partial=True)
class CondInstMaskHead(nn.Module):
    def __init__(self,
                 in_channels=8,
                 in_stride=8,
                 out_stride=4,
                 dynamic_convs=3,
                 dynamic_channels=8,
                 disable_rel_coors=False,
                 bbox_head_channels=256,
                 sizes_of_interest=[64, 128, 256, 512, 1024],
                 max_proposals=500,
                 topk_per_img=-1,
                 boxinst_enabled=False,
                 bottom_pixels_removed=10,
                 pairwise_size=3,
                 pairwise_dilation=2,
                 pairwise_color_thresh=0.3,
                 pairwise_warmup=10000,
                 norm_cfg=dict(type='BN', requires_grad=True),
                 init_cfg=dict(type='Normal', layer='Conv2d', std=0.01, bias=0)):
        super().__init__()
        assert in_stride >= out_stride and in_stride % out_stride == 0
        assert dynamic_channels > 1
        assert max_proposals == -1 or topk_per_img == -1, \
            'max_proposals and topk_per_img cannot be used at the same time'
        self.in_channels = in_channels
        self.in_stride = in_stride
        self.out_stride = out_stride
        self.dynamic_convs = dynamic_convs
        self.dynamic_channels = dynamic_channels
        self.disable_rel_coors = disable_rel_coors
        first = in_channels if disable_rel_coors else in_channels + 2
        self.dy_weights, self.dy_biases = [], []
        for i in range(dynamic_convs):
            cin = first if i == 0 else dynamic_channels
            cout = 1 if i == dynamic_convs - 1 else dynamic_channels
            self.dy_weights.append(cin * cout)
            self.dy_biases.append(cout)
        self.num_gen_params = sum(self.dy_weights) + sum(self.dy_biases)
        self.bbox_head_channels = bbox_head_channels
        self.register_buffer('sizes_of_interest', torch.tensor(sizes_of_interest))
        self.max_proposals = max_proposals
        self.topk_per_img = topk_per_img
        self.boxinst_enabled = boxinst_enabled
        self.bottom_pixels_removed = bottom_pixels_removed
        self.pairwise_size = pairwise_size
        self.pairwise_dilation = pairwise_dilation
        self.pairwise_color_thresh = pairwise_color_thresh
        self.register_buffer('_iter', torch.zeros([1]))
        self._warmup_iters = pairwise_warmup
        self.norm_cfg = norm_cfg
        self.init_cfg = init_cfg
        self.fp16_enable = False
        self.param_conv = nn.Conv2d(bbox_head_channels, self.num_gen_params, 3, stride=1, padding=1)
        if init_cfg and init_cfg.get('type') == 'Normal':
            nn.init.normal_(self.param_conv.weight, std=init_cfg.get('std', 0.01))
            nn.init.constant_(self.param_conv.bias, init_cfg.get('bias', 0))

    # ------------------------------------------------------------------ a1
    def forward(self, feat, params, coors, level_inds, img_inds):
        from ...ops.condinst import dynamic_mask_head
        return dynamic_mask_head(feat, params, coors, level_inds, img_inds,
                                 sizes_of_interest=self.sizes_of_interest, in_stride=self.in_stride,
                                 out_stride=self.out_stride, channels=self.dynamic_channels,
                                 num_layers=self.dynamic_convs, rel_coors=not self.disable_rel_coors)

    # ------------------------------------------------------------------ f2 (SURVEY 8f rank 2)
    def training_sample(self, cls_scores, centernesses, param_preds, coors, level_inds, img_inds, gt_inds):
        """Instance sampling of condinst_head.py:1166-1232, index-exact, without the reference's Python loop over images and
        ground truths (one ``.any()`` / ``.unique()`` / boolean-index host sync per image and per GT there; here: one sort, one
        size read).  ``topk_per_img``: per image every GT that has positives keeps its ``inst_per_gt = max(int(topk /
        #GTs of the image), 1)`` best positives by ``sigmoid(max class score) * sigmoid(centerness)`` (all of them, in their
        original order, when it has no more than that); output order = image, GT index, then top-k order, as the reference.
        ``max_proposals``: the reference's random permutation of the first ``min(max_proposals, P)`` positives (:1186-1189)."""
        params = torch.cat([p.permute(0, 2, 3, 1).flatten(end_dim=2) for p in param_preds], dim=0)
        pos = torch.nonzero(gt_inds != -1, as_tuple=False).squeeze(1)
        params, coors, level_inds, img_inds, gt_inds = params[pos], coors[pos], level_inds[pos], img_inds[pos], gt_inds[pos]
        P = params.size(0)
        if self.max_proposals != -1:
            sel = torch.randperm(min(self.max_proposals, P), device=params.device).long()
        elif self.topk_per_img != -1 and P > 0:
            cls = torch.cat([c.permute(0, 2, 3, 1).flatten(end_dim=2) for c in cls_scores], dim=0)[pos]
            ctr = torch.cat([c.permute(0, 2, 3, 1).reshape(-1) for c in centernesses], dim=0)[pos]
            score = cls.sigmoid().max(dim=1)[0] * ctr.sigmoid()
            big = int(gt_inds.max().item()) + 1 if P else 1                     # the one size read of this function
            key = img_inds.long() * big + gt_inds.long()                       # (image, GT) group, ascending like the reference's loops
            uniq, inv, counts = torch.unique(key, return_inverse=True, return_counts=True)
            gts_per_img = torch.zeros(int(img_inds.max().item()) + 1, dtype=torch.long, device=key.device)
            gts_per_img.scatter_add_(0, torch.div(uniq, big, rounding_mode='floor'), torch.ones_like(uniq))
            per_gt = torch.clamp(torch.div(self.topk_per_img, gts_per_img.clamp(min=1), rounding_mode='floor'), min=1)
            limit_g = per_gt[torch.div(uniq, big, rounding_mode='floor')]       # inst_per_gt of each group's image
            topk_g = counts > limit_g                                          # groups that are cut down by score
            # order inside a group: descending score where the group is cut (torch.topk's order), original order otherwise
            arange = torch.arange(P, device=key.device)
            first = torch.argsort(torch.where(topk_g[inv], -score, score.new_zeros(()).expand(P)), stable=True)
            order = first[torch.argsort(inv[first], stable=True)]              # stable: by group, then by the key above
            start = torch.cumsum(counts, 0) - counts
            rank = arange - start[inv[order]]
            sel = order[rank < torch.minimum(counts, limit_g)[inv[order]]]
        else:
            sel = torch.arange(P, device=params.device)
        return params[sel], coors[sel], level_inds[sel], img_inds[sel], gt_inds[sel]

    def simple_test(self, mask_feat, det_labels, det_params, det_coors, det_level_inds, img_metas, num_classes,
                    rescale=False):
        """condinst_head.py:1234-1286, same arguments and return value (per image, per class, uint8 numpy masks): the
        dynamic head once for the batch and the fused paste ``ops.condinst.paste_masks`` per image.  An image without a
        detection in a batch with some gets one entry of empty class lists (INTEGRATION.md section 11)."""
        from .condinst_infer import simple_test
        return simple_test(self, mask_feat, det_labels, det_params, det_coors, det_level_inds, img_metas, num_classes,
                           rescale)

    # ------------------------------------------------------------------ a5
    def get_targets(self, gt_bboxes, gt_masks, img, img_metas):
        """BoxInst: returns a BoxInstTargets (per-image similarity bits + per-GT rectangles) instead of
        the reference's G-fold duplicated similarity list; ``.bitmasks()`` gives the dense masks."""
        if not self.boxinst_enabled:
            start = int(self.out_stride // 2)
            bitmasks = [m[:, start::self.out_stride, start::self.out_stride] for m in gt_masks]
            return None, bitmasks, gt_masks
        return boxinst_ops.boxinst_targets(
            img, img_metas, gt_bboxes, stride=self.out_stride, pairwise_size=self.pairwise_size,
            pairwise_dilation=self.pairwise_dilation, pairwise_color_thresh=self.pairwise_color_thresh,
            bottom_pixels_removed=self.bottom_pixels_removed)

    # ------------------------------------------------------------------ a6+a7+a8
    def loss(self, imgs, img_metas, mask_logits, gt_inds, gt_bboxes, gt_masks, gt_labels):
        self._iter += 1
        mask_logits = mask_logits.float()                      # force_fp32(apply_to=('mask_logits',))
        losses = {}
        if len(mask_logits) == 0:                              # condinst_head.py:1306-1312
            dummy = 0 * mask_logits.sum()
            if self.boxinst_enabled:
                return {'loss_prj': dummy, 'loss_pairwise': dummy}
            return {'loss_mask': dummy}
        if self.boxinst_enabled:
            targets = self.get_targets(gt_bboxes, gt_masks, imgs, img_metas)
            if self.pairwise_size == 3:
                prj, pair = boxinst_ops.boxinst_mask_loss(mask_logits, targets, gt_inds, self._iter,
                                                          self._warmup_iters, self.pairwise_dilation)
            else:
                prj, pair = self._unfused_boxinst_loss(mask_logits, targets, gt_inds)
            losses['loss_prj'] = prj
            losses['loss_pairwise'] = pair
        else:
            from ...ops.condinst import dice_mask_loss
            losses['loss_mask'] = dice_mask_loss(mask_logits, gt_masks, gt_inds, self.out_stride)
        return losses

    def _unfused_boxinst_loss(self, mask_logits, targets, gt_inds):
        """pairwise_size != 3: composition of the fine-grained CUDA ops (no bit-packed similarity)."""
        from ...ops.pairwise import pairwise_nlog
        from ..losses.box_projection_loss import projection_losses
        bm = torch.cat(targets.bitmasks(), dim=0)[gt_inds].unsqueeze(1)
        prj = projection_losses(mask_logits.sigmoid(), bm).mean()
        sim = targets.similarity[targets.gt_img.long()[gt_inds]]
        w = (sim >= self.pairwise_color_thresh).float() * bm
        pl = pairwise_nlog(mask_logits, self.pairwise_size, self.pairwise_dilation)
        warm = (self._iter / float(self._warmup_iters)).clamp(max=1.0)
        return prj, (pl * w).sum() / w.sum().clamp(min=1.0) * warm
