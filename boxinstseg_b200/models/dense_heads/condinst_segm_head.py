"""``CondInstSegmHead`` (mmdet/models/dense_heads/condinst_head.py:877-968), the optional ``segm_head`` of
``CondInst.forward_train`` (detectors/condinst.py:62-65): its ``get_targets`` and ``loss`` on the device.

The reference builds, per image, int64 ``[G, H, W]`` copies of the areas and labels and a bool ``[G, H, W]`` mask at full
input resolution, only to keep every ``in_stride``-th pixel.  Here ``get_targets`` is ``ops.condinst.semantic_targets``
(csrc/condinst_sup.cu: the masks read in place, labels written at the sampled pixels only) and ``loss`` hands them to the
focal-loss kernel (``ops.focal.sigmoid_focal_loss_levels``) with the positive count kept on the device.

Registered as a *partial* head: with mmdet importable the registered class inherits the reference's constructor, towers
(``segm_branch``, ``segm_conv``) and state dict.  Stand-alone it carries what ``get_targets`` and ``loss`` read and builds no
towers.
"""
import torch

from ...ops.condinst import semantic_targets
from ...ops.focal import sigmoid_focal_loss_levels
from ..builder import HEADS, register
from .condinst_box_head import _loss_cfg

_DEFAULT_LOSS_SEGM = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)


def segm_loss_envelope(loss_segm):
    """(gamma, alpha, loss_weight) of ``loss_segm``, or a string naming it when ``CondInstSegmHead.loss`` does not run it
    natively: the envelope is ``FocalLoss(use_sigmoid=True)`` on logits with reduction 'mean'."""
    kind, c = _loss_cfg(loss_segm, 'FocalLoss')
    if kind != 'FocalLoss' or not c.get('use_sigmoid', True) or c.get('activated', False) or c.get('reduction', 'mean') != 'mean':
        return f'loss_segm {kind} {c}'
    return float(c.get('gamma', 2.0)), float(c.get('alpha', 0.25)), float(c.get('loss_weight', 1.0))


@register(HEADS, partial=True)
class CondInstSegmHead:
    """The target builder and the loss of the reference's ``CondInstSegmHead``; with mmdet importable everything else is
    the reference's class (``register(partial=True)``)."""

    def __init__(self, num_classes, in_channels=256, in_stride=8, stacked_convs=2, feat_channels=128,
                 loss_segm=_DEFAULT_LOSS_SEGM, **kwargs):
        self.num_classes = num_classes
        self.in_channels = in_channels
        self.in_stride = in_stride
        self.stacked_convs = stacked_convs
        self.feat_channels = feat_channels
        self.loss_segm = dict(loss_segm)
        self._bxs_post_init()

    def _bxs_post_init(self):
        """Also runs after the REFERENCE class's ``__init__`` on the loss module it built.  Never raises: a loss outside the
        envelope is recorded, and ``loss`` then defers to the reference or raises."""
        self.segm_loss = segm_loss_envelope(self.loss_segm)

    def forward(self, x):
        """condinst_head.py:931-932; needs the towers the reference constructor builds."""
        missing = [n for n in ('segm_branch', 'segm_conv') if not hasattr(self, n)]
        if missing:
            raise RuntimeError('CondInstSegmHead.forward needs the modules the reference constructor builds (mmdet '
                               f'installed); this head has no {", ".join(missing)}')
        return self.segm_conv(self.segm_branch(x))

    def get_targets(self, gt_masks, gt_labels):
        """condinst_head.py:950-968, same arguments and value: int64 [B, oh, ow] labels at the pixels (s/2 + s*i, s/2 + s*j),
        s = ``in_stride``, of the per-image uint8 [G_b, H, W] masks.  An image without ground truth gives all
        ``num_classes`` (the reference raises)."""
        return semantic_targets(gt_masks, gt_labels, self.in_stride, self.num_classes)

    def loss(self, segm_pred, gt_masks, gt_labels):
        """condinst_head.py:935-948, same arguments and value: ``{'loss_segm': ...}``.  Inside the envelope
        (``segm_loss_envelope``) the targets, the positive count (``clamp(min=1)``) and the focal loss stay on the device;
        float16 / bfloat16 ``segm_pred`` is promoted (the reference's ``@force_fp32``) and its gradient returns in the input
        dtype.  Outside the envelope this calls the reference's own ``loss`` when mmdet is importable and raises
        NotImplementedError otherwise."""
        if isinstance(self.segm_loss, str):
            ref = getattr(type(self), '_bxs_reference_class', None)
            if ref is not None:
                return ref.loss(self, segm_pred, gt_masks, gt_labels)
            raise NotImplementedError(f'CondInstSegmHead.loss: unsupported {self.segm_loss}')
        targets = self.get_targets(gt_masks, gt_labels)
        B, C, h, w = segm_pred.shape
        if tuple(targets.shape) != (B, h, w):
            raise ValueError(f'segm_pred {tuple(segm_pred.shape)} does not match the semantic targets {tuple(targets.shape)}')
        num_pos = (targets != self.num_classes).sum().float().clamp(min=1.)
        return dict(loss_segm=sigmoid_focal_loss_levels([segm_pred], [targets], num_pos, *self.segm_loss))
