"""f2: the target side and the loss of ``CondInstBoxHead`` (mmdet/models/dense_heads/condinst_head.py:247-548):
``get_targets`` + ``_get_target_single`` -- the FCOS point assignment that runs immediately before ``training_sample`` and
the mask loss -- and ``loss`` (:364-476), the classification, regression and centerness losses of the box branch.

The reference loops over the images (``multi_apply``), builds ~25 ``[points, gts]`` tensors per image, then splits per
level, concatenates per image and divides by the stride.  Here the whole batch is ONE launch of ``bxs_fcos_targets``
(`csrc/assign_targets.cu`): one thread per (image, location), results written in the reference's output layout, bit-exact.
No host synchronisation and no host-to-device copy: the level table and the per-image ground-truth offsets (host-known
lengths) travel in the kernel parameters, so the call can be captured in a CUDA graph.

``loss`` keeps the reference's signature and return value and runs on the device end to end: the points, one
``bxs_fcos_targets`` launch, the positive count and centerness-target sum (``bxs_fcos_loss_stats``), ONE all-reduce of both
when torch.distributed is initialised, the focal loss over the rectangular levels (``bxs_sigmoid_focal_loss_cells_forward``)
and the GIoU + centerness losses (``bxs_fcos_loss_forward``).  Nothing is read back to the host, so ``loss`` and its
backward can be captured in a CUDA graph.

Registered as a *partial* head: with mmdet importable the registered class inherits everything else (layers, forward,
simple_test) from the reference's own ``CondInstBoxHead``; ``get_bboxes`` runs on csrc/condinst_infer.cu (condinst_infer.py).
"""
import ctypes

import torch
import torch.distributed as dist
import torch.nn as nn

from ... import _lib as L
from ...ops.fcos import fcos_box_losses, fcos_box_stats, fcos_points
from ...ops.focal import sigmoid_focal_loss_levels
from ..builder import HEADS, register

INF = 1e8      # condinst_head.py:16


def fcos_get_targets(points, gt_bboxes_list, gt_labels_list, regress_ranges, strides, num_classes, center_sampling=True,
                     center_sample_radius=1.5, norm_on_bbox=True):
    """points: list (one per level) of [P_l, 2] float32 CUDA tensors; gt_bboxes_list / gt_labels_list: per image [G_b, 4]
    float32 / [G_b] int64.  Returns the three per-level lists of condinst_head.py:546-548: labels [B*P_l] int64,
    bbox_targets [B*P_l, 4] float32, gt_inds [B*P_l] int64 (offset by the ground truths of the preceding images)."""
    num_levels = len(points)
    assert num_levels == len(regress_ranges) == len(strides)
    assert len(gt_bboxes_list) == len(gt_labels_list) and len(gt_bboxes_list) > 0
    B = len(gt_bboxes_list)
    pts = torch.cat([p.reshape(-1, 2) for p in points], 0).contiguous().float()
    L.require_cuda(pts)
    dev = pts.device
    counts = [int(p.shape[0]) for p in points]
    level_off = [0]
    for c in counts:
        level_off.append(level_off[-1] + c)
    P = level_off[-1]
    gts = [int(g.shape[0]) for g in gt_bboxes_list]
    off = [0]
    for g in gts:
        off.append(off[-1] + g)
    boxes = torch.cat([g.reshape(-1, 4) for g in gt_bboxes_list], 0).to(device=dev, dtype=torch.float32).contiguous()
    labs = torch.cat([g.reshape(-1) for g in gt_labels_list], 0).to(device=dev, dtype=torch.int64).contiguous()
    labels = torch.empty(B * P, dtype=torch.int64, device=dev)
    targets = torch.empty((B * P, 4), dtype=torch.float32, device=dev)
    inds = torch.empty(B * P, dtype=torch.int64, device=dev)
    if P:
        f32 = lambda v: torch.tensor(v, dtype=torch.float64).to(torch.float32)        # double -> fp32, like a tensor assignment
        lo = f32([float(r[0]) for r in regress_ranges])
        hi = f32([float(r[1]) for r in regress_ranges])
        sr = f32([float(s) * center_sample_radius for s in strides])                   # :595 (Python float product, then fp32)
        st = f32([float(s) for s in strides])
        lvl = (ctypes.c_int64 * (num_levels + 1))(*level_off)
        gt_off = (ctypes.c_int64 * (B + 1))(*off)
        with torch.cuda.device(dev):
            L.check(L.lib().bxs_fcos_targets(
                L.ptr(pts), L.ptr(boxes) if boxes.numel() else None, L.ptr(labs) if labs.numel() else None,
                ctypes.cast(gt_off, ctypes.c_void_p),
                L.ptr(labels), L.ptr(targets), L.ptr(inds), B, num_levels, ctypes.cast(lvl, ctypes.c_void_p),
                L.c_p(lo.data_ptr()), L.c_p(hi.data_ptr()), L.c_p(sr.data_ptr()), L.c_p(st.data_ptr()),
                int(bool(center_sampling)), int(bool(norm_on_bbox)), int(num_classes), L.stream()), 'fcos_targets')
    sizes = [B * c for c in counts]
    return list(labels.split(sizes)), list(targets.split(sizes)), list(inds.split(sizes))


def _loss_cfg(module_or_cfg, default_type):
    """(type name, dict of the attributes the envelope checks) of a built loss module or a config dict."""
    if isinstance(module_or_cfg, nn.Module):
        m = module_or_cfg
        keys = ('use_sigmoid', 'activated', 'gamma', 'alpha', 'reduction', 'loss_weight', 'eps', 'use_mask', 'class_weight',
                'ignore_index')
        return type(m).__name__, {k: getattr(m, k) for k in keys if hasattr(m, k)}
    cfg = dict(module_or_cfg or {})
    return cfg.pop('type', default_type), cfg


def box_loss_envelope(loss_cls, loss_bbox, loss_centerness):
    """((gamma, alpha, loss_weight) of the focal loss, GIoU loss_weight, centerness loss_weight), or a string naming the
    first loss outside what ``CondInstBoxHead.loss`` runs natively: ``FocalLoss(use_sigmoid=True)`` on logits,
    ``GIoULoss(eps=1e-6)`` and ``CrossEntropyLoss(use_sigmoid=True)`` without class weights or ignore index, all with
    reduction 'mean' -- what every BoxInst config uses."""
    kind, c = _loss_cfg(loss_cls, 'FocalLoss')
    if kind != 'FocalLoss' or not c.get('use_sigmoid', True) or c.get('activated', False) or c.get('reduction', 'mean') != 'mean':
        return f'loss_cls {kind} {c}'
    focal = (float(c.get('gamma', 2.0)), float(c.get('alpha', 0.25)), float(c.get('loss_weight', 1.0)))
    kind, b = _loss_cfg(loss_bbox, 'IoULoss')
    if kind != 'GIoULoss' or b.get('reduction', 'mean') != 'mean' or float(b.get('eps', 1e-6)) != 1e-6:
        return f'loss_bbox {kind} {b}'
    kind, e = _loss_cfg(loss_centerness, 'CrossEntropyLoss')
    if (kind != 'CrossEntropyLoss' or not e.get('use_sigmoid', False) or e.get('use_mask', False)
            or e.get('reduction', 'mean') != 'mean' or e.get('class_weight') is not None or e.get('ignore_index') is not None):
        return f'loss_centerness {kind} {e}'
    return focal, float(b.get('loss_weight', 1.0)), float(e.get('loss_weight', 1.0))


def reduce_mean_clamped(stats):
    """``(max(reduce_mean(num_pos), 1.0), max(reduce_mean(sum ct), 1e-6))`` of condinst_head.py:443, 452-453 on the device:
    ONE all-reduce of both values when torch.distributed is initialised, each divided by the world size first and then
    summed, as mmdet's reduce_mean does; then the two clamps (a NaN stays NaN, as in the reference's Python ``max``),
    without a host-to-device copy so that the step can be captured in a CUDA graph."""
    if dist.is_available() and dist.is_initialized():
        stats = stats.clone()
        dist.all_reduce(stats.div_(dist.get_world_size()), op=dist.ReduceOp.SUM)
    return torch.cat((stats[:1].clamp(min=1.0), stats[1:].clamp(min=1e-6)))


_DEFAULT_LOSS_CLS = dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
_DEFAULT_LOSS_BBOX = dict(type='IoULoss', loss_weight=1.0)
_DEFAULT_LOSS_CENTERNESS = dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0)


@register(HEADS, partial=True)
class CondInstBoxHead:
    """The target builder and the loss of the reference's ``CondInstBoxHead``; everything else is inherited from the
    reference's class when mmdet is importable (``register(partial=True)``).  Stand-alone it carries the attributes
    ``get_targets`` and ``loss`` read and builds no conv towers."""

    def __init__(self, num_classes, in_channels=256, regress_ranges=((-1, 64), (64, 128), (128, 256), (256, 512), (512, INF)),
                 strides=(8, 16, 32, 64, 128), center_sampling=True, center_sample_radius=1.5, norm_on_bbox=True,
                 loss_cls=_DEFAULT_LOSS_CLS, loss_bbox=_DEFAULT_LOSS_BBOX, loss_centerness=_DEFAULT_LOSS_CENTERNESS,
                 test_cfg=None, **kwargs):
        self.num_classes = num_classes
        self.in_channels = in_channels
        self.regress_ranges = regress_ranges
        self.strides = strides
        self.center_sampling = center_sampling
        self.center_sample_radius = center_sample_radius
        self.norm_on_bbox = norm_on_bbox
        self.loss_cls, self.loss_bbox, self.loss_centerness = dict(loss_cls), dict(loss_bbox), dict(loss_centerness)
        self.test_cfg = test_cfg
        self._bxs_post_init()

    def _bxs_post_init(self):
        """Also runs after the REFERENCE class's ``__init__`` when mmdet is importable, on the loss modules it built.  Never
        raises: a loss outside the envelope is recorded, and ``loss`` then defers to the reference or raises."""
        self.box_losses = box_loss_envelope(self.loss_cls, self.loss_bbox, self.loss_centerness)

    def get_targets(self, points, gt_bboxes_list, gt_labels_list):
        """condinst_head.py:477-548, same arguments and return value."""
        assert len(points) == len(self.regress_ranges)
        return fcos_get_targets(points, gt_bboxes_list, gt_labels_list, self.regress_ranges, self.strides, self.num_classes,
                                self.center_sampling, self.center_sample_radius, self.norm_on_bbox)

    def loss(self, cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels, img_metas, gt_bboxes_ignore=None):
        """condinst_head.py:364-476, same arguments and return value: ({loss_cls, loss_bbox, loss_centerness},
        flatten_points, flatten_level_inds, flatten_img_inds, flatten_gt_inds).

        Inside the envelope (``box_loss_envelope``) every step runs on the device with no host read, and the number of
        launches does not depend on the ground truths or positives.  float16 / bfloat16 predictions are promoted to float32
        (the reference's ``@force_fp32``) and their gradients return in the input dtype.  Without a positive, loss_bbox and
        loss_centerness are zeros attached to the graph and loss_cls uses avg_factor 1.  Outside the envelope this calls the
        reference's own ``loss`` when mmdet is importable and raises NotImplementedError otherwise."""
        if isinstance(self.box_losses, str):
            ref = getattr(type(self), '_bxs_reference_class', None)
            if ref is not None:
                return ref.loss(self, cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels, img_metas,
                                gt_bboxes_ignore)
            raise NotImplementedError(f'CondInstBoxHead.loss: unsupported {self.box_losses}')
        focal, lw_bbox, lw_ctr = self.box_losses
        assert len(cls_scores) == len(bbox_preds) == len(centernesses)
        sizes = [tuple(int(v) for v in c.shape[-2:]) for c in cls_scores]
        dev = bbox_preds[0].device
        strides = [int(s[0]) if isinstance(s, (tuple, list)) else s for s in self.strides]
        points = fcos_points(sizes, strides, dev)
        labels, bbox_targets, gt_inds = self.get_targets(points, gt_bboxes, gt_labels)
        B = cls_scores[0].shape[0]
        den = reduce_mean_clamped(fcos_box_stats(labels, bbox_targets, sizes, strides, B, self.num_classes))
        loss_cls = sigmoid_focal_loss_levels(cls_scores, [t.reshape(B, -1) for t in labels], den[0], *focal)
        loss_bbox, loss_centerness = fcos_box_losses(bbox_preds, centernesses, labels, bbox_targets, den, strides,
                                                     self.num_classes, lw_bbox, lw_ctr)
        flatten_points = torch.cat([p.repeat(B, 1) for p in points])
        flatten_img_inds = torch.cat([torch.arange(B, device=dev).view(B, 1).expand(B, h * w).reshape(-1) for h, w in sizes])
        flatten_level_inds = torch.cat([torch.full((B * h * w,), i, device=dev).long() for i, (h, w) in enumerate(sizes)])
        losses = dict(loss_cls=loss_cls, loss_bbox=loss_bbox, loss_centerness=loss_centerness)
        return losses, flatten_points, flatten_level_inds, flatten_img_inds, torch.cat(gt_inds)

    def get_bboxes(self, cls_scores, bbox_preds, centernesses, param_preds, img_metas, cfg=None, rescale=False, with_nms=True):
        """condinst_head.py:640-853, same arguments and return value: per image (det_bboxes [n,5], det_labels int64,
        det_params [n,P], det_coors [n,2], det_level_inds int64), or with ``with_nms=False`` the reference's 6-tuple of
        every kept point.  ``cfg=None`` means ``self.test_cfg``.  Every image at once on the kernels of
        csrc/condinst_infer.cu (``condinst_infer.get_bboxes``), with two host reads per call; equal top-k keys keep the
        lower point and equal scores the candidate order (INTEGRATION.md section 11)."""
        from .condinst_infer import get_bboxes
        return get_bboxes(cls_scores, bbox_preds, centernesses, param_preds, img_metas,
                          self.test_cfg if cfg is None else cfg, self.strides, rescale, with_nms)
