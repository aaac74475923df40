"""CondInstBoxHead's regression and centerness losses over every FCOS level and image in one kernel
(condinst_head.py:437-469): ``GIoULoss`` weighted by the centerness targets and ``CrossEntropyLoss(use_sigmoid=True)`` on
the centerness logits, both with reduction 'mean', without the permute / cat, ``nonzero()`` and gathers of the reference
and without a host synchronisation.

``fcos_box_stats`` (bxs_fcos_loss_stats) gives the positive count and the sum of the positives' centerness targets on the
device; ``fcos_box_losses`` (bxs_fcos_loss_forward) writes both losses and their gradients, each level's in that level's own
[B,4,H,W] / [B,1,H,W] layout, in the same pass; the backward scales them in place by the upstream gradients (nothing to do
for an upstream gradient of 1).  Deterministic (no atomics).
"""
import ctypes

import torch

from .. import _lib as L

MAX_LEVELS = 8


def fcos_points(featmap_sizes, strides, device):
    """``MlvlPointGenerator(strides, offset=0.5).grid_priors(featmap_sizes, torch.float32, device)``: per level [H*W, 2]
    float32 ``((x + 0.5) * stride, (y + 0.5) * stride)``, x fastest, computed on the device (exact in fp32)."""
    out = []
    for (h, w), s in zip(featmap_sizes, strides):
        xs = (torch.arange(w, device=device) + 0.5) * s
        ys = (torch.arange(h, device=device) + 0.5) * s
        yy, xx = torch.meshgrid(ys, xs, indexing='ij')
        out.append(torch.stack([xx.reshape(-1), yy.reshape(-1)], -1))
    return out


class _Shapes:
    """The level table's host arrays: H_l, W_l, stride_l."""

    def __init__(self, featmap_sizes, strides):
        n = len(featmap_sizes)
        if not 0 < n <= MAX_LEVELS or len(strides) != n:
            raise ValueError(f'1 to {MAX_LEVELS} levels with one stride each, got {n} levels and {len(strides)} strides')
        self.n = n
        self.h = (ctypes.c_int64 * n)(*[int(s[0]) for s in featmap_sizes])
        self.w = (ctypes.c_int64 * n)(*[int(s[1]) for s in featmap_sizes])
        self.stride = (ctypes.c_float * n)(*[float(s) for s in strides])

    def workspace(self, lib, B, device):
        return torch.empty(lib.bxs_fcos_loss_workspace_bytes(self.h, self.w, self.n, B), dtype=torch.uint8, device=device)


def _ptrs(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _level_inputs(labels, bbox_targets, B, featmap_sizes, device):
    labels = [t.reshape(-1).to(device=device, dtype=torch.int64).contiguous() for t in labels]
    targets = [t.reshape(-1, 4).to(device=device, dtype=torch.float32).contiguous() for t in bbox_targets]
    for lab, tgt, (h, w) in zip(labels, targets, featmap_sizes):
        if lab.shape[0] != B * h * w or tgt.shape[0] != B * h * w:
            raise ValueError(f'labels / bbox_targets of a {h}x{w} level must hold B*H*W = {B * h * w} points')
    return labels, targets


def fcos_box_stats(labels, bbox_targets, featmap_sizes, strides, B, num_classes):
    """[2] float32 on the device: (number of positives, sum of the positives' centerness targets) over every level and
    image.  labels / bbox_targets: per level [B*H_l*W_l] / [B*H_l*W_l, 4], as ``get_targets`` returns them; a label in
    [0, num_classes) is a positive."""
    shapes = _Shapes(featmap_sizes, strides)
    dev = labels[0].device
    labels, targets = _level_inputs(labels, bbox_targets, B, featmap_sizes, dev)
    L.require_cuda(*labels, *targets)
    stats = torch.empty(2, dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        lib = L.lib()
        L.check(lib.bxs_fcos_loss_stats(_ptrs(labels), _ptrs(targets), shapes.h, shapes.w, shapes.stride, L.ptr(stats),
                                        L.ptr(shapes.workspace(lib, B, dev)), shapes.n, B, int(num_classes), L.stream()),
                'fcos_loss_stats')
    return stats


def _forward(lib, shapes, meta, labels, targets, den, bbox, ctr, g_pred, g_ctr):
    B, C, lw_bbox, lw_ctr = meta
    loss_bbox, loss_ctr = den.new_empty(()), den.new_empty(())
    L.check(lib.bxs_fcos_loss_forward(_ptrs(bbox), _ptrs(ctr), _ptrs(labels), _ptrs(targets),
                                      _ptrs(g_pred) if g_pred is not None else None,
                                      _ptrs(g_ctr) if g_ctr is not None else None, shapes.h, shapes.w, shapes.stride,
                                      L.ptr(den), L.ptr(loss_bbox), L.ptr(loss_ctr), L.ptr(shapes.workspace(lib, B, den.device)),
                                      shapes.n, B, C, lw_bbox, lw_ctr, L.stream()), 'fcos_loss_forward')
    return loss_bbox, loss_ctr


def _grad_buffers(ts):
    """One flat buffer for the gradients of every level (one scale launch in the backward) and its per-level views."""
    flat = ts[0].new_empty(sum(t.numel() for t in ts))
    return flat, [v.view(t.shape) for v, t in zip(flat.split([t.numel() for t in ts]), ts)]


class _FcosBoxLosses(torch.autograd.Function):
    @staticmethod
    def forward(ctx, shapes, meta, labels, targets, den, *preds):
        n = shapes.n
        bbox, ctr = preds[:n], preds[n:]
        need_b, need_c = any(ctx.needs_input_grad[5:5 + n]), any(ctx.needs_input_grad[5 + n:])
        gb, gb_views = _grad_buffers(bbox) if need_b else (None, None)
        gc, gc_views = _grad_buffers(ctr) if need_c else (None, None)
        with torch.cuda.device(den.device):
            out = _forward(L.lib(), shapes, meta, labels, targets, den, bbox, ctr, gb_views, gc_views)
        ctx.set_materialize_grads(False)
        ctx.shapes, ctx.meta, ctx.calls = shapes, meta, 0
        ctx.save_for_backward(den, *labels, *targets, *preds, *([gb] if need_b else []), *([gc] if need_c else []))
        ctx.need = (need_b, need_c)
        return out

    @staticmethod
    def backward(ctx, g_bbox, g_ctr):
        shapes, n = ctx.shapes, ctx.shapes.n
        saved = ctx.saved_tensors
        den, labels, targets, preds = saved[0], saved[1:1 + n], saved[1 + n:1 + 2 * n], saved[1 + 2 * n:1 + 4 * n]
        bbox, ctr = preds[:n], preds[n:]
        rest = list(saved[1 + 4 * n:])
        need_b, need_c = ctx.need
        gb = rest.pop(0) if need_b else None
        gc = rest.pop(0) if need_c else None
        ctx.calls += 1
        with torch.cuda.device(den.device):
            lib = L.lib()
            if ctx.calls > 1:       # a second backward (retain_graph): the saved gradients were scaled in place, recompute
                gb, gb_views = _grad_buffers(bbox) if need_b else (None, None)
                gc, gc_views = _grad_buffers(ctr) if need_c else (None, None)
                _forward(lib, shapes, ctx.meta, labels, targets, den, bbox, ctr, gb_views, gc_views)
            use_b = need_b and g_bbox is not None
            use_c = need_c and g_ctr is not None
            sb = g_bbox.detach().to(torch.float32).contiguous() if use_b else None
            sc = g_ctr.detach().to(torch.float32).contiguous() if use_c else None
            L.check(lib.bxs_fcos_loss_backward(L.ptr(gb) if use_b else None, gb.numel() if use_b else 0, L.ptr(sb),
                                               L.ptr(gc) if use_c else None, gc.numel() if use_c else 0, L.ptr(sc),
                                               L.stream()), 'fcos_loss_backward')
        gbs = [v.view(t.shape) for v, t in zip(gb.split([t.numel() for t in bbox]), bbox)] if use_b else [None] * n
        gcs = [v.view(t.shape) for v, t in zip(gc.split([t.numel() for t in ctr]), ctr)] if use_c else [None] * n
        gbs = [g if need else None for g, need in zip(gbs, ctx.needs_input_grad[5:5 + n])]
        gcs = [g if need else None for g, need in zip(gcs, ctx.needs_input_grad[5 + n:])]
        return (None,) * 5 + tuple(gbs) + tuple(gcs)


def fcos_box_losses(bbox_preds, centernesses, labels, bbox_targets, den, strides, num_classes, loss_weight_bbox=1.0,
                    loss_weight_centerness=1.0):
    """(loss_bbox, loss_centerness), float32 scalars: condinst_head.py:447-469 with ``GIoULoss(eps=1e-6)`` and
    ``CrossEntropyLoss(use_sigmoid=True)``, reduction 'mean':

        loss_bbox = loss_weight_bbox * sum_pos ct (1 - GIoU(distance2bbox(point, pred), distance2bbox(point, target)))
                    / (den[1] + FLT_EPSILON)
        loss_centerness = loss_weight_centerness * sum_pos BCE_with_logits(centerness, ct) / (den[0] + FLT_EPSILON)

    with ct the centerness target of the positive's regression target and point ((x + 0.5) * stride, (y + 0.5) * stride).
    Zero when there is no positive.  bbox_preds / centernesses: per level [B,4,H_l,W_l] / [B,1,H_l,W_l] CUDA tensors
    (at most 8 levels; other dtypes are promoted to float32, any layout); labels / bbox_targets: per level [B*H_l*W_l] /
    [B*H_l*W_l, 4] as ``get_targets`` returns them, a label in [0, num_classes) marks a positive; den: [2] float32 on the
    device, (avg_factor of the centerness loss, avg_factor of the GIoU loss), read on the device.  loss_bbox is
    differentiable with respect to bbox_preds, loss_centerness with respect to centernesses."""
    bbox = [p.float().contiguous() for p in bbox_preds]
    ctr = [c.float().contiguous() for c in centernesses]
    if not bbox or len(ctr) != len(bbox) or len(labels) != len(bbox) or len(bbox_targets) != len(bbox):
        raise ValueError('bbox_preds, centernesses, labels and bbox_targets must hold one entry per level')
    L.require_cuda(*bbox, *ctr)
    B = bbox[0].shape[0]
    sizes = []
    for p, c in zip(bbox, ctr):
        if p.dim() != 4 or p.shape[:2] != (B, 4) or c.shape != (B, 1) + tuple(p.shape[2:]):
            raise ValueError(f'bbox_preds must be [B,4,H,W] and centernesses [B,1,H,W], got {tuple(p.shape)} and '
                             f'{tuple(c.shape)}')
        sizes.append(tuple(p.shape[2:]))
    shapes = _Shapes(sizes, strides)
    dev = bbox[0].device
    labels, targets = _level_inputs(labels, bbox_targets, B, sizes, dev)
    den = den.detach().to(device=dev, dtype=torch.float32).reshape(2).contiguous()
    meta = (B, int(num_classes), float(loss_weight_bbox), float(loss_weight_centerness))
    return _FcosBoxLosses.apply(shapes, meta, labels, targets, den, *bbox, *ctr)
