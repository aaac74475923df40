"""mmdet's ``FocalLoss(use_sigmoid=True)`` over every FPN level in one kernel -- BoxSOLOv2's category loss
(box_solov2_head.py:370-383) and CondInstBoxHead's classification loss (condinst_head.py:404-445) -- without the permute /
reshape / cat of the reference and without a host synchronisation.

The forward (bxs_sigmoid_focal_loss_cells_forward) writes the loss and d loss / d logits in the same pass, each level's
gradient in that level's own [B,C,H,W] layout; the backward is ``saved_grad * g_out``.  Deterministic (no atomics).
"""
import ctypes

import torch

from .. import _lib as L


class _FocalLevels(torch.autograd.Function):
    @staticmethod
    def forward(ctx, params, labels, avg_factor, *preds):
        gamma, alpha, loss_weight = params
        B, C = preds[0].shape[:2]
        n = len(preds)
        need_grad = any(ctx.needs_input_grad[3:])
        grads = [torch.empty_like(p) for p in preds] if need_grad else None
        loss = preds[0].new_empty(())
        cells = (ctypes.c_int64 * n)(*[p.shape[2] * p.shape[3] for p in preds])
        ptrs = lambda ts: (ctypes.c_void_p * n)(*[t.data_ptr() for t in ts])    # noqa: E731
        with torch.cuda.device(preds[0].device):
            lib = L.lib()
            ws = torch.empty(lib.bxs_sigmoid_focal_loss_cells_forward_workspace_bytes(cells, n, B), dtype=torch.uint8,
                             device=preds[0].device)
            L.check(lib.bxs_sigmoid_focal_loss_cells_forward(ptrs(preds), ptrs(labels), cells, ptrs(grads) if need_grad else None,
                                                             L.ptr(avg_factor), L.ptr(loss), L.ptr(ws), n, B, C, gamma, alpha,
                                                             loss_weight, L.stream()), 'sigmoid_focal_loss_cells_forward')
        if need_grad:
            ctx.save_for_backward(*grads)
        return loss

    @staticmethod
    def backward(ctx, g_out):
        return (None, None, None, *[g * g_out for g in ctx.saved_tensors])


def sigmoid_focal_loss_levels(cate_preds, cate_labels, avg_factor, gamma=2.0, alpha=0.25, loss_weight=1.0):
    """``loss_weight * FocalLoss(cat_l(cate_preds[l].permute(0,2,3,1).reshape(-1,C)), cat_l(cate_labels[l].reshape(-1)),
    avg_factor=avg_factor)`` with mmdet's sigmoid focal loss and reduction 'mean' (sum / (avg_factor + FLT_EPSILON)).

    cate_preds: per level [B,C,H_l,W_l] logits (at most 8 levels; other dtypes are promoted to float32); cate_labels: per
    level [B,H_l,W_l] or [B,H_l*W_l] integer labels (cell y*W_l + x), a label outside [0, C) -- C is the background --
    makes the cell all-negative; avg_factor: a number or a device scalar tensor (read on the device).  The element loss is the numerically
    stable form of ``py_sigmoid_focal_loss`` (softplus for the logs).  Differentiable with respect to cate_preds."""
    preds = [p.contiguous().float() for p in cate_preds]
    L.require_cuda(*preds)
    dev = preds[0].device
    B, C = preds[0].shape[:2]
    for p in preds:
        if p.dim() != 4 or p.shape[:2] != (B, C):
            raise ValueError(f'cate_preds must be [B,C,H,W] with one B and C, got {tuple(p.shape)}')
    labels = [t.reshape(B, -1).to(device=dev, dtype=torch.int64).contiguous() for t in cate_labels]
    if len(labels) != len(preds) or any(t.shape[1] != p.shape[2] * p.shape[3] for t, p in zip(labels, preds)):
        raise ValueError('cate_labels must hold one [B,H*W] tensor per level')
    if torch.is_tensor(avg_factor):
        avg = avg_factor.detach().reshape(()).to(device=dev, dtype=torch.float32)
    else:
        avg = torch.full((), float(avg_factor), dtype=torch.float32, device=dev)
    return _FocalLevels.apply((float(gamma), float(alpha), float(loss_weight)), labels, avg, *preds)
