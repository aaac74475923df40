"""Box2Mask's classification loss: mmdet's ``CrossEntropyLoss(use_sigmoid=False, reduction='mean', class_weight=w)`` of every
decoder layer in one kernel (box2mask_head.py:248-258), with ``avg_factor = w[labels].sum()`` computed on the device and no
host synchronisation.

The forward (bxs_softmax_cross_entropy_layers_forward) writes the losses and d loss_l / d scores_l in the same pass, each
layer's gradient in that layer's own [B,Q,K] layout; the backward scales them in place by the upstream gradients (nothing to
do for an upstream gradient of 1).  Deterministic (no atomics).
"""
import ctypes

import torch

from .. import _lib as L

MAX_LAYERS = 16


def _forward(lib, preds, labels, cw, loss, grads, loss_weight):
    n = len(preds)
    B, Q, K = preds[0].shape
    ptrs = lambda ts: (ctypes.c_void_p * n)(*[t.data_ptr() for t in ts])    # noqa: E731
    ws = torch.empty(lib.bxs_softmax_cross_entropy_layers_forward_workspace_bytes(n, B, Q), dtype=torch.uint8,
                     device=preds[0].device)
    L.check(lib.bxs_softmax_cross_entropy_layers_forward(ptrs(preds), L.ptr(labels), L.ptr(cw),
                                                         ptrs(grads) if grads is not None else None, L.ptr(loss), L.ptr(ws),
                                                         n, B, Q, K, loss_weight, L.stream()),
            'softmax_cross_entropy_layers_forward')


class _CrossEntropyLayers(torch.autograd.Function):
    @staticmethod
    def forward(ctx, loss_weight, labels, cw, *preds):
        need_grad = any(ctx.needs_input_grad[3:])
        grads = [torch.empty_like(p) for p in preds] if need_grad else None
        loss = preds[0].new_empty((len(preds),))
        with torch.cuda.device(preds[0].device):
            _forward(L.lib(), preds, labels, cw, loss, grads, loss_weight)
        if need_grad:
            ctx.save_for_backward(labels, cw, *preds, *grads)
            ctx.loss_weight, ctx.calls = loss_weight, 0
        return loss

    @staticmethod
    def backward(ctx, g_out):
        saved = ctx.saved_tensors
        labels, cw, rest = saved[0], saved[1], saved[2:]
        n = len(rest) // 2
        preds, grads = rest[:n], rest[n:]
        ctx.calls += 1
        B, Q, K = preds[0].shape
        g = g_out.detach().to(torch.float32).contiguous()
        with torch.cuda.device(preds[0].device):
            lib = L.lib()
            if ctx.calls > 1:       # a second backward (retain_graph): the saved gradients were scaled in place, recompute
                grads = [torch.empty_like(p) for p in preds]
                _forward(lib, preds, labels, cw, preds[0].new_empty((n,)), grads, ctx.loss_weight)
            L.check(lib.bxs_softmax_cross_entropy_layers_backward((ctypes.c_void_p * n)(*[t.data_ptr() for t in grads]),
                                                                  L.ptr(g), n, B, Q, K, L.stream()),
                    'softmax_cross_entropy_layers_backward')
        return (None, None, None, *[gr if need else None for gr, need in zip(grads, ctx.needs_input_grad[3:])])


def softmax_cross_entropy_layers(scores_list, labels, class_weight=None, loss_weight=1.0):
    """[L] float32 losses: ``loss_weight * CrossEntropyLoss(class_weight=w)(scores_list[l].flatten(0, 1), labels[l].flatten(),
    avg_factor=w[labels[l]].sum())`` for every layer l, mmdet's softmax cross-entropy with reduction 'mean'
    (sum / (avg_factor + FLT_EPSILON)).

    scores_list: L <= 16 CUDA tensors [B,Q,K] (one B, Q, K), K = num_classes + 1; float16 / bfloat16 scores are promoted to
    float32 (what the reference's ``@force_fp32`` on ``loss`` does).  labels: integer [L,B,Q] (or a list of L [B,Q]); a label
    outside [0, K) adds nothing to the loss, to avg_factor or to the gradient (torch asserts there instead).  class_weight:
    [K] (list or tensor) or None for all ones.  Differentiable with respect to every entry of scores_list."""
    preds = [p.float().contiguous() for p in scores_list]
    if not preds:
        raise ValueError('scores_list is empty')
    if len(preds) > MAX_LAYERS:
        raise ValueError(f'at most {MAX_LAYERS} layers, got {len(preds)}')
    L.require_cuda(*preds)
    dev = preds[0].device
    shape = preds[0].shape
    for p in preds:
        if p.dim() != 3 or p.shape != shape:
            raise ValueError(f'scores_list must hold [B,Q,K] tensors of one shape, got {tuple(p.shape)}')
    if not torch.is_tensor(labels):
        labels = torch.stack([torch.as_tensor(t, device=dev) for t in labels])
    labels = labels.to(device=dev, dtype=torch.int64).reshape(len(preds), shape[0], shape[1]).contiguous()
    cw = None
    if class_weight is not None:
        cw = torch.as_tensor(class_weight, dtype=torch.float32, device=dev).reshape(-1).contiguous()
        if cw.numel() != shape[2]:
            raise ValueError(f'class_weight must hold K = {shape[2]} weights, got {cw.numel()}')
    return _CrossEntropyLayers.apply(float(loss_weight), labels, cw, *preds)
