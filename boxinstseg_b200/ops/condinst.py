"""a1: CondInst dynamic mask head on the C ABI (replaces CondInstMaskHead.forward,
mmdet/models/dense_heads/condinst_head.py:1139-1164; differentiable wrt mask_feat and params)."""
import ctypes

import torch

from .. import _lib as L


class _DynamicMaskHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, params, coors, soi, img_inds, in_stride, factor, rel):
        feat = feat.contiguous().float()
        params = params.contiguous().float()
        L.require_cuda(feat, params, coors, soi, img_inds)
        N, P = params.shape
        B, C, h, w = feat.shape
        out = torch.empty((N, 1, factor * h, factor * w), dtype=torch.float32, device=feat.device)
        if N:
            with torch.cuda.device(feat.device):
                L.check(L.lib().bxs_condinst_head_forward(L.ptr(feat), L.ptr(params), L.ptr(coors), L.ptr(soi),
                                                          L.ptr(img_inds), L.ptr(out), N, B, C, h, w, P, in_stride,
                                                          factor, int(rel), L.stream()), 'condinst_head_forward')
        ctx.save_for_backward(feat, params, coors, soi, img_inds)
        ctx.cfg = (in_stride, factor, int(rel))
        return out

    @staticmethod
    def backward(ctx, g_out):
        feat, params, coors, soi, img_inds = ctx.saved_tensors
        in_stride, factor, rel = ctx.cfg
        N, P = params.shape
        B, C, h, w = feat.shape
        g_feat = torch.empty_like(feat)
        g_params = torch.empty_like(params)
        if N == 0:
            return g_feat.zero_(), g_params, None, None, None, None, None, None
        g_out = g_out.contiguous().float()
        lib = L.lib()
        ws = torch.empty(lib.bxs_condinst_head_workspace_bytes(N, B, h, w, P), dtype=torch.uint8, device=feat.device)
        with torch.cuda.device(feat.device):
            L.check(lib.bxs_condinst_head_backward(L.ptr(feat), L.ptr(params), L.ptr(coors), L.ptr(soi),
                                                   L.ptr(img_inds), L.ptr(g_out), L.ptr(g_feat), L.ptr(g_params),
                                                   L.ptr(ws), N, B, C, h, w, P, in_stride, factor, rel, L.stream()),
                    'condinst_head_backward')
        return g_feat, g_params, None, None, None, None, None, None


def dynamic_mask_head(feat, params, coors, level_inds, img_inds, sizes_of_interest, in_stride=8, out_stride=4,
                      channels=8, num_layers=3, rel_coors=True):
    """feat [B,C,h,w], params [N,P], coors [N,2], level_inds/img_inds [N] -> mask logits [N,1,f*h,f*w]."""
    if channels != 8 or num_layers != 3:
        raise NotImplementedError('libboxseg_b200 implements dynamic_channels=8, dynamic_convs=3 '
                                  '(every CondInst/BoxInst config of the reference)')
    if feat.shape[1] > 32:
        raise NotImplementedError('mask_feat channels > 32')
    dev = feat.device
    soi = sizes_of_interest.to(device=dev, dtype=torch.float32)[level_inds.long()].contiguous() if rel_coors else None
    coors = coors.to(device=dev, dtype=torch.float32).contiguous() if rel_coors else None
    img32 = img_inds.to(device=dev, dtype=torch.int32).contiguous()
    return _DynamicMaskHead.apply(feat, params, coors, soi, img32, in_stride, in_stride // out_stride, rel_coors)


def paste_masks(mask_logits, factor, img_shape, ori_shape=None):
    """The mask lines of CondInstMaskHead.simple_test (condinst_head.py:1261-1281) in one pass: mask_logits [n,1,h,w] ->
    bool [n, H, W] = aligned_bilinear(sigmoid(mask_logits), factor)[:, :, :H_img, :W_img] > 0.5, resized bilinearly
    (align_corners=False) to ``ori_shape[:2]`` before the threshold when ``ori_shape`` is given (``rescale=True``)."""
    n, _, h, w = mask_logits.shape
    logits = mask_logits.detach().float().contiguous()
    L.require_cuda(logits)
    H_img, W_img = [int(v) for v in img_shape[:2]]
    H, W = [int(v) for v in ori_shape[:2]] if ori_shape is not None else (H_img, W_img)
    out = torch.empty((n, H, W), dtype=torch.bool, device=logits.device)
    with torch.cuda.device(logits.device):
        L.check(L.lib().bxs_condinst_paste_masks(L.ptr(logits), n, h, w, int(factor), H_img, W_img, H, W,
                                                 int(ori_shape is not None), L.ptr(out), L.stream()), 'condinst_paste_masks')
    return out


MAX_MASK_IMAGES = 64            # the per-image mask table of csrc/condinst_sup.cu travels in the kernel parameters


def _mask_table(gt_masks):
    """(mask pointers, element strides [3B], ground-truth offsets [B+1]) as ctypes arrays, and the shared (H, W), of the
    per-image uint8 / bool [G_b, H, W] CUDA masks, read in place by csrc/condinst_sup.cu."""
    if not 0 < len(gt_masks) <= MAX_MASK_IMAGES:
        raise NotImplementedError(f'libboxseg_b200 reads the masks of 1 to {MAX_MASK_IMAGES} images per call, got '
                                  f'{len(gt_masks)}')
    H, W = (int(v) for v in gt_masks[0].shape[-2:])
    off = [0]
    for m in gt_masks:
        if m.dim() != 3 or tuple(m.shape[-2:]) != (H, W):
            raise ValueError(f'gt_masks must be [G_b, H, W] with one H and W, got {tuple(m.shape)}')
        if m.dtype not in (torch.uint8, torch.bool):
            raise TypeError(f'gt_masks must be uint8 or bool, got {m.dtype}')
        if not m.is_cuda:
            raise RuntimeError('boxinstseg_b200: tensor must be a CUDA tensor')
        off.append(off[-1] + int(m.shape[0]))
    B = len(gt_masks)
    masks = (ctypes.c_void_p * B)(*[m.data_ptr() if m.numel() else None for m in gt_masks])
    strides = (ctypes.c_int64 * (3 * B))(*[s for m in gt_masks for s in m.stride()])
    return masks, strides, (ctypes.c_int64 * (B + 1))(*off), H, W


class _DiceMaskLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, gt_inds, gt_masks, start, stride):
        N, h, w = logits.shape
        masks, strides, off, H, W = _mask_table(gt_masks)
        dev = logits.device
        sums = torch.empty((N, 3), dtype=torch.float32, device=dev)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        lib = L.lib()
        ws = torch.empty(lib.bxs_condinst_dice_workspace_bytes(N, h, w), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            L.check(lib.bxs_condinst_dice_forward(L.ptr(logits), L.ptr(gt_inds), N, h, w, masks, strides, off, len(gt_masks),
                                                  H, W, start, stride, L.ptr(sums), L.ptr(loss), L.ptr(ws), L.stream()),
                    'condinst_dice_forward')
        ctx.save_for_backward(logits, gt_inds, sums)
        ctx.masks, ctx.cfg = list(gt_masks), (start, stride)
        ctx.mark_non_differentiable(sums)
        return loss, sums

    @staticmethod
    def backward(ctx, g_loss, _g_sums):
        logits, gt_inds, sums = ctx.saved_tensors
        N, h, w = logits.shape
        masks, strides, off, H, W = _mask_table(ctx.masks)
        g = g_loss.detach().reshape(()).float().contiguous()
        g_logits = torch.empty_like(logits)
        with torch.cuda.device(logits.device):
            L.check(L.lib().bxs_condinst_dice_backward(L.ptr(logits), L.ptr(gt_inds), N, h, w, masks, strides, off,
                                                       len(ctx.masks), H, W, *ctx.cfg, L.ptr(sums), L.ptr(g),
                                                       L.ptr(g_logits), L.stream()), 'condinst_dice_backward')
        return g_logits, None, None, None, None


def dice_mask_loss(mask_logits, gt_masks, gt_inds, out_stride, return_sums=False):
    """``dice_coefficient(mask_logits.sigmoid(), cat(bitmasks)[gt_inds]).mean()`` of CondInstMaskHead.loss with
    boxinst_enabled=False (condinst_head.py:117-131, 1298-1341), without the [N, h, w] target: ``bitmasks`` are
    ``m[:, s // 2::s, s // 2::s]`` (s = out_stride) of ``gt_masks``, the per-image uint8 [G_b, H, W] CUDA masks of
    ``CondInst.forward_train``, read in place at any strides.

    mask_logits: [N, 1, h, w] or [N, h, w], any float dtype (float16 / bfloat16 are promoted, as ``@force_fp32`` does; the
    gradient returns in the input dtype), any strides; gt_inds: [N] global ground-truth indices.  Returns the float32 loss
    (and, with ``return_sums``, the per-instance float32 [N, 3] sums (I, S, T)).  N == 0 gives the reference's
    ``0 * sigmoid(mask_logits).sum()``, attached to the graph.  Deterministic, no host synchronisation."""
    logits = mask_logits.float()
    N = logits.shape[0]
    logits = logits.reshape(N, *logits.shape[-2:])
    h, w = int(logits.shape[1]), int(logits.shape[2])
    s, start = int(out_stride), int(out_stride) // 2
    H, W = (int(v) for v in gt_masks[0].shape[-2:])
    if (len(range(start, H, s)), len(range(start, W, s))) != (h, w):
        raise ValueError(f'mask logits of {h}x{w} do not match masks of {H}x{W} sampled every {s} from {start}')
    if N == 0:
        loss = 0 * logits.sigmoid().sum()
        return (loss, logits.new_zeros((0, 3))) if return_sums else loss
    x = logits.contiguous()
    L.require_cuda(x)
    gt32 = gt_inds.to(device=x.device, dtype=torch.int32).contiguous()
    loss, sums = _DiceMaskLoss.apply(x, gt32, list(gt_masks), start, s)
    return (loss, sums) if return_sums else loss


def semantic_targets(gt_masks, gt_labels, stride, num_classes, return_areas=False):
    """CondInstSegmHead.get_targets (condinst_head.py:950-968) on the device: int64 [B, oh, ow] labels at the pixels
    (s/2 + s*i, s/2 + s*j), s = ``stride``, of the per-image uint8 [G_b, H, W] ``gt_masks`` (read in place) and int64
    [G_b] ``gt_labels``: the label of the first ground truth of least area among those whose mask is non-zero there,
    ``num_classes`` where none is (areas are int64 sums of the byte values, bit-exact with the reference's ``torch.sum``
    and its ``INF = 1e8`` sentinel).  An image without ground truth is all ``num_classes`` (the reference raises).  With
    ``return_areas`` also the int64 [sum G_b] areas.  Images are processed 64 per launch pair; no host synchronisation."""
    s = int(stride)
    H, W = (int(v) for v in gt_masks[0].shape[-2:])
    dev = gt_masks[0].device
    oh, ow = len(range(s // 2, H, s)), len(range(s // 2, W, s))
    out = torch.empty((len(gt_masks), oh, ow), dtype=torch.int64, device=dev)
    areas = torch.empty(sum(int(m.shape[0]) for m in gt_masks), dtype=torch.int64, device=dev)
    labels = [t.to(device=dev, dtype=torch.int64).contiguous() for t in gt_labels]
    if len(labels) != len(gt_masks) or any(t.numel() != m.shape[0] for t, m in zip(labels, gt_masks)):
        raise ValueError('gt_labels must hold one [G_b] tensor per image')
    lib = L.lib()
    b0 = g0 = 0
    while b0 < len(gt_masks):
        group = gt_masks[b0:b0 + MAX_MASK_IMAGES]
        masks, strides, off, _, _ = _mask_table(group)
        lab = (ctypes.c_void_p * len(group))(*[t.data_ptr() if t.numel() else None for t in labels[b0:b0 + len(group)]])
        with torch.cuda.device(dev):
            L.check(lib.bxs_condinst_semantic_targets(masks, strides, lab, off, len(group), H, W, s, int(num_classes),
                                                      L.ptr(areas[g0:]) if off[len(group)] else None, L.ptr(out[b0:]),
                                                      L.stream()), 'condinst_semantic_targets')
        b0 += len(group)
        g0 += off[len(group)]
    return (out, areas) if return_areas else out
