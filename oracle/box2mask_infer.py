"""Box2Mask inference restated in torch / numpy on the CPU: ``Box2MaskHead.simple_test`` (mmdet/models/dense_heads/
box2mask_head.py:445-459), ``MaskFormerFusionHead.simple_test`` / ``instance_postprocess`` (mmdet/models/seg_heads/
panoptic_fusion_heads/maskformer_fusion_head.py:112-241) and ``mask2bbox`` (mmdet/core/mask/utils.py:68-89).  Pinned to the
reference's own functions by tests/golden/box2mask_infer.npz (oracle/make_golden_box2mask_infer.py).

Two choices the reference leaves open are fixed here as the package's kernels fix them:
- the top ``max_per_image`` (query, class) pairs come from a stable descending sort (equal scores: the lower flat index
  q*K + c first), where the reference's ``topk(sorted=False)`` promises no order;
- every bilinear resize is ATen's upsample_bilinear2d arithmetic restated in float32 (oracle/solo_seg.py's taps), each
  product and sum rounded on its own (on CUDA tensors: ATen's kernel itself).  Equal input and output sizes copy, as ATen
  does.
Every function runs on CPU or CUDA tensors."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle.solo_seg import _lerp2, _tap


def resize(x, out_hw):
    """interpolate(x, out_hw, mode='bilinear', align_corners=False) of x [n, h, w] (float32 or float16 torch tensor; a
    float16 result is rounded to float16, as ATen computes on a half tensor).  A CUDA tensor goes through ATen's CUDA kernel
    itself, which the restatement restates (and which copies when the sizes are equal)."""
    if x.is_cuda:
        return F.interpolate(x[None], (int(out_hw[0]), int(out_hw[1])), mode='bilinear', align_corners=False)[0]
    dtype = x.dtype
    a = x.float().numpy()
    n, h, w = a.shape
    H, W = int(out_hw[0]), int(out_hw[1])
    if (h, w) == (H, W):
        return x.clone()
    ty = [_tap(np.float32(h) / np.float32(H), d, h) for d in range(H)]
    tx = [_tap(np.float32(w) / np.float32(W), d, w) for d in range(W)]
    col = lambda ts, k, t: np.array([v[k] for v in ts], t)
    y0, yp, x0, xp = col(ty, 0, np.int64), col(ty, 1, np.int64), col(tx, 0, np.int64), col(tx, 1, np.int64)
    wy = (None, None, col(ty, 2, np.float32)[:, None], col(ty, 3, np.float32)[:, None])
    wx = (None, None, col(tx, 2, np.float32)[None, :], col(tx, 3, np.float32)[None, :])
    Y0, Y1, X0, X1 = y0[:, None], (y0 + yp)[:, None], x0[None, :], (x0 + xp)[None, :]
    out = _lerp2(wy, wx, a[:, Y0, X0], a[:, Y0, X1], a[:, Y1, X0], a[:, Y1, X1]).astype(np.float32)
    return torch.from_numpy(out).to(dtype)


def interpolate(x, size=None, mode='bilinear', align_corners=False, **kw):
    """F.interpolate's signature for [N, C, h, w] with ``resize``'s arithmetic."""
    assert mode == 'bilinear' and not align_corners and not kw
    N, C, h, w = x.shape
    return resize(x.reshape(N * C, h, w), size).reshape(N, C, int(size[0]), int(size[1]))


def mask2bbox(masks):
    """[n, 4] float32 tight boxes [x_min, y_min, x_max + 1, y_max + 1] of bool masks [n, h, w], zeros when empty."""
    n = masks.shape[0]
    x_any, y_any = masks.any(1), masks.any(2)
    box = torch.zeros((n, 4), dtype=torch.float32, device=masks.device)
    for i in range(n):
        x, y = torch.where(x_any[i])[0], torch.where(y_any[i])[0]
        if len(x) and len(y):
            box[i] = torch.stack([x[0], y[0], x[-1] + 1, y[-1] + 1]).float()
    return box


def head_simple_test(all_cls_scores, all_mask_preds):
    """Box2MaskHead.simple_test after its forward, as this package returns it: the last layer, low resolution."""
    return all_cls_scores[-1], all_mask_preds[-1]


def instance_postprocess(mask_cls, mask_pred, num_things, max_per_image=100):
    """(labels, query, bboxes [n, 5], masks bool [n, h, w]) of one image (:112-152, stable order)."""
    num_classes = mask_cls.shape[-1] - 1
    scores = F.softmax(mask_cls, dim=-1)[:, :-1]
    if max_per_image > scores.numel():
        raise RuntimeError('selected index k out of range')
    s, top = torch.sort(scores.flatten(0, 1), descending=True, stable=True)
    scores_per_image, top = s[:max_per_image], top[:max_per_image]
    labels = top % num_classes
    query = top // num_classes
    is_thing = labels < num_things
    scores_per_image, labels, query = scores_per_image[is_thing], labels[is_thing], query[is_thing]
    mask_pred = mask_pred[query]
    binary = (mask_pred > 0).float()
    mask_scores = (mask_pred.sigmoid() * binary).flatten(1).sum(1) / (binary.flatten(1).sum(1) + 1e-6)
    det_scores = scores_per_image * mask_scores
    binary = binary.bool()
    bboxes = torch.cat([mask2bbox(binary), det_scores[:, None]], dim=-1)
    return labels, query, bboxes, binary


def fusion_simple_test(mask_cls_results, mask_pred_results, img_metas, num_things, max_per_image=100, rescale=False):
    """MaskFormerFusionHead.simple_test (instance output) per image; mask_pred_results at the mask-feature resolution are
    first upsampled to img_metas[0]['batch_input_shape'] (the reference head's F.interpolate)."""
    pad = tuple(img_metas[0]['batch_input_shape'][:2])
    if tuple(mask_pred_results.shape[-2:]) != pad:
        mask_pred_results = interpolate(mask_pred_results, pad)
    out = []
    for mask_cls, mask_pred, meta in zip(mask_cls_results, mask_pred_results, img_metas):
        H, W = meta['img_shape'][:2]
        mask_pred = mask_pred[:, :H, :W]
        if rescale:
            mask_pred = resize(mask_pred, meta['ori_shape'][:2])
        out.append(instance_postprocess(mask_cls, mask_pred, num_things, max_per_image))
    return out
