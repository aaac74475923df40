"""SOLOv2 inference restated line by line: ``mask_matrix_nms`` (mmdet/core/post_processing/matrix_nms.py:5-121) and
``get_seg`` / ``get_seg_single`` of BoxSOLOv2Head (mmdet/models/dense_heads/box_solov2_head.py:475-590) and
DiscoBoxSOLOv2Head (mmdet/models/dense_heads/discobox_head.py:1531-1660).  Pinned to the reference's own functions by
tests/golden/solo_seg.npz (oracle/make_golden_solo_seg.py).

Two switches the reference does not have: ``stable`` makes both sorts of ``mask_matrix_nms`` stable (the package's kernels
keep the candidates' order among equal scores), and ``half_inter`` rounds the intersection matrix to float16 once (what the
reference's ``torch.mm`` yields under DiscoBox's ``@autocast()``, without cuBLAS's reduced-precision reductions).  ``head``
is anything with the attributes the reference reads: ``cate_out_channels``, ``seg_num_grids``, ``strides`` and, for DiscoBox,
``kernel_out_channels``.  ``InstanceData`` is a plain namespace holding the image meta fields."""
import types

import numpy as np

import torch
import torch.nn.functional as F


def _sort(x, stable):
    return torch.sort(x, descending=True, stable=True) if stable else torch.sort(x, descending=True)


def mask_matrix_nms(masks, labels, scores, filter_thr=-1, nms_pre=-1, max_num=-1, kernel='gaussian', sigma=2.0,
                    mask_area=None, stable=False, half_inter=False):
    assert len(labels) == len(masks) == len(scores)
    if len(labels) == 0:
        return scores.new_zeros(0), labels.new_zeros(0), masks.new_zeros(0, *masks.shape[-2:]), labels.new_zeros(0)
    if mask_area is None:
        mask_area = masks.sum((1, 2)).float()
    else:
        assert len(masks) == len(mask_area)
    scores, sort_inds = _sort(scores, stable)
    keep_inds = sort_inds
    if nms_pre > 0 and len(sort_inds) > nms_pre:
        sort_inds = sort_inds[:nms_pre]
        keep_inds = keep_inds[:nms_pre]
        scores = scores[:nms_pre]
    masks = masks[sort_inds]
    mask_area = mask_area[sort_inds]
    labels = labels[sort_inds]
    num_masks = len(labels)
    flatten_masks = masks.reshape(num_masks, -1).float()
    inter_matrix = torch.mm(flatten_masks, flatten_masks.transpose(1, 0))
    if half_inter:
        inter_matrix = inter_matrix.half()
    expanded_mask_area = mask_area.expand(num_masks, num_masks)
    iou_matrix = (inter_matrix / (expanded_mask_area + expanded_mask_area.transpose(1, 0) - inter_matrix)).triu(diagonal=1)
    expanded_labels = labels.expand(num_masks, num_masks)
    label_matrix = (expanded_labels == expanded_labels.transpose(1, 0)).triu(diagonal=1)
    compensate_iou, _ = (iou_matrix * label_matrix).max(0)
    compensate_iou = compensate_iou.expand(num_masks, num_masks).transpose(1, 0)
    decay_iou = iou_matrix * label_matrix
    if kernel == 'gaussian':
        decay_matrix = torch.exp(-1 * sigma * (decay_iou ** 2))
        compensate_matrix = torch.exp(-1 * sigma * (compensate_iou ** 2))
        decay_coefficient, _ = (decay_matrix / compensate_matrix).min(0)
    elif kernel == 'linear':
        decay_matrix = (1 - decay_iou) / (1 - compensate_iou)
        decay_coefficient, _ = decay_matrix.min(0)
    else:
        raise NotImplementedError(f'{kernel} kernel is not supported in matrix nms!')
    scores = scores * decay_coefficient
    if filter_thr > 0:
        keep = scores >= filter_thr
        keep_inds = keep_inds[keep]
        if not keep.any():
            return scores.new_zeros(0), labels.new_zeros(0), masks.new_zeros(0, *masks.shape[-2:]), labels.new_zeros(0)
        masks = masks[keep]
        scores = scores[keep]
        labels = labels[keep]
    scores, sort_inds = _sort(scores, stable)
    keep_inds = keep_inds[sort_inds]
    if max_num > 0 and len(sort_inds) > max_num:
        sort_inds = sort_inds[:max_num]
        keep_inds = keep_inds[:max_num]
        scores = scores[:max_num]
    masks = masks[sort_inds]
    labels = labels[sort_inds]
    return scores, labels, masks, keep_inds


def InstanceData(img_meta):
    return types.SimpleNamespace(**img_meta)


def _empty_results(results, cls_scores):
    results.scores = cls_scores.new_ones(0)
    results.masks = cls_scores.new_zeros(0, *results.ori_shape[:2])
    results.labels = cls_scores.new_ones(0)
    return results


def _strides(head, cate_labels, like, inds):
    size_trans = cate_labels.new_tensor(head.seg_num_grids).pow(2).cumsum(0)
    strides = like.new_ones(size_trans[-1])
    n_stage = len(head.seg_num_grids)
    strides[:size_trans[0]] *= head.strides[0]
    for ind_ in range(1, n_stage):
        strides[size_trans[ind_ - 1]:size_trans[ind_]] *= head.strides[ind_]
    return strides[inds[:, 0]]


def _nms(seg_masks, cate_labels, cate_scores, sum_masks, cfg, stable, half_inter):
    return mask_matrix_nms(seg_masks, cate_labels, cate_scores, filter_thr=cfg.filter_thr, nms_pre=cfg.nms_pre,
                           max_num=cfg.max_per_img, kernel=cfg.kernel, sigma=cfg.sigma, mask_area=sum_masks, stable=stable,
                           half_inter=half_inter)


def box_get_seg(head, seg_preds, cate_preds, levelset_feats, img_metas, cfg, rescale=None, stable=False):   # :475-500
    assert len(seg_preds) == len(cate_preds)
    num_levels = len(cate_preds)
    featmap_size = seg_preds[0].size()[-2:]
    result_list = []
    for img_id in range(len(img_metas)):
        cate_pred_list = [cate_preds[i][img_id].view(-1, head.cate_out_channels).detach() for i in range(num_levels)]
        seg_pred_list = [seg_preds[i][img_id].detach() for i in range(num_levels)]
        cate_pred_list = torch.cat(cate_pred_list, dim=0)
        seg_pred_list = torch.cat(seg_pred_list, dim=0)
        result_list.append(box_get_seg_single(head, cate_pred_list, seg_pred_list, featmap_size, img_metas[img_id], cfg,
                                              stable))
    return result_list


def box_get_seg_single(head, cate_preds, seg_preds, featmap_size, img_meta, cfg, stable=False):          # :503-590
    assert len(cate_preds) == len(seg_preds)
    results = InstanceData(img_meta)
    h, w, _ = results.img_shape
    ori_shape = results.ori_shape
    upsampled_size_out = (featmap_size[0] * 4, featmap_size[1] * 4)
    inds = (cate_preds > cfg.score_thr)
    cate_scores = cate_preds[inds]
    if len(cate_scores) == 0:
        return _empty_results(results, cate_scores)
    inds = inds.nonzero()
    cate_labels = inds[:, 1]
    strides = _strides(head, cate_labels, cate_scores, inds)
    seg_preds = seg_preds[inds[:, 0]]
    seg_masks = seg_preds > cfg.mask_thr
    sum_masks = seg_masks.sum((1, 2)).float()
    keep = sum_masks > strides
    if keep.sum() == 0:
        return _empty_results(results, cate_scores)
    seg_masks = seg_masks[keep, ...]
    seg_preds = seg_preds[keep, ...]
    sum_masks = sum_masks[keep]
    cate_scores = cate_scores[keep]
    cate_labels = cate_labels[keep]
    seg_scores = (seg_preds * seg_masks.float()).sum((1, 2)) / sum_masks
    cate_scores *= seg_scores
    scores, labels, _, keep_inds = _nms(seg_masks, cate_labels, cate_scores, sum_masks, cfg, stable, False)
    seg_preds = seg_preds[keep_inds]
    seg_preds = F.interpolate(seg_preds.unsqueeze(0), size=upsampled_size_out, mode='bilinear')[:, :, :h, :w]
    seg_masks = F.interpolate(seg_preds, size=ori_shape[:2], mode='bilinear').squeeze(0)
    results.masks = seg_masks > cfg.mask_thr
    results.labels = labels
    results.scores = scores
    return results


def disco_get_seg(head, cate_preds, kernel_preds, seg_pred, img_metas, cfg, rescale=None, img=None, stable=False,
                  autocast=True, half_inter=None):                                                        # :1531-1557
    num_levels = len(cate_preds)
    featmap_size = seg_pred.size()[-2:]
    result_list = []
    for img_id in range(len(img_metas)):
        cate_pred_list = [cate_preds[i][img_id].view(-1, head.cate_out_channels).detach() for i in range(num_levels)]
        seg_pred_list = seg_pred[img_id, ...].unsqueeze(0)
        kernel_pred_list = [kernel_preds[i][img_id].permute(1, 2, 0).view(-1, head.kernel_out_channels).detach()
                            for i in range(num_levels)]
        cate_pred_list = torch.cat(cate_pred_list, dim=0)
        kernel_pred_list = torch.cat(kernel_pred_list, dim=0)
        result_list.append(disco_get_seg_single(head, cate_pred_list, seg_pred_list, kernel_pred_list, featmap_size,
                                                img_metas[img_id], cfg, stable, autocast, half_inter))
    return result_list


def disco_get_seg_single(head, cate_preds, seg_preds, kernel_preds, featmap_size, img_meta, cfg, stable=False,
                         autocast=True, half_inter=None):                                                 # :1559-1660
    """``autocast``: run under ``torch.autocast('cuda', float16)`` as the reference's ``@autocast()`` does (on CPU tensors
    the body runs in float32).  ``half_inter``: compute the intersection matrix in float32 and round it to float16 once,
    instead of leaving the ``torch.mm`` to autocast."""
    on = autocast and seg_preds.is_cuda
    with torch.autocast('cuda', dtype=torch.float16, enabled=on):
        return _disco_body(head, cate_preds, seg_preds, kernel_preds, featmap_size, img_meta, cfg, stable, bool(half_inter))


def _disco_body(head, cate_preds, seg_preds, kernel_preds, featmap_size, img_meta, cfg, stable, half_inter):
    assert len(cate_preds) == len(kernel_preds)
    results = InstanceData(img_meta)
    h, w, _ = results.img_shape
    ori_shape = results.ori_shape
    upsampled_size_out = (featmap_size[0] * 4, featmap_size[1] * 4)
    inds = (cate_preds > cfg.score_thr)
    cate_scores = cate_preds[inds]
    if len(cate_scores) == 0:
        return _empty_results(results, cate_scores)
    inds = inds.nonzero()
    cate_labels = inds[:, 1]
    kernel_preds = kernel_preds[inds[:, 0]]
    strides = _strides(head, cate_labels, kernel_preds, inds)
    I, N = kernel_preds.shape
    kernel_preds = kernel_preds.view(I, N, 1, 1)
    seg_preds = F.conv2d(seg_preds, kernel_preds, stride=1).squeeze(0).sigmoid()
    seg_masks = seg_preds > cfg.mask_thr
    sum_masks = seg_masks.sum((1, 2)).float()
    keep = sum_masks > strides
    if keep.sum() == 0:
        return _empty_results(results, cate_scores)
    seg_masks = seg_masks[keep, ...]
    seg_preds = seg_preds[keep, ...]
    sum_masks = sum_masks[keep]
    cate_scores = cate_scores[keep]
    cate_labels = cate_labels[keep]
    seg_scores = (seg_preds * seg_masks.float()).sum((1, 2)) / sum_masks
    cate_scores *= seg_scores
    if half_inter:              # the mm in float32 (exact integer counts), rounded to float16 once
        with torch.autocast('cuda', dtype=torch.float16, enabled=False):
            scores, labels, _, keep_inds = _nms(seg_masks, cate_labels, cate_scores, sum_masks, cfg, stable, True)
    else:
        scores, labels, _, keep_inds = _nms(seg_masks, cate_labels, cate_scores, sum_masks, cfg, stable, False)
    seg_preds = seg_preds[keep_inds]
    if seg_preds.shape[0] == 0:
        return _empty_results(results, cate_scores)
    seg_preds = F.interpolate(seg_preds.unsqueeze(0), size=upsampled_size_out, mode='bilinear')[:, :, :h, :w]
    seg_masks = F.interpolate(seg_preds, size=ori_shape[:2], mode='bilinear').squeeze(0)
    results.masks = seg_masks > cfg.mask_thr
    results.labels = labels
    results.scores = scores
    return results


def _tap(scale, d, n):
    """ATen's bilinear source tap (align_corners=False) in float32: (i0, 0/1 offset of the second tap, l0, l1)."""
    r = max(scale * (np.float32(d) + np.float32(0.5)) - np.float32(0.5), np.float32(0))
    i0 = int(r)
    l1 = np.float32(r - np.float32(i0))
    return i0, 1 if i0 < n - 1 else 0, np.float32(1) - l1, l1


def _lerp2(ty, tx, v00, v01, v10, v11):
    return ty[2] * (tx[2] * v00 + tx[3] * v01) + ty[3] * (tx[2] * v10 + tx[3] * v11)


def paste_plane(p, img_hw, ori_hw):
    """interpolate(interpolate(p, (4h, 4w))[:H_img, :W_img], (H_ori, W_ori)) of one float32 numpy plane, with ATen's
    upsample_bilinear2d arithmetic restated per output pixel in float32, each product and sum rounded on its own (no fused
    multiply-add).  Torch's CPU kernel agrees to a few units in the last place; this is the reference the host build of the
    paste arithmetic is held to bit for bit."""
    p = np.asarray(p, np.float32)
    h, w = p.shape
    (H_img, W_img), (H_ori, W_ori) = img_hw, ori_hw
    s1h, s1w = np.float32(h) / np.float32(4 * h), np.float32(w) / np.float32(4 * w)
    s2h, s2w = np.float32(H_img) / np.float32(H_ori), np.float32(W_img) / np.float32(W_ori)
    out = np.empty((H_ori, W_ori), np.float32)
    for y in range(H_ori):
        ty2 = _tap(s2h, y, H_img)
        for x in range(W_ori):
            tx2 = _tap(s2w, x, W_img)
            v = []
            for yy in (ty2[0], ty2[0] + ty2[1]):
                ty = _tap(s1h, yy, h)
                for xx in (tx2[0], tx2[0] + tx2[1]):
                    tx = _tap(s1w, xx, w)
                    i, j = ty[0], tx[0]
                    v.append(_lerp2(ty, tx, p[i, j], p[i, j + tx[1]], p[i + ty[1], j], p[i + ty[1], j + tx[1]]))
            out[y, x] = _lerp2(ty2, tx2, *v)
    return out
