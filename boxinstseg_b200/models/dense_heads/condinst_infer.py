"""CondInst inference for the whole batch: CondInstBoxHead.get_bboxes (condinst_head.py:640-853 with nms_with_others :18-83)
and CondInstMaskHead.simple_test (:1234-1286).

get_bboxes:
  1. ``bxs_condinst_point_scores``: the key the per-level top-k ranks, read in place from every level's predictions;
  2. a stable descending sort of each level's keys (the top-k; equal keys: the lower point first);
  3. ``bxs_condinst_decode``: boxes, sigmoid(centerness), and per class the candidate flag and score of every kept point;
  4. the candidates in the reference's order (image, level, top-k rank, class), batched_nms's offset boxes, one sort into
     (image, class) segments by descending score, ``bxs_box_nms`` for every image and class at once;
  5. a stable descending sort of each image's kept candidates, the cut at ``max_per_img`` and ``bxs_condinst_gather`` of
     the parameters, points and levels of the detections.
Two device-to-host reads per call, whatever the batch and the candidate counts: the per-(image, class) candidate counts
(which size the candidate buffers and the NMS workspace) and the kept counts (which size the outputs)."""
import ctypes

import numpy as np
import torch

from ... import _lib as L
from ...ops.box_nms import _nms_threshold, segment_nms
from ...ops.condinst import paste_masks


def cfg_get(cfg, key, default=None):
    if isinstance(cfg, dict):
        return cfg.get(key, default)
    return getattr(cfg, key, default)


class _Levels:
    """The level table's host arrays for a list of per-level [B,c,H,W] float32 tensors (any strides)."""

    def __init__(self, tensors):
        self.tensors = tensors
        n = len(tensors)
        self.ptrs = (ctypes.c_void_p * n)(*[t.data_ptr() for t in tensors])
        self.strides = (ctypes.c_int64 * (4 * n))(*[s for t in tensors for s in t.stride()])


def _f32(ts):
    """force_fp32: float16 / bfloat16 predictions promoted to float32; float32 ones read as they lie."""
    return [t.detach() if t.dtype == torch.float32 else t.detach().float() for t in ts]


def get_bboxes(cls_scores, bbox_preds, centernesses, param_preds, img_metas, cfg, strides, rescale=False, with_nms=True):
    assert len(cls_scores) == len(bbox_preds) == len(centernesses) == len(param_preds)
    cls, bbox, ctr, prm = _f32(cls_scores), _f32(bbox_preds), _f32(centernesses), _f32(param_preds)
    L.require_cuda(*[t.contiguous() for t in cls[:1]])
    n_lv = len(cls)
    B, C = int(cls[0].shape[0]), int(cls[0].shape[1])
    P = int(prm[0].shape[1])
    dev = cls[0].device
    sizes = [(int(t.shape[-2]), int(t.shape[-1])) for t in cls]
    hw = [h * w for h, w in sizes]
    nms_pre = int(cfg_get(cfg, 'nms_pre', -1))
    k = [nms_pre if 0 < nms_pre < n else n for n in hw]                 # get_k_for_topk: no top-k -> every point in order
    S, P_max = sum(k), max(hw)
    i64 = lambda v: (ctypes.c_int64 * n_lv)(*v)
    Hs, Ws, ks = i64([h for h, _ in sizes]), i64([w for _, w in sizes]), i64(k)
    st = (ctypes.c_float * n_lv)(*[float(s[0] if isinstance(s, (tuple, list)) else s) for s in strides])
    lc, lt, lb, lp = _Levels(cls), _Levels(ctr), _Levels(bbox), _Levels(prm)
    lib = L.lib()
    with torch.cuda.device(dev):
        order = None
        if any(kk < n for kk, n in zip(k, hw)):
            key = torch.empty((B, n_lv, P_max), dtype=torch.float32, device=dev)
            L.check(lib.bxs_condinst_point_scores(lc.ptrs, lc.strides, lt.ptrs, lt.strides, Hs, Ws, n_lv, B, C, P_max,
                                                  L.ptr(key), L.stream()), 'condinst_point_scores')
            order = torch.sort(key, dim=-1, descending=True, stable=True)[1]
        img_hw = (ctypes.c_float * (2 * B))(*[float(v) for m in img_metas for v in m['img_shape'][:2]])
        scale = None
        if rescale:
            sf = [np.broadcast_to(np.asarray(m['scale_factor'], dtype=np.float32).reshape(-1), (4,)) for m in img_metas]
            scale = (ctypes.c_float * (4 * B))(*[float(v) for s in sf for v in s])
        box = torch.empty((B, S, 4), dtype=torch.float32, device=dev)
        ctr_s = torch.empty((B, S), dtype=torch.float32, device=dev)
        point = torch.empty((B, S), dtype=torch.int64, device=dev)
        cand = torch.empty((B, S, C), dtype=torch.bool, device=dev)
        score = torch.empty((B, S, C), dtype=torch.float32, device=dev)
        sig = None if with_nms else torch.empty((B, S, C), dtype=torch.float32, device=dev)
        L.check(lib.bxs_condinst_decode(lc.ptrs, lc.strides, lt.ptrs, lt.strides, lb.ptrs, lb.strides, Hs, Ws, st, ks, n_lv, B,
                                        C, L.ptr(order), P_max, img_hw, scale, float(cfg_get(cfg, 'score_thr')), L.ptr(box),
                                        L.ptr(ctr_s), L.ptr(point), L.ptr(cand), L.ptr(score), L.ptr(sig), L.stream()),
                'condinst_decode')

        def gather(rows):
            n = rows.numel()
            params = torch.empty((n, P), dtype=torch.float32, device=dev)
            coors = torch.empty((n, 2), dtype=torch.float32, device=dev)
            level = torch.empty(n, dtype=torch.int64, device=dev)
            L.check(lib.bxs_condinst_gather(lp.ptrs, lp.strides, Hs, Ws, st, ks, n_lv, B, P, L.ptr(point), L.ptr(rows), n,
                                            L.ptr(params), L.ptr(coors), L.ptr(level), L.stream()), 'condinst_gather')
            return params.to(param_preds[0].dtype), coors, level      # params keep their dtype (no force_fp32 there)

        if not with_nms:
            params, coors, level = gather(torch.arange(B * S, device=dev))
            scores = torch.cat([sig, sig.new_zeros(B, S, 1)], -1)
            return list(zip(box, scores, ctr_s, params.view(B, S, P), coors.view(B, S, 2), level.view(B, S)))

        thr = _nms_threshold(cfg_get(cfg, 'nms'), False)
        max_num = int(cfg_get(cfg, 'max_per_img', -1))
        seg_counts_dev = cand.sum(1).flatten()                          # [B*C] candidates per (image, class)
        seg_counts = seg_counts_dev.tolist()                            # host read 1
        img_counts = [sum(seg_counts[b * C:(b + 1) * C]) for b in range(B)]
        K = sum(img_counts)
        if K == 0:
            return [_empty(P, param_preds[0].dtype, dev) for _ in range(B)]
        flat = torch.nonzero_static(cand.view(-1), size=K).squeeze(1)  # (image, slot, class) order
        slot, label = flat // C, flat % C
        img = slot // S
        cand_score = score.view(-1)[flat]
        cand_box = box.view(-1, 4)[slot]
        # batched_nms's offset boxes, per image over that image's candidates (mmcv's lines)
        first = np.concatenate([[0], np.cumsum(img_counts)]).tolist()
        max_coord = torch.stack([cand_box[first[b]:first[b + 1]].max() if img_counts[b] else cand_box.new_zeros(())
                                 for b in range(B)])
        offsets = label.to(cand_box) * (max_coord[img] + 1)         # mmcv's + torch.tensor(1): the same fp32 sum, no copy
        boxes_for_nms = cand_box + offsets[:, None]
        order = torch.sort(cand_score, descending=True, stable=True)[1]
        order = order[torch.sort((img * C + label)[order], stable=True)[1]]
        keep_sorted = segment_nms(boxes_for_nms[order], seg_counts_dev, seg_counts, thr)
        keep = torch.zeros(K, dtype=torch.bool, device=dev).index_put_((order,), keep_sorted)
        # per image, kept candidates by descending score, equal scores in candidate order
        K_max = max(img_counts)
        img_counts_dev = seg_counts_dev.view(B, C).sum(1)
        pos = torch.arange(K, device=dev) - (torch.cumsum(img_counts_dev, 0) - img_counts_dev)[img]
        padded = torch.full((B, K_max), float('-inf'), device=dev).index_put_((img, pos), cand_score.masked_fill(~keep, float('-inf')))
        kept_pad = torch.zeros((B, K_max), dtype=torch.bool, device=dev).index_put_((img, pos), keep)
        cand_of = torch.zeros((B, K_max), dtype=torch.int64, device=dev).index_put_((img, pos), torch.arange(K, device=dev))
        s2, o2 = torch.sort(padded, dim=1, descending=True, stable=True)
        n_kept = kept_pad.sum(1)
        if max_num > 0:
            n_kept = n_kept.clamp(max=max_num)
        n_kept = n_kept.tolist()                                        # host read 2
        sel = torch.cat([cand_of[b].gather(0, o2[b, :n]) for b, n in enumerate(n_kept)])
        params, coors, level = gather(slot[sel])
        dets = torch.cat([cand_box[sel], cand_score[sel][:, None]], -1)
        out = zip(dets.split(n_kept), label[sel].split(n_kept), params.split(n_kept), coors.split(n_kept), level.split(n_kept))
        return [tuple(o) for o in out]


def _empty(P, param_dtype, dev):
    return (torch.zeros((0, 5), device=dev), torch.zeros(0, dtype=torch.int64, device=dev),
            torch.zeros((0, P), dtype=param_dtype, device=dev), torch.zeros((0, 2), device=dev), torch.zeros(0, dtype=torch.int64, device=dev))


def simple_test(head, mask_feat, det_labels, det_params, det_coors, det_level_inds, img_metas, num_classes, rescale=False):
    """The dynamic head once for every detection of the batch, the fused paste per image, then ONE host copy of each image's
    masks and labels, split per class on the host into the reference's uint8 numpy masks."""
    num_imgs = len(img_metas)
    num_inst = [int(p.size(0)) for p in det_params]
    if sum(num_inst) == 0:
        return [[[] for _ in range(num_classes)] for _ in range(num_imgs)]
    dev = mask_feat.device
    img_inds = torch.cat([torch.full((n,), i, dtype=torch.long, device=dev) for i, n in enumerate(num_inst)])
    logits = head.forward(mask_feat, torch.cat(det_params), torch.cat(det_coors), torch.cat(det_level_inds), img_inds)
    masks = []
    for logit, meta in zip(logits.split(num_inst), img_metas):
        masks.append(paste_masks(logit, head.out_stride, meta['img_shape'], meta['ori_shape'] if rescale else None)
                     if logit.shape[0] else None)
    segm_results = []
    for m, labels in zip(masks, det_labels):
        if m is None:                       # the reference appends an entry here and falls through (see INTEGRATION.md)
            segm_results.append([[] for _ in range(num_classes)])
            continue
        m = m.cpu().numpy().view(np.uint8)
        labels = labels.detach().cpu().numpy()
        segm_results.append([m[labels == i] for i in range(num_classes)])
    return segm_results
