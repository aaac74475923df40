"""Greedy box NMS per (image, class) on the kernels of csrc/condinst_infer.cu: mmcv's ``batched_nms`` with ``type='nms'``.

mmcv separates the classes by offsetting every box by ``label * (max_coordinate + 1)`` and runs one NMS on the result;
its CUDA test is ``interS > iou_threshold * (Sa + Sb - interS)`` (offset 0).  Here the candidates are sorted into (image,
class) segments, each by descending score with ties in input order, the suppression bits are computed only inside a
segment (cost and workspace grow with the sum of n_s^2, not with (sum n_s)^2) and the greedy pass runs on the device.  The
offset boxes are kept, because the offset changes how the IoU rounds."""
import ctypes

import torch

from .. import _lib as L


def segment_nms(boxes_sorted, counts, counts_host, iou_thr):
    """Greedy NMS of N offset boxes [N,4] float32 sorted into segments of ``counts`` (int64 device tensor, one per segment;
    ``counts_host`` the same values on the host), each in descending score order -> keep bool [N] in that order."""
    N = boxes_sorted.shape[0]
    keep = torch.zeros(N, dtype=torch.uint8, device=boxes_sorted.device)
    if N == 0:
        return keep.bool()
    boxes_sorted = L.dense_aligned(boxes_sorted.float())
    counts = counts.to(torch.int64)
    seg_start = torch.cat([counts.new_zeros(1), torch.cumsum(counts, 0)])
    words = (counts + 63) // 64 * counts
    mask_off = torch.cumsum(words, 0) - words
    host = (ctypes.c_int64 * len(counts_host))(*counts_host)
    lib = L.lib()
    nbytes = lib.bxs_box_nms_workspace_bytes(host, len(counts_host))
    ws = torch.empty(max(nbytes, 8), dtype=torch.uint8, device=boxes_sorted.device)
    with torch.cuda.device(boxes_sorted.device):
        L.check(lib.bxs_box_nms(L.ptr(boxes_sorted), L.ptr(seg_start), L.ptr(mask_off), N, len(counts_host), max(counts_host),
                                float(iou_thr), L.ptr(ws), L.ptr(keep), L.stream()), 'box_nms')
    return keep.bool()


def _nms_threshold(nms_cfg, class_agnostic):
    cfg = dict(nms_cfg)
    if cfg.pop('class_agnostic', class_agnostic):
        raise NotImplementedError('batched_nms: class_agnostic is not supported')
    kind = cfg.pop('type', 'nms')
    if kind != 'nms':
        raise NotImplementedError(f'batched_nms: type {kind!r} is not supported')
    cfg.pop('split_thr', None)                  # both sorts are stable: the per-class branch would give the same result
    thr = cfg.pop('iou_threshold')
    if cfg.pop('offset', 0) != 0 or cfg:
        raise NotImplementedError(f'batched_nms: unsupported settings {cfg}')
    return float(thr)


def batched_nms(boxes, scores, idxs, nms_cfg, class_agnostic=False):
    """mmcv's ``batched_nms`` (mmcv/ops/nms.py) for ``type='nms'``: same signature, same ``(dets [k,5], keep [k])``.
    ``keep`` is ordered by descending score, equal scores in input order; ``split_thr`` is accepted and changes nothing.
    Other NMS types and ``class_agnostic=True`` raise NotImplementedError."""
    thr = _nms_threshold(nms_cfg, class_agnostic)
    L.require_cuda(boxes.contiguous(), scores.contiguous(), idxs.contiguous())
    if boxes.dtype != torch.float32:
        raise TypeError(f'batched_nms: boxes must be float32, got {boxes.dtype}')
    if boxes.shape[0] == 0:
        return torch.cat([boxes, scores[:, None]], -1), idxs.new_zeros(0, dtype=torch.int64)
    max_coordinate = boxes.max()                                   # mmcv's lines: the offset trick
    offsets = idxs.to(boxes) * (max_coordinate + 1)               # mmcv adds torch.tensor(1): the same fp32 sum
    boxes_for_nms = boxes + offsets[:, None]
    order = torch.sort(scores, descending=True, stable=True)[1]
    order = order[torch.sort(idxs[order], stable=True)[1]]
    _, counts = torch.unique_consecutive(idxs[order], return_counts=True)
    keep_sorted = segment_nms(boxes_for_nms[order], counts, counts.tolist(), thr)
    kept = torch.sort(order[keep_sorted])[0]                       # input order, so that the stable sort keeps it for ties
    s, o = torch.sort(scores[kept], descending=True, stable=True)
    keep = kept[o]
    return torch.cat([boxes[keep], s[:, None]], -1), keep
