"""SOLOv2 inference on the kernels of csrc/solo_seg.cu: per-row mask statistics, Matrix NMS (mmdet/core/post_processing/
matrix_nms.py) and the fused mask paste of get_seg_single (box_solov2_head.py:576-585, discobox_head.py:1645-1653); and
Box2Mask's instance masks on the same paste (maskformer_fusion_head.py:112-241), with their statistics; and the area and
box of finished masks, for the detectors' ``format_results``.

Row sources: the mask rows the kernels read are given as a list of tensors [rows_s, h, w] (float32 or float16, any layout:
made dense here) and addressed by a row id into their concatenation, so that BoxSOLOv2's per-level [B,S^2,h,w] predictions are
read in place, without a gather copy.  ``logits=True``: the rows hold logits and the sigmoid is applied in the kernels as torch
computes it for that dtype.  Thresholds are compared in the rows' dtype, as torch compares a tensor with a Python float."""
import ctypes

import torch

from .. import _lib as L

_DTYPE = {torch.float32: 0, torch.float16: 1}
_KERNEL = {'gaussian': 0, 'linear': 1}
MAX_SOURCES = 8


class RowSources:
    """Tensors [rows_s, h, w] of one dtype and plane size, addressed by row ids into their concatenation."""

    def __init__(self, tensors):
        ts = [t.contiguous() for t in tensors]
        L.require_cuda(*ts)
        if not ts or len(ts) > MAX_SOURCES:
            raise ValueError(f'between 1 and {MAX_SOURCES} row sources, got {len(ts)}')
        if len({t.dtype for t in ts}) != 1 or ts[0].dtype not in _DTYPE:
            raise TypeError(f'row sources must all be float32 or all float16, got {[t.dtype for t in ts]}')
        if len({tuple(t.shape[1:]) for t in ts}) != 1:
            raise ValueError('row sources must share one plane size')
        self.tensors = ts
        self.h, self.w = int(ts[0].shape[1]), int(ts[0].shape[2])
        self.dtype = ts[0].dtype
        self.device = ts[0].device
        self.ptrs = (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])
        self.rows = (ctypes.c_int64 * len(ts))(*[int(t.shape[0]) for t in ts])


def mask_stats(src, rows, mask_thr, logits=False):
    """(bits int32 [n, ceil(h*w/32)] -- the packed masks p > mask_thr, area int32 [n], masked sum float32 [n]) of the rows
    ``rows`` (int64 ids) of ``src``."""
    rows = rows.to(device=src.device, dtype=torch.int64).contiguous()
    n, hw = rows.numel(), src.h * src.w
    words = -(-hw // 32)
    bits = torch.empty((n, words), dtype=torch.int32, device=src.device)
    area = torch.empty(n, dtype=torch.int32, device=src.device)
    msum = torch.empty(n, dtype=torch.float32, device=src.device)
    with torch.cuda.device(src.device):
        L.check(L.lib().bxs_solo_mask_stats(src.ptrs, src.rows, len(src.tensors), hw, _DTYPE[src.dtype], int(logits),
                                            L.ptr(rows), n, float(mask_thr), L.ptr(bits), L.ptr(area), L.ptr(msum),
                                            L.stream()), 'solo_mask_stats')
    return bits, area, msum


def matrix_nms_sorted(bits, row, label, area, score, n_valid, kernel='gaussian', sigma=2.0, filter_thr=-1.0,
                      half_inter=False):
    """Matrix NMS of B images of N score-sorted candidate slots each ([B,N] row ids into ``bits``, labels, float32 areas and
    scores; ``n_valid`` [B] device counts of the valid leading slots) -> [B,N] float32 decayed scores, -inf for an invalid
    or filtered slot."""
    if kernel not in _KERNEL:
        raise NotImplementedError(f'{kernel} kernel is not supported in matrix nms!')
    B, N = score.shape
    out = torch.empty((B, N), dtype=torch.float32, device=score.device)
    if B * N == 0:
        return out
    args = [t.contiguous() for t in (row.long(), label.long(), area.float(), score.float(), n_valid.long())]
    bits = bits.contiguous()
    L.require_cuda(bits, *args)
    with torch.cuda.device(score.device):
        ws = torch.empty(L.lib().bxs_matrix_nms_workspace_bytes(B, N), dtype=torch.uint8, device=score.device)
        L.check(L.lib().bxs_matrix_nms(L.ptr(bits), bits.shape[1], *[L.ptr(t) for t in args], B, N, _KERNEL[kernel],
                                       float(sigma), float(filter_thr), int(half_inter), L.ptr(ws), L.ptr(out), L.stream()),
                'matrix_nms')
    return out


def paste_rows(src, rows, img_hw, ori_hw, mask_thr, logits=False, interp_f32=False):
    """bool [n, H_ori, W_ori] = interpolate(interpolate(p, (4h, 4w))[:H_img, :W_img], (H_ori, W_ori)) > mask_thr for the
    rows ``rows`` of ``src`` (bilinear, align_corners=False), in one pass.  ``interp_f32``: float16 probabilities are
    interpolated and compared in float32, as under ``torch.autocast`` (which runs upsample_bilinear2d in float32)."""
    rows = rows.to(device=src.device, dtype=torch.int64).contiguous()
    n = rows.numel()
    (H_img, W_img), (H_ori, W_ori) = [int(v) for v in img_hw[:2]], [int(v) for v in ori_hw[:2]]
    out = torch.empty((n, H_ori, W_ori), dtype=torch.bool, device=src.device)
    with torch.cuda.device(src.device):
        L.check(L.lib().bxs_solo_paste_masks(src.ptrs, src.rows, len(src.tensors), src.h, src.w, _DTYPE[src.dtype],
                                             int(logits), int(interp_f32), L.ptr(rows), n, H_img, W_img, H_ori, W_ori, float(mask_thr),
                                             L.ptr(out), L.stream()), 'solo_paste_masks')
    return out


def maskformer_paste_rows(src, rows, pad_hw, img_hw, ori_hw=None):
    """MaskFormer's instance masks of the LOGIT rows ``rows`` of ``src`` and their statistics, in one pass: masks bool
    [n, H, W] = interpolate(interpolate(x, pad_hw)[:H_img, :W_img], ori_hw) > 0 (bilinear, align_corners=False; a stage
    whose sizes match is skipped, so ``ori_hw=None`` gives the crop at ``img_hw``), area int32 [n], masked_sum float32 [n]
    (the sum of sigmoid over the set pixels) and box float32 [n, 4] (mask2bbox).  Two launches, no host read."""
    rows = rows.to(device=src.device, dtype=torch.int64).contiguous()
    n = rows.numel()
    (H_pad, W_pad), (H_img, W_img) = [int(v) for v in pad_hw[:2]], [int(v) for v in img_hw[:2]]
    H_out, W_out = (H_img, W_img) if ori_hw is None else [int(v) for v in ori_hw[:2]]
    dev = src.device
    out = torch.empty((n, H_out, W_out), dtype=torch.bool, device=dev)
    area = torch.empty(n, dtype=torch.int32, device=dev)
    msum = torch.empty(n, dtype=torch.float32, device=dev)
    box = torch.empty((n, 4), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws = torch.empty(L.lib().bxs_maskformer_paste_workspace_bytes(n), dtype=torch.uint8, device=dev)
        L.check(L.lib().bxs_maskformer_paste_masks(src.ptrs, src.rows, len(src.tensors), src.h, src.w, _DTYPE[src.dtype],
                                                   L.ptr(rows), n, H_pad, W_pad, H_img, W_img, int(ori_hw is not None),
                                                   H_out, W_out, L.ptr(ws), L.ptr(out), L.ptr(area), L.ptr(msum),
                                                   L.ptr(box), L.stream()), 'maskformer_paste_masks')
    return out, area, msum, box


def mask_extents(masks):
    """(area int32 [n], box float32 [n, 4]) of bool or uint8 masks [n, H, W]: each mask's count of set (non-zero) pixels and
    [x_min, y_min, x_max + 1, y_max + 1] of them, zeros for an empty mask.  Two launches, no host read."""
    if masks.dtype not in (torch.bool, torch.uint8):
        raise TypeError(f'masks must be bool or uint8, got {masks.dtype}')
    if masks.dim() != 3:
        raise ValueError(f'masks must be [n, H, W], got {tuple(masks.shape)}')
    masks = masks.contiguous()
    L.require_cuda(masks)
    n, H, W = masks.shape
    dev = masks.device
    area = torch.empty(n, dtype=torch.int32, device=dev)
    box = torch.empty((n, 4), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        ws = torch.empty(L.lib().bxs_mask_extents_workspace_bytes(n, H, W), dtype=torch.uint8, device=dev)
        L.check(L.lib().bxs_mask_extents(L.ptr(masks), n, H, W, L.ptr(ws), L.ptr(area), L.ptr(box), L.stream()),
                'mask_extents')
    return area, box


def paste_masks(rows, featmap_size, img_shape, ori_shape, mask_thr):
    """The mask paste of get_seg_single on its own: rows [n,h,w] probabilities (float32 or float16) with (h, w) ==
    featmap_size -> bool [n, H_ori, W_ori] = interpolate(interpolate(rows, (4h, 4w))[:, :H_img, :W_img], ori_shape[:2]) >
    mask_thr, bit for bit what ATen computes for that dtype (16-bit rows are rounded after each stage)."""
    if tuple(int(s) for s in featmap_size) != tuple(rows.shape[-2:]):
        raise ValueError(f'featmap_size {tuple(featmap_size)} is not the rows\' plane size {tuple(rows.shape[-2:])}')
    src = RowSources([rows])
    return paste_rows(src, torch.arange(rows.shape[0], device=src.device), img_shape, ori_shape, mask_thr)


def mask_matrix_nms(masks, labels, scores, filter_thr=-1, nms_pre=-1, max_num=-1, kernel='gaussian', sigma=2.0,
                    mask_area=None):
    """mmdet's ``mask_matrix_nms`` (matrix_nms.py:5-121): same signature, same 4-tuple (scores, labels, masks, keep_inds).
    ``masks`` [n,h,w] boolean (non-zero = set) are bit-packed on the device; both sorts are stable (equal scores keep the
    input order).  One host read: the number of masks kept, which sizes the outputs."""
    if kernel not in _KERNEL:
        raise NotImplementedError(f'{kernel} kernel is not supported in matrix nms!')
    assert len(labels) == len(masks) == len(scores)
    L.require_cuda(*[t.contiguous() for t in (masks, labels, scores)])
    empty = (scores.new_zeros(0), labels.new_zeros(0), masks.new_zeros(0, *masks.shape[-2:]), labels.new_zeros(0))
    n = len(labels)
    if n == 0:
        return empty
    dev = scores.device
    h, w = masks.shape[-2:]
    src = RowSources([(masks != 0).to(torch.float16).reshape(n, h, w)])
    bits, area, _ = mask_stats(src, torch.arange(n, device=dev), 0.5)
    mask_area = area.float() if mask_area is None else mask_area.float()
    sorted_scores, sort_inds = torch.sort(scores, descending=True, stable=True)
    N = min(nms_pre, n) if nms_pre > 0 else n
    sort_inds = sort_inds[:N]
    n_valid = torch.full((1,), N, dtype=torch.int64, device=dev)
    out = matrix_nms_sorted(bits, sort_inds[None], labels[sort_inds][None], mask_area[sort_inds][None],
                            sorted_scores[:N][None].float(), n_valid, kernel, sigma, filter_thr)[0]
    out = out.to(torch.promote_types(scores.dtype, torch.float32))
    s2, o2 = torch.sort(out, descending=True, stable=True)
    M = min(max_num, N) if max_num > 0 else N
    kept = int((s2[:M] > float('-inf')).sum())          # the one host read
    if kept == 0:
        return empty
    keep_inds = sort_inds[o2[:kept]]
    return s2[:kept], labels[keep_inds], masks[keep_inds], keep_inds
