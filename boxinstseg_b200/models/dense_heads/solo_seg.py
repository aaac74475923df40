"""SOLOv2 inference shared by BoxSOLOv2Head.get_seg (box_solov2_head.py:475-590) and DiscoBoxSOLOv2Head.get_seg
(discobox_head.py:1531-1660): the reference's per-image ``get_seg_single`` for the whole batch at once.

  1. candidates ``cate > score_thr`` of every image; the distinct candidate rows (level, image, cell) -- a cell above the
     threshold for several classes is one row;
  2. the rows' packed masks, areas and masked sums (``bxs_solo_mask_stats``; BoxSOLOv2 reads its per-level predictions in
     place, DiscoBox convolves each distinct cell once);
  3. the stride filter and mask scores per candidate, one stable descending sort per image with invalid slots at -inf,
     Matrix NMS for every image in one call (``bxs_matrix_nms``), a second stable sort;
  4. per image, the fused paste of the kept masks (``bxs_solo_paste_masks``).

Two device-to-host reads per call, whatever the batch and the candidate counts: the candidate counts (which size
``nonzero_static``) and the kept counts (which size the outputs).  Everything between is padded per image."""
import types

import torch

from ...ops import solo_seg as S
from ...ops.dynconv import PACK_MAX_ROWS, _CellPack, dynconv1x1, row_chunks

try:                                            # pragma: no cover - mmdet is absent in this image
    from mmdet.core import InstanceData
except ImportError:
    InstanceData = None


def cfg_get(cfg, key):
    return cfg[key] if isinstance(cfg, dict) else getattr(cfg, key)


def _results(img_meta):
    return InstanceData(img_meta) if InstanceData is not None else types.SimpleNamespace(**img_meta)


def _empty_results(results, like):
    """empty_results of get_seg_single (box_solov2_head.py:509-513): float tensors in the category scores' dtype."""
    results.scores = like.new_ones(0)
    results.masks = like.new_zeros(0, *results.ori_shape[:2])
    results.labels = like.new_ones(0)
    return results


class Candidates:
    """The candidates of a batch and their distinct rows, after the one host read of the candidate counts.

    rows are ordered level-major, then image-major, then by cell; ``row_level`` / ``row_img`` / ``row_cell`` describe them,
    ``seg_counts[l][b]`` counts those of (level, image).  Candidates are ordered as the reference's ``nonzero`` orders them
    per image, images in turn: ``cand_img``, ``cand_label``, ``cand_score`` (category dtype), ``cand_row`` (index into the
    distinct rows), ``cand_stride`` (float32); ``img_counts[b]`` per image."""

    def __init__(self, cate_preds, grids, strides, score_thr):
        n_lv = len(cate_preds)
        B, C = cate_preds[0].shape[0], cate_preds[0].shape[-1]
        dev = cate_preds[0].device
        sq = [g * g for g in grids]
        cate = torch.cat([c.reshape(B, s, C) for c, s in zip(cate_preds, sq)], 1)            # [B, P, C]
        P = cate.shape[1]
        cand = cate > score_thr
        cell_any = cand.any(2)                                                                # [B, P]
        off = [sum(sq[:l]) for l in range(n_lv + 1)]
        per_lv = [cell_any[:, off[l]:off[l + 1]] for l in range(n_lv)]
        counts = torch.cat([torch.stack([p.sum(1) for p in per_lv]).flatten(), cand.flatten(1).sum(1)])
        counts = counts.tolist()                                                              # host read 1
        self.seg_counts = [counts[l * B:(l + 1) * B] for l in range(n_lv)]
        self.img_counts = counts[n_lv * B:]
        R, K = sum(counts[:n_lv * B]), sum(self.img_counts)
        self.B, self.C, self.n_rows, self.n_cand, self.device, self.dtype = B, C, R, K, dev, cate.dtype
        # distinct rows: positions in the level-major (level, image, cell) concatenation
        mask_cat = torch.cat([p.reshape(-1) for p in per_lv])
        pos = torch.nonzero_static(mask_cat, size=R).squeeze(1)
        self.row_pos = pos
        lv_of = torch.cat([torch.full((B * s,), l, dtype=torch.int64, device=dev) for l, s in enumerate(sq)])
        idx_in = torch.cat([torch.arange(B * s, device=dev) for s in sq])
        sq_of = torch.cat([torch.full((B * s,), s, dtype=torch.int64, device=dev) for s in sq])
        self.row_level = lv_of[pos]
        self.row_img = idx_in[pos] // sq_of[pos]
        self.row_cell = idx_in[pos] % sq_of[pos]
        row_id = torch.cumsum(mask_cat, 0) - 1
        starts = [B * o for o in off]
        row_of = torch.cat([row_id[starts[l]:starts[l + 1]].view(B, s) for l, s in enumerate(sq)], 1)    # [B, P]
        # candidates, per image in the reference's (cell, class) order
        flat = torch.nonzero_static(cand.reshape(-1), size=K).squeeze(1)
        b, rem = flat // (P * C), flat % (P * C)
        p = rem // C
        self.cand_img, self.cand_label = b, rem % C
        self.cand_score = cate.reshape(-1)[flat]
        self.cand_row = row_of.reshape(-1)[b * P + p]
        stride_of = torch.cat([torch.full((s,), float(st), device=dev) for s, st in zip(sq, strides)])
        self.cand_stride = stride_of[p]


def _disco_sources(cands, kernel_preds, seg_pred):
    """DiscoBox's candidate convolution: every distinct cell once, packed per image (``bxs_disco_cells_pack``, at most
    PACK_MAX_ROWS rows per image and call: ``row_chunks``) and convolved by ``dynconv1x1`` under the caller's autocast.
    Returns the row sources (one [B*I_pad, h, w] logit tensor per chunk) and the source row id of every distinct row."""
    B, n_lv = cands.B, len(kernel_preds)
    dev = seg_pred.device
    h, w = seg_pred.shape[-2:]
    seg_start = [0]
    for l in range(n_lv):
        for b in range(B):
            seg_start.append(seg_start[-1] + cands.seg_counts[l][b])
    chunks = row_chunks(cands.seg_counts)
    if len(chunks) > S.MAX_SOURCES:
        raise NotImplementedError(f'DiscoBoxSOLOv2Head.get_seg: more than {S.MAX_SOURCES * PACK_MAX_ROWS} distinct '
                                  'candidate cells in one image')
    dt = kernel_preds[0].dtype if kernel_preds[0].dtype in (torch.float32, torch.float16, torch.bfloat16) else torch.float32
    grids = [k.detach().to(dt).contiguous() for k in kernel_preds]
    cells = cands.row_cell.to(torch.int32)
    sources, src_start = [], 0
    pieces = []                                   # (distinct-row start, length, source id base) of every sub-range
    for i_pad, counts, parts in chunks:
        cell_parts = []
        for l, b, j, n, r in parts:
            r0 = seg_start[l * B + b] + j
            cell_parts.append(cells[r0:r0 + n])
            pieces.append((r0, n, src_start + b * i_pad + r))
        packed = _CellPack.apply(counts, i_pad, torch.cat(cell_parts), *grids)
        logits = dynconv1x1(seg_pred.detach(), packed)                                      # [B, i_pad, h, w]
        sources.append(logits.reshape(B * i_pad, h, w))
        src_start += B * i_pad
    pieces.sort()
    ids = torch.cat([torch.arange(n, device=dev) + base for _, n, base in pieces])
    return sources, ids


def get_seg(cate_preds, grids, strides, img_metas, cfg, sources_of):
    """The batch body.  ``sources_of(cands)`` -> (row tensors [n_s,h,w], source row id of every distinct row, logits?)."""
    score_thr, mask_thr = cfg_get(cfg, 'score_thr'), cfg_get(cfg, 'mask_thr')
    nms_pre, max_num = cfg_get(cfg, 'nms_pre'), cfg_get(cfg, 'max_per_img')
    kernel, sigma, filter_thr = cfg_get(cfg, 'kernel'), cfg_get(cfg, 'sigma'), cfg_get(cfg, 'filter_thr')
    if kernel not in S._KERNEL:
        raise NotImplementedError(f'{kernel} kernel is not supported in matrix nms!')
    cands = Candidates(cate_preds, grids, strides, score_thr)
    B, dev = cands.B, cands.device
    results = [_results(m) for m in img_metas]
    if cands.n_cand == 0:
        return [_empty_results(r, cands.cand_score) for r in results]
    tensors, src_ids, logits, half_inter = sources_of(cands)
    src = S.RowSources(tensors)
    bits, area, msum = S.mask_stats(src, src_ids, mask_thr, logits)

    # per candidate (box_solov2_head.py:541-561): stride filter, mask score
    a = area.float()[cands.cand_row]
    keep = a > cands.cand_stride
    seg_score = msum[cands.cand_row] / a
    score = (cands.cand_score.float() * seg_score).to(cands.dtype)                  # cate_scores *= seg_scores
    # padded per image, filtered slots at -inf; stable sorts keep the reference's candidate order among equal scores
    K_max = max(cands.img_counts)
    first = [sum(cands.img_counts[:b]) for b in range(B)]
    slot = torch.arange(cands.n_cand, device=dev) - torch.cat(
        [torch.full((n,), f, dtype=torch.int64, device=dev) for n, f in zip(cands.img_counts, first)])
    padded = torch.full((B, K_max), float('-inf'), device=dev)
    padded.index_put_((cands.cand_img, slot), torch.where(keep, score.float(), float('-inf')))
    cand_of = torch.zeros((B, K_max), dtype=torch.int64, device=dev)
    cand_of.index_put_((cands.cand_img, slot), torch.arange(cands.n_cand, device=dev))
    s1, o1 = torch.sort(padded, dim=1, descending=True, stable=True)
    N = min(nms_pre, K_max) if nms_pre > 0 else K_max
    s1, slot_cand = s1[:, :N].contiguous(), cand_of.gather(1, o1[:, :N])
    n_valid = (s1 > float('-inf')).sum(1)
    decayed = S.matrix_nms_sorted(bits, cands.cand_row[slot_cand], cands.cand_label[slot_cand], a[slot_cand], s1, n_valid,
                                  kernel, sigma, filter_thr, half_inter)
    s2, o2 = torch.sort(decayed, dim=1, descending=True, stable=True)
    M = min(max_num, N) if max_num > 0 else N
    kept = (s2[:, :M] > float('-inf')).sum(1).tolist()                                # host read 2
    out = []
    for b, r in enumerate(results):
        n = kept[b]
        if n == 0:
            out.append(_empty_results(r, cands.cand_score))
            continue
        cand = slot_cand[b].gather(0, o2[b, :n])
        r.masks = S.paste_rows(src, src_ids[cands.cand_row[cand]], r.img_shape, r.ori_shape, mask_thr, logits,
                               interp_f32=torch.is_autocast_enabled('cuda'))
        r.labels = cands.cand_label[cand]
        r.scores = s2[b, :n]
        out.append(r)
    return out


def box_solov2_get_seg(seg_preds, cate_preds, strides, img_metas, cfg):
    """BoxSOLOv2Head: ``seg_preds`` per level [B,S^2,h,w] probabilities (``forward(eval=True)``), read in place."""
    assert len(seg_preds) == len(cate_preds)
    grids = [int(c.shape[1]) for c in cate_preds]
    dt = seg_preds[0].dtype if len({p.dtype for p in seg_preds}) == 1 and seg_preds[0].dtype in S._DTYPE else torch.float32

    def sources_of(cands):
        tensors = [p.detach().to(dt).reshape(-1, *p.shape[-2:]) for p in seg_preds]
        return tensors, cands.row_pos, False, False
    return get_seg(cate_preds, grids, strides, img_metas, cfg, sources_of)


def discobox_get_seg(cate_preds, kernel_preds, seg_pred, strides, img_metas, cfg, autocast=True):
    """DiscoBoxSOLOv2Head: the distinct candidate cells of ``kernel_preds`` (per level [B,E,S,S]) convolved with
    ``seg_pred`` [B,E,h,w] once each.  ``autocast``: under float16 autocast, as the reference's ``@autocast()`` runs
    get_seg_single: float16 logits, the intersection counts rounded to float16 as its ``torch.mm`` rounds them, the paste
    interpolated in float32; ``autocast=False`` runs the same lines in float32."""
    grids = [int(c.shape[1]) for c in cate_preds]

    def sources_of(cands):
        tensors, ids = _disco_sources(cands, kernel_preds, seg_pred)
        return tensors, ids, True, autocast
    with torch.autocast('cuda', dtype=torch.float16, enabled=autocast):
        return get_seg(cate_preds, grids, strides, img_metas, cfg, sources_of)
