"""Oracle of CondInst inference: CondInstBoxHead.get_bboxes / _get_bboxes (condinst_head.py:640-853), nms_with_others
(:18-83), CondInstMaskHead.forward / parse_dynamic_params / simple_test (:1100-1286), restated in torch on the CPU.

mmcv (not installed here) is restated from mmcv-full >= 1.3.17 (requirements/mminstall.txt):
  * ``batched_nms`` (mmcv/ops/nms.py): the offset trick ``boxes + idxs * (boxes.max() + 1)`` in float32, one ``nms`` call
    below ``split_thr`` candidates, else one per class (``torch.unique``) and a final sort of the kept scores;
  * ``nms`` with its CUDA kernel (mmcv/ops/csrc/common/cuda/nms_cuda_kernel.cuh, offset 0): candidates sorted by
    descending score, then greedy, box j dropped by a kept box i when ``interS > iou_threshold * (Sa + Sb - interS)``
    with ``left = fmaxf(..)``, ``width = fmaxf(right - left, 0)``, ``interS = width * height``, every operation one
    float32 rounding.  This predicate is the contract ``bxs_box_nms`` implements (INTEGRATION.md section 11).
    torchvision's ``nms`` divides instead (``inter / union > thr``); the two differ only on exact-boundary pairs.
``stable=True`` makes every sort stable and the top-k break ties by the lower index (the library's documented order);
``stable=False`` uses torch.topk and torch.sort as the reference does."""
import torch
import torch.nn.functional as F


def suppresses(a, b, thr):
    """mmcv's devIoU test (offset 0) of boxes b by boxes a (broadcast [..., 4] float32)."""
    left, right = torch.fmax(a[..., 0], b[..., 0]), torch.fmin(a[..., 2], b[..., 2])
    top, bottom = torch.fmax(a[..., 1], b[..., 1]), torch.fmin(a[..., 3], b[..., 3])
    zero = torch.zeros((), dtype=torch.float32, device=a.device)
    width, height = torch.fmax(right - left, zero), torch.fmax(bottom - top, zero)
    inter = width * height
    sa = (a[..., 2] - a[..., 0]) * (a[..., 3] - a[..., 1])
    sb = (b[..., 2] - b[..., 0]) * (b[..., 3] - b[..., 1])
    return inter > torch.tensor(thr, dtype=torch.float32, device=a.device) * ((sa + sb) - inter)


def nms(boxes, scores, iou_threshold, stable=True):
    """mmcv's ``nms`` (CUDA kernel semantics) -> (dets [k,5], inds [k]) in descending score order."""
    order = torch.sort(scores, descending=True, stable=stable)[1]
    b = boxes[order].float()
    n = len(order)
    sup = (suppresses(b[:, None], b[None], iou_threshold) & torch.triu(torch.ones(n, n, dtype=torch.bool, device=b.device), 1)).cpu()
    removed = torch.zeros(n, dtype=torch.bool)
    keep = []
    for i in range(n):
        if not removed[i]:
            keep.append(i)
            removed |= sup[i]
    inds = order[torch.tensor(keep, dtype=torch.long, device=order.device)]
    return torch.cat((boxes[inds], scores[inds].reshape(-1, 1)), dim=1), inds


def batched_nms(boxes, scores, idxs, nms_cfg, class_agnostic=False, stable=True):
    """mmcv's ``batched_nms`` lines (mmcv/ops/nms.py)."""
    nms_cfg_ = nms_cfg.copy()
    class_agnostic = nms_cfg_.pop('class_agnostic', class_agnostic)
    if class_agnostic:
        boxes_for_nms = boxes
    else:
        max_coordinate = boxes.max()
        offsets = idxs.to(boxes) * (max_coordinate + torch.tensor(1).to(boxes))
        boxes_for_nms = boxes + offsets[:, None]
    assert nms_cfg_.pop('type', 'nms') == 'nms'
    split_thr = nms_cfg_.pop('split_thr', 10000)
    if boxes_for_nms.shape[0] < split_thr:
        dets, keep = nms(boxes_for_nms, scores, stable=stable, **nms_cfg_)
        boxes = boxes[keep]
        scores = dets[:, -1]
    else:
        max_num = nms_cfg_.pop('max_num', -1)
        total_mask = scores.new_zeros(scores.size(), dtype=torch.bool)
        scores_after_nms = scores.new_zeros(scores.size())
        for id in torch.unique(idxs):
            mask = (idxs == id).nonzero(as_tuple=False).view(-1)
            dets, keep = nms(boxes_for_nms[mask], scores[mask], stable=stable, **nms_cfg_)
            total_mask[mask[keep]] = True
            scores_after_nms[mask[keep]] = dets[:, -1]
        keep = total_mask.nonzero(as_tuple=False).view(-1)
        scores, inds = torch.sort(scores_after_nms[keep], descending=True, stable=stable)
        keep = keep[inds]
        boxes = boxes[keep]
        if max_num > 0:
            keep, boxes, scores = keep[:max_num], boxes[:max_num], scores[:max_num]
    return torch.cat([boxes, scores[:, None]], -1), keep


def points(featmap_sizes, strides, device=None):
    """MlvlPointGenerator(strides, offset=0.5).grid_priors: per level [H*W, 2] float32, x fastest."""
    out = []
    for (h, w), s in zip(featmap_sizes, strides):
        xs = (torch.arange(w, device=device) + 0.5) * s
        ys = (torch.arange(h, device=device) + 0.5) * s
        yy, xx = torch.meshgrid(ys, xs, indexing='ij')
        out.append(torch.stack([xx.reshape(-1), yy.reshape(-1)], -1).float())
    return out


def distance2bbox(points, distance, max_shape):
    """transforms.py:153-184 for batched points [B,N,2] and per-image max_shape."""
    x1 = points[..., 0] - distance[..., 0]
    y1 = points[..., 1] - distance[..., 1]
    x2 = points[..., 0] + distance[..., 2]
    y2 = points[..., 1] + distance[..., 3]
    bboxes = torch.stack([x1, y1, x2, y2], -1)
    max_shape = x1.new_tensor(max_shape)[..., :2].type_as(x1)
    min_xy = x1.new_tensor(0)
    max_xy = torch.cat([max_shape, max_shape], dim=-1).flip(-1).unsqueeze(-2)
    bboxes = torch.where(bboxes < min_xy, min_xy, bboxes)
    return torch.where(bboxes > max_xy, max_xy, bboxes)


def topk_inds(key, k, stable):
    if stable:
        return torch.sort(key, dim=-1, descending=True, stable=True)[1][..., :k]
    return key.topk(k)[1]


def nms_with_others(bboxes, scores, centerness, others, cfg, stable=True):
    """nms_with_others (:18-83) with the background column already dropped."""
    n, C = scores.shape
    boxes = bboxes[:, None].expand(n, C, 4).reshape(-1, 4)
    positions = torch.arange(n, device=scores.device).view(-1, 1).expand(n, C).reshape(-1)
    labels = torch.arange(C, device=scores.device).view(1, -1).expand(n, C).reshape(-1)
    valid = scores.reshape(-1) > cfg['score_thr']
    s = (scores * centerness.view(-1, 1)).reshape(-1)
    inds = valid.nonzero(as_tuple=False).squeeze(1)
    boxes, s, positions, labels = boxes[inds], s[inds], positions[inds], labels[inds]
    if boxes.numel() == 0:
        return torch.cat([boxes, s[:, None]], -1), labels, [o[positions] for o in others]
    dets, keep = batched_nms(boxes, s, labels, cfg['nms'], stable=stable)
    if cfg['max_per_img'] > 0:
        dets, keep = dets[:cfg['max_per_img']], keep[:cfg['max_per_img']]
    return dets, labels[keep], [o[positions][keep] for o in others]


def get_bboxes(cls_scores, bbox_preds, centernesses, param_preds, img_metas, cfg, strides, rescale=False, with_nms=True,
               stable=True):
    """_get_bboxes (:749-853) on per-level [B,c,H,W] tensors."""
    B, C = cls_scores[0].shape[:2]
    sizes = [tuple(c.shape[-2:]) for c in cls_scores]
    nms_pre = cfg.get('nms_pre', -1)
    mlvl = []
    for lvl, (cls, bbox, ctr, prm, pts) in enumerate(zip(cls_scores, bbox_preds, centernesses, param_preds,
                                                          points(sizes, strides, cls_scores[0].device))):
        scores = cls.permute(0, 2, 3, 1).reshape(B, -1, C).float().sigmoid()
        centerness = ctr.permute(0, 2, 3, 1).reshape(B, -1).float().sigmoid()
        bbox = bbox.permute(0, 2, 3, 1).reshape(B, -1, 4).float()
        prm = prm.permute(0, 2, 3, 1).reshape(B, -1, prm.shape[1])
        pts = pts.expand(B, -1, 2)
        if 0 < nms_pre < bbox.shape[1]:
            max_scores, _ = (scores * centerness[..., None]).max(-1)
            ti = topk_inds(max_scores, nms_pre, stable)
            bi = torch.arange(B, device=ti.device).view(-1, 1).expand_as(ti)
            pts, bbox, scores, centerness, prm = pts[bi, ti], bbox[bi, ti], scores[bi, ti], centerness[bi, ti], prm[bi, ti]
        boxes = distance2bbox(pts, bbox, [m['img_shape'] for m in img_metas])
        mlvl.append((pts, boxes, scores, centerness, prm, torch.full_like(centerness, lvl).long()))
    coors, boxes, scores, centerness, prm, lvl = [torch.cat(x, 1) for x in zip(*mlvl)]
    if rescale:
        boxes = boxes / boxes.new_tensor([m['scale_factor'] for m in img_metas]).unsqueeze(1)
    if not with_nms:
        scores = torch.cat([scores, scores.new_zeros(B, scores.shape[1], 1)], -1)
        return [tuple(x) for x in zip(boxes, scores, centerness, prm, coors, lvl)]
    out = []
    for b in range(B):
        dets, labels, others = nms_with_others(boxes[b], scores[b], centerness[b], [prm[b], coors[b], lvl[b]], cfg, stable)
        out.append((dets, labels) + tuple(others))
    return out


def aligned_bilinear(tensor, factor):
    """condinst_head.py:146-167."""
    if factor == 1:
        return tensor
    h, w = tensor.size()[2:]
    tensor = F.pad(tensor, pad=(0, 1, 0, 1), mode='replicate')
    oh, ow = factor * h + 1, factor * w + 1
    tensor = F.interpolate(tensor, size=(oh, ow), mode='bilinear', align_corners=True)
    tensor = F.pad(tensor, pad=(factor // 2, 0, factor // 2, 0), mode='replicate')
    return tensor[:, :, :oh - 1, :ow - 1]


def mask_head_forward(feat, params, coors, level_inds, img_inds, sizes_of_interest, in_stride=8, out_stride=4, channels=8,
                      num_convs=3):
    """CondInstMaskHead.forward (:1139-1164) with parse_dynamic_params (:1100-1137), rel coords on."""
    mask_feat = feat[img_inds]
    N, _, H, W = mask_feat.size()
    shift_x = torch.arange(0, W * in_stride, step=in_stride, dtype=mask_feat.dtype, device=feat.device)
    shift_y = torch.arange(0, H * in_stride, step=in_stride, dtype=mask_feat.dtype, device=feat.device)
    shift_y, shift_x = torch.meshgrid(shift_y, shift_x, indexing='ij')
    locations = torch.stack([shift_x, shift_y], dim=0) + in_stride // 2
    rel = (coors[..., None, None] - locations[None]) / sizes_of_interest.float()[level_inds][..., None, None, None]
    x = torch.cat([rel, mask_feat], dim=1).reshape(1, -1, H, W)
    cin = feat.shape[1] + 2
    shapes = [(channels, cin), (channels, channels), (1, channels)]
    w_n = [o * i for o, i in shapes]
    split = torch.split_with_sizes(params, w_n + [o for o, _ in shapes], dim=1)
    for i, (o, c) in enumerate(shapes):
        wt = split[i].reshape(N * o, c, 1, 1)
        bs = split[num_convs + i].reshape(N * o)
        x = F.conv2d(x, wt, bias=bs, groups=N)
        if i < num_convs - 1:
            x = F.relu(x)
    return aligned_bilinear(x.permute(1, 0, 2, 3), in_stride // out_stride)


def paste(mask_logits, out_stride, img_shape, ori_shape=None):
    """The mask lines of simple_test (:1261-1281) for one image -> bool [n, H, W]."""
    m = aligned_bilinear(mask_logits.sigmoid(), out_stride)[:, :, :img_shape[0], :img_shape[1]]
    if ori_shape is not None:
        m = F.interpolate(m, tuple(ori_shape[:2]), mode='bilinear', align_corners=False)
    return m.squeeze(1) > 0.5


COCO_SIZES = ((100, 168), (50, 84), (25, 42), (13, 21), (7, 11))      # 800x1344 padded input, strides 8 .. 128
COCO_STRIDES = (8, 16, 32, 64, 128)
COCO_TEST_CFG = dict(nms_pre=2000, min_bbox_size=0, score_thr=0.05, nms=dict(type='nms', iou_threshold=0.5), max_per_img=2000)
COCO_META = dict(img_shape=(800, 1067, 3), ori_shape=(480, 640, 3), pad_shape=(800, 1344, 3))


def workload(seed, B, n_obj, size, extra, C=80, P=233, mask_ch=16, device='cuda'):
    """Seeded COCO-test-shaped head outputs: n_obj objects per image, square-ish boxes of ``size`` = (min, max) pixels in
    the 800x1067 image, each of one class plus ``extra`` other classes.  Points inside an object predict its box (plus 0.5 px
    of noise) with class logits N(1, 1) for its classes; every other logit is N(-7, 1) and centerness N(0, 1).  Dynamic
    parameters N(0, 0.3); mask_feat [B,16,100,168]; img_metas of an 800x1067 image from a 480x640 original."""
    import numpy as np
    gen = torch.Generator(device='cpu').manual_seed(seed)
    cls, bbox, ctr, prm = [], [], [], []
    objs = []
    for b in range(B):
        wh = torch.rand(n_obj, 2, generator=gen) * (size[1] - size[0]) + size[0]
        c0 = torch.rand(n_obj, 2, generator=gen) * torch.tensor([1067., 800.])
        box = torch.cat([c0 - wh / 2, c0 + wh / 2], 1)
        labels = torch.stack([torch.randperm(C, generator=gen)[:1 + extra] for _ in range(n_obj)])
        objs.append((box, labels))
    for (h, w), s in zip(COCO_SIZES, COCO_STRIDES):
        c = torch.randn(B, C, h, w, generator=gen) - 7
        d = torch.rand(B, 4, h, w, generator=gen) * 3 * s + s / 2
        xs, ys = (torch.arange(w) + 0.5) * s, (torch.arange(h) + 0.5) * s
        for b, (box, labels) in enumerate(objs):
            for o in range(n_obj):
                x0, y0, x1, y1 = box[o].tolist()
                ix = ((xs > x0) & (xs < x1)).nonzero().flatten()
                iy = ((ys > y0) & (ys < y1)).nonzero().flatten()
                if len(ix) == 0 or len(iy) == 0:
                    continue
                yy, xx = torch.meshgrid(iy, ix, indexing='ij')
                for lab in labels[o].tolist():
                    c[b, lab, yy, xx] = torch.randn(yy.shape, generator=gen) + 1
                px, py = xs[xx], ys[yy]
                for k, v in enumerate((px - x0, py - y0, x1 - px, y1 - py)):
                    d[b, k, yy, xx] = v + torch.randn(yy.shape, generator=gen) * 0.5
        cls.append(c.to(device))
        bbox.append(d.clamp(min=0).to(device))
        ctr.append(torch.randn(B, 1, h, w, generator=gen).to(device))
        prm.append((torch.randn(B, P, h, w, generator=gen) * 0.3).to(device))
    feat = torch.randn(B, mask_ch, 100, 168, generator=gen).to(device)
    sf = [1067 / 640, 800 / 480, 1067 / 640, 800 / 480]
    metas = [dict(COCO_META, scale_factor=np.array(sf, dtype=np.float32)) for _ in range(B)]
    return cls, bbox, ctr, prm, feat, metas


# (name, workload args): about 3k candidates and 100 detections per image; about 20k candidates and 300 detections
WORKLOADS = [('3k_cand', (30, (24, 80), 1)), ('20k_cand', (40, (80, 260), 2))]
