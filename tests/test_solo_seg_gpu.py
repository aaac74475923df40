"""SOLOv2 inference on the GPU (csrc/solo_seg.cu, ops/solo_seg.py, models/dense_heads/solo_seg.py) against the oracle's
restatement of the reference (oracle/solo_seg.py) on the same CUDA tensors: Matrix NMS bit for bit (float32 intersections
and float16-rounded ones), the row statistics, the fused paste against two bilinear resizes, both heads' ``get_seg`` end to
end, the number of synchronising calls, determinism, layouts and the empty cases."""
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import solo_seg as oss
from oracle.make_golden_solo_seg import case, cfg_of, nms_case

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _big_nms_case(seed, n, h=40, w=56, classes=3):
    masks, labels, scores = nms_case(seed, n=n, h=h, w=w, classes=classes)
    g = torch.Generator().manual_seed(seed)
    for i in range(n):                                   # larger, overlapping blobs
        y0, x0 = int(torch.randint(0, h // 2, (1,), generator=g)), int(torch.randint(0, w // 2, (1,), generator=g))
        masks[i, y0:y0 + h // 3, x0:x0 + w // 3] = True
    if n > 7:
        scores[3] = scores[7]                            # ties: the stable order decides
    return masks.to(DEV), labels.to(DEV), scores.to(DEV)


@pytest.mark.parametrize('n', [1, 37, 300, 1100])
@pytest.mark.parametrize('kw', [dict(), dict(kernel='linear'), dict(nms_pre=200, max_num=50), dict(filter_thr=0.3),
                                dict(sigma=0.5, filter_thr=0.5, kernel='gaussian')])
def test_matrix_nms_equals_oracle(n, kw):
    from boxinstseg_b200.ops.solo_seg import mask_matrix_nms
    masks, labels, scores = _big_nms_case(n, n)
    got = mask_matrix_nms(masks, labels, scores, **kw)
    ref = oss.mask_matrix_nms(masks, labels, scores, stable=True, **kw)
    for a, b in zip(got, ref):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)


def _sorted_nms(masks, labels, scores, half_inter, **kw):
    from boxinstseg_b200.ops import solo_seg as S
    n = len(labels)
    src = S.RowSources([masks.to(torch.float16)])
    bits, area, _ = S.mask_stats(src, torch.arange(n, device=DEV), 0.5)
    s, order = torch.sort(scores, descending=True, stable=True)
    out = S.matrix_nms_sorted(bits, order[None], labels[order][None], area.float()[order][None], s[None],
                              torch.full((1,), n, device=DEV), half_inter=half_inter, **kw)[0]
    s2, o2 = torch.sort(out, descending=True, stable=True)
    keep = s2 > float('-inf')
    return s2[keep], order[o2[keep]]


@pytest.mark.parametrize('kernel', ['gaussian', 'linear'])
def test_matrix_nms_half_intersections_equal_oracle(kernel):
    """Intersections above 2048 pixels, where float16 rounding changes them: the kernel's once-rounded counts against the
    oracle's float32 torch.mm rounded to float16 once."""
    masks, labels, scores = _big_nms_case(5, 200, h=160, w=200, classes=2)
    s, k = _sorted_nms(masks, labels, scores, True, kernel=kernel)
    so, _, _, ko = oss.mask_matrix_nms(masks, labels, scores, kernel=kernel, stable=True, half_inter=True)
    assert torch.equal(k, ko) and torch.equal(s, so)
    s32, _ = _sorted_nms(masks, labels, scores, False, kernel=kernel)
    assert not torch.equal(s32, s)                       # the rounding is exercised


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('logits', [False, True])
@pytest.mark.parametrize('hw', [(50, 84), (11, 13)])
def test_mask_stats(dtype, logits, hw):
    from boxinstseg_b200.ops import solo_seg as S
    g = torch.Generator(device=DEV).manual_seed(1)
    x = (torch.randn((2, 7) + hw, generator=g, device=DEV) * 3).to(dtype)
    p = torch.sigmoid(x) if logits else torch.sigmoid(x.float()).to(dtype)
    rows_of = (x if logits else p)
    src = S.RowSources([rows_of.reshape(-1, *hw), rows_of[1, 2:]])                  # two sources, row ids across them
    rows = torch.tensor([0, 3, 13, 8, 7, 9], device=DEV)
    bits, area, msum = S.mask_stats(src, rows, 0.55, logits)
    allp = torch.cat([p.reshape(-1, *hw), p[1, 2:]])[rows]
    m = allp > 0.55
    assert torch.equal(area, m.flatten(1).sum(1).int())
    packed = np.packbits(m.flatten(1).cpu().numpy(), axis=1, bitorder='little')
    words = bits.cpu().numpy().view(np.uint8)[:, :packed.shape[1]]
    assert np.array_equal(words, packed)
    ref = (allp * m.float()).sum((1, 2))
    assert torch.allclose(msum, ref, rtol=1e-6, atol=0)


def _paste_ref(p, img_hw, ori_hw):
    from boxinstseg_b200.ops.resize import bilinear_resize
    h, w = p.shape[-2:]
    r1 = bilinear_resize(p.float(), (4 * h, 4 * w)).to(p.dtype)[:, :img_hw[0], :img_hw[1]]
    return bilinear_resize(r1.float(), ori_hw).to(p.dtype)


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16])
@pytest.mark.parametrize('shape', [((50, 84), (200, 336), (480, 640)), ((11, 13), (40, 50), (31, 45)), ((24, 32), (90, 120), (90, 120))])
def test_paste_equals_two_bilinear_resizes(dtype, shape, capsys):
    from boxinstseg_b200.ops.solo_seg import paste_masks
    hw, img_hw, ori_hw = shape
    g = torch.Generator(device=DEV).manual_seed(2)
    p = torch.sigmoid(torch.randn((9,) + hw, generator=g, device=DEV) * 2).to(dtype)
    got = paste_masks(p.transpose(1, 2).contiguous().transpose(1, 2), hw, img_hw + (3,), ori_hw + (3,), 0.55)
    v = _paste_ref(p, img_hw, ori_hw)
    assert got.dtype == torch.bool and torch.equal(got, v > 0.55)
    ti = F.interpolate(F.interpolate(p[None], (4 * hw[0], 4 * hw[1]), mode='bilinear')[:, :, :img_hw[0], :img_hw[1]],
                       ori_hw, mode='bilinear')[0]
    diff = got != (ti > 0.55)
    assert ((ti.float()[diff] - 0.55).abs() <= 1e-6).all()
    with capsys.disabled():
        print(f'\npaste {dtype} {shape}: {int(diff.sum())} of {diff.numel()} bits differ from F.interpolate')


def test_paste_float32_interpolation_under_autocast():
    """DiscoBox's paste under autocast: float16 probabilities interpolated in float32 (autocast's rule for
    upsample_bilinear2d), compared with the oracle's F.interpolate under real autocast."""
    from boxinstseg_b200.ops import solo_seg as S
    g = torch.Generator(device=DEV).manual_seed(3)
    x = (torch.randn(6, 24, 32, generator=g, device=DEV) * 3).half()
    src = S.RowSources([x])
    got = S.paste_rows(src, torch.arange(6, device=DEV), (90, 120), (70, 100), 0.4, logits=True, interp_f32=True)
    with torch.autocast('cuda', dtype=torch.float16):
        p = x.sigmoid()
        r = F.interpolate(F.interpolate(p[None], (96, 128), mode='bilinear')[:, :, :90, :120], (70, 100), mode='bilinear')[0]
    assert r.dtype == torch.float32
    assert torch.equal(got, r > 0.4)


def _match(got, ref, score_rtol, min_iou):
    """Same instance count; per position the same label and score within score_rtol, except inside a run of equal-within-
    tolerance scores, where the instances are matched by label and mask IoU."""
    assert len(got.scores) == len(ref.scores), (len(got.scores), len(ref.scores))
    n = len(ref.scores)
    if n == 0:
        return
    assert torch.allclose(got.scores.float(), ref.scores.float(), rtol=score_rtol, atol=0)
    gm, rm = got.masks.flatten(1).float(), ref.masks.flatten(1).float()
    inter = gm @ rm.t()
    iou = inter / (gm.sum(1)[:, None] + rm.sum(1)[None] - inter).clamp(min=1)
    close = (got.scores.float()[:, None] - ref.scores.float()[None]).abs() <= score_rtol * ref.scores.float().abs()[None]
    same = got.labels[:, None] == ref.labels[None]
    best = torch.where(close & same, iou, torch.zeros_like(iou)).max(1).values
    assert (best >= min_iou).all(), best.min().item()


def _solo_head_case(seed=0, B=2, C=64):
    from oracle import solo_head as osh
    from boxinstseg_b200.models import build_head
    head = osh.attach_towers(build_head(dict(osh.GOLDEN_HEAD, in_channels=C, seg_feat_channels=C)), C, C, 80, seed=seed)
    head = head.to(DEV)
    g = torch.Generator().manual_seed(seed)
    H, W = 256, 320
    feats = [torch.randn(B, C, -(-H // s), -(-W // s), generator=g).to(DEV) for s in (4, 8, 16, 32, 64)]
    return head, feats


def _quantile_thr(cate_preds, k):
    flat = torch.cat([c.reshape(-1) for c in cate_preds])
    return float(flat.topk(k + 1).values[-1]) if k else 1.0


def test_box_solov2_get_seg_on_forward_eval():
    head, feats = _solo_head_case()
    with torch.no_grad():
        seg, cate, lst = head.forward(feats, eval=True)
    cfg = dict(score_thr=_quantile_thr(cate, 600), mask_thr=0.5, nms_pre=500, max_per_img=100, kernel='gaussian', sigma=2.0,
               filter_thr=0.0)
    metas = [dict(img_shape=(250, 310, 3), ori_shape=(480, 600, 3))] * 2
    got = head.get_seg(seg, cate, lst, metas, cfg)
    ref = oss.box_get_seg(head, seg, cate, lst, metas, cfg_of(cfg), stable=True)
    for g_, r in zip(got, ref):
        assert g_.masks.dtype == torch.bool and g_.labels.dtype == torch.int64 and g_.scores.dtype == torch.float32
        _match(g_, r, 1e-5, 0.999)
    again = head.get_seg(seg, cate, lst, metas, cfg)
    for a, b in zip(got, again):
        assert torch.equal(a.masks, b.masks) and torch.equal(a.scores, b.scores) and torch.equal(a.labels, b.labels)


def _disco_case(seed, B=2, h=48, w=64, K=400):
    head, (cate, kern, feat), metas = case(seed, 'disco', B=B, h=h, w=w, C=80, E=32, grids=(40, 36, 24, 16, 12),
                                           strides=(8, 8, 16, 32, 32), img_shape=(180, 250, 3), ori_shape=(300, 420, 3),
                                           device=DEV)
    return head, cate, kern, feat, metas, _quantile_thr(cate, K)


@pytest.mark.parametrize('autocast', [False, True])
def test_discobox_get_seg(autocast):
    """Against the oracle on the same tensors; with autocast the oracle runs under real float16 autocast (cuDNN's float16
    convolution, cuBLAS's float16 intersections).  Tolerance: the convolutions (cuDNN against the wgmma kernel, TF32 or
    float16 operands) differ in the last bits of the logits, so a mask can differ by the pixels at the threshold and a
    score in its fourth digit."""
    from boxinstseg_b200.models import build_head
    from boxinstseg_b200.models.dense_heads.solo_seg import discobox_get_seg
    head, cate, kern, feat, metas, thr = _disco_case(7)
    cfg = dict(score_thr=thr, mask_thr=0.4, nms_pre=500, max_per_img=100, kernel='gaussian', sigma=2.0, filter_thr=0.0)
    if autocast:
        dh = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, num_grids=list(head.seg_num_grids),
                             strides=list(head.strides)))
        got = dh.get_seg(cate, kern, feat, metas, cfg)
    else:
        got = discobox_get_seg(cate, kern, feat, head.strides, metas, cfg, autocast=False)
    ref = oss.disco_get_seg(head, cate, kern, feat, metas, cfg_of(cfg), stable=True, autocast=autocast)
    for g_, r in zip(got, ref):
        assert abs(len(g_.scores) - len(r.scores)) <= 1
        n = min(len(g_.scores), len(r.scores))
        sub = lambda x: type('R', (), dict(scores=x.scores[:n], labels=x.labels[:n], masks=x.masks[:n]))   # noqa: E731
        _match(sub(g_), sub(r), 2e-3, 0.98)


def _count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return sum('synchroniz' in str(r.message) for r in rec)


@pytest.mark.parametrize('B', [1, 2])
@pytest.mark.parametrize('K', [0, 40, 3200])
def test_at_most_two_syncs(B, K, capsys):
    head, (seg, cate, _), metas = case(11, 'box', B=B, h=24, w=32, C=80, grids=(40, 36, 24, 16, 12), strides=(8, 8, 16, 32, 32),
                                       device=DEV)
    from boxinstseg_b200.models import build_head
    bh = build_head(dict(type='BoxSOLOv2Head', num_classes=80, num_grids=list(head.seg_num_grids), strides=list(head.strides)))
    cfg = dict(score_thr=_quantile_thr(cate, K), mask_thr=0.5, nms_pre=-1, max_per_img=100, kernel='gaussian', sigma=2.0,
               filter_thr=0.05)
    bh.get_seg(seg, cate, None, metas, cfg)                                                  # warm up
    n = _count_syncs(lambda: bh.get_seg(seg, cate, None, metas, cfg))
    n_ref = _count_syncs(lambda: oss.box_get_seg(head, seg, cate, None, metas, cfg_of(cfg))) if K else None
    with capsys.disabled():
        print(f'\nsyncs per get_seg (B={B}, K~{K}): {n}; reference lines: {n_ref}')
    assert n <= 2


def test_noncontiguous_inputs_and_empty_cases():
    from boxinstseg_b200.models import build_head
    head, (seg, cate, _), metas = case(3, 'box', device=DEV)
    bh = build_head(dict(type='BoxSOLOv2Head', num_classes=5, num_grids=list(head.seg_num_grids), strides=list(head.strides)))
    cfg = dict(cfg_of({}).__dict__)
    perm = [c.permute(0, 3, 1, 2).contiguous().permute(0, 2, 3, 1) for c in cate]             # forward(eval)'s layout
    a, b = bh.get_seg(seg, cate, None, metas, cfg), bh.get_seg(seg, perm, None, metas, cfg)
    for x, y in zip(a, b):
        assert torch.equal(x.masks, y.masks) and torch.equal(x.scores, y.scores)
    for over, kw in ((dict(score_thr=0.999), {}), ({}, dict(strides=(5000, 5000, 5000)))):
        head, (seg, cate, _), metas = case(4, 'box', device=DEV, **kw)
        bh.strides = list(head.strides)
        got = bh.get_seg(seg, cate, None, metas, dict(cfg, **over))
        ref = oss.box_get_seg(head, seg, cate, None, metas, cfg_of(over))
        for g_, r in zip(got, ref):
            for k in ('masks', 'labels', 'scores'):
                assert getattr(g_, k).dtype == getattr(r, k).dtype and getattr(g_, k).shape == getattr(r, k).shape
    # Matrix NMS keeps nothing: the reference raises for BoxSOLOv2, returns empty_results for DiscoBox
    head, (seg, cate, _), metas = case(5, 'box', device=DEV)
    bh.strides = list(head.strides)
    got = bh.get_seg(seg, cate, None, metas, dict(cfg, filter_thr=2.0))
    assert all(len(r.scores) == 0 and r.masks.dtype == cate[0].dtype and r.masks.shape == (0, 44, 60) for r in got)
