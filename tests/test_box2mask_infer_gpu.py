"""Box2Mask inference on the GPU (csrc/solo_seg.cu's maskformer paste, ops/solo_seg.py, models/dense_heads/
box2mask_infer.py): the golden cases against the oracle (oracle/box2mask_infer.py) on the same CUDA tensors, COCO-shaped
inputs against the reference's lines on CUDA and against two bilinear_resize passes, both input resolutions, float16
predictions, the edge cases, the number of synchronising calls, determinism and the detector's post-head lines."""
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import box2mask_infer as obi
from oracle.make_golden_box2mask_infer import CASES, case

pytestmark = pytest.mark.gpu
DEV = 'cuda'
COCO = dict(hw=(200, 272), pad=(800, 1088), img=(800, 1067), ori=(480, 640), Q=100, K=80)


def _head(things, stuff=0, max_per_image=100):
    from boxinstseg_b200.models.dense_heads.box2mask_infer import MaskFormerFusionHead
    return MaskFormerFusionHead(things, stuff, test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True,
                                                             max_per_image=max_per_image))


def _results(head, mask_cls, mask_pred, metas, rescale):
    from boxinstseg_b200.models.dense_heads.box2mask_infer import instance_results
    return instance_results(mask_cls, mask_pred, metas, head.num_things_classes, head.test_cfg['max_per_image'], rescale)


def _coco(B, seed=0, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    c = COCO
    mask_cls = (torch.randn(B, c['Q'], c['K'] + 1, generator=g) * 3).to(DEV)
    low = torch.randn(B, c['Q'], 25, 34, generator=g) * 4          # smooth logits, so that masks are blobs
    mask_pred = F.interpolate(low, c['hw'], mode='bilinear', align_corners=False).to(DEV, dtype)
    ori = [c['ori'], (427, 640)][:B]
    metas = [dict(img_shape=c['img'] + (3,), ori_shape=o + (3,), batch_input_shape=c['pad']) for o in ori]
    return mask_cls, mask_pred, metas


def _assert_same_as_oracle(res, ora):
    for (labels, query, bboxes, masks), (ol, oq, ob, om) in zip(res, ora):
        assert torch.equal(labels, ol) and torch.equal(query, oq)
        assert torch.equal(masks, om)
        assert torch.equal(bboxes[:, :4], ob[:, :4])
        assert ((bboxes[:, 4] - ob[:, 4]).abs() <= 1e-6 * ob[:, 4].abs()).all()


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_golden_cases_equal_oracle_on_cuda(i):
    mask_cls, mask_pred, metas, cfg = case(i)
    mask_cls, mask_pred = mask_cls.to(DEV), mask_pred.to(DEV)
    head = _head(cfg['things'], cfg['stuff'], cfg['max_per_image'])
    res = _results(head, mask_cls, mask_pred, metas, cfg['rescale'])
    ora = obi.fusion_simple_test(mask_cls, mask_pred, metas, cfg['things'], cfg['max_per_image'], cfg['rescale'])
    _assert_same_as_oracle(res, ora)
    if CASES[i][0] == 'base':                                        # the all-negative query: box and score zero
        labels, query, bboxes, masks = res[1]
        k = query.tolist().index(4)
        assert not masks[k].any() and not bboxes[k].any()


def _reference_lines(mask_cls, mask_pred, metas, max_per_image, rescale):
    """Box2MaskHead.simple_test's upsample and MaskFormerFusionHead.simple_test / instance_postprocess as the reference
    writes them (topk(sorted=False), mask2bbox), on CUDA; per image (labels, query, bboxes, masks, final logits)."""
    K = mask_cls.shape[-1] - 1
    pred = F.interpolate(mask_pred, metas[0]['batch_input_shape'], mode='bilinear', align_corners=False)
    out = []
    for cls, mp, meta in zip(mask_cls, pred, metas):
        mp = mp[:, :meta['img_shape'][0], :meta['img_shape'][1]]
        if rescale:
            mp = F.interpolate(mp[:, None], meta['ori_shape'][:2], mode='bilinear', align_corners=False)[:, 0]
        scores = F.softmax(cls, dim=-1)[:, :-1]
        s, top = scores.flatten(0, 1).topk(max_per_image, sorted=False)
        labels, query = top % K, top // K
        mp = mp[query]
        binary = (mp > 0).float()
        det = s * ((mp.sigmoid() * binary).flatten(1).sum(1) / (binary.flatten(1).sum(1) + 1e-6))
        out.append((labels, query, torch.cat([obi.mask2bbox(binary.bool()), det[:, None]], -1), binary.bool(), mp))
    return out


DELTA = 1e-5


@pytest.mark.parametrize('B', [1, 2])
def test_coco_shapes_against_reference_lines_and_resize_passes(B):
    from boxinstseg_b200.ops.resize import bilinear_resize
    mask_cls, mask_pred, metas = _coco(B, seed=B)
    res = _results(_head(80), mask_cls, mask_pred, metas, True)
    ref = _reference_lines(mask_cls, mask_pred, metas, 100, True)
    up = bilinear_resize(mask_pred, COCO['pad'])
    for b, ((labels, query, bboxes, masks), (rl, rq, rb, rm, rv)) in enumerate(zip(res, ref)):
        key = (query * 80 + labels).tolist()
        rkey = (rq * 80 + rl).tolist()
        assert sorted(key) == sorted(rkey)
        o = torch.tensor([rkey.index(k) for k in key], device=DEV)
        diff = masks != rm[o]
        assert (rv[o][diff].abs() <= DELTA).all()                   # a pixel may differ only within DELTA of 0
        assert torch.equal(bboxes[:, :4], obi.mask2bbox(masks))     # boxes follow from the masks
        assert ((bboxes[:, 4] - rb[o, 4]).abs() <= 1e-6 * rb[o, 4].abs() + 1e-12).all()
        # the masks are two bilinear_resize passes and the threshold, bit for bit
        crop = up[b, :, :metas[b]['img_shape'][0], :metas[b]['img_shape'][1]].contiguous()
        two = bilinear_resize(crop, metas[b]['ori_shape'][:2]) > 0
        assert torch.equal(masks, two[query])


def test_low_and_batch_input_resolution_give_identical_results():
    from boxinstseg_b200.ops.resize import bilinear_resize
    mask_cls, mask_pred, metas = _coco(2, seed=5)
    head = _head(80)
    for rescale in (True, False):
        a = head.simple_test(mask_cls, mask_pred, metas, rescale=rescale)
        b = head.simple_test(mask_cls, bilinear_resize(mask_pred, COCO['pad']), metas, rescale=rescale)
        for x, y in zip(a, b):
            assert all(torch.equal(u, v) for u, v in zip(x['ins_results'], y['ins_results']))


def test_float16_rounds_after_each_stage():
    mask_cls, mask_pred, metas = _coco(2, seed=7, dtype=torch.float16)
    res = _results(_head(80), mask_cls, mask_pred, metas, True)
    ora = obi.fusion_simple_test(mask_cls, mask_pred, metas, 80, 100, True)       # ATen's half kernel, both stages
    _assert_same_as_oracle(res, ora)


def test_instance_postprocess_and_edge_cases():
    head = _head(3, 0, max_per_image=8)
    g = torch.Generator().manual_seed(3)
    cls = torch.randn(4, 4, generator=g).to(DEV)
    cls[1] = cls[2]                                                  # tied class scores: the lower q*K + c first
    pred = (torch.randn(4, 20, 24, generator=g) * 2).to(DEV)
    pred[3] = -1.0                                                   # an all-negative query, picked
    cls[3, 0] = 9.0
    labels, bboxes, masks = head.instance_postprocess(cls, pred)
    ol, oq, ob, om = obi.instance_postprocess(cls, pred, 3, 8)
    assert torch.equal(labels, ol) and torch.equal(masks, om) and torch.equal(bboxes[:, :4], ob[:, :4])
    s = F.softmax(cls, -1)[:, :-1].flatten()
    assert torch.equal(s[oq * 3 + ol], s.sort(descending=True, stable=True)[0][:8])
    k = oq.tolist().index(3)
    assert not masks[k].any() and not bboxes[k].any()
    with pytest.raises(RuntimeError, match='out of range'):
        _head(3, 0, max_per_image=13).instance_postprocess(cls, pred)


def test_strided_and_offset_views():
    mask_cls, mask_pred, metas = _coco(2, seed=9)
    head = _head(80)
    want = head.simple_test(mask_cls, mask_pred, metas, rescale=True)
    big = torch.zeros(2, 101, 81, device=DEV)
    big[:, 1:] = mask_cls
    cls_t = mask_cls.transpose(1, 2).contiguous().transpose(1, 2)     # strided
    pred_off = torch.cat([mask_pred[:, :1], mask_pred], 1)[:, 1:]     # offset view (contiguous)
    pred_t = mask_pred.transpose(2, 3).contiguous().transpose(2, 3)   # strided
    for c, p in ((big[:, 1:], pred_off), (cls_t, pred_t)):
        got = head.simple_test(c, p, metas, rescale=True)
        for x, y in zip(got, want):
            assert all(torch.equal(u, v) for u, v in zip(x['ins_results'], y['ins_results']))


def _count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    # the message of a synchronising call; the once-per-process notice that the debug mode is a prototype does not count
    return sum('called a synchronizing' in str(r.message) for r in rec)


@pytest.mark.parametrize('B', [1, 2])
def test_synchronising_calls(B, capsys):
    mask_cls, mask_pred, metas = _coco(B, seed=11)
    head = _head(80)
    head.simple_test(mask_cls, mask_pred, metas, rescale=True)        # warm
    assert _count_syncs(lambda: head.simple_test(mask_cls, mask_pred, metas, rescale=True)) == 0
    torch.cuda.set_sync_debug_mode('error')
    try:
        head.simple_test(mask_cls, mask_pred, metas, rescale=True)
    finally:
        torch.cuda.set_sync_debug_mode('default')
    stuff = _head(60, 20)
    stuff.simple_test(mask_cls, mask_pred, metas, rescale=True)       # warm
    n = _count_syncs(lambda: stuff.simple_test(mask_cls, mask_pred, metas, rescale=True))
    with capsys.disabled():
        print(f'\nsyncs per simple_test (B={B}): 0 things only, {n} with stuff classes')
    assert n <= 1


def test_deterministic():
    mask_cls, mask_pred, metas = _coco(2, seed=13)
    head = _head(80)
    a = head.simple_test(mask_cls, mask_pred, metas, rescale=True)
    b = head.simple_test(mask_cls, mask_pred, metas, rescale=True)
    for x, y in zip(a, b):
        assert all(torch.equal(u, v) for u, v in zip(x['ins_results'], y['ins_results']))


def test_detector_post_head_lines_on_registered_heads():
    """MaskFormer.simple_test (detectors/maskformer.py:156-177) after the two registered heads."""
    from boxinstseg_b200.models import build_head
    mask_cls, mask_pred, metas = _coco(2, seed=17)
    box2mask = build_head(dict(type='Box2MaskHead', num_things_classes=80, num_stuff_classes=0, num_queries=100))
    box2mask.forward = lambda feats, img_metas: ([mask_cls * 0, mask_cls], [mask_pred * 0, mask_pred], [None, None])
    fusion = build_head(dict(type='MaskFormerFusionHead', num_things_classes=80, num_stuff_classes=0,
                             test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True, max_per_image=100)))
    cls_r, pred_r = box2mask.simple_test(None, metas, rescale=True)
    assert cls_r is mask_cls and pred_r is mask_pred
    results = fusion.simple_test(cls_r, pred_r, metas, rescale=True)
    for i, meta in enumerate(metas):
        labels, bboxes, masks = results[i]['ins_results']
        bl, bb = labels.cpu().numpy(), bboxes.cpu().numpy()
        bbox_results = [bb[bl == c, :] for c in range(80)]                   # bbox2result
        mask_results = [[] for _ in range(80)]
        for j, label in enumerate(labels):
            mask_results[label].append(masks[j].detach().cpu().numpy())
        assert sum(len(r) for r in bbox_results) == sum(len(m) for m in mask_results) == 100
        for c in range(80):
            assert bbox_results[c].shape == (len(mask_results[c]), 5) and bbox_results[c].dtype == np.float32
            for m in mask_results[c]:
                assert m.dtype == bool and m.shape == meta['ori_shape'][:2]
