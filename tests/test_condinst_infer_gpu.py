"""CondInst inference on the GPU (csrc/condinst_infer.cu, ops/box_nms.py, ops/condinst.py, models/dense_heads/
condinst_infer.py) against the oracle's restatement of the reference (oracle/condinst_infer.py) on the same CUDA tensors:
get_bboxes bit for bit (boxes, scores, labels, params, coors, level indices), batched_nms against the oracle and
torchvision, the fused paste against bxs_bilinear_resize_forward passes, simple_test end to end against the reference's
cuDNN dynamic convolutions, the number of synchronising calls, determinism, layouts and the empty cases."""
import warnings

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import condinst_infer as oci
from oracle.make_golden_condinst_infer import CASES, MASK_CH, NUM_CLASSES, SOI, STRIDES, case, cfg_of

pytestmark = pytest.mark.gpu
DEV = 'cuda'
MASK_DELTA = 1e-3        # a mask pixel may differ from the reference only where its reference probability is this close to 0.5


def _box_head(cfg, strides=STRIDES, C=NUM_CLASSES):
    from boxinstseg_b200.models.dense_heads.condinst_box_head import CondInstBoxHead
    return CondInstBoxHead(num_classes=C, strides=strides, test_cfg=cfg)


def _mask_head(in_channels=MASK_CH):
    from boxinstseg_b200.models.dense_heads.condinst_mask_head import CondInstMaskHead
    return CondInstMaskHead(in_channels=in_channels, sizes_of_interest=list(SOI)).to(DEV)


def _assert_equal(got, ref):
    assert len(got) == len(ref)
    for g_img, r_img in zip(got, ref):
        assert len(g_img) == len(r_img)
        for i, (g, r) in enumerate(zip(g_img, r_img)):
            assert g.dtype == r.dtype and g.shape == r.shape, (i, g.dtype, r.dtype, g.shape, r.shape)
            assert torch.equal(g, r), i


@pytest.mark.parametrize('seed', range(len(CASES)), ids=[c[0] for c in CASES])
def test_get_bboxes_bit_exact_with_oracle(seed):
    name, kw, over, rescale, with_nms = CASES[seed]
    cls, bbox, ctr, prm, feat, metas = case(seed, device=DEV, **kw)
    cfg = cfg_of(over)
    got = _box_head(cfg).get_bboxes(cls, bbox, ctr, prm, metas, rescale=rescale, with_nms=with_nms)
    _assert_equal(got, oci.get_bboxes(cls, bbox, ctr, prm, metas, cfg, STRIDES, rescale, with_nms))


def _coco(name, B):
    args = dict(oci.WORKLOADS)[name]
    return oci.workload(7, B, *args, device=DEV)


@pytest.mark.parametrize('B', [1, 2])
@pytest.mark.parametrize('name', [w[0] for w in oci.WORKLOADS])
def test_get_bboxes_coco_shapes(name, B, capsys):
    cls, bbox, ctr, prm, feat, metas = _coco(name, B)
    head = _box_head(oci.COCO_TEST_CFG, oci.COCO_STRIDES, 80)
    got = head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True)
    ref = oci.get_bboxes(cls, bbox, ctr, prm, metas, oci.COCO_TEST_CFG, oci.COCO_STRIDES, True, True)
    _assert_equal(got, ref)
    raw = head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True, with_nms=False)
    n_cand = [int((r[1][:, :-1] > 0.05).sum()) for r in raw]
    with capsys.disabled():
        print(f'\n{name} B={B}: candidates {n_cand}, detections {[len(g[0]) for g in got]}')
    if name == '20k_cand':
        assert min(n_cand) > 10000                        # mmcv's per-class branch in the oracle
    again = head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True)
    _assert_equal(again, got)                             # run to run


def _count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return sum('called a synchronizing' in str(r.message) for r in rec)


@pytest.mark.parametrize('B', [1, 2])
def test_at_most_two_syncs_and_none_in_the_mask_device_part(B, capsys):
    cls, bbox, ctr, prm, feat, metas = _coco('20k_cand', B)
    head = _box_head(oci.COCO_TEST_CFG, oci.COCO_STRIDES, 80)
    dets = head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True)            # warm up
    n_box = _count_syncs(lambda: head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True))
    n_empty = _count_syncs(lambda: head.get_bboxes([c - 100 for c in cls], bbox, ctr, prm, metas, rescale=True))
    mh = _mask_head(16)
    args = (feat, [d[1] for d in dets], [d[2] for d in dets], [d[3] for d in dets], [d[4] for d in dets], metas, 80)
    mh.simple_test(*args, rescale=True)
    n_mask = _count_syncs(lambda: mh.simple_test(*args, rescale=True))
    with capsys.disabled():
        print(f'\nsyncs (B={B}): get_bboxes {n_box}, without candidates {n_empty}; simple_test {n_mask} '
              f'(the host copies of masks and labels: {2 * B})')
    assert n_box <= 2 and n_empty <= 1
    assert n_mask <= 2 * B


def test_batched_nms_equals_oracle_and_torchvision():
    torchvision = pytest.importorskip('torchvision')
    from boxinstseg_b200.ops.box_nms import batched_nms
    g = torch.Generator(device=DEV).manual_seed(11)
    for n, classes, split in ((3000, 5, 10000), (12000, 7, 10000), (500, 3, 50)):
        xy = torch.rand(n, 2, generator=g, device=DEV) * 300
        boxes = torch.cat([xy, xy + torch.rand(n, 2, generator=g, device=DEV) * 60 + 1], 1)
        scores = torch.rand(n, generator=g, device=DEV)
        idxs = torch.randint(0, classes, (n,), generator=g, device=DEV)
        cfg = dict(type='nms', iou_threshold=0.5, split_thr=split)
        dets, keep = batched_nms(boxes, scores, idxs, cfg)
        r_dets, r_keep = oci.batched_nms(boxes, scores, idxs, cfg)
        assert torch.equal(keep, r_keep) and torch.equal(dets, r_dets)
        assert torch.equal(keep, torchvision.ops.batched_nms(boxes, scores, idxs, 0.5))
    # equal scores keep the input order; an empty input gives empty outputs
    scores = torch.full((n,), 0.5, device=DEV)
    assert torch.equal(batched_nms(boxes, scores, idxs, cfg)[1], oci.batched_nms(boxes, scores, idxs, cfg)[1])
    d, k = batched_nms(boxes[:0], scores[:0], idxs[:0], cfg)
    assert d.shape == (0, 5) and k.shape == (0,)


def _paste_passes(logits, f, img_hw, ori_hw):
    """The reference's mask lines with the library's bilinear kernel for both interpolations."""
    from boxinstseg_b200.ops.resize import bilinear_resize
    p = logits.sigmoid()
    h, w = p.shape[-2:]
    u = bilinear_resize(F.pad(p, (0, 1, 0, 1), mode='replicate'), (f * h + 1, f * w + 1), align_corners=True)
    u = F.pad(u, (f // 2, 0, f // 2, 0), mode='replicate')[:, :, :f * h, :f * w][:, :, :img_hw[0], :img_hw[1]]
    if ori_hw is not None:
        u = bilinear_resize(u.contiguous(), ori_hw, align_corners=False)
    return u[:, 0]


@pytest.mark.parametrize('shape', [((200, 336), 4, (800, 1067), (480, 640)), ((200, 336), 4, (800, 1067), None),
                                   ((13, 17), 4, (50, 61), (37, 45)), ((10, 12), 2, (19, 24), None)])
def test_paste_equals_bilinear_resize_passes(shape):
    from boxinstseg_b200.ops.condinst import paste_masks
    hw, f, img_hw, ori_hw = shape
    g = torch.Generator(device=DEV).manual_seed(5)
    logits = torch.randn((6, 1) + hw, generator=g, device=DEV) * 3
    got = paste_masks(logits, f, img_hw, ori_hw)
    assert got.dtype == torch.bool and torch.equal(got, _paste_passes(logits, f, img_hw, ori_hw) > 0.5)


def _reference_probs(feat, dets, metas, rescale):
    """The reference's simple_test lines before the threshold, with cuDNN's dynamic convolutions (TF32 off)."""
    out = []
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        for b, d in enumerate(dets):
            if len(d[2]) == 0:
                out.append(None)
                continue
            logits = oci.mask_head_forward(feat, d[2], d[3], d[4], torch.full((len(d[2]),), b, dtype=torch.long, device=DEV),
                                           torch.tensor(SOI, device=DEV))
            m = oci.aligned_bilinear(logits.sigmoid(), 4)[:, :, :metas[b]['img_shape'][0], :metas[b]['img_shape'][1]]
            if rescale:
                m = F.interpolate(m, tuple(metas[b]['ori_shape'][:2]), mode='bilinear', align_corners=False)
            out.append(m[:, 0])
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    return out


@pytest.mark.parametrize('rescale', [True, False])
def test_simple_test_end_to_end_against_cudnn_reference(rescale, capsys):
    cls, bbox, ctr, prm, feat, metas = _coco('3k_cand', 2)
    dets = _box_head(oci.COCO_TEST_CFG, oci.COCO_STRIDES, 80).get_bboxes(cls, bbox, ctr, prm, metas, rescale=rescale)
    mh = _mask_head(16)
    segm = mh.simple_test(feat, [d[1] for d in dets], [d[2] for d in dets], [d[3] for d in dets], [d[4] for d in dets],
                          metas, 80, rescale=rescale)
    probs = _reference_probs(feat, dets, metas, rescale)
    for b, (s, p) in enumerate(zip(segm, probs)):
        labels = dets[b][1].cpu().numpy()
        assert len(s) == 80
        ref = (p > 0.5).cpu().numpy().astype(np.uint8)
        got = np.zeros_like(ref)
        for c in range(80):
            assert s[c].dtype == np.uint8 and s[c].shape[1:] == ref.shape[1:]
            got[labels == c] = s[c]
        diff = got != ref
        near = (p.cpu().numpy()[diff] - 0.5).__abs__()
        with capsys.disabled():
            print(f'\nsimple_test rescale={rescale} image {b}: {int(diff.sum())} of {diff.size} pixels differ, '
                  f'max |p - 0.5| there {near.max() if near.size else 0:.2e}')
        assert (near <= MASK_DELTA).all()
    again = mh.simple_test(feat, [d[1] for d in dets], [d[2] for d in dets], [d[3] for d in dets], [d[4] for d in dets],
                           metas, 80, rescale=rescale)
    assert all(np.array_equal(x, y) for s1, s2 in zip(segm, again) for x, y in zip(s1, s2))


def test_layouts_dtypes_and_alignment():
    cls, bbox, ctr, prm, feat, metas = case(0, device=DEV)
    cfg = cfg_of({})
    head = _box_head(cfg)
    ref = head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True)
    cl = lambda ts: [t.contiguous(memory_format=torch.channels_last) for t in ts]            # noqa: E731
    _assert_equal(head.get_bboxes(cl(cls), cl(bbox), cl(ctr), cl(prm), metas, rescale=True), ref)

    def shifted(ts):                     # one element into a bigger buffer: element-aligned only, and strided
        out = []
        for t in ts:
            big = torch.empty(t.numel() * 2 + 1, device=DEV)
            v = big[1:1 + 2 * t.numel()].view(*t.shape[:-1], 2 * t.shape[-1])[..., ::2]
            v.copy_(t)
            out.append(v)
        return out
    _assert_equal(head.get_bboxes(shifted(cls), shifted(bbox), shifted(ctr), shifted(prm), metas, rescale=True), ref)
    half = lambda ts: [t.half() for t in ts]                                                 # noqa: E731
    got = head.get_bboxes(half(cls), half(bbox), half(ctr), prm, metas, rescale=True)
    f32 = lambda ts: [t.half().float() for t in ts]                                          # noqa: E731
    _assert_equal(got, oci.get_bboxes(f32(cls), f32(bbox), f32(ctr), prm, metas, cfg, STRIDES, True, True))


def test_empty_cases():
    cls, bbox, ctr, prm, feat, metas = case(6, device=DEV, empty_img=1)
    head, mh = _box_head(cfg_of({})), _mask_head()
    dets = head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True)
    assert len(dets[0][0]) > 0 and len(dets[1][0]) == 0
    assert [t.shape for t in dets[1]] == [(0, 5), (0,), (0, 169), (0, 2), (0,)]
    segm = mh.simple_test(feat, *[[d[i] for d in dets] for i in (1, 2, 3, 4)], metas, NUM_CLASSES, rescale=True)
    assert len(segm) == 2 and segm[1] == [[] for _ in range(NUM_CLASSES)]
    assert sum(len(m) for m in segm[0]) == len(dets[0][0])
    none = head.get_bboxes([c - 100 for c in cls], bbox, ctr, prm, metas)
    assert all(len(d[0]) == 0 for d in none)
    segm = mh.simple_test(feat, *[[d[i] for d in none] for i in (1, 2, 3, 4)], metas, NUM_CLASSES)
    assert segm == [[[] for _ in range(NUM_CLASSES)] for _ in range(2)]
