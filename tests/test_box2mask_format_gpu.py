"""Box2Mask's test-result formatting on the GPU (models/detectors/box2mask.py ``format_instance_results`` and the registered
``Box2Mask.simple_test``) against the oracle's restatement of the reference's tail (oracle/box2mask_format.py) on the same
CUDA results of ``MaskFormerFusionHead.simple_test``: every golden case, COCO shapes with two original sizes, 0, 1 and 100
detections in one call, non-contiguous, misaligned and uint8 masks, earlier results intact after later calls, the host
waits per call, and the whole ``simple_test`` on stub features and head outputs."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import box2mask_format as obf
from oracle.make_golden_box2mask_infer import CASES, case
from tools.benchkit import syncs

pytestmark = pytest.mark.gpu
DEV = 'cuda'
PAD, IMG, ORI = (800, 1088), (800, 1067), ((480, 640), (427, 640))


def _fusion(things, stuff=0, max_per_image=100):
    from boxinstseg_b200.models.dense_heads.box2mask_infer import MaskFormerFusionHead
    return MaskFormerFusionHead(things, stuff, test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True,
                                                             max_per_image=max_per_image))


def _coco(B, seed):
    """mask_cls [B,100,81], smooth mask_pred [B,100,200,272] and COCO test metas, original 480 x 640 then 427 x 640."""
    g = torch.Generator().manual_seed(seed)
    mask_cls = (torch.randn(B, 100, 81, generator=g) * 3).to(DEV)
    low = torch.randn(B, 100, 25, 34, generator=g) * 4
    mask_pred = F.interpolate(low, (200, 272), mode='bilinear', align_corners=False).to(DEV)
    metas = [dict(img_shape=IMG + (3,), ori_shape=ORI[b % 2] + (3,), batch_input_shape=PAD) for b in range(B)]
    return mask_cls, mask_pred, metas


def _coco_ins(B, seed, max_per_image=100):
    mask_cls, mask_pred, metas = _coco(B, seed)
    return [r['ins_results'] for r in _fusion(80, 0, max_per_image).simple_test(mask_cls, mask_pred, metas, rescale=True)]


def _format(ins, C=80):
    from boxinstseg_b200.models.detectors import format_instance_results
    return format_instance_results(ins, C)


def _check(ins, C=80, what=''):
    got = _format(ins, C)
    obf.assert_same(got, obf.maskformer_simple_test_tail(ins, C), what)
    return got


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_golden_cases_equal_oracle(i):
    mask_cls, mask_pred, metas, cfg = case(i)
    res = _fusion(cfg['things'], cfg['stuff'], cfg['max_per_image']).simple_test(mask_cls.to(DEV), mask_pred.to(DEV),
                                                                                  metas, rescale=cfg['rescale'])
    ins = [r['ins_results'] for r in res]
    got = _check(ins, cfg['things'], CASES[i][0])
    for (bbox, masks), (labels, _, m) in zip(got, ins):
        assert all(b.dtype.name == 'float32' for b in bbox)
        assert sum(len(x) for x in masks) == len(labels)
        assert all(x.dtype == bool and x.shape == tuple(m.shape[1:]) for xs in masks for x in xs)


def test_coco_two_original_sizes():
    ins = _coco_ins(2, seed=1)
    got = _check(ins, what='coco B=2')
    for (bbox, masks), ori in zip(got, ORI):
        assert sum(len(b) for b in bbox) == sum(len(m) for m in masks) == 100
        assert {x.shape for xs in masks for x in xs} == {ori}


def test_zero_one_and_hundred_detections_in_one_call():
    a, b = _coco_ins(2, seed=2)
    ins = [tuple(t[:0] for t in a), tuple(t[:1] for t in b), a, tuple(t[:0] for t in b), b]
    got = _check(ins, what='0 / 1 / 100')
    assert [sum(len(m) for m in masks) for _, masks in got] == [0, 1, 100, 0, 100]


def test_max_per_image_20_and_voc_classes():
    _check(_coco_ins(1, seed=3, max_per_image=20), what='max 20')
    labels, bboxes, masks = _coco_ins(1, seed=4)[0]
    _check([(labels % 20, bboxes, masks)], 20, 'voc')


def test_noncontiguous_misaligned_and_uint8_masks_and_other_box_layouts():
    (labels, bboxes, masks), = _coco_ins(1, seed=5, max_per_image=30)
    n, H, W = masks.shape
    big = torch.zeros(n, W, 2 * H, dtype=torch.bool, device=DEV)
    big[:, :, ::2] = masks.transpose(1, 2)
    strided = big[:, :, ::2].transpose(1, 2)
    assert not strided.is_contiguous()
    flat = torch.zeros(n * H * W + 1, dtype=torch.bool, device=DEV)
    flat[1:] = masks.flatten()
    offset = flat[1:].view(n, H, W)
    assert offset.is_contiguous() and offset.data_ptr() % 16
    box_t = bboxes.t().contiguous().t()                                  # strided boxes
    lab_s = torch.stack([labels, labels], 1)[:, 0]                       # strided labels
    for what, ins in (('strided', (labels, bboxes, strided)), ('offset', (labels, bboxes, offset)),
                      ('uint8', (labels, bboxes, masks.to(torch.uint8) * 3)), ('strided boxes', (lab_s, box_t, masks)),
                      ('float64 boxes', (labels, bboxes.double(), masks)),
                      ('one float64 box', (labels[:1], bboxes[:1].double(), masks[:1]))):
        got = _check([ins], what=what)
        if what == 'uint8':
            assert got[0][1][int(labels[0])][0].dtype.name == 'uint8'


def test_results_intact_after_later_calls():
    """Each call writes into buffers of its own: a later call, even one whose inputs have the same shapes and whose
    earlier buffers are free again, never changes results that are still held."""
    ins_a, ins_b = _coco_ins(2, seed=6), _coco_ins(2, seed=7)
    first = _format(ins_a)
    snapshot = copy.deepcopy(first)
    second = _format(ins_b)
    del second
    third = _format(ins_b)
    torch.cuda.synchronize()
    obf.assert_same(first, snapshot, 'first call after two more')
    obf.assert_same(third, obf.maskformer_simple_test_tail(ins_b, 80), 'third call')
    obf.assert_same(first, obf.maskformer_simple_test_tail(ins_a, 80), 'first call against the oracle')


def _host_waits(fn, monkeypatch):
    """(synchronising calls sync-debug mode flags, the names of Event / Stream waits) of one call of fn."""
    waits = []
    for cls in (torch.cuda.Event, torch.cuda.Stream):
        orig = cls.synchronize
        monkeypatch.setattr(cls, 'synchronize', lambda *a, _o=orig, _n=cls.__name__: (waits.append(_n), _o(*a))[1])
    n = syncs(fn)
    monkeypatch.undo()
    return n, waits


@pytest.mark.parametrize('B', [1, 2])
def test_one_host_wait_per_call(B, monkeypatch, capsys):
    ins = _coco_ins(B, seed=8)
    _format(ins)                                                                   # warm up
    n_sync, waits = _host_waits(lambda: _format(ins), monkeypatch)
    n_ref = syncs(lambda: obf.maskformer_simple_test_tail(ins, 80))
    with capsys.disabled():
        print(f'\nB={B}: synchronising calls {n_sync}, event / stream waits {waits}; reference lines: {n_ref}')
    assert n_sync == 0 and waits == ['Event']
    assert n_ref >= 100 * B                                                       # one blocking copy per mask at least
    empty = [tuple(t[:0] for t in i) for i in ins]
    assert _host_waits(lambda: _format(empty), monkeypatch) == (0, [])           # no detections: no device work


def _detector(name, mask_cls, mask_pred, calls):
    """The registered detector on a stub backbone and the registered Box2MaskHead (forward stubbed) and fusion head."""
    from boxinstseg_b200.models import HEADS, build_head
    det = HEADS.get(name)()
    head = build_head(dict(type='Box2MaskHead', num_things_classes=80, num_stuff_classes=0, num_queries=100))
    head.forward = lambda feats, img_metas: (calls.append('forward'),
                                             ([mask_cls * 0, mask_cls], [mask_pred * 0, mask_pred], [None, None]))[1]
    det.extract_feat = lambda imgs: (calls.append('extract_feat'), ['feat'])[1]
    det.panoptic_head = head
    det.panoptic_fusion_head = build_head(dict(type='MaskFormerFusionHead', num_things_classes=80, num_stuff_classes=0,
                                               test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True,
                                                             max_per_image=100)))
    det.num_things_classes, det.num_stuff_classes = 80, 0
    return det


@pytest.mark.parametrize('name', ['Box2Mask', 'MaskFormer'])
def test_simple_test_equals_reference_tail(name, monkeypatch):
    mask_cls, mask_pred, metas = _coco(2, seed=9)
    calls = []
    det = _detector(name, mask_cls, mask_pred, calls)
    got = det.simple_test(torch.zeros(2, 3, 8, 8, device=DEV), metas, rescale=True)
    assert calls == ['extract_feat', 'forward']
    ins = [r['ins_results'] for r in det.panoptic_fusion_head.simple_test(mask_cls, mask_pred, metas, rescale=True)]
    obf.assert_same(got, obf.maskformer_simple_test_tail(ins, 80), name)
    assert len(got) == 2 and all(len(bbox) == len(masks) == 80 for bbox, masks in got)
    n_sync, waits = _host_waits(lambda: det.simple_test(None, metas, rescale=True), monkeypatch)
    assert n_sync == 0 and waits == ['Event']
