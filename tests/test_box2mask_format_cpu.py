"""Box2Mask's test-result formatting, CPU side: (1) the oracle (oracle/box2mask_format.py) on hand-built inputs -- an empty
image, every detection in one class, classes without detections, labels out of class order, VOC's 20 classes; (2) the
oracle on the golden Box2Mask inference cases (tests/golden/box2mask_infer.npz) against the golden labels, boxes and masks;
(3) what ``format_instance_results`` and ``Box2Mask.simple_test`` do without a device: empty images, the type checks, the
registration, and the merge with a reference class.  The GPU twin of this file is tests/test_box2mask_format_gpu.py."""
import types

import numpy as np
import pytest
import torch

from oracle import box2mask_format as obf
from oracle import box2mask_infer as obi
from oracle.make_golden_box2mask_infer import CASES, case


def _image(labels, H=6, W=7, seed=0):
    g = torch.Generator().manual_seed(seed)
    n = len(labels)
    bboxes = torch.rand(n, 5, generator=g) * 40
    masks = torch.rand(n, H, W, generator=g) < 0.3
    return torch.tensor(labels, dtype=torch.int64), bboxes, masks


def _expected(labels, bboxes, masks, C):
    """Per class the rows and masks of that class in detection order, grouped without the oracle's code."""
    lab = labels.tolist()
    rows = [[j for j, l in enumerate(lab) if l == c] for c in range(C)]
    return ([bboxes.numpy()[r].reshape(-1, 5) for r in rows], [[masks[j].numpy() for j in r] for r in rows])


@pytest.mark.parametrize('labels,C', [([2, 2, 2, 2], 4),            # every detection in one class
                                      ([3, 0, 3, 1, 0], 6),         # classes 2, 4, 5 without detection, out of order
                                      ([0], 1),
                                      ([19, 0, 7, 7, 19, 12, 3, 3, 0, 18, 11], 20)])     # VOC
def test_oracle_on_hand_built_images(labels, C):
    img = _image(labels, seed=len(labels))
    out = obf.maskformer_simple_test_tail([img], C)
    obf.assert_same(out, [_expected(*img, C)])
    bbox, masks = out[0]
    assert len(bbox) == len(masks) == C
    assert all(b.dtype == np.float32 and b.shape[1:] == (5,) for b in bbox)
    assert all(m.dtype == bool and m.shape == (6, 7) for ms in masks for m in ms)


def test_oracle_empty_image_has_one_array_per_class():
    out = obf.maskformer_simple_test_tail([(torch.zeros(0, dtype=torch.int64), torch.zeros(0, 5),
                                            torch.zeros(0, 4, 4, dtype=torch.bool))], 20)
    bbox, masks = out[0]
    assert [b.shape for b in bbox] == [(0, 5)] * 20 and all(b.dtype == np.float32 for b in bbox)
    assert len({id(b) for b in bbox}) == 20 and masks == [[] for _ in range(20)]


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_on_golden_inference_cases(golden, i):
    g = golden('box2mask_infer')
    name = CASES[i][0]
    mask_cls, mask_pred, metas, cfg = case(i)
    ora = obi.fusion_simple_test(mask_cls, mask_pred, metas, cfg['things'], cfg['max_per_image'], cfg['rescale'])
    out = obf.maskformer_simple_test_tail([(l, b, m) for l, _, b, m in ora], cfg['things'])
    assert len(out) == 2
    for b, (bbox, masks) in enumerate(out):
        gl, gb = g[f'{name}_{b}_labels'], g[f'{name}_{b}_bboxes']
        shape = tuple(g[f'{name}_{b}_mask_shape'])
        gm = np.unpackbits(g[f'{name}_{b}_masks'], axis=-1, count=shape[-1]).astype(bool)
        assert len(bbox) == len(masks) == cfg['things']
        for c in range(cfg['things']):
            want = gb[gl == c]
            assert bbox[c].dtype == np.float32 and bbox[c].shape == want.shape and bbox[c].tobytes() == want.tobytes()
            assert len(masks[c]) == len(want)
            for m, w in zip(masks[c], gm[gl == c]):
                assert m.dtype == bool and np.array_equal(m, w)
        assert sum(len(m) for m in masks) == len(gl)


def test_format_instance_results_without_device_work():
    """Images without detections need no device, whatever their tensors; detections on the CPU or in masks that are
    neither bool nor uint8 raise."""
    from boxinstseg_b200.models.detectors import format_instance_results
    empty = (torch.zeros(0, dtype=torch.int64), torch.zeros(0, 5), torch.zeros(0, 5, 6))
    out = format_instance_results([empty, empty], 3)
    obf.assert_same(out, obf.maskformer_simple_test_tail([empty, empty], 3))
    assert len({id(b) for b in out[0][0] + out[1][0]}) == 6
    assert format_instance_results([], 3) == []
    labels, bboxes, masks = _image([0, 1])
    with pytest.raises(TypeError):
        format_instance_results([(labels, bboxes, masks.float())], 3)
    with pytest.raises(RuntimeError, match='CUDA'):
        format_instance_results([(labels, bboxes, masks)], 3)


class _Stub:
    """extract_feat / panoptic_head / panoptic_fusion_head of a detector, recording their calls."""

    def __init__(self, results):
        self.calls, self.results = [], results
        self.panoptic_head = types.SimpleNamespace(simple_test=self.head)
        self.panoptic_fusion_head = types.SimpleNamespace(simple_test=self.fusion)

    def extract_feat(self, imgs):
        self.calls.append(('extract_feat', imgs))
        return 'feats'

    def head(self, feats, img_metas, **kw):
        self.calls.append(('panoptic_head', feats, img_metas, kw))
        return 'cls', 'pred'

    def fusion(self, cls, pred, img_metas, **kw):
        self.calls.append(('panoptic_fusion_head', cls, pred, img_metas, kw))
        return self.results()


@pytest.mark.parametrize('name', ['Box2Mask', 'MaskFormer'])
def test_simple_test_on_stubs_without_detections(name):
    from boxinstseg_b200.models import HEADS
    det = HEADS.get(name)()
    empty = lambda: (torch.zeros(0, dtype=torch.int64), torch.zeros(0, 5), torch.zeros(0, 3, 4, dtype=torch.bool))  # noqa
    stub = _Stub(lambda: [dict(ins_results=empty()), dict(ins_results=empty())])
    det.extract_feat, det.panoptic_head, det.panoptic_fusion_head = (stub.extract_feat, stub.panoptic_head,
                                                                     stub.panoptic_fusion_head)
    det.num_things_classes, det.num_stuff_classes = 4, 0
    out = det.simple_test('imgs', ['m0', 'm1'], rescale=True)
    obf.assert_same(out, obf.maskformer_simple_test_tail([empty(), empty()], 4))
    assert [c[0] for c in stub.calls] == ['extract_feat', 'panoptic_head', 'panoptic_fusion_head']
    assert stub.calls[1] == ('panoptic_head', 'feats', ['m0', 'm1'], dict(rescale=True))
    assert stub.calls[2] == ('panoptic_fusion_head', 'cls', 'pred', ['m0', 'm1'], dict(rescale=True))
    # with stuff classes the per-image dicts stay; a panoptic map is copied to numpy; semantic output is refused
    det.num_stuff_classes = 2
    stub.results = lambda: [dict(ins_results=empty(), pan_results=torch.ones(3, 4, dtype=torch.int32))]
    (res,) = det.simple_test('imgs', ['m0'])
    assert isinstance(res['pan_results'], np.ndarray) and res['pan_results'].shape == (3, 4)
    obf.assert_same([res['ins_results']], obf.maskformer_simple_test_tail([empty()], 4))
    stub.results = lambda: [dict(sem_results=None)]
    with pytest.raises(AssertionError):
        det.simple_test('imgs', ['m0'])


def test_registered_detectors():
    from boxinstseg_b200.models import HEADS
    from boxinstseg_b200.models.detectors import Box2Mask, MaskFormer
    assert HEADS.get('Box2Mask') is Box2Mask and HEADS.get('MaskFormer') is MaskFormer
    assert issubclass(Box2Mask, MaskFormer) and Box2Mask.simple_test is MaskFormer.simple_test


def test_registration_merges_with_the_reference_detectors():
    """With mmdet importable, the registered Box2Mask is this package's class and the reference's: the reference's
    constructor and every other method, this package's simple_test.  Simulated with stand-in reference classes."""
    from boxinstseg_b200.models import builder as b
    from boxinstseg_b200.models.detectors import box2mask
    if b.HAVE_MMDET:
        return
    reg = b.Registry('sim')

    class RefMaskFormer:
        def __init__(self, backbone=None, test_cfg=None):
            self.backbone, self.test_cfg = backbone, test_cfg

        def simple_test(self, imgs, img_metas, **kwargs):
            return 'reference simple_test'

        def aug_test(self, imgs, img_metas, **kwargs):
            return 'reference aug_test'

    class RefBox2Mask(RefMaskFormer):
        pass
    reg.register_module(name='MaskFormer', module=RefMaskFormer)
    reg.register_module(name='Box2Mask', module=RefBox2Mask)
    MF = b.register(reg, partial=True)(type('MaskFormer', (), {'simple_test': box2mask.MaskFormer.simple_test}))
    B2M = b.register(reg, partial=True)(type('Box2Mask', (MF,), {}))
    det = reg.build(dict(type='Box2Mask', backbone='r50', test_cfg={}))
    assert isinstance(det, RefBox2Mask) and isinstance(det, RefMaskFormer) and isinstance(det, MF)
    assert type(det) is B2M and det.backbone == 'r50'
    assert det.aug_test(None, None) == 'reference aug_test'
    assert type(det).simple_test is box2mask.MaskFormer.simple_test
