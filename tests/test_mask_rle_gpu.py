"""COCO RLE of mask results on the GPU (csrc/mask_rle.cu, ops/mask_rle.py, core/mask.py ``encode_mask_results``) against
the golden vectors of the reference's ``encode_mask_results`` and the oracle's restatement of pycocotools (oracle/
mask_rle.py): every golden case from host and CUDA inputs, the run counts on their own, COCO-sized and odd-sized masks,
more masks than one grid dimension holds, every pixel a run, non-contiguous, misaligned and uint8 masks, the real outputs of
the three inference paths, the host waits, no device work for no masks, determinism, and pycocotools itself where it can be
imported."""

import numpy as np
import pytest
import torch

from oracle import mask_rle as omr
from oracle.make_golden_mask_rle import CASES, case, segms_of
from tests.test_mask_rle_cpu import golden_case, oracle_encode
from tools.benchkit import launches, syncs

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _blobs(n, H, W, seed):
    """n seeded bool masks [n, H, W] on the device: thresholded smooth noise, so that each holds a few blobs."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    low = torch.randn(n, 1, max(2, H // 40), max(2, W // 40), generator=g, device=DEV)
    up = torch.nn.functional.interpolate(low, (H, W), mode='bilinear', align_corners=False)[:, 0]
    return up > 0.8


def _alternating(H, W):
    """[H, W] with every pixel its own column-major run, the first pixel set: H * W + 1 counts."""
    j = torch.arange(W, device=DEV)[None, :] * H + torch.arange(H, device=DEV)[:, None]
    return (j % 2 == 0)


def _oracle(masks):
    """The oracle's RLE dicts of [n, H, W] masks (any device), as the reference's encode_mask_results calls it."""
    return [oracle_encode(m) for m in masks.cpu().numpy()]


def _as_host_and_cuda(results, to_cuda):
    """A case's mask results with every mask as it is (host) or moved to CUDA (per-class [k, H, W] arrays whole)."""
    if not to_cuda:
        return results
    segms = segms_of(results)
    moved = [torch.as_tensor(np.asarray(per)).to(DEV) if isinstance(per, np.ndarray)
             else [torch.as_tensor(m).to(DEV) for m in per] for per in segms]
    return (moved, results[1]) if isinstance(results, tuple) else moved


@pytest.mark.parametrize('to_cuda', [False, True], ids=['host', 'cuda'])
@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_golden_cases(golden, i, to_cuda):
    from boxinstseg_b200.core import encode_mask_results
    name = CASES[i][0]
    _, per_class, expected = golden_case(golden('mask_rle'), name)
    results = _as_host_and_cuda(case(i), to_cuda)
    out = encode_mask_results(results)
    if isinstance(results, tuple):
        assert isinstance(out, tuple) and out[1] is results[1]
        out = out[0]
    assert [len(per) for per in out] == per_class.tolist()
    rles = [r for per in out for r in per]
    masks = [m for per in segms_of(results) for m in per]
    assert [r['counts'] for r in rles] == expected
    for r, m in zip(rles, masks):
        assert r['size'] == list(m.shape) and all(type(v) is int for v in r['size'])
    assert encode_mask_results(out) == out                                  # already encoded: unchanged


@pytest.mark.parametrize('shape', [(100, 480, 640), (9, 427, 641), (70000, 3, 5), (3, 1, 33), (4, 31, 1)])
@pytest.mark.parametrize('dtype', [torch.bool, torch.uint8])
def test_counts_and_strings_equal_oracle(shape, dtype):
    """Seeded blob masks at COCO size and an odd size, more than 65535 tiny masks, one-row and one-column masks."""
    from boxinstseg_b200.ops import mask_rle
    n, H, W = shape
    masks = _blobs(n, H, W, seed=sum(shape)) if H * W > 100 else \
        torch.rand(shape, generator=torch.Generator(device=DEV).manual_seed(n), device=DEV) < 0.5
    masks[::5] = False
    masks[1::7] = True
    if dtype == torch.uint8:
        masks = masks.to(torch.uint8)
    counts, offsets = mask_rle.rle_counts(masks)
    host = masks.cpu().numpy()
    ref = [omr.counts(m.T) for m in host]
    assert counts.dtype == torch.int32 and offsets.dtype == torch.int64 and offsets.shape == (n + 1,)
    assert offsets.cpu().tolist() == np.concatenate(([0], np.cumsum([len(c) for c in ref]))).tolist()
    assert np.array_equal(counts.cpu().numpy(), np.concatenate(ref).astype(np.int32))
    got = mask_rle.encode(masks)
    assert got == _oracle(masks)


def test_every_pixel_a_run():
    from boxinstseg_b200.ops import mask_rle
    m = torch.stack([_alternating(480, 640), ~_alternating(480, 640)])
    counts, offsets = mask_rle.rle_counts(m)
    assert offsets.cpu().tolist() == [0, 307201, 307201 + 307200]
    assert counts[0].item() == 0 and bool((counts[1:] == 1).all())
    assert mask_rle.encode(m) == _oracle(m)


def test_layouts_and_uint8_values():
    """Non-contiguous views, a base one byte into its buffer (the byte path), W % 4 != 0, and uint8 values above 1 with
    changes between non-zero values."""
    from boxinstseg_b200.ops import mask_rle
    base = _blobs(6, 64, 96, seed=3)
    t = base.transpose(1, 2).contiguous().transpose(1, 2)                   # same values, column-major strides
    assert not t.is_contiguous()
    assert mask_rle.encode(t) == _oracle(base)
    strided = torch.zeros(6, 64, 192, dtype=torch.bool, device=DEV)
    strided[:, :, ::2] = base
    assert mask_rle.encode(strided[:, :, ::2]) == _oracle(base)
    flat = torch.zeros(6 * 64 * 96 + 1, dtype=torch.uint8, device=DEV)
    mis = flat[1:].view(6, 64, 96)
    mis.copy_(base)
    assert mis.is_contiguous() and mis.data_ptr() % 4
    assert mask_rle.encode(mis) == _oracle(base)
    g = torch.Generator(device=DEV).manual_seed(9)
    vals = base.to(torch.uint8) * torch.randint(1, 256, (6, 1, 1), generator=g, device=DEV, dtype=torch.uint8)
    vals[2] = torch.randint(0, 4, (64, 96), generator=g, device=DEV, dtype=torch.uint8)
    vals[3, 10:40, 20:50] = 9
    for v in (vals, vals[:, :, :93]):
        assert mask_rle.encode(v) == _oracle(v)
        counts, _ = mask_rle.rle_counts(v)
        assert np.array_equal(counts.cpu().numpy(), np.concatenate([omr.counts(m.T) for m in v.cpu().numpy()]))


def test_zero_sized_masks():
    from boxinstseg_b200.ops import mask_rle
    for shape in ((3, 0, 5), (2, 4, 0)):
        m = torch.zeros(shape, dtype=torch.bool, device=DEV)
        assert mask_rle.encode(m) == _oracle(m)


def _count_waits(fn, monkeypatch):
    """(synchronising calls sync-debug mode flags, [event / stream waits]) of one call of fn.  Sync-debug mode does not
    flag an event wait, so Event.synchronize and Stream.synchronize are wrapped and counted."""
    waits = []
    for cls in (torch.cuda.Event, torch.cuda.Stream):
        orig = cls.synchronize
        monkeypatch.setattr(cls, 'synchronize', lambda *a, _o=orig, _n=cls.__name__: (waits.append(_n), _o(*a))[1])
    n = syncs(fn)
    monkeypatch.undo()
    return n, waits


@pytest.mark.parametrize('form', ['host', 'cuda', 'device_op'])
def test_two_host_waits_per_group(form, monkeypatch, capsys):
    from boxinstseg_b200.core import encode_mask_results
    from boxinstseg_b200.ops import mask_rle
    masks = _blobs(100, 480, 640, seed=1)
    if form == 'device_op':
        fn = lambda: mask_rle.encode(masks)                                   # noqa: E731
    else:
        src = masks.cpu().numpy() if form == 'host' else masks
        per_class = [list(src[c::7]) for c in range(7)]
        fn = lambda: encode_mask_results(per_class)                          # noqa: E731
    fn()                                                                       # warm up
    n, waits = _count_waits(fn, monkeypatch)
    with capsys.disabled():
        print(f'\n{form}: synchronising calls {n}, event / stream waits {waits}')
    assert n == 0 and waits == ['Event', 'Event']
    two_groups = [list(masks[:3]), [masks[0, :, :320]]]
    n, waits = _count_waits(lambda: encode_mask_results(two_groups), monkeypatch)
    assert n == 0 and waits == ['Event'] * 4


def test_no_device_work_without_masks():
    from boxinstseg_b200.core import encode_mask_results
    from boxinstseg_b200.ops import mask_rle
    empty = torch.zeros(0, 480, 640, dtype=torch.bool, device=DEV)
    assert launches(lambda: mask_rle.encode(empty)) == 0
    assert launches(lambda: encode_mask_results([[], np.zeros((0, 4, 4), np.uint8), []])) == 0
    assert mask_rle.encode(empty) == []


def test_deterministic():
    from boxinstseg_b200.ops import mask_rle
    m = _blobs(100, 480, 640, seed=5)
    noise = torch.rand(20, 480, 640, device=DEV) < 0.5
    for x in (m, noise):
        a, b = mask_rle.encode(x), mask_rle.encode(x)
        assert a == b
        c1, o1 = mask_rle.rle_counts(x)
        c2, o2 = mask_rle.rle_counts(x)
        assert torch.equal(c1, c2) and torch.equal(o1, o2)


def _check_against_oracle(per_class):
    from boxinstseg_b200.core import encode_mask_results
    ref = [[oracle_encode(np.asarray(m.cpu() if isinstance(m, torch.Tensor) else m)) for m in per] for per in per_class]
    assert encode_mask_results(per_class) == ref
    assert sum(len(r) for r in ref) > 0
    return ref


def test_end_to_end_solov2_format_results():
    from boxinstseg_b200.core import encode_mask_results
    from boxinstseg_b200.models import build_head
    from boxinstseg_b200.models.detectors.solo import format_results
    from oracle.make_golden_solo_seg import case as seg_case, cfg_of
    head, (seg, cate, _), metas = seg_case(0, 'box', B=2, h=24, w=32, img_shape=(90, 120, 3), ori_shape=(75, 101, 3),
                                           device=DEV)
    bh = build_head(dict(type='BoxSOLOv2Head', num_classes=5, num_grids=list(head.seg_num_grids), strides=list(head.strides)))
    outs = bh.get_seg(seg, cate, None, metas, dict(cfg_of({}).__dict__))
    assert sum(len(r.labels) for r in outs) > 0
    for r in outs:
        _, (mask_results, score_results) = format_results(r, 5)              # pinned host views, 0-d scores
        out = encode_mask_results((mask_results, score_results))
        assert out[1] is score_results
        assert out[0] == [[oracle_encode(m.numpy()) for m in per] for per in mask_results]


def test_end_to_end_condinst_simple_test():
    from boxinstseg_b200.models.dense_heads.condinst_box_head import CondInstBoxHead
    from boxinstseg_b200.models.dense_heads.condinst_mask_head import CondInstMaskHead
    from oracle.make_golden_condinst_infer import MASK_CH, NUM_CLASSES, SOI, STRIDES, case as ci_case, cfg_of
    cls, bbox, ctr, prm, feat, metas = ci_case(0, device=DEV)
    dets = CondInstBoxHead(num_classes=NUM_CLASSES, strides=STRIDES, test_cfg=cfg_of({})).get_bboxes(
        cls, bbox, ctr, prm, metas, rescale=True)
    mh = CondInstMaskHead(in_channels=MASK_CH, sizes_of_interest=list(SOI)).to(DEV)
    segm = mh.simple_test(feat, *[[d[i] for d in dets] for i in (1, 2, 3, 4)], metas, NUM_CLASSES, rescale=True)
    for s in segm:                                                            # per class [k, H, W] uint8 arrays
        if sum(len(m) for m in s):
            _check_against_oracle(s)


def test_end_to_end_maskformer_fusion():
    from boxinstseg_b200.models.dense_heads.box2mask_infer import MaskFormerFusionHead
    g = torch.Generator().manual_seed(17)
    mask_cls = (torch.randn(2, 100, 81, generator=g) * 3).to(DEV)
    low = torch.randn(2, 100, 25, 34, generator=g) * 4
    mask_pred = torch.nn.functional.interpolate(low, (200, 272), mode='bilinear', align_corners=False).to(DEV)
    metas = [dict(img_shape=(800, 1067, 3), ori_shape=o + (3,), batch_input_shape=(800, 1088)) for o in ((480, 640),
                                                                                                          (427, 640))]
    fusion = MaskFormerFusionHead(80, 0, test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True,
                                                       max_per_image=100))
    for r in fusion.simple_test(mask_cls, mask_pred, metas, rescale=True):
        labels, _, masks = r['ins_results']
        assert masks.dtype == torch.bool and masks.is_cuda
        on_device = [[] for _ in range(80)]
        on_host = [[] for _ in range(80)]
        for j, label in enumerate(labels.tolist()):
            on_device[label].append(masks[j])
            on_host[label].append(masks[j].detach().cpu().numpy())            # the reference's per-mask copy
        ref = _check_against_oracle(on_device)
        from boxinstseg_b200.core import encode_mask_results
        assert encode_mask_results(on_host) == ref


def test_pycocotools_cross_check(golden):
    """Everything above against pycocotools.mask.encode itself, where it is installed."""
    mask_util = pytest.importorskip('pycocotools.mask')
    from boxinstseg_b200.ops import mask_rle

    def ref(masks):
        host = np.asfortranarray(masks.cpu().numpy().astype(np.uint8).transpose(1, 2, 0))
        return [{'size': list(r['size']), 'counts': r['counts']} for r in mask_util.encode(host)]
    for i, (name, _) in enumerate(CASES):
        _, _, expected = golden_case(golden('mask_rle'), name)
        masks = [np.asarray(m) for per in segms_of(case(i)) for m in per]
        assert [mask_util.encode(np.array(m[:, :, None], order='F', dtype='uint8'))[0]['counts'] for m in masks] \
            == expected, name
    vals = _blobs(6, 64, 96, seed=3).to(torch.uint8) * 3
    vals[2, 10:40, 20:50] = 200
    for m in (_blobs(100, 480, 640, seed=1), _blobs(9, 427, 641, seed=2), torch.stack([_alternating(480, 640)]), vals):
        assert mask_rle.encode(m) == ref(m)
