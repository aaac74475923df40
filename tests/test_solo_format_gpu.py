"""``format_results`` of BoxLevelSet / DiscoBoxSOLOv2 on the GPU (csrc/solo_seg.cu ``bxs_mask_extents``, ops/solo_seg.py
``mask_extents``, models/detectors/solo.py) against the oracle's restatement of the reference (oracle/solo_format.py) on the
same CUDA results: every golden case, uint8 masks, more masks than one grid dimension holds, non-contiguous and misaligned
masks, the host waits per image, both heads' ``get_seg`` output end to end, and determinism."""
import types

import pytest
import torch

from oracle import solo_format as osf
from oracle import solo_seg as oss
from oracle.make_golden_solo_format import CASES, assert_same, case
from oracle.make_golden_solo_seg import case as seg_case, cfg_of
from tools.benchkit import syncs

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _extents_ref(masks):
    """area and box of [n, H, W] masks from whole-tensor torch reductions."""
    on = masks != 0
    area = on.sum((1, 2)).int()
    rows, cols = on.any(2), on.any(1)
    H, W = masks.shape[1:]
    ar = lambda k: torch.arange(k, device=masks.device)                     # noqa: E731
    y0 = torch.where(rows, ar(H), H).min(1).values
    y1 = torch.where(rows, ar(H), -1).max(1).values + 1
    x0 = torch.where(cols, ar(W), W).min(1).values
    x1 = torch.where(cols, ar(W), -1).max(1).values + 1
    box = torch.stack([x0, y0, x1, y1], 1).float() * (area > 0)[:, None]
    return area, box


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_golden_cases_equal_oracle(i):
    from boxinstseg_b200.models.detectors.solo import format_results
    results, C = case(i, device=DEV)
    assert_same(format_results(results, C), osf.format_results(results, C), CASES[i][0])


@pytest.mark.parametrize('shape', [(70000, 4, 16), (66000, 3, 7), (100, 480, 640), (9, 427, 641), (5, 1, 16)])
@pytest.mark.parametrize('dtype', [torch.bool, torch.uint8])
def test_mask_extents_equal_torch(shape, dtype):
    """The vector path (W % 16 == 0), the byte path, more masks than 65535, COCO size, uint8 values above 1."""
    from boxinstseg_b200.ops.solo_seg import mask_extents
    g = torch.Generator(device=DEV).manual_seed(sum(shape))
    n, H, W = shape
    masks = (torch.rand(shape, generator=g, device=DEV) < torch.rand(n, 1, 1, generator=g, device=DEV) ** 8)
    masks[::4] = False
    if dtype == torch.uint8:
        masks = masks.to(torch.uint8) * torch.randint(1, 256, (n, 1, 1), generator=g, device=DEV, dtype=torch.uint8)
    area, box = mask_extents(masks)
    ra, rb = _extents_ref(masks)
    assert area.dtype == torch.int32 and box.dtype == torch.float32
    assert torch.equal(area, ra) and torch.equal(box, rb)


def test_mask_extents_misaligned_base():
    """A dense view that starts one byte into its buffer is read byte by byte."""
    from boxinstseg_b200.ops.solo_seg import mask_extents
    n, H, W = 7, 48, 64
    flat = torch.rand(n * H * W + 1, device=DEV) < 0.001
    masks = flat[1:].view(n, H, W)
    assert masks.is_contiguous() and masks.data_ptr() % 16
    area, box = mask_extents(masks)
    ra, rb = _extents_ref(masks)
    assert torch.equal(area, ra) and torch.equal(box, rb)


def test_noncontiguous_masks():
    from boxinstseg_b200.models.detectors.solo import format_results
    results, C = case(0, device=DEV)
    big = torch.zeros(results.masks.shape[0], results.masks.shape[2], results.masks.shape[1] * 2, dtype=torch.bool,
                      device=DEV)
    big[:, :, ::2] = results.masks.transpose(1, 2)
    results.masks = big[:, :, ::2].transpose(1, 2)
    assert not results.masks.is_contiguous()
    assert_same(format_results(results, C), osf.format_results(results, C), 'noncontiguous')


@pytest.mark.parametrize('i', [0, 1, 6, 8], ids=[CASES[i][0] for i in (0, 1, 6, 8)])
def test_one_host_wait_per_image(i, monkeypatch, capsys):
    """No synchronising call that sync-debug mode flags, and one event wait for an image with detections (none for
    n == 0).  Sync-debug mode does not flag an event wait, so Event.synchronize (and Stream.synchronize) are wrapped and
    counted."""
    from boxinstseg_b200.models.detectors.solo import format_results
    results, C = case(i, device=DEV)
    format_results(results, C)                                                   # warm up
    waits = []
    for cls in (torch.cuda.Event, torch.cuda.Stream):
        orig = cls.synchronize
        monkeypatch.setattr(cls, 'synchronize', lambda *a, _o=orig, _n=cls.__name__: (waits.append(_n), _o(*a))[1])
    n_sync = syncs(lambda: format_results(results, C))
    monkeypatch.undo()
    n_ref = syncs(lambda: osf.format_results(results, C))
    with capsys.disabled():
        print(f'\n{CASES[i][0]}: synchronising calls {n_sync}, event / stream waits {waits}; reference lines: {n_ref}')
    assert n_sync == 0
    assert waits == (['Event'] if len(results.labels) else [])


def _check_detectors(outs, C):
    from boxinstseg_b200.models import HEADS
    from boxinstseg_b200.models.detectors.solo import format_results
    dets = [HEADS.get(n)() for n in ('BoxLevelSet', 'DiscoBoxSOLOv2')]
    for d in dets:
        d.bbox_head = types.SimpleNamespace(num_classes=C)
    for r in outs:
        ref = osf.format_results(r, C)
        assert_same(format_results(r, C), ref, 'format_results')
        for d in dets:
            assert_same(d.format_results(r), ref, type(d).__name__)
    return [format_results(r, C) for r in outs]


def test_end_to_end_box_solov2():
    from boxinstseg_b200.models import build_head
    head, (seg, cate, _), metas = seg_case(0, 'box', B=2, h=24, w=32, img_shape=(90, 120, 3), ori_shape=(75, 101, 3),
                                           device=DEV)
    bh = build_head(dict(type='BoxSOLOv2Head', num_classes=5, num_grids=list(head.seg_num_grids), strides=list(head.strides)))
    cfg = dict(cfg_of({}).__dict__)
    outs = bh.get_seg(seg, cate, None, metas, cfg)
    assert sum(len(r.scores) for r in outs) > 0
    a = _check_detectors(outs, 5)
    b = _check_detectors(bh.get_seg(seg, cate, None, metas, cfg), 5)
    for x, y in zip(a, b):                                                        # determinism across two runs
        assert_same(x, y, 'determinism')


def test_end_to_end_discobox_autocast():
    from boxinstseg_b200.models import build_head
    head, (cate, kern, feat), metas = seg_case(7, 'disco', B=2, h=48, w=64, C=80, E=32, grids=(40, 36, 24, 16, 12),
                                               strides=(8, 8, 16, 32, 32), img_shape=(180, 250, 3),
                                               ori_shape=(300, 420, 3), device=DEV)
    flat = torch.cat([c.reshape(-1) for c in cate])
    cfg = dict(score_thr=float(flat.topk(401).values[-1]), mask_thr=0.4, nms_pre=500, max_per_img=100, kernel='gaussian',
               sigma=2.0, filter_thr=0.0)
    dh = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, num_grids=list(head.seg_num_grids),
                         strides=list(head.strides)))
    outs = dh.get_seg(cate, kern, feat, metas, cfg)                               # float16 autocast inside
    assert sum(len(r.scores) for r in outs) > 0
    a = _check_detectors(outs, 80)
    b = _check_detectors(outs, 80)
    for x, y in zip(a, b):
        assert_same(x, y, 'determinism')
