"""CondInst inference, CPU side: (1) the oracle (oracle/condinst_infer.py) reproduces the golden vectors minted from the
reference's own ``get_bboxes`` / ``_get_bboxes`` / ``nms_with_others`` and ``CondInstMaskHead.simple_test``
(oracle/make_golden_condinst_infer.py); (2) the HOST build of the kernels' arithmetic (csrc/box_nms_core.cuh through
tests/host_harness/box_nms_host.cpp) against the oracle: the decode bit for bit, mmcv's suppression test on pairs built to
sit exactly on ``interS == thr * union`` after the class offset, equal scores and NaN boxes, and the aligned_bilinear
taps; (3) the argument checks of the new C entry points and ops without a GPU.  The GPU twin is
tests/test_condinst_infer_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import condinst_infer as oci
from oracle.make_golden_condinst_infer import CASES, NUM_CLASSES, STRIDES, case, cfg_of, oracle_masks
from tests.helpers import host_twin


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize('seed', range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_reproduces_reference_golden(golden, seed):
    g = golden('condinst_infer')
    name, kw, over, rescale, with_nms = CASES[seed]
    cls, bbox, ctr, prm, feat, metas = case(seed, **kw)
    out = oci.get_bboxes(cls, bbox, ctr, prm, metas, cfg_of(over), STRIDES, rescale, with_nms)
    for b, r in enumerate(out):
        for i, v in enumerate(r):
            assert np.array_equal(v.numpy(), g[f'{name}_{b}_{i}']), (b, i)
    if with_nms:
        keep = [b for b in range(len(out)) if len(out[b][0])]
        masks = oracle_masks([out[b] for b in keep], feat[keep], [metas[b] for b in keep], rescale)
        for b, m in zip(keep, masks):
            assert tuple(m.shape) == tuple(g[f'{name}_{b}_mask_shape'])
            assert np.array_equal(np.packbits(m.numpy(), axis=-1), g[f'{name}_{b}_masks'])


def test_golden_covers_the_issue_cases(golden):
    g = golden('condinst_infer')
    assert len(g['truncate_0_0']) == 4 and len(g['no_candidate_0_0']) == 0
    assert len(g['one_empty_0_0']) > 0 and len(g['one_empty_1_0']) == 0 and 'one_empty_1_masks' not in g
    assert g['no_nms_0_1'].shape[-1] == NUM_CLASSES + 1


def test_host_twin_decode_equals_oracle():
    lib = host_twin('box_nms_host')
    gen = torch.Generator().manual_seed(3)
    pts = oci.points([(9, 13)], [16])[0]
    d = torch.rand(len(pts), 4, generator=gen) * 200 - 20
    d[5, 0] = float('nan')
    sf = torch.tensor([1.37, 1.21, 1.37, 1.21])
    for scale in (None, sf):
        out = torch.empty(len(pts), 4)
        lib.host_decode(len(pts), _p(pts), _p(d), ctypes.c_float(100.), ctypes.c_float(150.), None if scale is None else _p(scale), _p(out))
        ref = oci.distance2bbox(pts[None], d[None], [(100, 150, 3)])[0]
        if scale is not None:
            ref = ref / scale
        assert torch.equal(out.isnan(), ref.isnan()) and torch.equal(out.nan_to_num(), ref.nan_to_num())


def _boundary_pairs():
    """Box pairs whose offset boxes (label 1, max coordinate 40) sit exactly on interS == 0.5 * union, and their
    neighbours one ulp away: [a, b] float32."""
    off = torch.tensor(1.) * (torch.tensor(40.) + 1)
    pairs = []
    for x1 in (0., 4., 10.):
        a = torch.tensor([x1, 0., x1 + 20., 10.])
        b = torch.tensor([x1, 0., x1 + 10., 10.])             # inter 100, union 200: exactly on the threshold
        pairs += [(a, b), (a, b + torch.tensor([0., 0., 1e-3, 0.])), (a, b - torch.tensor([0., 0., 1e-3, 0.]))]
        pairs.append((a, torch.tensor([x1 + 30., 0., x1 + 31., 1.])))                  # disjoint
        pairs.append((a, torch.tensor([float('nan'), 0., x1 + 20., 10.])))              # a NaN coordinate
    return torch.stack([torch.stack([a + off, b + off]) for a, b in pairs])


def test_host_twin_suppression_equals_oracle_on_boundary_and_nan_pairs():
    lib = host_twin('box_nms_host')
    pairs = _boundary_pairs()
    gen = torch.Generator().manual_seed(5)
    xy = torch.rand(60, 2, generator=gen) * 50
    rand = torch.cat([xy, xy + torch.rand(60, 2, generator=gen) * 30 + 1], 1)
    for boxes in [p for p in pairs] + [rand]:
        boxes = boxes.contiguous()
        n = len(boxes)
        for thr in (0.5, 0.3, 0.7):
            sup = torch.empty(n, n, dtype=torch.uint8)
            lib.host_suppress(n, _p(boxes), ctypes.c_float(thr), _p(sup))
            assert torch.equal(sup.bool(), oci.suppresses(boxes[:, None], boxes[None], thr))
    on = pairs[0]
    assert not oci.suppresses(on[0], on[1], 0.5) and oci.suppresses(on[0], on[1], 0.4999)   # strict '>' at the boundary


def test_host_twin_greedy_equals_oracle_nms_with_equal_scores():
    lib = host_twin('box_nms_host')
    gen = torch.Generator().manual_seed(7)
    xy = torch.rand(80, 2, generator=gen) * 60
    boxes = torch.cat([xy, xy + torch.rand(80, 2, generator=gen) * 25 + 1], 1)
    scores = (torch.rand(80, generator=gen) * 8).floor() / 8                # many equal scores
    order = torch.sort(scores, descending=True, stable=True)[1]
    keep = torch.empty(80, dtype=torch.uint8)
    sorted_boxes = boxes[order].contiguous()
    lib.host_greedy(80, _p(sorted_boxes), ctypes.c_float(0.5), _p(keep))
    _, inds = oci.nms(boxes, scores, 0.5, stable=True)
    assert torch.equal(order[keep.bool()], inds)


@pytest.mark.parametrize('shape', [((5, 7), 4, (18, 25)), ((8, 10), 4, (32, 40)), ((6, 6), 2, (11, 9))])
def test_host_twin_aligned_bilinear_equals_oracle(shape):
    (h, w), f, (H, W) = shape
    lib = host_twin('box_nms_host')
    p = torch.rand(h, w, generator=torch.Generator().manual_seed(h * w))
    out = torch.empty(H, W)
    lib.host_aligned(_p(p), h, w, f, H, W, _p(out))
    ref = oci.aligned_bilinear(p[None, None], f)[0, 0, :H, :W]
    assert (out - ref).abs().max() <= 1e-6


def test_ops_reject_unsupported_settings_and_cpu_tensors():
    from boxinstseg_b200.ops import box_nms
    from boxinstseg_b200.ops.condinst import paste_masks
    b, s, i = torch.rand(3, 4), torch.rand(3), torch.zeros(3, dtype=torch.long)
    with pytest.raises(NotImplementedError):
        box_nms.batched_nms(b, s, i, dict(type='soft_nms', iou_threshold=0.5))
    with pytest.raises(NotImplementedError):
        box_nms.batched_nms(b, s, i, dict(type='nms', iou_threshold=0.5), class_agnostic=True)
    with pytest.raises(RuntimeError):
        box_nms.batched_nms(b, s, i, dict(type='nms', iou_threshold=0.5, split_thr=2))
    with pytest.raises(RuntimeError):
        paste_masks(torch.rand(2, 1, 4, 4), 4, (16, 16, 3))


def test_c_abi_argument_checks():
    from boxinstseg_b200 import _lib
    h = _lib.lib()
    buf = ctypes.cast((ctypes.c_float * 4096)(), ctypes.c_void_p)
    ptrs = (ctypes.c_void_p * 2)(buf.value, buf.value)
    nul = (ctypes.c_void_p * 2)(None, None)
    st = (ctypes.c_int64 * 8)(*[1] * 8)
    H, W = (ctypes.c_int64 * 2)(4, 2), (ctypes.c_int64 * 2)(4, 2)
    strides = (ctypes.c_float * 2)(8., 16.)
    k_ok, k_bad = (ctypes.c_int64 * 2)(5, 4), (ctypes.c_int64 * 2)(17, 4)
    hw = (ctypes.c_float * 2)(32., 32.)
    ps = h.bxs_condinst_point_scores
    assert ps(nul, st, ptrs, st, H, W, 2, 1, 3, 16, buf, None) == -1              # NULL level pointer
    assert ps(ptrs, st, ptrs, st, H, W, 2, 1, 3, 15, buf, None) == -1             # P_max below a level's size
    assert ps(ptrs, st, ptrs, st, H, W, 9, 1, 3, 16, buf, None) == -3             # more than 8 levels
    assert ps(ptrs, st, ptrs, st, H, W, 2, 33, 3, 16, buf, None) == -3            # more than 32 images
    dec = h.bxs_condinst_decode
    args = lambda k, order: (ptrs, st, ptrs, st, ptrs, st, H, W, strides, k, 2, 1, 3, order, 16, hw, None, ctypes.c_float(0.05),
                             buf, buf, buf, buf, buf, None, None)
    assert dec(*args(k_bad, buf)) == -1                                           # k above the level's size
    assert dec(*args(k_ok, None)) == -1                                           # level 0 cut but no order
    assert h.bxs_condinst_gather(ptrs, st, H, W, strides, k_ok, 2, 1, 0, buf, buf, 1, buf, buf, buf, None) == -1   # P = 0
    counts = (ctypes.c_int64 * 3)(3, 0, 70)
    assert h.bxs_box_nms_workspace_bytes(counts, 3) == (3 * 1 + 70 * 2) * 8
    assert h.bxs_box_nms(buf, buf, buf, 4, 0, 4, ctypes.c_float(0.5), buf, buf, None) == -1           # no segment
    assert h.bxs_box_nms(buf, buf, buf, 4, 1, 400000, ctypes.c_float(0.5), buf, buf, None) == -3      # segment too long
    off = ctypes.c_void_p(buf.value + 4)
    assert h.bxs_box_nms(off, buf, buf, 4, 1, 4, ctypes.c_float(0.5), buf, buf, None) == -1           # misaligned boxes
    paste = h.bxs_condinst_paste_masks
    assert paste(buf, 1, 4, 4, 4, 17, 16, 17, 16, 0, buf, None) == -1             # crop beyond factor * h
    assert paste(buf, 1, 4, 4, 4, 16, 16, 10, 10, 0, buf, None) == -1             # resize without rescale
    assert paste(None, 1, 4, 4, 4, 16, 16, 10, 10, 1, buf, None) == -1            # NULL logits
