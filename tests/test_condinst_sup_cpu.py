"""CondInst's mask-supervised losses, CPU side: the oracle (oracle/condinst_sup.py) reproduces the golden vectors minted
from the reference's own code (oracle/make_golden_condinst_sup.py) -- label maps exactly, losses and gradients to 1e-6 --
and its label maps equal an explicit first-index scan; ``CondInstSegmHead`` builds from its config dict through the
registry and keeps to its loss envelope; the C entry points reject bad arguments before any device call.  The GPU twin of
this file is tests/test_condinst_sup_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import condinst_sup as ocs
from oracle.make_golden_condinst_sup import CASES, IN_STRIDE, OUT_STRIDE, case


@pytest.mark.parametrize('seed,kw', CASES)
def test_oracle_reproduces_reference_golden(golden, seed, kw):
    g = golden('condinst_sup')
    masks, labels, logits, gt_inds, segm = case(seed, **kw)
    C = kw.get('C', 5)
    x = logits.clone().requires_grad_(True)
    lm = ocs.mask_loss(x, masks, gt_inds, OUT_STRIDE)['loss_mask']
    (gx,) = torch.autograd.grad(lm, x)
    assert abs(float(lm.detach()) - float(g[f's{seed}_loss_mask'])) <= 1e-6
    assert np.abs(gx.numpy() - g[f's{seed}_g_mask']).max(initial=0) <= 1e-6
    t = ocs.semantic_targets(masks, labels, IN_STRIDE, C)
    assert np.array_equal(t.numpy(), g[f's{seed}_targets'].astype(np.int64))
    assert torch.equal(t, ocs.first_min_targets(masks, labels, IN_STRIDE, C))
    p = segm.clone().requires_grad_(True)
    ls = ocs.segm_loss(p, masks, labels, IN_STRIDE, C)['loss_segm']
    (gp,) = torch.autograd.grad(ls, p)
    assert abs(float(ls.detach()) - float(g[f's{seed}_loss_segm'])) <= 1e-6
    assert np.abs(gp.numpy() - g[f's{seed}_g_segm']).max() <= 1e-6


def test_golden_cases_cover_the_edges():
    """Area ties, bytes above 1, empty and full masks, images of different G and N = 0 are all in the golden cases."""
    kinds = {kw.get('kind', 'random') for _, kw in CASES}
    assert {'ties', 'bytes', 'extremes'} <= kinds
    assert any(len(set(kw.get('G', (3, 5)))) > 1 for _, kw in CASES) and any(kw.get('N') == 0 for _, kw in CASES)
    masks, labels, *_ = case(1, kind='ties', G=(4, 3))
    areas = [int(a) for a in masks[0].long().sum(dim=(1, 2))]
    assert areas[0] == areas[1] == areas[3] and (masks[0][0] & masks[0][1]).any()
    masks, *_ = case(2, kind='bytes')
    assert int(masks[0].max()) > 1


def test_segm_head_builds_from_config():
    from boxinstseg_b200.models import HEADS, build_head
    head = build_head(dict(type='CondInstSegmHead', num_classes=80, in_channels=256, in_stride=8, stacked_convs=2,
                           feat_channels=128, loss_segm=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25,
                                                             loss_weight=1.0),
                           norm_cfg=dict(type='BN', requires_grad=True)))
    assert type(head) is HEADS.get('CondInstSegmHead')
    assert (head.num_classes, head.in_stride, head.segm_loss) == (80, 8, (2.0, 0.25, 1.0))
    with pytest.raises(RuntimeError, match='segm_branch, segm_conv'):
        head.forward(torch.zeros(1, 256, 4, 4))


def test_segm_head_outside_envelope_raises():
    from boxinstseg_b200.models import build_head
    for loss in (dict(type='FocalLoss', use_sigmoid=True, reduction='sum'), dict(type='CrossEntropyLoss')):
        head = build_head(dict(type='CondInstSegmHead', num_classes=3, loss_segm=loss))
        assert isinstance(head.segm_loss, str)
        with pytest.raises(NotImplementedError, match='loss_segm'):
            head.loss(torch.zeros(1, 3, 2, 2), [torch.zeros(1, 16, 16, dtype=torch.uint8)], [torch.zeros(1).long()])


def test_c_entry_points_reject_bad_arguments():
    from boxinstseg_b200 import _lib as L
    lib = L.lib()
    one = ctypes.c_void_p(16)
    masks = (ctypes.c_void_p * 65)(*([16] * 65))
    strides = (ctypes.c_int64 * 195)(*([1] * 195))
    off = (ctypes.c_int64 * 66)(*range(66))
    labs = (ctypes.c_void_p * 65)(*([16] * 65))
    sums = loss = ws = one
    # 65 images: more than the table holds
    assert lib.bxs_condinst_dice_forward(one, one, 1, 4, 4, masks, strides, off, 65, 16, 16, 2, 4, sums, loss, ws,
                                         None) == -3
    assert lib.bxs_condinst_semantic_targets(masks, strides, labs, off, 65, 16, 16, 8, 3, one, one, None) == -3
    # a sampled pixel outside the masks, a non-positive stride, a first offset that is not 0, a NULL mask
    assert lib.bxs_condinst_dice_forward(one, one, 1, 5, 4, masks, strides, off, 1, 16, 16, 2, 4, sums, loss, ws, None) == -1
    assert lib.bxs_condinst_dice_forward(one, one, 1, 4, 4, masks, strides, off, 1, 16, 16, 2, 0, sums, loss, ws, None) == -1
    bad_off = (ctypes.c_int64 * 2)(1, 2)
    assert lib.bxs_condinst_dice_backward(one, one, 1, 4, 4, masks, strides, bad_off, 1, 16, 16, 2, 4, sums, one, one,
                                          None) == -1
    null_mask = (ctypes.c_void_p * 1)(None)
    assert lib.bxs_condinst_semantic_targets(null_mask, strides, labs, off, 1, 16, 16, 8, 3, one, one, None) == -1
    assert lib.bxs_condinst_semantic_targets(masks, strides, None, off, 1, 16, 16, 8, 3, one, one, None) == -1
    assert lib.bxs_condinst_dice_workspace_bytes(500, 200, 256) == 156160      # 500 instances x 13 chunks x 3 doubles, 256-byte aligned
    assert lib.bxs_condinst_dice_workspace_bytes(-1, 200, 256) == 0
