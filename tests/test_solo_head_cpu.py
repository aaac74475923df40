"""CPU: BoxSOLOv2Head's construction surface, the training ``forward``'s deferred ``SoloInsPreds`` against the reference's
dense shapes (oracle/solo_head.py on the same stand-in towers), and the focal entry points' argument checks."""
import ctypes

import pytest
import torch

from oracle import solo_head as osh

GRIDS = [40, 36, 24, 16, 12]
# configs/boxlevelset/box_levelset_coco_r50_fpn_3x.py:17-39
CONFIG_HEAD = dict(type='BoxSOLOv2Head', num_classes=80, in_channels=256, stacked_convs=4, seg_feat_channels=256,
                   strides=[8, 8, 16, 32, 32], scale_ranges=((1, 96), (48, 192), (96, 384), (192, 768), (384, 2048)),
                   sigma=0.2, num_grids=GRIDS, cate_down_pos=0,
                   loss_cate=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                   loss_boxpro=dict(type='BoxProjectionLoss', loss_weight=3.0),
                   loss_levelset=dict(type='LevelsetLoss', loss_weight=1.0))


def _build(**over):
    from boxinstseg_b200.models import build_head
    return build_head({**CONFIG_HEAD, **over})


def test_config_head_builds_with_loss_cate():
    head = _build()
    assert head.seg_num_grids == GRIDS and list(head.strides) == [8, 8, 16, 32, 32] and head.sigma == 0.2
    assert head.scale_ranges[0] == (1, 96)
    assert head.focal == (2.0, 0.25, 1.0)
    assert _build(loss_cate=dict(type='FocalLoss', use_sigmoid=True, gamma=1.5, alpha=0.5, loss_weight=2.0)).focal == (1.5, 0.5, 2.0)


@pytest.mark.parametrize('bad', [dict(use_sigmoid=False), dict(use_sigmoid=True, reduction='sum')])
def test_unsupported_category_loss_raises(bad):
    with pytest.raises(NotImplementedError):
        _build(loss_cate=dict(type='FocalLoss', **bad))


def test_forward_needs_the_towers():
    with pytest.raises(RuntimeError, match='feature_convs'):
        _build().forward([torch.zeros(1, 256, 8, 8)] * 5)


def _feats(B, C, H, W, gen):
    return [torch.randn(B, C, -(-H // s), -(-W // s), generator=gen) for s in (4, 8, 16, 32, 64)]


def test_solo_ins_preds_report_the_reference_shapes():
    """Training ``forward`` on the stand-in towers: cate_preds and levelset_feats equal the restated reference's, and every
    ``SoloInsPreds`` entry reports the shape of the reference's dense ins_pred without computing it."""
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import SoloInsPreds
    head = osh.attach_towers(_build(in_channels=64), 64, 64, 80, seed=1)
    feats = _feats(2, 64, 128, 160, torch.Generator().manual_seed(0))
    with torch.no_grad():
        ins, cate, lst = head.forward(feats)
        r_ins, r_cate, r_lst = osh.forward(head, feats)
    assert isinstance(ins, SoloInsPreds) and len(ins) == 5
    for p, r in zip(ins, r_ins):
        assert p.shape == r.shape and p.size() == r.size() and p.size()[-2:] == r.size()[-2:] and p.size(1) == r.size(1)
        assert p.kernel_pred.shape[-1] == r.shape[1] ** 0.5
    assert ins.feature_pred.shape == (2, 64, 32, 40)
    for c, rc in zip(cate, r_cate):
        assert torch.equal(c, rc)
    assert torch.equal(lst, r_lst)


def test_focal_entry_points_reject_bad_arguments_without_gpu():
    from boxinstseg_b200 import _lib
    h = _lib.lib()
    p = ctypes.cast((ctypes.c_float * 64)(), ctypes.c_void_p)
    arr = lambda v: (ctypes.c_void_p * len(v))(*v)              # noqa: E731
    i64 = lambda v: (ctypes.c_int64 * len(v))(*v)              # noqa: E731
    ptrs, grid = arr([p.value] * 9), i64(GRIDS + [8] * 4)
    call = lambda *a: h.bxs_sigmoid_focal_loss_levels_forward(*a)    # noqa: E731
    ok = (ptrs, ptrs, grid, ptrs, p, p, p, 5, 2, 80, 2.0, 0.25, 1.0, None)
    rc = lambda **k: call(*[k.get(n, v) for n, v in zip(('lg', 'lb', 'gr', 'gd', 'avg', 'loss', 'ws', 'L', 'B', 'C', 'gamma',
                                                          'alpha', 'w', 's'), ok)])  # noqa: E731
    assert rc(lg=None) == -1 and rc(lb=None) == -1 and rc(avg=None) == -1 and rc(loss=None) == -1 and rc(ws=None) == -1
    assert rc(lg=arr([p.value] * 4 + [None])) == -1                      # one level's logits missing
    assert rc(B=0) == -1 and rc(C=0) == -1 and rc(L=0) == -1 and rc(gamma=-0.5) == -1 and rc(gamma=float('nan')) == -1
    assert rc(gr=i64([40, 36, 0, 16, 12])) == -1
    assert rc(L=9) == -3                                                 # more than 8 levels
    assert h.bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(grid, 5, 2) >= 4 * 2 * (25 + 21 + 9 + 4 + 3)
    assert h.bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(grid, 9, 2) == 0
    assert h.bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(None, 5, 2) == 0


def test_focal_op_rejects_cpu_tensors():
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    with pytest.raises(RuntimeError):
        sigmoid_focal_loss_levels([torch.zeros(1, 80, 4, 4)], [torch.zeros(1, 16, dtype=torch.long)], 1.0)


def _golden_run(case, loss_fn):
    head, feats, img, bboxes, labels, masks = case
    xs = [f.clone().requires_grad_(True) for f in feats]
    out = loss_fn(head, xs, img, bboxes, labels, masks)
    grads = torch.autograd.grad(out['loss_boxpro'] + out['loss_levelset'] + out['loss_cate'],
                                xs + [head.levelset_bottom.weight])
    return out, grads


def test_oracle_reproduces_the_reference_golden():
    """oracle/solo_head.py's forward + loss (CPU oracle parts) against tests/golden/solo_head.npz, minted from the
    reference's own BoxSOLOv2Head methods and FocalLoss by oracle/make_golden_solo_head.py."""
    import os
    import numpy as np
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'solo_head.npz'))

    def lines(head, xs, img, bboxes, labels, masks):
        ins, cate, lst = osh.forward(head, xs)
        return osh.loss(head, ins, cate, lst, bboxes, labels, masks, img, parts=osh.cpu_parts(head))
    out, grads = _golden_run(osh.golden_case(), lines)
    for k in ('loss_boxpro', 'loss_levelset', 'loss_cate'):
        assert abs(out[k].item() - float(gold[k])) <= 1e-4 * abs(float(gold[k])), (k, out[k].item(), float(gold[k]))
    for i, g in enumerate(grads):
        ref = torch.from_numpy(gold[f'grad_{i}'])
        assert g.shape == ref.shape and ((g - ref).norm() / ref.norm()).item() < 1e-4, i
