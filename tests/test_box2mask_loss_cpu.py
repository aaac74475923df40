"""CPU: Box2MaskHead's training loss -- the restated reference lines (oracle/box2mask_loss.py) against the golden vectors
minted from the reference's own ``loss`` / ``loss_single`` / ``get_targets``, the cross-entropy entry points' argument checks,
and the head's classification-loss configuration."""
import ctypes
import os

import numpy as np
import pytest
import torch

from oracle import box2mask_loss as obl

# configs/box2mask/box2mask_r50_lsj_8x2_50e_coco.py:92-97
CONFIG_LOSS_CLS = dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=2.0, reduction='mean',
                       class_weight=[1.0] * 80 + [0.1])


def _build(**over):
    from boxinstseg_b200.models import build_head
    return build_head({**dict(type='Box2MaskHead', num_queries=100, num_things_classes=80, num_stuff_classes=0,
                              loss_cls=CONFIG_LOSS_CLS), **over})


def test_oracle_reproduces_the_reference_golden():
    """oracle/box2mask_loss.py with the CPU oracle parts against tests/golden/box2mask_loss.npz (3 layers, an image without
    ground truth): the same matching, every loss and every gradient within 1e-5."""
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'box2mask_loss.npz'))
    cls, masks, lsts, labels, gts, img = obl.golden_case()
    parts = obl.cpu_parts()
    got = torch.stack([m for c, mp in zip(cls, masks) for m in obl.assignments(parts, list(c), list(mp), labels, gts)])
    assert torch.equal(got, torch.from_numpy(gold['matches']))
    leaves = [[t.clone().requires_grad_(True) for t in ts] for ts in (cls, masks, lsts)]
    out = obl.loss(parts, 8, obl.GOLDEN_NUM_CLASSES, obl.GOLDEN_CLASS_WEIGHT, 2.0, *leaves, labels, gts, img)
    assert list(out) == list(gold['keys'])
    assert list(out)[:3] == ['loss_cls', 'loss_project', 'loss_levelset'] and list(out)[3] == 'd0.loss_cls'
    for k, v in out.items():
        assert abs(v.item() - float(gold[k])) <= 1e-5 * abs(float(gold[k])), (k, v.item(), float(gold[k]))
    grads = torch.autograd.grad(sum(out.values()), [t for ts in leaves for t in ts])
    for i, g in enumerate(grads):
        ref = torch.from_numpy(gold[f'grad_{i}'])
        assert g.shape == ref.shape and ((g - ref).norm() / ref.norm()).item() < 1e-5, i


def test_cross_entropy_entry_points_are_exported():
    from boxinstseg_b200 import _lib
    names = ['bxs_softmax_cross_entropy_layers_forward', 'bxs_softmax_cross_entropy_layers_forward_workspace_bytes',
             'bxs_softmax_cross_entropy_layers_backward']
    handle = ctypes.CDLL(_lib.LIB_PATH)
    for n in names:
        assert n in _lib.SIGNATURES and hasattr(handle, n)


def test_cross_entropy_entry_points_reject_bad_arguments_without_gpu():
    from boxinstseg_b200 import _lib
    h = _lib.lib()
    p = ctypes.cast((ctypes.c_float * 64)(), ctypes.c_void_p)
    arr = lambda v: (ctypes.c_void_p * len(v))(*v)              # noqa: E731
    ptrs = arr([p.value] * 17)
    names = ('sc', 'lab', 'cw', 'gd', 'loss', 'ws', 'L', 'B', 'Q', 'K', 'w', 's')
    ok = (ptrs, p, None, ptrs, p, p, 10, 2, 100, 81, 2.0, None)
    rc = lambda **k: h.bxs_softmax_cross_entropy_layers_forward(*[k.get(n, v) for n, v in zip(names, ok)])  # noqa: E731
    assert rc(sc=None) == -1 and rc(lab=None) == -1 and rc(loss=None) == -1 and rc(ws=None) == -1
    assert rc(sc=arr([p.value] * 9 + [None])) == -1                        # one layer's scores missing
    assert rc(gd=arr([p.value] * 9 + [None])) == -1                        # one layer's gradient missing
    assert rc(L=0) == -1 and rc(B=0) == -1 and rc(Q=-1) == -1 and rc(K=0) == -1
    assert rc(L=17) == -3                                                  # more than 16 layers
    bwd = lambda **k: h.bxs_softmax_cross_entropy_layers_backward(          # noqa: E731
        *[k.get(n, v) for n, v in zip(('gd', 'g', 'L', 'B', 'Q', 'K', 's'), (ptrs, p, 10, 2, 100, 81, None))])
    assert bwd(gd=None) == -1 and bwd(g=None) == -1 and bwd(gd=arr([p.value] * 9 + [None])) == -1
    assert bwd(K=0) == -1 and bwd(L=17) == -3
    ws = h.bxs_softmax_cross_entropy_layers_forward_workspace_bytes
    assert ws(10, 2, 100) >= 4 * (10 * 7 + 10) and ws(17, 2, 100) == 0 and ws(10, 0, 100) == 0


def test_cross_entropy_op_rejects_bad_inputs():
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    with pytest.raises(RuntimeError):
        softmax_cross_entropy_layers([torch.zeros(1, 4, 5)], torch.zeros(1, 1, 4, dtype=torch.long))
    with pytest.raises(ValueError):
        softmax_cross_entropy_layers([torch.zeros(1, 4, 5)] * 17, torch.zeros(17, 1, 4, dtype=torch.long))


def test_head_builds_from_the_config_loss_cls():
    head = _build()
    assert head.cls_loss_weight == 2.0 and head.cls_class_weight == [1.0] * 80 + [0.1]
    default = _build(loss_cls=None)                                       # no value: the reference config's loss_cls
    assert default.cls_loss_weight == 2.0 and default.cls_class_weight == [1.0] * 80 + [0.1]
    plain = _build(loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=1.0))
    assert plain.cls_loss_weight == 1.0 and plain.cls_class_weight is None
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import Box2MaskHead
    bare = Box2MaskHead(num_queries=100)
    assert bare.num_queries == 100 and bare.cls_class_weight == [1.0] * 80 + [0.1]


@pytest.mark.parametrize('bad', [dict(use_sigmoid=True), dict(use_mask=True), dict(reduction='sum'),
                                 dict(reduction='none'), dict(avg_non_ignore=True)])
def test_unsupported_classification_loss_raises(bad):
    with pytest.raises(NotImplementedError):
        _build(loss_cls={**CONFIG_LOSS_CLS, **bad})
