"""Golden vectors for BoxSOLOv2Head's training ``forward`` + ``loss``, minted from the REFERENCE's own methods (authoring
container only).

``BoxSOLOv2Head.forward``, ``forward_single``, ``split_feats``, ``loss`` and ``solo_target_single`` are AST-extracted from
mmdet/models/dense_heads/box_solov2_head.py; ``FocalLoss`` / ``py_sigmoid_focal_loss`` from mmdet/models/losses/focal_loss.py,
``weight_reduce_loss`` / ``reduce_loss`` from utils.py, ``BoxProjectionLoss`` and ``LevelsetLoss`` from their files.  They are
bound to a stand-in head holding the seeded stand-in towers of oracle/solo_head.py; third-party pieces are stand-ins:
``multi_apply`` (mmdet/core/utils/misc.py, restated), ``mmcv.imrescale`` (oracle/solo_targets.py), ``mmcv.jit`` (identity),
``mst`` / ``tree_filter`` (the CPU tree oracle).  On CPU tensors ``FocalLoss.forward`` takes its one-hot / py branch.

Asserts that oracle/solo_head.py (forward + loss with ``cpu_parts``) equals the reference, and writes
tests/golden/solo_head.npz: the three losses and the gradients of their sum with respect to the FPN inputs and the level-set
branch (``levelset_bottom.weight``).      python -m oracle.make_golden_solo_head"""
import ast
import os
import types
from functools import partial

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from scipy import ndimage

from oracle import solo_head as osh
from oracle import solo_targets as ost
from oracle import tree as ot
from oracle.make_golden import _Registry, extract

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'solo_head.npz')
METHODS = ['forward', 'forward_single', 'split_feats', 'loss', 'solo_target_single']


def multi_apply(func, *args, **kwargs):
    pfunc = partial(func, **kwargs) if kwargs else func
    return tuple(map(list, zip(*map(pfunc, *args))))


def reference_head(head):
    """A stand-in ``self`` whose methods are the reference's own, sharing ``head``'s tower modules."""
    mmcv = types.SimpleNamespace(imrescale=ost.imrescale, jit=lambda **k: (lambda fn: fn))
    src = open(os.path.join(REF, 'mmdet/models/dense_heads/box_solov2_head.py')).read()
    cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == 'BoxSOLOv2Head'][0]
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in METHODS]
    assert {f.name for f in fns} == set(METHODS)
    g = dict(torch=torch, F=F, nn=nn, np=np, ndimage=ndimage, mmcv=mmcv, multi_apply=multi_apply)
    exec(compile(ast.Module(body=fns, type_ignores=[]), 'box_solov2_head.py', 'exec'), g)
    ut = extract('mmdet/models/losses/utils.py', ['reduce_loss', 'weight_reduce_loss'], dict(mmcv=mmcv))
    fl = extract('mmdet/models/losses/focal_loss.py', ['py_sigmoid_focal_loss', 'FocalLoss'],
                 dict(LOSSES=_Registry(), weight_reduce_loss=ut.weight_reduce_loss, _sigmoid_focal_loss=None))
    bp = extract('mmdet/models/losses/box_projection_loss.py', ['BoxProjectionLoss'], dict(LOSSES=_Registry()))
    ls = extract('mmdet/models/losses/levelset_loss.py', ['LevelsetLoss', 'region_levelset', 'length_regularization'],
                 dict(LOSSES=_Registry()))
    Ref = type('RefBoxSOLOv2Head', (), {n: g[n] for n in METHODS})
    me = Ref()
    for name in osh_towers():
        setattr(me, name, getattr(head, name))
    me.num_classes = me.cate_out_channels = head.num_classes
    me.seg_num_grids, me.strides, me.scale_ranges, me.sigma = head.seg_num_grids, head.strides, head.scale_ranges, head.sigma
    me.cate_down_pos = head.cate_down_pos
    me.loss_cate = fl.FocalLoss(use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
    me.loss_boxpro = bp.BoxProjectionLoss(loss_weight=3.0)
    me.loss_levelset = ls.LevelsetLoss(loss_weight=1.0)
    me.mst = lambda fm: ot.mst(fm.detach())              # the reference MST has no gradient (functions/mst.py)
    me.tree_filter = ot.tree_filter
    return me


def osh_towers():
    return ('feature_convs', 'kernel_convs', 'cate_convs', 'solo_kernel', 'solo_cate', 'solo_mask', 'levelset_bottom')


def run(head, feats, img, bboxes, labels, masks, ref=None):
    """(losses, gradients of their sum w.r.t. the FPN inputs and levelset_bottom's weight).  Not its bias: the losses see
    only differences between the level-set channels, so that gradient is 0 and its computed value is rounding noise."""
    xs = [f.clone().requires_grad_(True) for f in feats]
    if ref is not None:
        ins, cate, lst = ref.forward(xs)
        out = ref.loss(ins, cate, lst, bboxes, labels, masks, img, None, None)
    else:
        ins, cate, lst = osh.forward(head, xs)
        out = osh.loss(head, ins, cate, lst, bboxes, labels, masks, img, parts=osh.cpu_parts(head))
    wrt = xs + [head.levelset_bottom.weight]
    grads = torch.autograd.grad(out['loss_boxpro'] + out['loss_levelset'] + out['loss_cate'], wrt)
    return {k: v.detach() for k, v in out.items()}, grads


def main():
    torch.set_grad_enabled(True)
    case = osh.golden_case()
    head = case[0]
    r_out, r_grads = run(*case, ref=reference_head(head))
    o_out, o_grads = run(*case)
    for k in r_out:
        err = abs(o_out[k].item() - r_out[k].item()) / abs(r_out[k].item())
        assert err < 1e-5, (k, o_out[k].item(), r_out[k].item())
    for i, (a, b) in enumerate(zip(o_grads, r_grads)):
        err = ((a - b).norm() / b.norm()).item()
        assert err < 1e-5, (i, err)
    arrays = {k: v.numpy() for k, v in r_out.items()}
    arrays.update({f'grad_{i}': g.numpy() for i, g in enumerate(r_grads)})
    np.savez_compressed(OUT, **arrays)
    print({k: float(v) for k, v in r_out.items()}, 'written', OUT)


if __name__ == '__main__':
    main()
