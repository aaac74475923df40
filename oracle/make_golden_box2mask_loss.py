"""Golden vectors for Box2MaskHead's training ``loss`` over several decoder layers, minted from the REFERENCE's own methods
(authoring container only).

``Box2MaskHead.loss``, ``loss_single``, ``get_targets`` and ``_get_target_single`` are AST-extracted from
mmdet/models/dense_heads/box2mask_head.py; ``cross_entropy`` / ``CrossEntropyLoss`` from cross_entropy_loss.py,
``weight_reduce_loss`` / ``reduce_loss`` from utils.py, ``BoxProjectionLoss``, ``LevelsetLoss`` and ``LCM`` from their files,
``_scale_target`` from models/utils/misc.py, ``MaskHungarianAssigner`` with ``ClassificationCost`` / ``BoxMatchingCost`` / ``FocalLossCost`` and
``AssignResult``, ``MaskPseudoSampler`` and ``MaskSamplingResult`` from mmdet/core/bbox.  They are bound to a stand-in head;
third-party pieces are stand-ins: ``multi_apply`` (restated), ``force_fp32`` (identity), the mixin / base classes (object),
``mst`` / ``tree_filter`` (the CPU tree oracle); the matching is scipy's, as in the reference.

Asserts that oracle/box2mask_loss.py (``cpu_parts``) matches the queries exactly as the reference does and equals its
losses and gradients, then writes tests/golden/box2mask_loss.npz: the 3*L losses, the gradients of their sum with respect to
every layer's scores, mask logits and level-set feature, and the reference's matching.
    python -m oracle.make_golden_box2mask_loss"""
import ast
import os
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

from oracle import box2mask_loss as obl
from oracle import tree as ot
from oracle.make_golden import _force_fp32, _Registry, extract

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'box2mask_loss.npz')
METHODS = ['loss', 'loss_single', 'get_targets', '_get_target_single']


def multi_apply(func, *args, **kwargs):
    from functools import partial
    pfunc = partial(func, **kwargs) if kwargs else func
    return tuple(map(list, zip(*map(pfunc, *args))))


def reference_head():
    """A stand-in ``self`` whose methods are the reference's own, with the reference's losses, assigner and sampler."""
    src = open(os.path.join(REF, 'mmdet/models/dense_heads/box2mask_head.py')).read()
    cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == 'Box2MaskHead'][0]
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in METHODS]
    assert {f.name for f in fns} == set(METHODS)
    stubs = dict(LOSSES=_Registry(), MATCH_COST=_Registry(), BBOX_ASSIGNERS=_Registry(), BBOX_SAMPLERS=_Registry())
    misc = extract('mmdet/models/utils/misc.py', ['_scale_target'])
    ls = extract('mmdet/models/losses/levelset_loss.py', ['LevelsetLoss', 'region_levelset', 'length_regularization', 'LCM',
                                                          'LocalConsistencyModule'], stubs)
    bp = extract('mmdet/models/losses/box_projection_loss.py', ['BoxProjectionLoss'], stubs)
    ut = extract('mmdet/models/losses/utils.py', ['reduce_loss', 'weight_reduce_loss'],
                 dict(mmcv=types.SimpleNamespace(jit=lambda **k: (lambda fn: fn))))
    ce = extract('mmdet/models/losses/cross_entropy_loss.py', ['cross_entropy', 'CrossEntropyLoss'],
                 dict(stubs, weight_reduce_loss=ut.weight_reduce_loss, warnings=__import__('warnings'),
                      binary_cross_entropy=None, mask_cross_entropy=None))
    mc = extract('mmdet/core/bbox/match_costs/match_cost.py', ['ClassificationCost', 'BoxMatchingCost', 'FocalLossCost'],
                 stubs)
    ar = extract('mmdet/core/bbox/assigners/assign_result.py', ['AssignResult'],
                 dict(util_mixins=types.SimpleNamespace(NiceRepr=object)))
    costs = dict(ClassificationCost=mc.ClassificationCost, BoxMatchingCost=mc.BoxMatchingCost,
                 FocalLossCost=mc.FocalLossCost)                 # the assigner's default mask_cost, weight 0
    build_match_cost = lambda cfg: costs[cfg['type']](**{k: v for k, v in cfg.items() if k != 'type'})   # noqa: E731
    asg = extract('mmdet/core/bbox/assigners/mask_hungarian_assigner.py', ['MaskHungarianAssigner'],
                  dict(stubs, BaseAssigner=object, AssignResult=ar.AssignResult, build_match_cost=build_match_cost,
                       linear_sum_assignment=linear_sum_assignment))
    msr = extract('mmdet/core/bbox/samplers/mask_sampling_result.py', ['MaskSamplingResult'], dict(SamplingResult=object))
    smp = extract('mmdet/core/bbox/samplers/mask_pseudo_sampler.py', ['MaskPseudoSampler'],
                  dict(stubs, BaseSampler=object, MaskSamplingResult=msr.MaskSamplingResult))
    g = dict(torch=torch, F=F, nn=nn, np=np, multi_apply=multi_apply, _scale_target=misc._scale_target, LCM=ls.LCM,
             force_fp32=_force_fp32)
    exec(compile(ast.Module(body=fns, type_ignores=[]), 'box2mask_head.py', 'exec'), g)
    me = type('RefBox2MaskHead', (), {n: g[n] for n in METHODS})()
    me.num_queries, me.num_classes = 8, obl.GOLDEN_NUM_CLASSES
    me.class_weight = obl.GOLDEN_CLASS_WEIGHT
    me.loss_cls = ce.CrossEntropyLoss(use_sigmoid=False, loss_weight=2.0, reduction='mean', class_weight=me.class_weight)
    me.loss_box = bp.BoxProjectionLoss(loss_weight=5.0)
    me.loss_mask = ls.LevelsetLoss(loss_weight=1.0)
    me.assigner = asg.MaskHungarianAssigner(**{k: v for k, v in obl.ASSIGNER.items() if k != 'type'})
    me.sampler = smp.MaskPseudoSampler()
    me.mst = lambda fm: ot.mst(fm.detach())              # the reference MST has no gradient (functions/mst.py)
    me.tree_filter = ot.tree_filter
    return me


def run(case, ref=None):
    """(losses, gradients of their sum w.r.t. every layer's scores, mask logits and level-set feature)."""
    cls, masks, lsts, labels, gts, img = case
    leaves = [[t.clone().requires_grad_(True) for t in ts] for ts in (cls, masks, lsts)]
    if ref is not None:
        out = ref.loss(*leaves, labels, gts, [dict() for _ in labels], img)
    else:
        out = obl.loss(obl.cpu_parts(), 8, obl.GOLDEN_NUM_CLASSES, obl.GOLDEN_CLASS_WEIGHT, 2.0, *leaves, labels, gts, img)
    flat = [t for ts in leaves for t in ts]
    grads = torch.autograd.grad(sum(out.values()), flat)
    return {k: v.detach() for k, v in out.items()}, grads


def reference_matches(ref, case):
    """The reference assigner's matched ground truth (-1: none) of every (layer, image) query."""
    cls, masks, _, labels, gts, _ = case
    out = []
    for c, m in zip(cls, masks):
        for b in range(c.shape[0]):
            mp = F.interpolate(m[b].unsqueeze(1), gts[b].shape[-2:], mode='bilinear', align_corners=False)    # :159-163
            res = ref.assigner.assign(c[b], mp, labels[b], gts[b].unsqueeze(1), None)
            out.append(res.gt_inds - 1)
    return torch.stack(out)


def main():
    torch.set_grad_enabled(True)
    case = obl.golden_case()
    ref = reference_head()
    want = reference_matches(ref, case)
    mine = torch.stack([m for c, mp in zip(case[0], case[1])
                        for m in obl.assignments(obl.cpu_parts(), list(c), list(mp), case[3], case[4])])
    assert torch.equal(want, mine), (want, mine)
    r_out, r_grads = run(case, ref=ref)
    o_out, o_grads = run(case)
    assert list(r_out) == list(o_out)
    for k in r_out:
        err = abs(o_out[k].item() - r_out[k].item()) / max(abs(r_out[k].item()), 1e-12)
        assert err < 1e-5 or abs(r_out[k].item()) == o_out[k].item() == 0.0, (k, o_out[k].item(), r_out[k].item())
    for i, (a, b) in enumerate(zip(o_grads, r_grads)):
        err = ((a - b).norm() / b.norm().clamp(min=1e-30)).item()
        assert err < 1e-5, (i, err)
    arrays = {k: v.numpy() for k, v in r_out.items()}
    arrays.update({f'grad_{i}': g.numpy() for i, g in enumerate(r_grads)})
    arrays['matches'] = want.numpy()
    arrays['keys'] = np.array(list(r_out))
    np.savez_compressed(OUT, **arrays)
    print({k: float(v) for k, v in r_out.items()}, 'written', OUT)


if __name__ == '__main__':
    main()
