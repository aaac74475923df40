"""Golden vectors for ``CondInstBoxHead.loss``, minted from the REFERENCE's own code (authoring container only).

AST-extracted and run on seeded float64 inputs: ``CondInstBoxHead.loss`` and ``centerness_target`` (condinst_head.py),
``bbox_overlaps`` / ``fp16_clamp`` (iou2d_calculator.py), ``giou_loss`` / ``GIoULoss`` (iou_loss.py) with
``weighted_loss`` / ``weight_reduce_loss`` / ``reduce_loss`` (losses/utils.py, ``mmcv.jit`` as the identity),
``py_sigmoid_focal_loss`` / ``FocalLoss`` (focal_loss.py, the CPU branch), ``binary_cross_entropy`` / ``CrossEntropyLoss``
(cross_entropy_loss.py), ``distance2bbox`` (transforms.py), ``MlvlPointGenerator`` (point_generator.py) and
``reduce_mean`` (dist_utils.py, world size 1).  ``get_targets`` is the float32 restatement pinned by
tests/golden/fcos_targets.npz, its regression targets handed to the float64 loss as the reference's ``@force_fp32`` run
would hand float32 ones.  Asserts the oracle (oracle/fcos_loss.py) == the reference bit for bit, and writes
tests/golden/fcos_loss.npz: the three losses, the gradients of the three prediction lists and the four returned index
tensors.      python -m oracle.make_golden_fcos_loss"""
import ast
import functools
import os
import types
import warnings

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import fcos_loss as ofl
from oracle import fcos_targets as oft

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'fcos_loss.npz')
STRIDES = (8, 16, 32, 64, 128)
RANGES = ((-1, 64), (64, 128), (128, 256), (256, 512), (512, oft.INF))


def case(seed, B=2, H=160, W=224, G=(5, 8), C=4, ties=True, no_pos=False, dtype=torch.float64):
    """Seeded CPU inputs of ``loss``: (cls_scores, bbox_preds, centernesses, gt_bboxes, gt_labels), predictions in
    ``dtype``.  ``ties`` plants, at the positives, predictions equal to their targets, sharing one edge with them,
    zero-width ones and ones that only touch the target box; ``no_pos`` gives every image ground truths no point is
    assigned to."""
    gen = torch.Generator().manual_seed(seed)
    sizes = [((H + s - 1) // s, (W + s - 1) // s) for s in STRIDES]
    boxes, labels = [], []
    for b in range(B):
        g = G[b % len(G)]
        x1 = torch.rand(g, generator=gen) * (W - 16)
        y1 = torch.rand(g, generator=gen) * (H - 16)
        bw = 8 + torch.rand(g, generator=gen) ** 2 * W
        bh = 8 + torch.rand(g, generator=gen) ** 2 * H
        bx = torch.stack([x1, y1, torch.clamp(x1 + bw, max=float(W)), torch.clamp(y1 + bh, max=float(H))], 1)
        if no_pos:                                       # zero-area boxes between locations: no point is inside any
            bx = torch.tensor([[1.0, 1.0, 1.0, 1.0]]).repeat(g, 1)
        boxes.append(bx)
        labels.append(torch.randint(0, C, (g,), generator=gen))
    cls = [torch.randn(B, C, h, w, generator=gen).to(dtype) for h, w in sizes]
    bbox = [(0.1 + 6 * torch.rand(B, 4, h, w, generator=gen)).to(dtype) for h, w in sizes]
    ctr = [torch.randn(B, 1, h, w, generator=gen).to(dtype) for h, w in sizes]
    if ties and not no_pos:
        pts = oft.grid_points(sizes, STRIDES)
        lab, tgt, _ = oft.get_targets(pts, boxes, labels, RANGES, STRIDES, C)
        k = 0
        for l, (h, w) in enumerate(sizes):
            pos = ((lab[l] >= 0) & (lab[l] < C)).nonzero().reshape(-1).tolist()
            for i in pos:
                b, p = divmod(i, h * w)
                y, x = divmod(p, w)
                t = tgt[l][i].to(dtype)
                kind = k % 6
                if kind == 0:                            # the prediction is its target
                    bbox[l][b, :, y, x] = t
                elif kind == 1:                          # one shared edge (left), the rest different
                    bbox[l][b, 0, y, x] = t[0]
                elif kind == 2:                          # zero width
                    bbox[l][b, 0, y, x] = 0.
                    bbox[l][b, 2, y, x] = 0.
                elif kind == 3:                          # touches the target's left edge from outside
                    bbox[l][b, 2, y, x] = -t[0]
                    bbox[l][b, 0, y, x] = t[0] + 1.
                k += 1
    return cls, bbox, ctr, boxes, labels


CASES = [(0, dict()), (1, dict(B=3, G=(1, 9, 4), C=3)), (2, dict(no_pos=True)), (3, dict(ties=False, H=96, W=128))]


def _extract(rel, names):
    """The named top-level functions / classes of a reference file, with decorators dropped except ``weighted_loss``."""
    tree = ast.parse(open(os.path.join(REF, rel)).read())
    out = []
    for n in tree.body:
        if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in names:
            n.decorator_list = [d for d in n.decorator_list if isinstance(d, ast.Name) and d.id == 'weighted_loss']
            out.append(n)
    assert {n.name for n in out} == set(names), (rel, names)
    return out


def reference():
    g = dict(torch=torch, nn=nn, F=F, np=np, functools=functools, warnings=warnings,
             mmcv=types.SimpleNamespace(jit=lambda **kw: (lambda f: f)), _pair=lambda v: (v, v),
             dist=types.SimpleNamespace(is_available=lambda: False, is_initialized=lambda: False))
    parts = [('mmdet/models/losses/utils.py', ['reduce_loss', 'weight_reduce_loss', 'weighted_loss']),
             ('mmdet/core/bbox/iou_calculators/iou2d_calculator.py', ['fp16_clamp', 'bbox_overlaps']),
             ('mmdet/models/losses/iou_loss.py', ['giou_loss', 'GIoULoss']),
             ('mmdet/models/losses/focal_loss.py', ['py_sigmoid_focal_loss', 'FocalLoss']),
             ('mmdet/models/losses/cross_entropy_loss.py', ['_expand_onehot_labels', 'binary_cross_entropy',
                                                            'CrossEntropyLoss']),
             ('mmdet/core/bbox/transforms.py', ['distance2bbox']),
             ('mmdet/core/anchor/point_generator.py', ['MlvlPointGenerator']),
             ('mmdet/core/utils/dist_utils.py', ['reduce_mean'])]
    for rel, names in parts:
        exec(compile(ast.Module(body=_extract(rel, names), type_ignores=[]), rel, 'exec'), g)
    g.update(cross_entropy=None, mask_cross_entropy=None, sigmoid_focal_loss=None, bbox_overlaps=g['bbox_overlaps'])
    src = open(os.path.join(REF, 'mmdet/models/dense_heads/condinst_head.py')).read()
    cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == 'CondInstBoxHead'][0]
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in ('loss', 'centerness_target')]
    for f in fns:
        f.decorator_list = []
    exec(compile(ast.Module(body=fns, type_ignores=[]), 'condinst_head.py', 'exec'), g)
    return g


def reference_head(g, C):
    """A stand-in ``self`` for the extracted ``loss``: the BoxInst config's losses, built by the reference's classes."""
    me = types.SimpleNamespace(num_classes=C, cls_out_channels=C, strides=STRIDES)
    me.prior_generator = g['MlvlPointGenerator'](STRIDES, offset=0.5)
    me.loss_cls = g['FocalLoss'](use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
    me.loss_bbox = g['GIoULoss'](loss_weight=1.0)
    me.loss_centerness = g['CrossEntropyLoss'](use_sigmoid=True, loss_weight=1.0)
    me.centerness_target = types.MethodType(g['centerness_target'], me)

    def get_targets(points, gt_bboxes, gt_labels):
        lab, tgt, ind = oft.get_targets([p.float() for p in points], gt_bboxes, gt_labels, RANGES, STRIDES, C)
        return lab, [t.to(points[0].dtype) for t in tgt], ind
    me.get_targets = get_targets
    return me


def run(fn, inputs):
    cls, bbox, ctr, boxes, labels = inputs
    leaves = [t.clone().requires_grad_(True) for t in cls + bbox + ctr]
    n = len(cls)
    out = fn(leaves[:n], leaves[n:2 * n], leaves[2 * n:], boxes, labels)
    losses = out[0]
    grads = torch.autograd.grad(losses['loss_cls'] + losses['loss_bbox'] + losses['loss_centerness'], leaves)
    return out, grads


def main():
    g = reference()
    res = {}
    for seed, kw in CASES:
        inputs = case(seed, **kw)
        C = kw.get('C', 4)
        me = reference_head(g, C)
        r_out, r_grads = run(lambda c, b, t, gb, gl: g['loss'](me, c, b, t, gb, gl, None), inputs)
        o_out, o_grads = run(lambda c, b, t, gb, gl: ofl.loss(c, b, t, gb, gl, STRIDES, C), inputs)
        for k in ('loss_cls', 'loss_bbox', 'loss_centerness'):
            assert torch.equal(r_out[0][k], o_out[0][k]), (seed, k, r_out[0][k], o_out[0][k])
        for a, b in zip(r_out[1:], o_out[1:]):
            assert a.dtype == b.dtype and torch.equal(a, b), 'index tensors'
        for a, b in zip(r_grads, o_grads):
            assert torch.equal(a, b), 'gradients'
        for k in ('loss_cls', 'loss_bbox', 'loss_centerness'):
            res[f's{seed}_{k}'] = r_out[0][k].detach().numpy()
        n = len(inputs[0])
        for j, name in enumerate(('cls', 'bbox', 'ctr')):
            res[f's{seed}_g_{name}'] = torch.cat([t.reshape(-1) for t in r_grads[j * n:(j + 1) * n]]).numpy()
        res[f's{seed}_points'] = r_out[1].float().numpy()
        for j, name in enumerate(('level_inds', 'img_inds', 'gt_inds')):
            res[f's{seed}_{name}'] = r_out[2 + j].numpy().astype(np.int16)
        if kw.get('no_pos'):
            assert float(r_out[0]['loss_bbox'].detach()) == 0 and float(r_out[0]['loss_centerness'].detach()) == 0
    np.savez_compressed(OUT, **res)
    print('oracle == reference on', len(CASES), 'cases;', os.path.getsize(OUT) // 1024, 'KiB ->', OUT)


if __name__ == '__main__':
    main()
