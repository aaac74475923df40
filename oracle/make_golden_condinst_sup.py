"""Golden vectors for CondInst's mask-supervised losses, minted from the REFERENCE's own code (authoring container only).

AST-extracted from condinst_head.py and run on seeded float64 CPU inputs: ``dice_coefficient``, ``INF``,
``CondInstMaskHead.loss`` and ``.get_targets`` (``boxinst_enabled=False``), ``CondInstSegmHead.get_targets`` and ``.loss``
with ``FocalLoss(use_sigmoid=True)`` / ``py_sigmoid_focal_loss`` (focal_loss.py, its CPU branch) and
``weight_reduce_loss`` / ``reduce_loss`` (losses/utils.py).  Asserts that the oracle (oracle/condinst_sup.py) equals the
reference bit for bit, and writes tests/golden/condinst_sup.npz: per case the two losses, their gradients and the semantic
label map.  At N = 0 the reference raises (``dice_coefficient`` reshapes zero instances with -1); that case records the
oracle's ``0 * sum()``, the dummy loss the reference sets just before.      python -m oracle.make_golden_condinst_sup"""
import ast
import functools
import os
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import condinst_sup as ocs

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'condinst_sup.npz')
OUT_STRIDE, IN_STRIDE = 4, 8


def case(seed, G=(3, 5), H=64, W=96, C=5, N=12, kind='random', dtype=torch.float64):
    """Seeded CPU inputs: (gt_masks per image uint8 [G_b, H, W], gt_labels per image int64 [G_b], mask_logits
    [N, 1, H/4, W/4], gt_inds int64 [N], segm_pred [B, C, H/8, W/8]).  ``kind``: 'random' rectangles and blobs;
    'ties' overlapping rectangles of equal area, and one mask nested inside another; 'bytes' mask values 1..255;
    'extremes' empty and full masks among ordinary ones."""
    gen = torch.Generator().manual_seed(seed)
    masks, labels = [], []
    for b, g in enumerate(G):
        m = torch.zeros(g, H, W, dtype=torch.uint8)
        for k in range(g):
            y0, x0 = int(torch.randint(0, H - 8, (1,), generator=gen)), int(torch.randint(0, W - 8, (1,), generator=gen))
            hh, ww = int(torch.randint(4, H - y0 + 1, (1,), generator=gen)), int(torch.randint(4, W - x0 + 1, (1,), generator=gen))
            if kind == 'ties':                     # every mask 16 x 24 = 384 pixels, shifted so that they overlap
                y0, x0, hh, ww = 4 + 5 * k, 6 + 7 * k, 16, 24
            m[k, y0:y0 + hh, x0:x0 + ww] = 1
            if kind == 'random' and k % 2:         # a blob with holes
                m[k] &= (torch.rand(H, W, generator=gen) < 0.7).to(torch.uint8)
        if kind == 'ties' and g >= 3:              # nested: mask 2 inside mask 0
            m[2] = 0
            m[2, 6:12, 8:14] = 1
        if kind == 'bytes':
            m = m * torch.randint(1, 256, (g, H, W), generator=gen, dtype=torch.int64).to(torch.uint8)
        if kind == 'extremes' and g >= 2:
            m[0] = 0
            m[1] = 1
        masks.append(m)
        labels.append(torch.randint(0, C, (g,), generator=gen))
    total = sum(G)
    gt_inds = torch.randint(0, max(total, 1), (N,), generator=gen) if total else torch.zeros(0, dtype=torch.int64)
    h, w = len(range(OUT_STRIDE // 2, H, OUT_STRIDE)), len(range(OUT_STRIDE // 2, W, OUT_STRIDE))
    logits = (3 * torch.randn(N, 1, h, w, generator=gen)).to(dtype)
    segm = torch.randn(len(G), C, len(range(IN_STRIDE // 2, H, IN_STRIDE)), len(range(IN_STRIDE // 2, W, IN_STRIDE)),
                       generator=gen).to(dtype)
    return masks, labels, logits, gt_inds, segm


CASES = [(0, dict()), (1, dict(kind='ties', G=(4, 3))), (2, dict(kind='bytes')), (3, dict(kind='extremes', G=(2, 6))),
         (4, dict(G=(1, 7, 2), N=20)), (5, dict(N=0))]


def _members(tree, cls_name, names):
    cls = [n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls_name][0]
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert {f.name for f in fns} == set(names), (cls_name, names)
    for f in fns:
        f.decorator_list = []
    return fns


def reference():
    """Namespace with the reference's functions; classes' methods prefixed with their class names."""
    g = dict(torch=torch, nn=nn, F=F, np=np, functools=functools)
    utils = ast.parse(open(os.path.join(REF, 'mmdet/models/losses/utils.py')).read())
    focal = ast.parse(open(os.path.join(REF, 'mmdet/models/losses/focal_loss.py')).read())
    head = ast.parse(open(os.path.join(REF, 'mmdet/models/dense_heads/condinst_head.py')).read())
    body = [n for n in utils.body if isinstance(n, ast.FunctionDef) and n.name in ('reduce_loss', 'weight_reduce_loss')]
    body += [n for n in focal.body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in
             ('py_sigmoid_focal_loss', 'FocalLoss')]
    body += [n for n in head.body if isinstance(n, ast.FunctionDef) and n.name == 'dice_coefficient']
    body += [n for n in head.body if isinstance(n, ast.Assign) and n.targets[0].id == 'INF']
    for n in body:
        n.decorator_list = []
    g['sigmoid_focal_loss'] = None                  # the CUDA op; never reached on CPU tensors
    exec(compile(ast.Module(body=body, type_ignores=[]), 'reference', 'exec'), g)
    for cls_name, names in (('CondInstMaskHead', ('loss', 'get_targets')), ('CondInstSegmHead', ('loss', 'get_targets'))):
        ns = dict(g)
        exec(compile(ast.Module(body=_members(head, cls_name, names), type_ignores=[]), cls_name, 'exec'), ns)
        for n in names:
            g[f'{cls_name}.{n}'] = ns[n]
    return g


def reference_mask_head(g):
    me = types.SimpleNamespace(_iter=torch.zeros([1]), boxinst_enabled=False, out_stride=OUT_STRIDE)
    me.get_targets = types.MethodType(g['CondInstMaskHead.get_targets'], me)
    return me


def reference_segm_head(g, C):
    me = types.SimpleNamespace(num_classes=C, in_stride=IN_STRIDE)
    me.loss_segm = g['FocalLoss'](use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
    me.get_targets = types.MethodType(g['CondInstSegmHead.get_targets'], me)
    return me


def main():
    g = reference()
    res = {}
    for seed, kw in CASES:
        masks, labels, logits, gt_inds, segm = case(seed, **kw)
        C = kw.get('C', 5)
        x = logits.clone().requires_grad_(True)
        x2 = logits.clone().requires_grad_(True)
        o = ocs.mask_loss(x2, masks, gt_inds, OUT_STRIDE)['loss_mask']
        (o_gx,) = torch.autograd.grad(o, x2)
        if len(logits):
            r = g['CondInstMaskHead.loss'](reference_mask_head(g), None, None, x, gt_inds, None, masks, labels)['loss_mask']
            (r_gx,) = torch.autograd.grad(r, x)
            assert torch.equal(r, o) and torch.equal(r_gx, o_gx), (seed, 'loss_mask')
        else:       # the reference sets its 0 * sum() dummy, then still reaches dice_coefficient, whose reshape raises
            try:
                g['CondInstMaskHead.loss'](reference_mask_head(g), None, None, x, gt_inds, None, masks, labels)
                raise AssertionError('the reference was expected to raise at N = 0')
            except RuntimeError:
                pass
            r, r_gx = o, o_gx
        me = reference_segm_head(g, C)
        r_t = me.get_targets(masks, labels)
        assert torch.equal(r_t, ocs.semantic_targets(masks, labels, IN_STRIDE, C)), (seed, 'targets')
        assert torch.equal(r_t, ocs.first_min_targets(masks, labels, IN_STRIDE, C)), (seed, 'first-index targets')
        p = segm.clone().requires_grad_(True)
        rs = g['CondInstSegmHead.loss'](me, p, masks, labels)['loss_segm']
        (r_gp,) = torch.autograd.grad(rs, p)
        p2 = segm.clone().requires_grad_(True)
        os_ = ocs.segm_loss(p2, masks, labels, IN_STRIDE, C)['loss_segm']
        (o_gp,) = torch.autograd.grad(os_, p2)
        assert torch.equal(rs, os_) and torch.equal(r_gp, o_gp), (seed, 'loss_segm', rs, os_)
        res[f's{seed}_loss_mask'] = r.detach().numpy()
        res[f's{seed}_g_mask'] = r_gx.numpy()
        res[f's{seed}_targets'] = r_t.numpy().astype(np.int16)
        res[f's{seed}_loss_segm'] = rs.detach().numpy()
        res[f's{seed}_g_segm'] = r_gp.numpy()
    np.savez_compressed(OUT, **res)
    print('oracle == reference on', len(CASES), 'cases;', os.path.getsize(OUT) // 1024, 'KiB ->', OUT)


if __name__ == '__main__':
    main()
