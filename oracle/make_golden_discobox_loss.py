"""Golden vectors for ``DiscoBoxSOLOv2Head.loss``, minted from the REFERENCE's own code (authoring container only).

AST-extracted from mmdet/models/dense_heads/discobox_head.py and run on seeded float64 CPU inputs: ``loss`` (its
``@autocast()`` dropped: it does not touch CPU tensors) and ``solov2_target_single`` bound to a stand-in ``self``, with the
module-level ``center_of_mass``, ``dice_loss``, ``mil_loss`` and ``MeanField``; the category loss is ``FocalLoss`` /
``py_sigmoid_focal_loss`` of mmdet/models/losses/focal_loss.py (the CPU branch) with ``weight_reduce_loss`` /
``reduce_loss`` of losses/utils.py.  ``multi_apply`` is mmdet's one-liner, ``mmcv.imrescale`` the restated ``cv2.resize``
of oracle/solo_targets.py, ``BitmapMasks`` the stand-in of oracle/make_golden_disco.py.  Asserts the oracle
(oracle/discobox_loss.py) equals the reference and writes tests/golden/discobox_loss.npz: the four losses and the gradients
to cate_preds (once per case: they do not depend on the flags), s_kernel_preds_raw and s_ins_pred (float32), for both
``use_loss_ts`` and both ``use_ind_teacher`` settings.
The correspondence branch is pinned by tests/golden/corr.npz.      python -m oracle.make_golden_discobox_loss"""
import ast
import functools
import os
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import discobox_loss as odl
from oracle import solo_targets as ost
from oracle.make_golden_disco import Masks

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'discobox_loss.npz')
# a 64x64 image with the grids and scale ranges shrunk to it (the COCO grids halved): small enough that the vectors stay
# small, with covered cells on four levels and the top level (48, 512) empty
CFG = dict(odl.CFG, scale_ranges=((1, 12), (6, 24), (12, 48), (24, 96), (48, 512)))
GRIDS = (20, 18, 12, 8, 6)
NUM_CLASSES = 4
FLAGS = [(ts, ind) for ts in (False, True) for ind in (False, True)]


def case(seed, H=64, W=64, G=(6, 4), C=32, empty_image=None):
    """Seeded float64 inputs (cate_preds, s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, boxes, labels,
    masks (uint8 numpy), img).  Ground truths 1 and 2 of every image have the same box and mask (two ground truths on the
    same cells); ``empty_image``: that image's ground truths are zero-area boxes, below every scale range (no covered cell)."""
    gen = torch.Generator().manual_seed(seed)
    B = len(G)
    boxes, labels, masks = [], [], []
    for b, g in enumerate(G):
        x1 = torch.rand(g, generator=gen) * (W - 20)
        y1 = torch.rand(g, generator=gen) * (H - 20)
        bw = 4 + torch.rand(g, generator=gen) * 36
        bh = 4 + torch.rand(g, generator=gen) * 36
        bx = torch.stack([x1, y1, torch.minimum(x1 + bw, torch.tensor(W - 1.)), torch.minimum(y1 + bh, torch.tensor(H - 1.))], 1)
        bx = bx.floor()
        if b == empty_image:
            bx[:, 2:] = bx[:, :2]
        bx[2] = bx[1]
        m = np.zeros((g, H, W), np.uint8)
        for i, r in enumerate(bx):
            m[i, int(r[1]):int(r[3]) + 1, int(r[0]):int(r[2]) + 1] = 1
        m[0, ::3, :] = 0                                                 # not a rectangle
        boxes.append(bx.float())
        labels.append(torch.randint(0, NUM_CLASSES, (g,), generator=gen))
        masks.append(m)
    fh, fw = H // 4, W // 4
    cate = [torch.randn(B, NUM_CLASSES, S, S, generator=gen, dtype=torch.float64) for S in GRIDS]
    s_k = [torch.randn(B, C, S, S, generator=gen, dtype=torch.float64) * 0.3 for S in GRIDS]
    t_k = [torch.randn(B, C, S, S, generator=gen, dtype=torch.float64) * 0.3 for S in GRIDS]
    s_in = torch.randn(B, C, fh, fw, generator=gen, dtype=torch.float64)
    t_in = torch.randn(B, C, fh, fw, generator=gen, dtype=torch.float64)
    img = F.interpolate(torch.randn(B, 3, H // 16, W // 16, generator=gen, dtype=torch.float64), size=(H, W),
                        mode='bilinear', align_corners=False)
    return cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img


# without use_loss_ts the teacher is unused, so (False, True) would repeat (False, False)
CASES = [(0, dict(), [(False, False), (True, False), (True, True)]), (1, dict(G=(5, 3), empty_image=1), [(True, True)])]


def _extract(rel, names, cls_name=None):
    tree = ast.parse(open(os.path.join(REF, rel)).read())
    body = tree.body
    if cls_name:
        body = [n for n in body if isinstance(n, ast.ClassDef) and n.name == cls_name][0].body
    out = [n for n in body if isinstance(n, (ast.FunctionDef, ast.ClassDef)) and n.name in names]
    for n in out:
        n.decorator_list = [d for d in n.decorator_list if isinstance(d, ast.Name) and d.id == 'weighted_loss']
    assert {n.name for n in out} == set(names), (rel, names)
    return out


def reference():
    g = dict(torch=torch, nn=nn, F=F, np=np, functools=functools, mmcv=types.SimpleNamespace(imrescale=ost.imrescale),
             sigmoid_focal_loss=None,
             multi_apply=lambda func, *args, **kw: tuple(map(list, zip(*map(functools.partial(func, **kw), *args)))))
    parts = [('mmdet/models/losses/utils.py', ['reduce_loss', 'weight_reduce_loss']),
             ('mmdet/models/losses/focal_loss.py', ['py_sigmoid_focal_loss', 'FocalLoss']),
             ('mmdet/models/dense_heads/discobox_head.py', ['center_of_mass', 'dice_loss', 'mil_loss', 'MeanField'])]
    for rel, names in parts:
        exec(compile(ast.Module(body=_extract(rel, names), type_ignores=[]), rel, 'exec'), g)
    fns = _extract('mmdet/models/dense_heads/discobox_head.py', ['loss', 'solov2_target_single'], 'DiscoBoxSOLOv2Head')
    exec(compile(ast.Module(body=fns, type_ignores=[]), 'discobox_head.py', 'exec'), g)
    return g


def reference_head(g):
    me = types.SimpleNamespace(num_classes=NUM_CLASSES, cate_out_channels=NUM_CLASSES, seg_num_grids=list(GRIDS),
                               strides=CFG['strides'], scale_ranges=CFG['scale_ranges'], sigma=CFG['sigma'],
                               ins_loss_weight=CFG['ins_loss_weight'], ts_loss_weight=CFG['ts_loss_weight'])
    mf = CFG['mf']
    me.alpha0, me.theta0, me.theta1, me.theta2 = mf['alpha0'], mf['theta0'], mf['theta1'], 20.0
    me.mkernel, me.crf_base, me.crf_max_iter = mf['kernel_size'], mf['base'], mf['iter']
    gamma, alpha, weight = CFG['focal']
    me.loss_cate = g['FocalLoss'](use_sigmoid=True, gamma=gamma, alpha=alpha, loss_weight=weight)
    me.solov2_target_single = types.MethodType(g['solov2_target_single'], me)
    return me


def run(fn, inputs):
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = inputs
    leaves = [t.clone().requires_grad_(True) for t in cate + s_k + [s_in]]
    n = len(cate)
    out = fn(leaves[:n], leaves[n:2 * n], leaves[2 * n])
    total = out['loss_ins'].sum() + out['loss_ts'] + out['loss_cate'] + out['loss_corr']
    grads = torch.autograd.grad(total, leaves, allow_unused=True)
    grads = [torch.zeros_like(x) if gr is None else gr for x, gr in zip(leaves, grads)]
    return {k: v.detach().reshape(()) if v.numel() == 1 else v.detach() for k, v in out.items()}, grads


def main():
    g = reference()
    res = {}
    for seed, kw, flags in CASES:
        inputs = case(seed, **kw)
        cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = inputs
        me = reference_head(g)
        for ts, ind in flags:
            r_out, r_grads = run(lambda c, k, f: g['loss'](me, c, k, t_k, f, t_in, boxes, labels, [Masks(m) for m in masks],
                                                           None, None, img=img, use_loss_ts=ts, use_ind_teacher=ind), inputs)
            o_out, o_grads = run(lambda c, k, f: odl.loss(c, k, t_k, f, t_in, boxes, labels, masks, img, GRIDS, NUM_CLASSES,
                                                          use_loss_ts=ts, use_ind_teacher=ind, cfg=CFG), inputs)
            tag = f's{seed}_ts{int(ts)}_ind{int(ind)}'
            for k in ('loss_ins', 'loss_ts', 'loss_cate', 'loss_corr'):
                assert torch.allclose(r_out[k].double(), o_out[k].double(), rtol=1e-12, atol=1e-14), (tag, k, r_out[k], o_out[k])
                res[f'{tag}_{k}'] = r_out[k].numpy()                  # float64
            for a, b in zip(r_grads, o_grads):
                assert torch.allclose(a, b, rtol=1e-10, atol=1e-14), (tag, 'gradients')
            n = len(cate)
            g_cate = torch.cat([t.reshape(-1) for t in r_grads[:n]]).float().numpy()     # float32: the tests compare to 1e-3
            if f's{seed}_g_cate' in res:                                                  # loss_cate ignores the flags
                assert np.array_equal(res[f's{seed}_g_cate'], g_cate)
            res[f's{seed}_g_cate'] = g_cate
            res[f'{tag}_g_kern'] = torch.cat([t.reshape(-1) for t in r_grads[n:2 * n]]).float().numpy()
            res[f'{tag}_g_ins'] = r_grads[2 * n].float().numpy()
    np.savez_compressed(OUT, **res)
    print('oracle == reference on', sum(len(c[2]) for c in CASES), 'runs;', os.path.getsize(OUT) // 1024, 'KiB ->', OUT)


if __name__ == '__main__':
    main()
