"""Golden vectors for CondInst inference, minted from the REFERENCE's own lines (authoring container only).

AST-extracted: ``nms_with_others`` and ``aligned_bilinear`` (mmdet/models/dense_heads/condinst_head.py), ``distance2bbox``
(mmdet/core/bbox/transforms.py), ``get_k_for_topk`` (mmdet/core/export/onnx_helper.py), ``CondInstBoxHead.get_bboxes`` /
``_get_bboxes`` and ``CondInstMaskHead.forward`` / ``parse_dynamic_params`` / ``simple_test``, bound to stand-in heads;
``batched_nms`` is the oracle's restatement of mmcv's (oracle/condinst_infer.py: mmcv is not installed) with the reference's
unstable sorts.  Asserts that the oracle (stable sorts) equals them and writes tests/golden/condinst_infer.npz.
                                                                            python -m oracle.make_golden_condinst_infer
"""
import ast
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

from oracle import condinst_infer as oci
from oracle.make_golden import _force_fp32, extract

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'condinst_infer.npz')

SIZES = ((8, 10), (4, 5), (2, 3))
STRIDES = (8, 16, 32)
NUM_CLASSES = 3
MASK_CH = 8
NUM_PARAMS = (MASK_CH + 2) * 8 + 8 + 8 * 8 + 8 + 8 + 1          # 169: dynamic_convs=3, dynamic_channels=8
SOI = (64, 128, 256, 512, 1024)


class Cfg(dict):
    """mmcv.Config stand-in: attribute and .get access."""
    __getattr__ = dict.__getitem__


BASE_CFG = dict(nms_pre=30, score_thr=0.3, nms=dict(type='nms', iou_threshold=0.5), max_per_img=100)

# (name, case kwargs, cfg overrides, rescale, with_nms)
CASES = [
    ('base', {}, {}, False, True),                                       # level 0 cut by nms_pre, levels 1 and 2 not
    ('split', {}, dict(nms=dict(type='nms', iou_threshold=0.5, split_thr=5)), False, True),   # mmcv's per-class branch
    ('truncate', {}, dict(max_per_img=4), False, True),
    ('rescale', {}, {}, True, True),
    ('nms_pre_all', {}, dict(nms_pre=-1), False, True),
    ('tight_iou', {}, dict(nms=dict(type='nms', iou_threshold=0.2)), True, True),
    ('no_candidate', {}, dict(score_thr=0.9999), False, True),
    ('one_empty', dict(empty_img=1), {}, True, True),
    ('no_nms', {}, {}, True, False),
]


def cfg_of(over):
    return Cfg(dict(BASE_CFG, **over))


def case(seed, B=2, empty_img=None, device='cpu'):
    """Seeded inputs: per level cls [B,C,H,W], bbox distances [B,4,H,W] (a few strides long, so boxes overlap), centerness
    [B,1,H,W], params [B,169,H,W]; mask_feat [B,8,8,10]; img_metas with a 60x75 image in the 64x80 padded input."""
    gen = torch.Generator().manual_seed(1000 + seed)
    cls, bbox, ctr, prm = [], [], [], []
    for (h, w), s in zip(SIZES, STRIDES):
        c = torch.randn(B, NUM_CLASSES, h, w, generator=gen) * 2 - 1.5
        if empty_img is not None:
            c[empty_img] = -20.
        cls.append(c)
        bbox.append(torch.rand(B, 4, h, w, generator=gen) * 3 * s + 1)
        ctr.append(torch.randn(B, 1, h, w, generator=gen))
        prm.append(torch.randn(B, NUM_PARAMS, h, w, generator=gen) * 0.5)
    feat = torch.randn(B, MASK_CH, 8, 10, generator=gen)
    metas = [dict(img_shape=(60, 75, 3), ori_shape=(45, 56, 3), pad_shape=(64, 80, 3),
                  scale_factor=np.array([75 / 56, 60 / 45, 75 / 56, 60 / 45], dtype=np.float32)) for _ in range(B)]
    to = lambda ts: [t.to(device) for t in ts]
    return to(cls), to(bbox), to(ctr), to(prm), feat.to(device), metas


def _methods(rel, cls_name, names, g):
    src = open(os.path.join(REF, rel)).read()
    cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == cls_name][0]
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert len(fns) == len(names), (cls_name, names)
    ns = dict(g)
    exec(compile(ast.Module(body=fns, type_ignores=[]), rel, 'exec'), ns)
    return {n: ns[n] for n in names}


def reference_heads():
    """(box head, mask head) stand-ins carrying the reference's own methods."""
    onnx = extract('mmdet/core/export/onnx_helper.py', ['get_k_for_topk'], {'os': os})
    sys.modules.setdefault('mmdet', types.ModuleType('mmdet'))
    sys.modules.setdefault('mmdet.core', types.ModuleType('mmdet.core'))
    sys.modules['mmdet.core.export'] = types.SimpleNamespace(get_k_for_topk=onnx.get_k_for_topk)
    d2b = extract('mmdet/core/bbox/transforms.py', ['distance2bbox']).distance2bbox
    top = extract('mmdet/models/dense_heads/condinst_head.py', ['nms_with_others', 'aligned_bilinear'],
                  {'batched_nms': lambda *a, **k: oci.batched_nms(*a, stable=False, **k)})
    g = dict(torch=torch, F=F, np=np, force_fp32=_force_fp32, distance2bbox=d2b, nms_with_others=top.nms_with_others,
             aligned_bilinear=top.aligned_bilinear)
    box = _methods('mmdet/models/dense_heads/condinst_head.py', 'CondInstBoxHead', ['get_bboxes', '_get_bboxes'], g)
    mask = _methods('mmdet/models/dense_heads/condinst_head.py', 'CondInstMaskHead',
                    ['forward', 'parse_dynamic_params', 'simple_test'], g)
    box_head = type('RefBoxHead', (), box)()
    box_head.prior_generator = types.SimpleNamespace(
        grid_priors=lambda sizes, dtype, device: oci.points([tuple(s) for s in sizes], STRIDES, device))
    box_head.cls_out_channels = NUM_CLASSES
    mask_head = type('RefMaskHead', (), mask)()
    first = MASK_CH + 2
    mask_head.__dict__.update(in_stride=8, out_stride=4, dynamic_convs=3, dynamic_channels=8, disable_rel_coors=False,
                              dy_weights=[first * 8, 8 * 8, 8], dy_biases=[8, 8, 1],
                              sizes_of_interest=torch.tensor(SOI))
    return box_head, mask_head


def oracle_masks(dets, feat, metas, rescale):
    """The oracle's simple_test for images with detections: bool [n, H, W] per image."""
    out = []
    for b, (d, lab, prm, coors, lvl) in enumerate(dets):
        logits = oci.mask_head_forward(feat, prm, coors, lvl, torch.full((len(prm),), b, dtype=torch.long),
                                       torch.tensor(SOI))
        out.append(oci.paste(logits, 4, metas[b]['img_shape'], metas[b]['ori_shape'] if rescale else None))
    return out


def main():
    box_head, mask_head = reference_heads()
    arrays = {}
    for seed, (name, kw, over, rescale, with_nms) in enumerate(CASES):
        cls, bbox, ctr, prm, feat, metas = case(seed, **kw)
        cfg = cfg_of(over)
        ref = box_head.get_bboxes(cls, bbox, ctr, prm, metas, cfg=cfg, rescale=rescale, with_nms=with_nms)
        ora = oci.get_bboxes(cls, bbox, ctr, prm, metas, cfg, STRIDES, rescale, with_nms)
        for b, (r, o) in enumerate(zip(ref, ora)):
            assert len(r) == len(o)
            for i, (rv, ov) in enumerate(zip(r, o)):
                assert rv.dtype == ov.dtype and torch.equal(rv, ov), (name, b, i)
                arrays[f'{name}_{b}_{i}'] = rv.numpy()
        if with_nms:
            keep = [b for b in range(len(ref)) if len(ref[b][0])]        # the reference mishandles an empty image in a batch
            if keep:
                sub = [ref[b] for b in keep]
                segm = mask_head.simple_test(feat[keep], [s[1] for s in sub], [s[2] for s in sub], [s[3] for s in sub],
                                             [s[4] for s in sub], [metas[b] for b in keep], NUM_CLASSES, rescale=rescale)
                mine = oracle_masks(sub, feat[keep], [metas[b] for b in keep], rescale)
                for j, b in enumerate(keep):
                    labels = sub[j][1].numpy()
                    m = mine[j].numpy().astype(np.uint8)
                    for c in range(NUM_CLASSES):
                        assert np.array_equal(segm[j][c], m[labels == c]), (name, b, c)
                    arrays[f'{name}_{b}_masks'] = np.packbits(m.astype(bool), axis=-1)
                    arrays[f'{name}_{b}_mask_shape'] = np.array(m.shape, np.int64)
        print(name, [len(r[0]) for r in ref])
    np.savez_compressed(OUT, **arrays)
    print('written', OUT)


if __name__ == '__main__':
    main()
