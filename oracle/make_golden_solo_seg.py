"""Golden vectors for SOLOv2 inference, minted from the REFERENCE's own functions (authoring container only).

``mask_matrix_nms`` is AST-extracted from mmdet/core/post_processing/matrix_nms.py, ``get_seg`` / ``get_seg_single`` from
BoxSOLOv2Head (mmdet/models/dense_heads/box_solov2_head.py) and DiscoBoxSOLOv2Head (discobox_head.py), and bound to stand-in
heads holding the grids and strides; ``InstanceData`` is a namespace of the meta fields and ``@autocast()`` the identity (CPU,
float32).  Asserts that oracle/solo_seg.py (with the reference's own unstable sorts) equals them, and writes
tests/golden/solo_seg.npz: per case and image the scores, labels and bit-packed masks.      python -m oracle.make_golden_solo_seg
"""
import ast
import os
import types

import numpy as np
import torch
import torch.nn.functional as F

from oracle import solo_seg as oss
from oracle.make_golden import extract

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'solo_seg.npz')

BASE_CFG = dict(score_thr=0.1, mask_thr=0.5, nms_pre=500, max_per_img=100, kernel='gaussian', sigma=2.0, filter_thr=0.05)

# (name, method, case kwargs, cfg overrides)
CASES = [
    ('gaussian', 'box', {}, {}),
    ('linear', 'box', {}, dict(kernel='linear')),
    ('truncate', 'box', {}, dict(nms_pre=5, max_per_img=3)),
    ('filter', 'box', {}, dict(filter_thr=0.35)),
    ('no_candidate', 'box', {}, dict(score_thr=0.999)),
    ('stride_filter', 'box', dict(strides=(5000, 5000, 5000)), {}),
    ('two_classes', 'box', dict(two_class_cell=True), {}),
    ('img_ne_ori', 'box', dict(img_shape=(37, 50, 3), ori_shape=(30, 41, 3)), {}),
    ('odd_hw', 'box', dict(h=11, w=13), {}),
    ('disco_gaussian', 'disco', {}, dict(mask_thr=0.4)),
    ('disco_linear_trunc', 'disco', dict(img_shape=(37, 50, 3), ori_shape=(30, 41, 3)),
     dict(mask_thr=0.4, kernel='linear', nms_pre=6, max_per_img=4)),
    ('disco_odd_hw', 'disco', dict(h=11, w=13), dict(mask_thr=0.4)),
]


def cfg_of(over):
    return types.SimpleNamespace(**dict(BASE_CFG, **over))


def case(seed, method='box', B=2, h=12, w=16, C=5, E=8, grids=(6, 4, 3), strides=(8, 8, 16), img_shape=(44, 60, 3),
         ori_shape=(44, 60, 3), two_class_cell=False, device='cpu'):
    """Seeded inputs of one golden case: (head stand-in, the head's get_seg arguments, img_metas).  BoxSOLOv2: probabilities of
    overlapping blobs [B,S^2,h,w] per level and local-max-style category maps [B,S,S,C]; DiscoBox: features [B,E,h,w] and raw
    kernel grids [B,E,S,S] whose products give blob-shaped logits."""
    gen = torch.Generator().manual_seed(seed)
    head = types.SimpleNamespace(cate_out_channels=C, kernel_out_channels=E, seg_num_grids=list(grids), strides=list(strides))
    cate = []
    for S in grids:
        c = torch.rand(B, S, S, C, generator=gen) ** 4
        if two_class_cell:
            c[0, 0, 0, :2] = torch.tensor([0.9, 0.8])
        cate.append(c)
    ys = torch.arange(h, dtype=torch.float32).view(h, 1)
    xs = torch.arange(w, dtype=torch.float32).view(1, w)
    metas = [dict(img_shape=img_shape, ori_shape=ori_shape, pad_shape=(4 * h, 4 * w, 3))] * B
    if method == 'box':
        seg = []
        for S in grids:
            cy = torch.rand(B, S * S, 1, 1, generator=gen) * h
            cx = torch.rand(B, S * S, 1, 1, generator=gen) * w
            r = 1.5 + torch.rand(B, S * S, 1, 1, generator=gen) * min(h, w) / 3
            d = ((ys - cy) ** 2 + (xs - cx) ** 2).sqrt()
            seg.append(torch.sigmoid((r - d) * 1.7))
        args = ([s.to(device) for s in seg], [c.to(device) for c in cate], None)
    else:
        feat = torch.randn(B, E, h, w, generator=gen)
        feat[:, 0] = (ys / h - 0.5) * 4            # coordinate-like channels make blob-like logits
        feat[:, 1] = (xs / w - 0.5) * 4
        kern = [torch.randn(B, E, S, S, generator=gen) for S in grids]
        args = ([c.to(device) for c in cate], [k.to(device) for k in kern], feat.to(device))
    return head, args, metas


def reference_fns():
    """The reference's own functions, bound to stand-in globals."""
    mnms = extract('mmdet/core/post_processing/matrix_nms.py', ['mask_matrix_nms']).mask_matrix_nms
    g = dict(torch=torch, F=F, np=np, InstanceData=oss.InstanceData, mask_matrix_nms=mnms,
             autocast=lambda *a, **k: (lambda fn: fn))
    out = {}
    for rel, cls_name, key in (('mmdet/models/dense_heads/box_solov2_head.py', 'BoxSOLOv2Head', 'box'),
                               ('mmdet/models/dense_heads/discobox_head.py', 'DiscoBoxSOLOv2Head', 'disco')):
        src = open(os.path.join(REF, rel)).read()
        cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == cls_name][0]
        fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in ('get_seg', 'get_seg_single')]
        assert len(fns) == 2
        ns = dict(g)
        exec(compile(ast.Module(body=fns, type_ignores=[]), rel, 'exec'), ns)
        out[key] = type(f'Ref{cls_name}', (), {'get_seg': ns['get_seg'], 'get_seg_single': ns['get_seg_single']})
    return out, mnms


def run_oracle(method, head, args, metas, cfg, stable=False):
    if method == 'box':
        return oss.box_get_seg(head, *args, metas, cfg, stable=stable)
    return oss.disco_get_seg(head, *args, metas, cfg, stable=stable)


def main():
    refs, mnms = reference_fns()
    arrays = {}
    for seed, (name, method, kw, over) in enumerate(CASES):
        head, args, metas = case(seed, method, **kw)
        cfg = cfg_of(over)
        me = refs[method]()
        me.__dict__.update(vars(head))
        ref = me.get_seg(*args, metas, cfg)
        ora = run_oracle(method, head, args, metas, cfg)
        for b, (r, o) in enumerate(zip(ref, ora)):
            for k in ('scores', 'labels', 'masks'):
                rv, ov = getattr(r, k), getattr(o, k)
                assert rv.dtype == ov.dtype and rv.shape == ov.shape and torch.equal(rv, ov), (name, b, k)
            arrays[f'{name}_{b}_scores'] = r.scores.numpy()
            arrays[f'{name}_{b}_labels'] = r.labels.numpy()
            arrays[f'{name}_{b}_masks'] = np.packbits(r.masks.numpy().astype(bool), axis=-1)
            arrays[f'{name}_{b}_shape'] = np.array(r.masks.shape, np.int64)
            arrays[f'{name}_{b}_dtype'] = np.array(str(r.masks.dtype))
        print(name, [len(r.scores) for r in ref])
    # the standalone mask_matrix_nms: both kernels, truncation and the filter, against the reference's own function
    for i, kw in enumerate(NMS_CASES):
        masks, labels, scores = nms_case(i)
        r = mnms(masks, labels, scores, **kw)
        o = oss.mask_matrix_nms(masks, labels, scores, **kw)
        for a, b in zip(r, o):
            assert a.dtype == b.dtype and torch.equal(a, b), (i, kw)
        arrays[f'nms{i}_scores'], arrays[f'nms{i}_labels'], arrays[f'nms{i}_keep'] = r[0].numpy(), r[1].numpy(), r[3].numpy()
    np.savez_compressed(OUT, **arrays)
    print('written', OUT)


NMS_CASES = [dict(), dict(kernel='linear'), dict(nms_pre=7, max_num=4), dict(filter_thr=0.4), dict(sigma=0.5, filter_thr=0.2)]


def nms_case(seed, n=20, h=9, w=13, classes=3):
    """Overlapping boolean rectangles with a few labels and distinct scores."""
    gen = torch.Generator().manual_seed(100 + seed)
    masks = torch.zeros(n, h, w, dtype=torch.bool)
    for i in range(n):
        y0, x0 = int(torch.randint(0, h - 3, (1,), generator=gen)), int(torch.randint(0, w - 3, (1,), generator=gen))
        masks[i, y0:y0 + 3 + int(torch.randint(0, 4, (1,), generator=gen)), x0:x0 + 3 + int(torch.randint(0, 5, (1,), generator=gen))] = True
    labels = torch.randint(0, classes, (n,), generator=gen)
    scores = torch.rand(n, generator=gen) * 0.9 + 0.1
    return masks, labels, scores


if __name__ == '__main__':
    main()
