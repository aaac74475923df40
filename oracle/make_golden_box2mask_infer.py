"""Golden vectors for Box2Mask inference, minted from the REFERENCE's own lines (authoring container only).

AST-extracted: ``Box2MaskHead.simple_test`` (mmdet/models/dense_heads/box2mask_head.py), ``MaskFormerFusionHead.simple_test``
/ ``instance_postprocess`` (mmdet/models/seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py) and ``mask2bbox``
(mmdet/core/mask/utils.py), bound to stand-in heads.  Their ``F.interpolate`` is the oracle's restatement of ATen's bilinear
arithmetic (what the CUDA kernels compute; torch's CPU kernel differs from it in the last bits, checked here to 1e-5), the
rest is torch.  Asserts that the oracle equals them -- the (label, score, box, mask) rows compared after a canonical sort,
because the reference's ``topk(sorted=False)`` promises no order -- and writes tests/golden/box2mask_infer.npz.
                                                                            python -m oracle.make_golden_box2mask_infer
"""
import os
import types

import numpy as np
import torch
import torch.nn.functional as F

from oracle import box2mask_infer as obi
from oracle.make_golden import extract

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'box2mask_infer.npz')

Q = 6
BASE = dict(things=3, stuff=0, hw=(8, 10), pad=(32, 40), max_per_image=10, rescale=True,
            shapes=(((30, 37), (20, 25)), ((25, 40), (40, 64))))
# (name, overrides): two images with different img_shape / ori_shape in every case; query 2 of image 0 is picked for two
# classes and query 4 of image 1 has no positive logit (see case())
CASES = [
    ('base', {}),
    ('no_rescale', dict(rescale=False)),
    ('pad_not_4h', dict(hw=(7, 9))),
    ('stuff', dict(stuff=2, max_per_image=12)),
    ('all_pairs', dict(max_per_image=Q * 3)),
]


def case_cfg(i):
    return dict(BASE, **CASES[i][1])


def case(i):
    """(mask_cls [2,Q,K+1], mask_pred [2,Q,h,w] at the mask-feature resolution, img_metas, cfg) of case i."""
    cfg = case_cfg(i)
    K = cfg['things'] + cfg['stuff']
    gen = torch.Generator().manual_seed(2000 + i)
    mask_cls = torch.randn(2, Q, K + 1, generator=gen) * 2
    mask_cls[0, 2, :2] = 6.0 + torch.rand(2, generator=gen)        # a query picked for two classes
    mask_cls[1, 4, 0] = 8.0                                          # ... and an empty mask picked
    mask_pred = torch.randn(2, Q, *cfg['hw'], generator=gen) * 3
    mask_pred[1, 4] = -2.0 - torch.rand(*cfg['hw'], generator=gen)
    metas = [dict(img_shape=img + (3,), ori_shape=ori + (3,), pad_shape=cfg['pad'] + (3,), batch_input_shape=cfg['pad'])
             for img, ori in cfg['shapes']]
    return mask_cls, mask_pred, metas, cfg


def reference_heads(cfg):
    """(Box2MaskHead, MaskFormerFusionHead) stand-ins carrying the reference's own methods."""
    m2b = extract('mmdet/core/mask/utils.py', ['mask2bbox']).mask2bbox
    Fi = types.SimpleNamespace(softmax=F.softmax, interpolate=obi.interpolate)
    head = extract('mmdet/models/dense_heads/box2mask_head.py', ['Box2MaskHead'],
                   {'AnchorFreeHead': object, 'HEADS': types.SimpleNamespace(register_module=lambda *a, **k: (lambda c: c)),
                    'F': Fi, 'force_fp32': lambda *a, **k: (lambda f: f)})
    fusion = extract('mmdet/models/seg_heads/panoptic_fusion_heads/maskformer_fusion_head.py', ['MaskFormerFusionHead'],
                     {'BasePanopticFusionHead': object, 'HEADS': types.SimpleNamespace(register_module=lambda *a, **k: (lambda c: c)),
                      'F': Fi, 'mask2bbox': m2b, 'INSTANCE_OFFSET': 1000})
    ref_head = type('RefBox2MaskHead', (), {'simple_test': head.Box2MaskHead.simple_test,
                                            '__call__': lambda self, feats, img_metas: self.forward_out})()
    ref_fusion = type('RefFusionHead', (), {'simple_test': fusion.MaskFormerFusionHead.simple_test,
                                            'instance_postprocess': fusion.MaskFormerFusionHead.instance_postprocess})()
    ref_fusion.__dict__.update(num_things_classes=cfg['things'], num_stuff_classes=cfg['stuff'],
                               num_classes=cfg['things'] + cfg['stuff'],
                               test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True,
                                             max_per_image=cfg['max_per_image']))
    return ref_head, ref_fusion


def canonical(labels, bboxes, masks):
    """Rows sorted by (label, score, box), as numpy arrays."""
    labels, bboxes, masks = labels.numpy(), bboxes.numpy(), masks.numpy()
    o = np.lexsort([bboxes[:, k] for k in (3, 2, 1, 0, 4)] + [labels])
    return labels[o], bboxes[o], masks[o]


def main():
    arrays = {}
    for i, (name, _) in enumerate(CASES):
        mask_cls, mask_pred, metas, cfg = case(i)
        ref_head, ref_fusion = reference_heads(cfg)
        ref_head.forward_out = ([mask_cls], [mask_pred], [None])     # what ``self(feats, img_metas)`` returns
        cls_r, pred_r = ref_head.simple_test(None, metas)
        up = F.interpolate(mask_pred, cfg['pad'], mode='bilinear', align_corners=False)
        assert (up - pred_r).abs().max() <= 1e-5                   # the restatement against torch's CPU kernel
        ref = ref_fusion.simple_test(cls_r, pred_r, metas, rescale=cfg['rescale'])
        ora = obi.fusion_simple_test(*obi.head_simple_test([mask_cls], [mask_pred]), metas, cfg['things'],
                                     cfg['max_per_image'], cfg['rescale'])
        ora_hi = obi.fusion_simple_test(cls_r, pred_r, metas, cfg['things'], cfg['max_per_image'], cfg['rescale'])
        for b, (r, o, oh) in enumerate(zip(ref, ora, ora_hi)):
            labels, query, bboxes, masks = o
            assert all(torch.equal(x, y) for x, y in zip(o, oh)), (name, b)
            for x, y in zip(canonical(*r['ins_results']), canonical(labels, bboxes, masks)):
                assert x.dtype == y.dtype and np.array_equal(x, y), (name, b)
            arrays[f'{name}_{b}_labels'] = labels.numpy()
            arrays[f'{name}_{b}_query'] = query.numpy()
            arrays[f'{name}_{b}_bboxes'] = bboxes.numpy()
            arrays[f'{name}_{b}_masks'] = np.packbits(masks.numpy(), axis=-1)
            arrays[f'{name}_{b}_mask_shape'] = np.array(masks.shape, np.int64)
        print(name, [len(o[0]) for o in ora])
    np.savez_compressed(OUT, **arrays)
    print('written', OUT)


if __name__ == '__main__':
    main()
