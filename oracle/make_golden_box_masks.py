"""Golden vectors for the box-mask pipeline, minted from the REFERENCE's own code (authoring container only).

AST-extracts ``GenerateBoxMask._generate_mask_from_box`` (mmdet/datasets/pipelines/loading.py) and the ``BitmapMasks``
class (mmdet/core/mask/structures.py) and runs them with ``mmcv`` bound to the restatement in oracle/box_masks.py, whose
``imresize`` is the real ``cv2.resize(INTER_NEAREST)`` (this script requires cv2).  Seeded chains as the configs build
them: DiscoBox / BoxLevelSet multiscale resize + flip + pad to a multiple of 32, and Box2Mask's large-scale jitter
(flip, resize by 0.1-2.0, RandomCrop with ``recompute_bbox``, FilterAnnotations, pad), at reduced image sizes; plus
boxes at rounding ties, negative and out-of-image boxes, one-pixel and whole-image boxes, rectangles that vanish under
downscaling, crops at the image edge and G = 0.  Asserts that the restatement equals the reference at every step and
writes tests/golden/box_masks.npz: per case the resolved chain (JSON) and, per step, the masks, ``get_bboxes()``,
``areas`` and the declared size.      python -m oracle.make_golden_box_masks"""
import ast
import json
import os
import types

import cv2  # noqa: F401  (the reference's resize; oracle.box_masks uses it when it imports)
import numpy as np

from oracle import box_masks as ob

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'box_masks.npz')


def reference():
    """(GenerateBoxMask, BitmapMasks) of the reference, built from its source with ``mmcv`` = the restatement."""
    mmcv = types.SimpleNamespace(rescale_size=lambda size, scale: ob.rescale_size(size, scale),
                                 imrescale=lambda img, scale, interpolation='nearest': ob.imrescale(img, scale,
                                                                                                     interpolation),
                                 imresize=lambda img, size, interpolation='nearest': ob.imresize(img, size, interpolation),
                                 imflip=lambda img, direction='horizontal': ob.imflip(img, direction),
                                 impad=lambda img, shape, pad_val=0: ob.impad(img, shape, pad_val))
    g = dict(np=np, mmcv=mmcv, BaseInstanceMasks=object)
    structures = ast.parse(open(os.path.join(REF, 'mmdet/core/mask/structures.py')).read())
    cls = [n for n in structures.body if isinstance(n, ast.ClassDef) and n.name == 'BitmapMasks'][0]
    exec(compile(ast.Module(body=[cls], type_ignores=[]), 'structures.py', 'exec'), g)
    loading = ast.parse(open(os.path.join(REF, 'mmdet/datasets/pipelines/loading.py')).read())
    gen = [n for n in loading.body if isinstance(n, ast.ClassDef) and n.name == 'GenerateBoxMask'][0]
    gen.decorator_list = []
    exec(compile(ast.Module(body=[gen], type_ignores=[]), 'loading.py', 'exec'), g)
    return g['GenerateBoxMask'], g['BitmapMasks']


def disco_chain(rng, G, h, w):
    """Resize(img_scale=[(1333, 800) .. (1333, 640)], multiscale 'value', keep_ratio) + RandomFlip + Pad(32), at 1/4."""
    scale = (333, int(rng.choice([200, 192, 184, 176, 168, 160])))
    c = [('generate', ob._boxes(rng, G, h, w), h, w), ('rescale', scale), ('flip', 'horizontal')]
    return c + [('pad', None)]


def lsj_chain(rng, G, h, w, side=128):
    """Box2Mask's large-scale jitter at image_size = side: flip, Resize(ratio 0.1-2.0, keep_ratio), RandomCrop(side)
    with recompute_bbox, FilterAnnotations(1e-5), Pad(side)."""
    r = rng.uniform(0.1, 2.0)
    c = [('generate', ob._boxes(rng, G, h, w), h, w), ('flip', str(rng.choice(['horizontal', 'vertical', 'diagonal']))),
         ('rescale', (int(side * r), int(side * r)))]
    return c + [('lsj_crop', side), ('filter', 1e-5), ('pad', (side, side))]


def resolve_lsj(chain, h, w, rng):
    """Replace 'lsj_crop' by RandomCrop's index of kept masks and its crop box, from the size after the rescale."""
    out = []
    for op in chain:
        if op[0] == 'lsj_crop':
            side = op[1]
            nw, nh = ob.rescale_size((w, h), out[-1][1])
            oy, ox = int(rng.integers(0, max(nh - side, 0) + 1)), int(rng.integers(0, max(nw - side, 0) + 1))
            out.append(('index', None))
            out.append(('crop', [ox, oy, ox + side, oy + side]))
        else:
            out.append(op)
    return out


def special_chain(rng):
    h, w = 37, 53
    b = np.array([[0.5, 0.5, 10.5, 10.5], [1.5, 2.5, 3.5, 4.5], [-7.2, -3.0, 5.4, 6.6], [-60, -40, -20, -10],
                  [60, 40, 80, 50], [0, 0, w - 1, h - 1], [12, 13, 12, 13], [40.49, 30.5, 52.5, 36.5],
                  [-0.5, -0.5, w - 0.5, h - 0.5], [20, 5, 21, 5]], dtype=np.float32)
    return [('generate', b, h, w), ('rescale', 0.1), ('resize', (37, 53)), ('flip', 'diagonal'),
            ('crop', [5, 3, 40, 30]), ('expand', (50, 60, 4, 6)), ('pad', (64, 64)), ('index', None)]


def edge_chain(rng):
    b = np.array([[1, 1, 5, 5], [0, 0, 9, 7]], dtype=np.float32)
    return [('generate', b, 8, 10), ('crop', [10, 2, 12, 6]), ('pad', (9, 4))]


def empty_chain(rng):
    return [('generate', np.zeros((0, 4), np.float32), 21, 17), ('rescale', (40, 30)), ('flip', 'vertical'),
            ('crop', [2, 3, 15, 11]), ('pad', (32, 32)), ('expand', (40, 40, 3, 5))]


def cases():
    out = []
    for s, G in enumerate((7, 20, 3)):
        rng = np.random.default_rng(100 + s)
        out.append(('disco_%d' % s, disco_chain(rng, G, int(rng.integers(90, 130)), int(rng.integers(140, 170))), rng))
    for s, G in enumerate((12, 40, 1)):
        rng = np.random.default_rng(200 + s)
        h, w = int(rng.integers(60, 130)), int(rng.integers(60, 130))
        out.append(('lsj_%d' % s, resolve_lsj(lsj_chain(rng, G, h, w), h, w, rng), rng))
    for name, fn in (('special', special_chain), ('edge', edge_chain), ('empty', empty_chain)):
        rng = np.random.default_rng(len(out))
        out.append((name, fn(rng), rng))
    for s in range(6):
        rng = np.random.default_rng(300 + s)
        out.append(('random_%d' % s, ob.random_chain(rng), rng))
    return out


def _jsonable(op):
    return [v.tolist() if isinstance(v, np.ndarray) else v for v in op]


def main():
    Gen, Ref = reference()
    gen = Gen()

    def make_ref(boxes, h, w):
        return gen._generate_mask_from_box({'gt_bboxes': boxes, 'img': np.zeros((h, w, 3), np.float32),
                                            'mask_fields': []})['gt_masks']

    data = {}
    names = []
    for name, chain, rng in cases():
        state = rng.bit_generator.state
        ref_steps, done = ob.run_chain(chain, make_ref, rng)
        rng.bit_generator.state = state
        orc_steps, _ = ob.run_chain(done, ob.generate_box_mask)
        assert isinstance(ref_steps[0], Ref)
        for i, (r, o) in enumerate(zip(ref_steps, orc_steps)):
            assert r.masks.shape == o.masks.shape and r.masks.dtype == o.masks.dtype, (name, i)
            assert np.array_equal(r.masks, o.masks) and (r.height, r.width) == (o.height, o.width), (name, i)
            assert np.array_equal(r.get_bboxes(), o.get_bboxes()) and np.array_equal(r.areas, o.areas), (name, i)
            assert r.areas.dtype == o.areas.dtype, (name, i)
            data[f'{name}/{i}/masks'] = r.masks
            data[f'{name}/{i}/bboxes'] = r.get_bboxes()
            data[f'{name}/{i}/areas'] = r.areas
            data[f'{name}/{i}/size'] = np.array([r.height, r.width], dtype=np.int64)
        data[f'{name}/chain'] = np.array(json.dumps([_jsonable(op) for op in done]))
        data[f'{name}/boxes'] = done[0][1]
        names.append(name)
    data['cases'] = np.array(names)
    np.savez_compressed(OUT, **data)
    print(f'wrote {OUT}: {len(names)} chains, {os.path.getsize(OUT)} bytes')


if __name__ == '__main__':
    main()
