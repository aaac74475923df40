"""Golden vectors for ``format_results`` of the SOLOv2-family detectors, minted from the REFERENCE's own function
(authoring container only).

``format_results`` is AST-extracted from SingleStageBoxInsDetector (mmdet/models/detectors/single_stage_boxseg.py, used by
BoxLevelSet) and SingleStageWSInsDetector (single_stage_ts.py, used by DiscoBoxSOLOv2); their ASTs are asserted identical,
so one restatement pins both.  It is bound to a stand-in detector whose ``bbox_head.num_classes`` is the case's, run on the
seeded results of ``CASES``, asserted equal to oracle/solo_format.py, and written to tests/golden/solo_format.npz: per case
the bbox rows of every class in class order, each row's class, the kept masks bit-packed and their scores.
    python -m oracle.make_golden_solo_format
"""
import ast
import os
import types

import numpy as np
import torch

from oracle import solo_format as osf

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'solo_format.npz')

# (name, n, H, W, num_classes, kind): kind picks the masks and scores of case()
CASES = [
    ('empty_between', 12, 24, 32, 5, 'empty_between'),
    ('all_empty', 5, 24, 32, 3, 'all_empty'),
    ('corners', 4, 24, 32, 2, 'corners'),
    ('full_frame', 3, 24, 32, 4, 'full'),
    ('equal_scores', 6, 24, 32, 3, 'equal_scores'),
    ('sparse_classes', 7, 24, 32, 9, 'sparse_classes'),
    ('odd_width', 6, 427, 641, 4, 'blobs'),
    ('uint8_values', 6, 20, 48, 3, 'uint8'),
    ('no_detection', 0, 24, 32, 3, 'none'),
]


def case(i, device='cpu'):
    """Seeded results of case i: a namespace with ``labels`` int64 [n], ``scores`` float32 [n] and ``masks`` [n, H, W]
    (bool; uint8 with values up to 255 for 'uint8'; empty float32 for 'none', as the reference's ``empty_results``)."""
    name, n, H, W, C, kind = CASES[i]
    gen = torch.Generator().manual_seed(1000 + i)
    labels = torch.randint(0, C, (n,), generator=gen)
    scores = torch.rand(n, generator=gen)
    ys = torch.arange(H).view(H, 1)
    xs = torch.arange(W).view(1, W)
    masks = torch.zeros(n, H, W, dtype=torch.bool)
    for k in range(n):                                       # rectangles of random extent
        y0, x0 = int(torch.randint(0, H, (1,), generator=gen)), int(torch.randint(0, W, (1,), generator=gen))
        y1 = y0 + 1 + int(torch.randint(0, H - y0, (1,), generator=gen))
        x1 = x0 + 1 + int(torch.randint(0, W - x0, (1,), generator=gen))
        masks[k] = (ys >= y0) & (ys < y1) & (xs >= x0) & (xs < x1)
    if kind == 'empty_between':
        masks[1::3] = False
    elif kind == 'all_empty':
        masks[:] = False
    elif kind == 'corners':
        masks[:] = False
        for k, (y, x) in enumerate(((0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1))):
            masks[k, y, x] = True
        labels[:] = 1
    elif kind == 'full':
        masks[:] = True
    elif kind == 'equal_scores':
        scores[:] = 0.5
        labels[:] = 2
    elif kind == 'sparse_classes':
        labels = torch.tensor([1, 5, 1, 8, 5, 1, 8])[:n]
    elif kind == 'uint8':
        masks = masks.to(torch.uint8) * torch.randint(1, 256, (n, 1, 1), generator=gen, dtype=torch.uint8)
        masks[2] = 0
    elif kind == 'none':
        masks = torch.zeros(0, H, W)
    return types.SimpleNamespace(labels=labels.to(device), scores=scores.to(device), masks=masks.to(device)), C


def reference_fn():
    """The reference's format_results, after asserting that both detector files define the same one."""
    fns = []
    for rel, cls_name in (('mmdet/models/detectors/single_stage_boxseg.py', 'SingleStageBoxInsDetector'),
                          ('mmdet/models/detectors/single_stage_ts.py', 'SingleStageWSInsDetector')):
        src = open(os.path.join(REF, rel)).read()
        cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == cls_name][0]
        fns.append(([n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name == 'format_results'][0], rel))
    assert ast.dump(fns[0][0]) == ast.dump(fns[1][0]), 'the two format_results differ'
    ns = dict(torch=torch, np=np)
    exec(compile(ast.Module(body=[fns[0][0]], type_ignores=[]), fns[0][1], 'exec'), ns)
    fn = ns['format_results']

    def run(results, num_classes):
        return fn(types.SimpleNamespace(bbox_head=types.SimpleNamespace(num_classes=num_classes)), results)
    return run


def flatten(out):
    """(bbox rows of every class in class order, each row's class, kept masks, their scores) of a format_results value."""
    bbox, (masks, scores) = out
    cls = np.concatenate([np.full(len(b), c, np.int64) for c, b in enumerate(bbox)])
    rows = np.concatenate([b.reshape(-1, 5) for b in bbox])
    m = [x for per in masks for x in per]
    s = [x for per in scores for x in per]
    return rows, cls, m, s


def assert_same(a, b, what):
    """Exact equality of two format_results values: structure, dtypes, devices, order and values."""
    (ba, (ma, sa)), (bb, (mb, sb)) = a, b
    assert len(ba) == len(bb) == len(ma) == len(mb) == len(sa) == len(sb), what
    for c in range(len(ba)):
        assert isinstance(ba[c], np.ndarray) and ba[c].dtype == bb[c].dtype == np.float64, (what, c)
        assert ba[c].shape == bb[c].shape and np.array_equal(ba[c], bb[c]), (what, c)
        assert len(ma[c]) == len(mb[c]) and len(sa[c]) == len(sb[c]), (what, c)
        for x, y in zip(ma[c] + sa[c], mb[c] + sb[c]):
            assert x.device == y.device and x.device.type == 'cpu', (what, c)
            assert x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y), (what, c)


def main():
    ref = reference_fn()
    arrays = {}
    for i, (name, *_rest) in enumerate(CASES):
        results, C = case(i)
        r = ref(results, C)
        assert_same(r, osf.format_results(results, C), name)
        rows, cls, m, s = flatten(r)
        arrays[f'{name}_bbox'] = rows
        arrays[f'{name}_cls'] = cls
        arrays[f'{name}_masks'] = np.packbits(np.stack([x.numpy() != 0 for x in m]), axis=-1) if m else np.zeros(0, np.uint8)
        arrays[f'{name}_mask_values'] = np.stack([x.numpy() for x in m]).astype(np.uint8).max((1, 2)) if m else np.zeros(0, np.uint8)
        arrays[f'{name}_scores'] = np.array([float(x) for x in s], np.float32)
        arrays[f'{name}_dtype'] = np.array(str(m[0].dtype) if m else '')
        print(name, [len(b) for b in r[0]])
    np.savez_compressed(OUT, **arrays)
    print('written', OUT)


if __name__ == '__main__':
    main()
