"""Golden vectors for ``encode_mask_results`` (COCO RLE of mask results), minted from the REFERENCE's own function
(authoring container only).

``encode_mask_results`` is AST-extracted from mmdet/core/mask/utils.py, its ``mask_util`` bound to oracle/mask_rle.py (the
restatement of pycocotools' ``encode``), and run on the seeded mask results of ``CASES``.  Written to
tests/golden/mask_rle.npz, per case: the masks in class order then detection order (bit-packed, or raw bytes when a uint8
mask holds values above 1), their shapes, the masks per class, and the expected strings concatenated with their offsets.
    python -m oracle.make_golden_mask_rle
"""
import ast
import os

import numpy as np

from oracle import mask_rle as omr

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'mask_rle.npz')

# (name, form): form is 'list' (per-class lists of 2-D masks), 'tuple' ((cls_segms, cls_mask_scores), SOLOv2's
# format_results) or 'array' (per-class [k, H, W] arrays, CondInst's simple_test)
CASES = [
    ('list_bool', 'list'),
    ('tuple_uint8', 'tuple'),
    ('array_per_class', 'array'),
    ('empty_classes', 'list'),
    ('odd_sizes', 'list'),
    ('edge_pixels', 'list'),
    ('checkerboard', 'list'),
    ('uint8_values', 'list'),
    ('long_runs', 'list'),
]


def blobs(gen, k, H, W):
    """k bool masks [H, W] of one to three seeded ellipses each."""
    ys, xs = np.mgrid[:H, :W]
    out = np.zeros((k, H, W), bool)
    for i in range(k):
        for _ in range(gen.integers(1, 4)):
            cy, cx = gen.uniform(0, H), gen.uniform(0, W)
            ry, rx = gen.uniform(1, H / 3 + 1), gen.uniform(1, W / 3 + 1)
            out[i] |= ((ys - cy) / ry) ** 2 + ((xs - cx) / rx) ** 2 <= 1
    return out


def long_run_mask():
    """One 4200 x 4200 uint8 mask whose column-major runs are 5, 3, 16777300, 1, 7, 600000, 3, 2 and the rest: deltas of
    6 and 5 characters, positive and negative."""
    H = W = 4200
    runs = [5, 3, 16777300, 1, 7, 600000, 3, 2]
    runs.append(H * W - sum(runs))
    flat = np.repeat(np.arange(len(runs)) % 2, runs).astype(np.uint8)
    return flat.reshape(W, H).T.copy()


def case(i):
    """The mask results of case i, on the host: numpy masks."""
    name, form = CASES[i]
    gen = np.random.default_rng(2000 + i)
    if name == 'list_bool':
        m = blobs(gen, 7, 60, 80)
        return [list(m[:3]), [], list(m[3:])]
    if name == 'tuple_uint8':
        m = blobs(gen, 5, 48, 64).astype(np.uint8)
        return [list(m[:2]), list(m[2:])], [[0.9, 0.5], [0.8, 0.7, 0.1]]
    if name == 'array_per_class':
        m = blobs(gen, 6, 40, 56).astype(np.uint8)
        return [m[:4], np.zeros((0, 40, 56), np.uint8), m[4:]]
    if name == 'empty_classes':
        return [[], [], [], []]
    if name == 'odd_sizes':
        big = blobs(gen, 2, 427, 641)
        return [list(big), [gen.random((1, 37)) < 0.5], [gen.random((29, 1)) < 0.5, big[0][:, :1].copy()]]
    if name == 'edge_pixels':
        H, W = 24, 32
        first, last, both = (np.zeros((H, W), bool) for _ in range(3))
        first[0, 0] = True
        last[H - 1, W - 1] = True
        both[0, 0] = both[H - 1, W - 1] = True
        return [[first, last, np.ones((H, W), bool), np.zeros((H, W), bool), both]]
    if name == 'checkerboard':
        c = (np.add.outer(np.arange(15), np.arange(20)) % 2 == 0)   # odd H: every pixel a run, the first one set
        return [[c, ~c]]
    if name == 'uint8_values':
        m = blobs(gen, 4, 30, 44).astype(np.uint8) * gen.integers(1, 256, (4, 1, 1)).astype(np.uint8)
        m[1, 5:20, 10:30] = 7                                   # a change between two non-zero values
        m[2] = gen.integers(0, 4, (30, 44))                     # 0, 1, 2, 3 at random
        return [list(m[:2]), list(m[2:])]
    if name == 'long_runs':
        m = long_run_mask()
        return [[m, (1 - m).astype(bool)]]
    raise KeyError(name)


def segms_of(results):
    """The per-class mask lists of a case's results (either form)."""
    return results[0] if isinstance(results, tuple) else results


def reference_fn():
    """The reference's encode_mask_results with ``mask_util`` bound to oracle/mask_rle.py."""
    rel = 'mmdet/core/mask/utils.py'
    src = open(os.path.join(REF, rel)).read()
    fn = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == 'encode_mask_results'][0]
    ns = dict(np=np, mask_util=omr)
    exec(compile(ast.Module(body=[fn], type_ignores=[]), rel, 'exec'), ns)
    return ns['encode_mask_results']


def flatten(encoded):
    """(per-class counts, concatenated strings uint8, offsets int64 [m + 1], sizes int64 [m, 2]) of an encoded value."""
    rles = [r for per in encoded for r in per]
    lens = [len(r['counts']) for r in rles]
    return (np.array([len(per) for per in encoded], np.int64),
            np.frombuffer(b''.join(r['counts'] for r in rles), np.uint8).copy(),
            np.concatenate(([0], np.cumsum(lens))).astype(np.int64),
            np.array([r['size'] for r in rles], np.int64).reshape(-1, 2))


def main():
    ref = reference_fn()
    arrays = {}
    for i, (name, form) in enumerate(CASES):
        results = case(i)
        out = ref(results)
        if form == 'tuple':
            assert isinstance(out, tuple) and out[1] is results[1]
            out = out[0]
        for per in out:
            for r in per:
                assert isinstance(r['counts'], bytes) and all(type(v) is int for v in r['size'])
        per_class, chars, offsets, sizes = flatten(out)
        masks = [np.asarray(m) for per in segms_of(results) for m in per]
        arrays[f'{name}_per_class'] = per_class
        arrays[f'{name}_chars'] = chars
        arrays[f'{name}_offsets'] = offsets
        arrays[f'{name}_sizes'] = sizes
        arrays[f'{name}_dtypes'] = np.array([str(m.dtype) for m in masks])
        flat = np.concatenate([m.reshape(-1).astype(np.uint8) for m in masks]) if masks else np.zeros(0, np.uint8)
        if flat.size and flat.max() > 1:
            arrays[f'{name}_raw'] = flat
        else:
            arrays[f'{name}_bits'] = np.packbits(flat)
        print(name, per_class.tolist(), 'chars', len(chars))
    np.savez_compressed(OUT, **arrays)
    print('written', OUT)


if __name__ == '__main__':
    main()
