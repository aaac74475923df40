"""CPU: ``BoxMasks`` and ``GenerateBoxMask`` against the reference's own ``BitmapMasks`` / ``GenerateBoxMask``
(tests/golden/box_masks.npz), the numpy restatement over random chains, and cv2's nearest resize."""
import json
import pickle
import subprocess
import sys

import numpy as np
import pytest

from boxinstseg_b200.core import BoxMasks
from boxinstseg_b200.core.box_masks import nearest_map
from oracle import box_masks as ob

ROOT = __import__('os').path.dirname(__import__('os').path.dirname(__import__('os').path.abspath(__file__)))


def make_box_masks(boxes, h, w):
    from boxinstseg_b200.datasets import GenerateBoxMask
    results = {'gt_bboxes': np.asarray(boxes, dtype=np.float32), 'img': np.zeros((h, w, 3), np.float32),
               'mask_fields': []}
    out = GenerateBoxMask()(results)
    assert out['mask_fields'] == ['gt_masks']
    return out['gt_masks']


def _chain(raw):
    ops = json.loads(str(raw))
    first = ops[0]
    return [('generate', np.asarray(first[1], dtype=np.float32), first[2], first[3])] + [tuple(op) for op in ops[1:]]


def _same(a, b, where):
    """``a`` (BoxMasks) equals ``b`` (any BitmapMasks-like object) in every observable."""
    assert isinstance(a, BoxMasks), where
    assert (a.height, a.width) == (b.height, b.width), where
    assert len(a) == len(b), where
    x, y = a.to_ndarray(), b.to_ndarray()
    assert x.shape == y.shape and x.dtype == y.dtype and np.array_equal(x, y), where
    assert a.get_bboxes().dtype == np.float32 and np.array_equal(a.get_bboxes(), b.get_bboxes()), where
    assert a.areas.dtype == b.areas.dtype and np.array_equal(a.areas, b.areas), where


def test_golden_chains(golden):
    g = golden('box_masks')
    names = list(g['cases'])
    assert len(names) >= 12
    for name in names:
        chain = _chain(g[f'{name}/chain'])
        steps, _ = ob.run_chain(chain, make_box_masks)
        for i, m in enumerate(steps):
            ref = g[f'{name}/{i}/masks']
            assert (m.height, m.width) == tuple(g[f'{name}/{i}/size']), (name, i)
            assert m.to_ndarray().shape == ref.shape and m.to_ndarray().dtype == ref.dtype, (name, i)
            assert np.array_equal(m.to_ndarray(), ref), (name, i)
            assert np.array_equal(m.get_bboxes(), g[f'{name}/{i}/bboxes']), (name, i)
            assert m.areas.dtype == g[f'{name}/{i}/areas'].dtype and np.array_equal(m.areas, g[f'{name}/{i}/areas'])


def test_golden_covers_the_edge_cases(golden):
    g = golden('box_masks')
    sizes = {n: [tuple(g[f'{n}/{i}/masks'].shape) for i in range(len(_chain(g[f'{n}/chain'])))] for n in g['cases']}
    assert sizes['empty'][0][0] == 0 and all(s[0] == 0 for s in sizes['empty'])
    assert sizes['edge'][1] == (0, 4, 1)                          # a crop at the image's edge: size 1, no mask left
    assert any(0 < a.sum() < len(a) for n in g['cases'] for a in [g[f'{n}/0/areas'] == 0])   # vanishing boxes


@pytest.mark.parametrize('block', range(4))
def test_random_chains_match_the_restatement(block):
    for s in range(block * 1000, (block + 1) * 1000):
        rng = np.random.default_rng(s)
        chain = ob.random_chain(rng)
        ref, done = ob.run_chain(chain, ob.generate_box_mask, np.random.default_rng(s + 10 ** 6))
        mine, _ = ob.run_chain(done, make_box_masks)
        for i, (a, b) in enumerate(zip(mine, ref)):
            _same(a, b, (s, i, done[i][0]))


def test_nearest_map_equals_cv2():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(7)
    pairs = [(1, 1), (1, 7), (7, 1), (3, 3), (2047, 1), (1, 2047)]
    pairs += [(int(a), int(b)) for a, b in rng.integers(1, 3000, (3000, 2))]
    pairs += [(int(s), max(1, int(s * r + 0.5))) for s, r in zip(rng.integers(1, 2000, 3000), rng.uniform(0.1, 2.0, 3000))]
    pairs += [(s, 2 * s + 1) for s in range(1, 200, 2)] + [(2 * s + 1, s) for s in range(1, 200, 2)]
    for src, dst in pairs:
        img = np.arange(src, dtype=np.float32).reshape(1, src)
        got = cv2.resize(img, (dst, 1), interpolation=cv2.INTER_NEAREST)[0].astype(np.int64)
        assert np.array_equal(nearest_map(src, dst), got), (src, dst)
        col = cv2.resize(img.T.copy(), (1, dst), interpolation=cv2.INTER_NEAREST)[:, 0].astype(np.int64)
        assert np.array_equal(nearest_map(src, dst), col), (src, dst)


def test_resize_equals_cv2_on_masks():
    cv2 = pytest.importorskip('cv2')
    rng = np.random.default_rng(8)
    for _ in range(300):
        h, w = (int(v) for v in rng.integers(1, 90, 2))
        m = make_box_masks(ob._boxes(rng, int(rng.integers(1, 5)), h, w), h, w)
        nh, nw = (int(v) for v in rng.integers(1, 180, 2))
        want = np.stack([cv2.resize(x, (nw, nh), interpolation=cv2.INTER_NEAREST) for x in m.to_ndarray()])
        assert np.array_equal(m.resize((nh, nw)).to_ndarray(), want), (h, w, nh, nw)


def test_generate_rounding_and_slicing():
    boxes = np.array([[0.5, 1.5, 2.5, 3.5],          # round half to even: 0, 2, 2, 4
                      [-3, -2, 1, 1],                # negative starts wrap: rows 8-2=6..1 -> empty
                      [-12, 0, 3, 2],                # a start past -W clips to 0
                      [5, 5, 20, 20]], np.float32)  # stops past the edge clip
    m = make_box_masks(boxes, 8, 10)
    ref = ob.generate_box_mask(boxes, 8, 10)
    assert np.array_equal(m.to_ndarray(), ref.masks)
    assert m.rects.tolist() == [[2, 0, 5, 3], [0, 0, 0, 0], [0, 0, 3, 4], [5, 5, 8, 10]]


def test_indexing_and_containers():
    m = BoxMasks([[1, 2, 5, 7], [0, 0, 3, 3], [2, 2, 2, 9]], 8, 10)
    ref = ob.Bitmap(m.to_ndarray().copy(), 8, 10)
    for idx in (1, -1, slice(0, 2), slice(None, None, -1), np.array([2, 0, 0]), np.array([True, False, True]),
                np.zeros(0, np.int64), [0, 2]):
        _same(m[idx], ref[idx], idx)
    assert len(m) == 3 and [x.sum() for x in m] == [20, 9, 0]
    assert repr(m) == 'BoxMasks(num_masks=3, height=8, width=10)'
    assert not m.masks.flags.writeable


def test_pickle_is_small_and_round_trips():
    rng = np.random.default_rng(3)
    m = make_box_masks(ob._boxes(rng, 100, 1024, 1024), 1024, 1024)
    blob = pickle.dumps(m)
    assert len(blob) < 8 * 1024
    back = pickle.loads(blob)
    assert np.array_equal(back.rects, m.rects) and (back.height, back.width) == (1024, 1024)
    m.masks                                                   # a materialised array does not travel
    assert len(pickle.dumps(m)) == len(blob)


def test_to_tensor_on_cpu():
    import torch
    m = BoxMasks([[1, 2, 5, 7], [0, 0, 0, 0]], 6, 9)
    for dt in (torch.uint8, torch.bool, torch.float32, torch.float16, torch.bfloat16, torch.int64):
        assert torch.equal(m.to_tensor(dt, 'cpu'), torch.tensor(m.to_ndarray(), dtype=dt))


def test_transforms_without_rectangles_need_bitmapmasks():
    from boxinstseg_b200.core import box_masks as bm
    if bm.HAVE_MMDET:
        pytest.skip('mmdet is importable: these defer to its BitmapMasks')
    m = BoxMasks([[1, 2, 5, 7]], 8, 10)
    for call in (lambda: m.rescale(0.5, 'bilinear'), lambda: m.pad((10, 12), pad_val=1), lambda: m.rotate((8, 10), 30),
                 lambda: m.translate((8, 10), 2), lambda: m.shear((8, 10), 0.1), lambda: m.crop(np.array([0., 0, 4, 4])),
                 lambda: m.crop_and_resize(np.zeros((1, 4)), (4, 4), np.zeros(1, np.int64))):
        with pytest.raises(NotImplementedError):
            call()


def test_registry_builds_generate_box_mask():
    from boxinstseg_b200.datasets import PIPELINES, GenerateBoxMask
    t = PIPELINES.build(dict(type='GenerateBoxMask'))
    assert isinstance(t, GenerateBoxMask)
    out = t({'gt_bboxes': np.array([[1, 1, 3, 4]], np.float32), 'img': np.zeros((6, 6, 3)), 'mask_fields': []})
    assert isinstance(out['gt_masks'], BoxMasks) and out['gt_masks'].rects.tolist() == [[1, 1, 5, 4]]


def test_importing_models_alone_does_not_register_it():
    code = ('import boxinstseg_b200.models as m\n'
            'from boxinstseg_b200.models.builder import HAVE_MMDET\n'
            'if HAVE_MMDET:\n'
            '    from mmdet.datasets.builder import PIPELINES\n'
            '    before = PIPELINES.get("GenerateBoxMask")\n'
            'else:\n'
            '    from boxinstseg_b200.models.builder import PIPELINES\n'
            '    assert PIPELINES.get("GenerateBoxMask") is None\n'
            '    before = None\n'
            'import boxinstseg_b200.datasets as d\n'
            'assert PIPELINES.get("GenerateBoxMask") is d.GenerateBoxMask is not before\n')
    subprocess.run([sys.executable, '-c', code], check=True, cwd=ROOT)


def test_rasterize_argument_checks_without_a_device():
    """Every check of bxs_box_masks_rasterize runs before any device call."""
    import ctypes
    from boxinstseg_b200 import _lib as L
    h = L.lib()

    def call(rects, sizes, es=1, one=1, ptr=16):
        r = np.ascontiguousarray(np.asarray(rects, np.int32).reshape(-1, 4))
        s = np.ascontiguousarray(np.asarray(sizes, np.int64).reshape(-1, 3))
        p = np.full(len(s), ptr, np.uint64)
        return h.bxs_box_masks_rasterize(p.ctypes.data, r.ctypes.data, s.ctypes.data, len(s), es, one, None)

    assert h.bxs_box_masks_rasterize(None, None, None, 0, 1, 1, None) == 0
    assert h.bxs_box_masks_rasterize(None, None, None, -1, 1, 1, None) == -1
    assert call(np.zeros((3, 4)), [[0, 5, 5], [3, 0, 7]], ptr=0) == 0        # nothing to write
    assert call([[0, 0, 6, 5]], [[1, 5, 5]]) == -1                           # y1 > H
    assert call([[2, 0, 1, 5]], [[1, 5, 5]]) == -1                           # y0 > y1
    assert call([[-1, 0, 1, 5]], [[1, 5, 5]]) == -1
    assert call([[0, 0, 1, 5]], [[-1, 5, 5]]) == -1
    assert call([[0, 0, 1, 5]], [[1, 5, 5]], es=3) == -1
    assert call([[0, 0, 1, 5]], [[1, 5, 5]], es=1, one=256) == -1
    assert call([[0, 0, 1, 5]], [[1, 5, 5]], es=4, one=2 ** 32) == -1
    assert call([[0, 0, 1, 5]], [[1, 5, 5]], es=2, ptr=17) == -1             # not aligned to the element
    assert call([[0, 0, 1, 5]], [[1, 5, 5]], ptr=0) == -1
    assert call([[0, 0, 1, 1]], [[1, 46341, 46341]]) == -3                   # H * W > 2^31 - 1
    assert ctypes.c_void_p is L.SIGNATURES['bxs_box_masks_rasterize'][0]
