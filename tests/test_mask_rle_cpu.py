"""COCO RLE of mask results, CPU side: (1) the oracle (oracle/mask_rle.py) reproduces the golden vectors minted from the
reference's own ``encode_mask_results`` (oracle/make_golden_mask_rle.py), and its ``decode`` inverts its ``encode``; (2) the
HOST build of the kernels' string arithmetic (csrc/mask_rle_core.cuh through tests/host_harness/mask_rle_host.cpp) against
the oracle on every delta at the edges of a character count; (3) the argument checks of the C entry points, none of which
launches; (4) the Python side's type checks and the cases that need no device.  The GPU twin is tests/test_mask_rle_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import mask_rle as omr
from oracle.make_golden_mask_rle import CASES, case, segms_of
from tests.helpers import host_twin


def _p(a):
    return ctypes.c_void_p(a.ctypes.data)


def golden_case(g, name):
    """(masks as stored, per-class counts, expected strings) of one golden case."""
    sizes, off, chars = g[f'{name}_sizes'], g[f'{name}_offsets'], g[f'{name}_chars'].tobytes()
    n_pix = int(sizes.prod(1).sum()) if len(sizes) else 0
    flat = g[f'{name}_raw'] if f'{name}_raw' in g else np.unpackbits(g[f'{name}_bits'])[:n_pix]
    masks, p = [], 0
    for h, w in sizes:
        masks.append(flat[p:p + h * w].reshape(h, w))
        p += h * w
    return masks, g[f'{name}_per_class'], [chars[off[k]:off[k + 1]] for k in range(len(sizes))]


def oracle_encode(m):
    """pycocotools' encode of one 2-D mask as the reference calls it."""
    return omr.encode(np.array(np.asarray(m)[:, :, np.newaxis], order='F', dtype='uint8'))[0]


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_reproduces_reference_golden(golden, i):
    g = golden('mask_rle')
    name = CASES[i][0]
    stored, per_class, expected = golden_case(g, name)
    segms = segms_of(case(i))
    assert [len(per) for per in segms] == per_class.tolist()
    masks = [np.asarray(m) for per in segms for m in per]
    assert [str(m.dtype) for m in masks] == g[f'{name}_dtypes'].tolist()
    for m, s, e in zip(masks, stored, expected):
        assert np.array_equal(m.astype(np.uint8), s)
        rle = oracle_encode(m)
        assert rle['size'] == list(m.shape) and rle['counts'] == e
        d = omr.decode(rle)                                          # runs alternate 0 / 1 from 0
        if m.max(initial=0) <= 1:
            assert np.array_equal(d, m.astype(np.uint8))
        assert oracle_encode(d)['counts'] == e or m.max(initial=0) > 1
        assert np.array_equal(omr.from_string(e), omr.counts(m.T))


def test_golden_cases_cover_their_edges(golden):
    g = golden('mask_rle')
    assert g['empty_classes_per_class'].tolist() == [0, 0, 0, 0] and g['list_bool_per_class'][1] == 0
    assert g['array_per_class_per_class'].tolist() == [4, 0, 2]
    assert {tuple(s) for s in g['odd_sizes_sizes']} == {(427, 641), (1, 37), (29, 1), (427, 1)}
    _, _, edge = golden_case(g, 'edge_pixels')
    assert [omr.from_string(e).tolist() for e in edge] == [[0, 1, 767], [767, 1], [0, 768], [768], [0, 1, 766, 1]]
    _, _, board = golden_case(g, 'checkerboard')
    assert [len(omr.from_string(e)) for e in board] == [301, 300]             # every pixel a run
    raw = g['uint8_values_raw']
    assert raw.max() > 1 and len(np.unique(raw)) > 3
    _, _, runs = golden_case(g, 'long_runs')
    c = omr.from_string(runs[0]).astype(np.int64)
    x = c.copy()
    x[3:] -= c[1:-2]
    assert x.min() < -(1 << 24) and x.max() >= 1 << 24 and ((x > -(1 << 24)) & (x <= -(1 << 19))).any()


def _edge_deltas():
    xs = {0}
    for p in range(30):
        for v in ((1 << p) - 1, 1 << p, (1 << p) + 1):
            xs |= {v, -v}
    return np.array(sorted(x for x in xs if -(1 << 29) <= x < (1 << 29)), np.int64)


def test_host_twin_characters_equal_oracle():
    lib = host_twin('mask_rle_host')
    x = _edge_deltas()
    assert {0, 15, -15, 16, -16, 511, -511, 512, -512, (1 << 29) - 1, -(1 << 29) + 1, -(1 << 29)} <= set(x.tolist())
    n = len(x)
    ln = np.zeros(n, np.int32)
    chars = np.zeros((n, 6), np.uint8)
    assert lib.host_rle_chars(ctypes.c_int64(n), _p(x), _p(ln), _p(chars)) == 0
    for i in range(n):
        ref = omr._to_string(np.array([x[i]], np.int64))             # one count: written as it is
        assert chars[i, :ln[i]].tobytes() == ref, int(x[i])
    assert ln.max() == 6 and ln[x == 0] == 1


def test_host_twin_deltas_equal_oracle(golden):
    lib = host_twin('mask_rle_host')
    g = golden('mask_rle')
    for name, _ in CASES:
        _, _, expected = golden_case(g, name)
        for e in expected:
            c = omr.from_string(e)
            x = np.zeros(len(c), np.int64)
            lib.host_rle_deltas(ctypes.c_int64(len(c)), _p(c), _p(x))
            ln = np.zeros(len(c), np.int32)
            chars = np.zeros((len(c), 6), np.uint8)
            assert lib.host_rle_chars(ctypes.c_int64(len(c)), _p(x), _p(ln), _p(chars)) == 0
            assert b''.join(chars[i, :ln[i]].tobytes() for i in range(len(c))) == e


def test_c_abi_argument_checks():
    from boxinstseg_b200 import _lib
    h = _lib.lib()
    buf = ctypes.cast((ctypes.c_int64 * 64)(), ctypes.c_void_p)
    assert h.bxs_mask_rle_runs(buf, -1, 4, 4, buf, buf, None) == -1                  # negative n
    assert h.bxs_mask_rle_runs(buf, 1, -4, 4, buf, buf, None) == -1                  # negative H
    assert h.bxs_mask_rle_runs(buf, 1, 4, -4, buf, buf, None) == -1                  # negative W
    assert h.bxs_mask_rle_runs(None, 1, 4, 4, buf, buf, None) == -1                  # NULL masks
    assert h.bxs_mask_rle_runs(buf, 1, 4, 4, None, buf, None) == -1                  # NULL workspace
    assert h.bxs_mask_rle_runs(buf, 1, 4, 4, buf, None, None) == -1                  # NULL offsets
    assert h.bxs_mask_rle_runs(buf, 1, 1 << 14, 1 << 15, buf, buf, None) == -3       # H * W == 2^29
    assert h.bxs_mask_rle_runs(None, 0, 4, 4, None, None, None) == 0                # n == 0: a no-op
    assert h.bxs_mask_rle_counts(buf, -1, 4, 4, buf, buf, buf, None) == -1
    assert h.bxs_mask_rle_counts(buf, 1, 4, 4, buf, None, buf, None) == -1          # NULL offsets
    assert h.bxs_mask_rle_counts(buf, 1, 4, 4, buf, buf, None, None) == -1          # NULL counts
    assert h.bxs_mask_rle_counts(buf, 1, 1 << 15, 1 << 14, buf, buf, buf, None) == -3
    assert h.bxs_mask_rle_counts(None, 0, 4, 4, None, None, None, None) == 0
    assert h.bxs_mask_rle_strings(buf, buf, -1, 4, buf, buf, buf, None) == -1        # negative n
    assert h.bxs_mask_rle_strings(buf, buf, 3, 2, buf, buf, buf, None) == -1         # R < n
    for k in range(5):                                                                 # each NULL pointer
        args = [buf] * 5
        args[k] = None
        assert h.bxs_mask_rle_strings(args[0], args[1], 1, 1, args[2], args[3], args[4], None) == -1
    assert h.bxs_mask_rle_strings(None, None, 0, 0, None, None, None, None) == 0
    assert h.bxs_mask_rle_counts_workspace_bytes(0, 480, 640) == 0
    assert h.bxs_mask_rle_counts_workspace_bytes(100, 480, 640) >= 100 * 640 * 8 * 8
    assert h.bxs_mask_rle_strings_workspace_bytes(2, 1) == 0
    assert h.bxs_mask_rle_strings_workspace_bytes(100, 50000) >= 8 * 2 * (50000 // 4096)


def test_python_checks_and_cases_without_a_device():
    from boxinstseg_b200.core import encode_mask_results
    from boxinstseg_b200.ops import mask_rle
    with pytest.raises(TypeError):
        mask_rle.encode(torch.zeros(2, 4, 4))                                 # float masks
    with pytest.raises(RuntimeError):
        mask_rle.encode(torch.zeros(2, 4, 4, dtype=torch.bool))               # CPU tensors
    with pytest.raises(RuntimeError):
        mask_rle.rle_counts(torch.zeros(2, 4, 4, dtype=torch.uint8))
    with pytest.raises(TypeError):
        encode_mask_results([[np.zeros((4, 4), np.float32)]])
    with pytest.raises(TypeError):
        encode_mask_results([[torch.zeros(4, 4, dtype=torch.int32)]])
    assert encode_mask_results([[], [], []]) == [[], [], []]                 # the reference's structure, no device
    scores = [[], []]
    out = encode_mask_results(([[], np.zeros((0, 5, 7), np.uint8)], scores))
    assert out == ([[], []], scores) and out[1] is scores
    rle = oracle_encode(np.eye(5, dtype=bool))
    again = encode_mask_results(([[rle], []], [[0.5], []]))                 # already encoded: returned unchanged
    assert again[0][0][0] is rle and again[1] == [[0.5], []]
