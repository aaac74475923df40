"""``format_results`` of the SOLOv2-family detectors, CPU side: (1) the oracle (oracle/solo_format.py) reproduces the golden
vectors minted from the reference's own ``format_results`` (oracle/make_golden_solo_format.py); (2) the argument checks of
``bxs_mask_extents`` through the C ABI, none of which launches; (3) the Python side's type checks and the empty case.  The
GPU twin of this file is tests/test_solo_format_gpu.py."""
import ctypes
import types

import numpy as np
import pytest
import torch

from oracle import solo_format as osf
from oracle.make_golden_solo_format import CASES, case, flatten


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_reproduces_reference_golden(golden, i):
    g = golden('solo_format')
    name = CASES[i][0]
    results, C = case(i)
    out = osf.format_results(results, C)
    rows, cls, masks, scores = flatten(out)
    assert len(out[0]) == C and all(b.dtype == np.float64 and b.shape[1:] == (5,) for b in out[0])
    assert np.array_equal(rows, g[f'{name}_bbox']) and np.array_equal(cls, g[f'{name}_cls'])
    assert np.array_equal(np.array([float(s) for s in scores], np.float32), g[f'{name}_scores'])
    if masks:
        assert str(masks[0].dtype) == str(g[f'{name}_dtype'])
        assert np.array_equal(np.packbits(np.stack([m.numpy() != 0 for m in masks]), axis=-1), g[f'{name}_masks'])
        assert np.array_equal(np.stack([m.numpy() for m in masks]).astype(np.uint8).max((1, 2)), g[f'{name}_mask_values'])
    else:
        assert g[f'{name}_masks'].size == 0


def test_golden_cases_cover_their_edges(golden):
    g = golden('solo_format')
    assert g['all_empty_bbox'].shape == (0, 5) and g['no_detection_bbox'].shape == (0, 5)
    assert sorted(map(tuple, g['corners_bbox'][:, :4].astype(int))) == [(0, 0, 1, 1), (0, 23, 1, 24), (31, 0, 32, 1),
                                                                        (31, 23, 32, 24)]
    assert (g['full_frame_bbox'][:, :4] == [0, 0, 32, 24]).all()
    assert len(set(g['equal_scores_scores'].tolist())) == 1 and len(g['equal_scores_scores']) == 6
    assert set(g['sparse_classes_cls'].tolist()) == {1, 5, 8}
    assert g['odd_width_bbox'][:, 2].max() <= 641 and 641 % 16
    assert g['uint8_values_mask_values'].max() > 1 and str(g['uint8_values_dtype']) == 'torch.uint8'
    assert len(g['empty_between_bbox']) < 12


def test_c_abi_argument_checks():
    from boxinstseg_b200 import _lib
    h = _lib.lib()
    buf = ctypes.cast((ctypes.c_float * 64)(), ctypes.c_void_p)
    assert h.bxs_mask_extents(buf, -1, 4, 4, buf, buf, buf, None) == -1                 # negative n
    assert h.bxs_mask_extents(buf, 1, -4, 4, buf, buf, buf, None) == -1                 # negative H
    assert h.bxs_mask_extents(buf, 1, 4, -4, buf, buf, buf, None) == -1                 # negative W
    assert h.bxs_mask_extents(None, 1, 4, 4, buf, buf, buf, None) == -1                 # NULL masks
    assert h.bxs_mask_extents(buf, 1, 4, 4, None, buf, buf, None) == -1                 # NULL workspace
    assert h.bxs_mask_extents(buf, 1, 4, 4, buf, None, buf, None) == -1                 # NULL area
    assert h.bxs_mask_extents(buf, 1, 4, 4, buf, buf, None, None) == -1                 # NULL box
    assert h.bxs_mask_extents(buf, 1, 65536, 32768, buf, buf, buf, None) == -3          # H * W > INT32_MAX
    assert h.bxs_mask_extents(None, 0, 4, 4, None, None, None, None) == 0               # n == 0: a no-op
    assert h.bxs_mask_extents_workspace_bytes(0, 480, 640) == 0
    assert h.bxs_mask_extents_workspace_bytes(100, 480, 640) >= 100 * 28


def test_format_results_checks_and_empty_case():
    from boxinstseg_b200.models import HEADS
    from boxinstseg_b200.models.detectors.solo import format_results
    r = types.SimpleNamespace(labels=torch.zeros(2, dtype=torch.long), scores=torch.rand(2), masks=torch.zeros(2, 4, 4))
    with pytest.raises(TypeError):
        format_results(r, 3)                                            # float masks with n > 0
    r.masks = torch.zeros(2, 4, 4, dtype=torch.bool)
    with pytest.raises(RuntimeError):
        format_results(r, 3)                                            # CPU tensors
    empty = types.SimpleNamespace(labels=torch.zeros(0), scores=torch.zeros(0), masks=torch.zeros(0, 4, 4))
    bbox, (masks, scores) = format_results(empty, 3)                    # the reference's empty_results: no device work
    assert [b.shape for b in bbox] == [(0, 5)] * 3 and masks == scores == [[], [], []]
    for name in ('BoxLevelSet', 'DiscoBoxSOLOv2'):
        det = HEADS.get(name)()
        det.bbox_head = types.SimpleNamespace(num_classes=2)
        assert [b.shape for b in det.format_results(empty)[0]] == [(0, 5)] * 2
