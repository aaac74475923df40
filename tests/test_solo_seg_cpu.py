"""SOLOv2 inference, CPU side: (1) the oracle (oracle/solo_seg.py) reproduces the golden vectors minted from the reference's
own ``get_seg`` / ``get_seg_single`` of both SOLOv2 heads and its ``mask_matrix_nms`` (oracle/make_golden_solo_seg.py);
(2) the HOST build of the kernels' arithmetic (csrc/solo_seg_core.cuh through tests/host_harness/matrix_nms_host.cpp)
against the oracle: the kept candidates and their order exactly, the decayed scores bit for bit with the linear kernel and
within one unit in the last place with the gaussian one (the C library's expf against torch's CPU exp); the two-stage
paste bit for bit against the float32 restatement of ATen's arithmetic and within rounding of torch's CPU interpolate;
(3) the ops' argument handling without a GPU.  The GPU twin of this file is tests/test_solo_seg_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import solo_seg as oss
from oracle.make_golden_solo_seg import CASES, NMS_CASES, case, cfg_of, nms_case, run_oracle
from tests.helpers import host_twin


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize('seed', range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_reproduces_reference_golden(golden, seed):
    g = golden('solo_seg')
    name, method, kw, over = CASES[seed]
    head, args, metas = case(seed, method, **kw)
    out = run_oracle(method, head, args, metas, cfg_of(over))
    for b, r in enumerate(out):
        assert np.array_equal(r.scores.numpy(), g[f'{name}_{b}_scores'])
        assert np.array_equal(r.labels.numpy(), g[f'{name}_{b}_labels'])
        assert tuple(r.masks.shape) == tuple(g[f'{name}_{b}_shape']) and str(r.masks.dtype) == str(g[f'{name}_{b}_dtype'])
        assert np.array_equal(np.packbits(r.masks.numpy().astype(bool), axis=-1), g[f'{name}_{b}_masks'])
        if len(r.scores) == 0:          # empty_results: float tensors, as the reference builds them
            assert r.masks.dtype == r.labels.dtype == r.scores.dtype == args[1 if method == 'box' else 0][0].dtype


@pytest.mark.parametrize('i', range(len(NMS_CASES)))
def test_oracle_nms_reproduces_reference_golden(golden, i):
    g = golden('solo_seg')
    masks, labels, scores = nms_case(i)
    s, l, _, k = oss.mask_matrix_nms(masks, labels, scores, **NMS_CASES[i])
    assert np.array_equal(s.numpy(), g[f'nms{i}_scores']) and np.array_equal(l.numpy(), g[f'nms{i}_labels'])
    assert np.array_equal(k.numpy(), g[f'nms{i}_keep'])


def _twin_nms(masks, labels, scores, kernel='gaussian', sigma=2.0, filter_thr=-1, tie_scores=False):
    """The host twin on the oracle's sorted candidates: decayed scores, then the stable second sort."""
    lib = host_twin('matrix_nms_host')
    s, order = torch.sort(scores, descending=True, stable=True)
    m = masks[order].reshape(len(order), -1).float()
    inter = (m @ m.t()).contiguous()
    area = m.sum(1).contiguous()
    lab = labels[order].contiguous()
    out = torch.empty(len(order))
    lib.host_matrix_nms(ctypes.c_int64(len(order)), _p(inter), _p(area), _p(lab), _p(s.contiguous()), {'gaussian': 0, 'linear': 1}[kernel],
                        ctypes.c_float(sigma), ctypes.c_float(filter_thr), _p(out))
    s2, o2 = torch.sort(out, descending=True, stable=True)
    keep = s2 > float('-inf')
    return s2[keep], order[o2[keep]]


@pytest.mark.parametrize('i', range(len(NMS_CASES)))
def test_host_twin_matrix_nms_equals_oracle(i):
    kw = dict(NMS_CASES[i])
    kw.pop('nms_pre', None), kw.pop('max_num', None)
    masks, labels, scores = nms_case(i, n=40)
    scores[5] = scores[9]                               # a tie: the stable order decides
    s, k = _twin_nms(masks, labels, scores, **kw)
    so, _, _, ko = oss.mask_matrix_nms(masks, labels, scores, stable=True, **kw)
    assert torch.equal(k, ko)
    if kw.get('kernel') == 'linear':
        assert torch.equal(s, so)
    else:
        # The host build's exp is the C library's expf; torch's CPU exp is SLEEF's, and the two differ in the last bit
        # on a few inputs.  On the GPU both sides call CUDA's expf, and the GPU test compares bit for bit.
        assert ((s - so).abs() <= so.abs() * 2.0 ** -23).all()


@pytest.mark.parametrize('shape', [((11, 13), (40, 50), (31, 45)), ((12, 16), (48, 64), (48, 64)), ((7, 9), (25, 36), (60, 70))])
def test_host_twin_paste_equals_oracle(shape):
    (h, w), img_hw, ori_hw = shape
    lib = host_twin('matrix_nms_host')
    p = torch.rand(h, w, generator=torch.Generator().manual_seed(h * w))
    out = torch.empty(ori_hw)
    lib.host_paste(_p(p), h, w, *img_hw, *ori_hw, _p(out))
    assert np.array_equal(out.numpy(), oss.paste_plane(p.numpy(), img_hw, ori_hw))
    ref = F.interpolate(F.interpolate(p[None, None], (4 * h, 4 * w), mode='bilinear')[:, :, :img_hw[0], :img_hw[1]], ori_hw,
                        mode='bilinear')[0, 0]
    assert (out - ref).abs().max() <= 1e-6


def test_ops_reject_cpu_tensors_and_unknown_kernels():
    from boxinstseg_b200.ops import solo_seg
    m = torch.zeros(2, 4, 4, dtype=torch.bool)
    with pytest.raises(NotImplementedError):
        solo_seg.mask_matrix_nms(m, torch.zeros(2, dtype=torch.long), torch.rand(2), kernel='box')
    with pytest.raises(RuntimeError):
        solo_seg.mask_matrix_nms(m, torch.zeros(2, dtype=torch.long), torch.rand(2))
    with pytest.raises(RuntimeError):
        solo_seg.paste_masks(torch.rand(2, 4, 4), (4, 4), (16, 16, 3), (10, 10, 3), 0.5)


def test_c_abi_argument_checks():
    from boxinstseg_b200 import _lib
    h = _lib.lib()
    ptrs = (ctypes.c_void_p * 1)(None)
    rows = (ctypes.c_int64 * 1)(4)
    buf = ctypes.cast((ctypes.c_float * 64)(), ctypes.c_void_p)
    assert h.bxs_solo_mask_stats(ptrs, rows, 1, 16, 0, 0, buf, 1, 0.5, buf, buf, buf, None) == -1      # NULL source
    ptrs = (ctypes.c_void_p * 1)(buf.value)
    assert h.bxs_solo_mask_stats(ptrs, rows, 1, 16, 2, 0, buf, 1, 0.5, buf, buf, buf, None) == -1      # unknown dtype
    assert h.bxs_solo_mask_stats(ptrs, rows, 9, 16, 0, 0, buf, 1, 0.5, buf, buf, buf, None) == -3      # > 8 sources
    assert h.bxs_matrix_nms(buf, 4, buf, buf, buf, buf, buf, 1, 4, 2, 2.0, -1.0, 0, buf, buf, None) == -1   # kernel 2
    assert h.bxs_matrix_nms_workspace_bytes(2, 500) >= 2 * 500 * 500 * 4
    assert h.bxs_solo_paste_masks(ptrs, rows, 1, 4, 4, 0, 0, 0, buf, 1, 17, 16, 10, 10, 0.5, buf, None) == -1   # crop > 4h
