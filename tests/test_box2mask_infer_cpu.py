"""Box2Mask inference, CPU side: (1) the oracle (oracle/box2mask_infer.py) reproduces the golden vectors minted from the
reference's own ``Box2MaskHead.simple_test``, ``MaskFormerFusionHead.simple_test`` / ``instance_postprocess`` and
``mask2bbox`` (oracle/make_golden_box2mask_infer.py); (2) the HOST build of the paste and statistics arithmetic
(csrc/solo_seg_core.cuh through tests/host_harness/box2mask_infer_host.cpp) against the oracle: the mask pixel for pixel,
area and box exactly, the masked sum within 1e-6 relative, with H_pad != 4h and with either stage skipped; (3) the C entry
point's and the head's argument errors without a GPU.  The GPU twin of this file is tests/test_box2mask_infer_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import box2mask_infer as obi
from oracle.make_golden_box2mask_infer import CASES, case
from tests.helpers import host_twin


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize('i', range(len(CASES)), ids=[c[0] for c in CASES])
def test_oracle_reproduces_reference_golden(golden, i):
    g = golden('box2mask_infer')
    name = CASES[i][0]
    mask_cls, mask_pred, metas, cfg = case(i)
    out = obi.fusion_simple_test(*obi.head_simple_test([mask_cls], [mask_pred]), metas, cfg['things'],
                                 cfg['max_per_image'], cfg['rescale'])
    for b, (labels, query, bboxes, masks) in enumerate(out):
        assert np.array_equal(labels.numpy(), g[f'{name}_{b}_labels'])
        assert np.array_equal(query.numpy(), g[f'{name}_{b}_query'])
        assert np.array_equal(bboxes.numpy(), g[f'{name}_{b}_bboxes'])
        assert tuple(masks.shape) == tuple(g[f'{name}_{b}_mask_shape'])
        assert np.array_equal(np.packbits(masks.numpy(), axis=-1), g[f'{name}_{b}_masks'])


def test_golden_cases_cover_their_edges(golden):
    g = golden('box2mask_infer')
    q0 = g['base_0_query'].tolist()
    assert q0.count(2) >= 2                                       # a query picked for two classes
    k = g['base_1_query'].tolist().index(4)                       # the all-negative query: no pixel, box and score 0
    assert not g['base_1_bboxes'][k].any() and not np.unpackbits(g['base_1_masks'][k]).any()
    assert tuple(g['no_rescale_0_mask_shape'][1:]) == (30, 37) and tuple(g['base_1_mask_shape'][1:]) == (40, 64)
    assert (g['stuff_0_labels'] < 3).all() and len(g['stuff_0_labels']) < 12
    assert len(g['all_pairs_0_labels']) == 18


GEOMS = [  # (h, w), (H_pad, W_pad), (H_img, W_img), (H_out, W_out) or None (no rescale)
    ((8, 10), (32, 40), (30, 37), (20, 25)),
    ((7, 9), (32, 40), (25, 40), (40, 64)),                       # H_pad != 4h, the crop upsampled
    ((8, 10), (32, 40), (30, 37), None),                          # second stage skipped
    ((32, 40), (32, 40), (30, 37), (45, 50)),                     # first stage skipped
    ((20, 24), (20, 24), (17, 21), None),                         # both skipped (instance_postprocess)
]


@pytest.mark.parametrize('geom', GEOMS)
@pytest.mark.parametrize('seed', [0, 1])
def test_host_twin_equals_oracle(geom, seed):
    (h, w), pad, img, ori = geom
    lib = host_twin('box2mask_infer_host')
    gen = torch.Generator().manual_seed(seed * 100 + h * w)
    x = torch.randn(h, w, generator=gen) * 3 - (0 if seed == 0 else 6)     # seed 1: mostly negative
    if seed == 1:
        x[:] = -1.0                                                          # ... and an empty mask
    v = obi.resize(obi.resize(x[None], pad)[:, :img[0], :img[1]], ori or img)[0]
    H, W = v.shape
    out = torch.empty((H, W), dtype=torch.uint8)
    area, msum, box = torch.zeros(1, dtype=torch.int32), torch.zeros(1), torch.zeros(4)
    lib.host_maskformer_paste(_p(x), h, w, *pad, *img, int(ori is not None), H, W, _p(out), _p(area), _p(msum), _p(box))
    ref = v > 0
    assert torch.equal(out.bool(), ref)
    assert int(area) == int(ref.sum())
    assert torch.equal(box, obi.mask2bbox(ref[None])[0])
    want = (v.sigmoid() * ref.float()).sum()
    assert abs(float(msum) - float(want)) <= 1e-6 * abs(float(want))


def test_head_rejects_unsupported_outputs_and_k():
    from boxinstseg_b200.models.dense_heads.box2mask_infer import MaskFormerFusionHead
    cls, pred = torch.zeros(1, 4, 3), torch.zeros(1, 4, 8, 8)
    metas = [dict(img_shape=(8, 8, 3), ori_shape=(8, 8, 3), batch_input_shape=(8, 8))]
    for key in ('panoptic_on', 'semantic_on'):
        head = MaskFormerFusionHead(2, 0, test_cfg=dict(dict(panoptic_on=False, instance_on=True), **{key: True}))
        with pytest.raises(NotImplementedError, match=key):
            head.simple_test(cls, pred, metas)
    with pytest.raises(NotImplementedError, match='panoptic_on'):                 # the reference's default is True
        MaskFormerFusionHead(2, 0, test_cfg=dict(instance_on=True)).simple_test(cls, pred, metas)
    head = MaskFormerFusionHead(2, 0, test_cfg=dict(panoptic_on=False, instance_on=True, max_per_image=9))
    with pytest.raises(RuntimeError, match='out of range'):                        # Q * K = 8
        head.simple_test(cls, pred, metas)
    with pytest.raises(RuntimeError):                                              # CPU tensors
        MaskFormerFusionHead(2, 0, test_cfg=dict(panoptic_on=False, instance_on=True, max_per_image=4)).simple_test(
            cls, pred, metas)


def test_c_abi_argument_checks():
    from boxinstseg_b200 import _lib
    h = _lib.lib()
    buf = ctypes.cast((ctypes.c_float * 64)(), ctypes.c_void_p)
    ptrs = (ctypes.c_void_p * 1)(buf.value)
    rows = (ctypes.c_int64 * 1)(4)

    def call(*, src=ptrs, n_src=1, hw=(8, 10), dtype=0, n=1, pad=(32, 40), img=(30, 37), rescale=1, out=(20, 25),
             ws=buf, dst=buf):
        return h.bxs_maskformer_paste_masks(src, rows, n_src, *hw, dtype, buf, n, *pad, *img, rescale, *out, ws, dst, buf,
                                            buf, buf, None)

    assert call(src=(ctypes.c_void_p * 1)(None)) == -1                    # NULL source
    assert call(n_src=9) == -3                                           # more than 8 sources
    assert call(dtype=2) == -1                                           # bfloat16 / unknown dtype
    assert call(img=(33, 37)) == -1                                      # crop taller than the padded plane
    assert call(img=(30, 41)) == -1
    assert call(hw=(33, 10)) == -1                                       # input larger than the first stage's output
    assert call(rescale=0) == -1                                         # no rescale: the output is the crop
    assert call(out=(0, 25)) == -1 and call(n=-1) == -1
    assert call(ws=None) == -1 and call(dst=None) == -1                  # NULL workspace / output
    assert call(pad=(2 ** 31, 40)) == -3 and call(out=(2 ** 16, 2 ** 16)) == -3   # beyond INT32_MAX
    assert call(n=0, ws=None, dst=None) == 0                             # nothing to do: no pointer read
    assert h.bxs_maskformer_paste_workspace_bytes(0) == 0
    assert h.bxs_maskformer_paste_workspace_bytes(100) >= 100 * 64 * 28
