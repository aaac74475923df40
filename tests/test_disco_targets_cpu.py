"""f2: DiscoBox's SOLO target builders (discobox_head.py:1362-1529).  (1) the oracle restatement reproduces the golden vectors
minted from the reference's own two methods (oracle/make_golden_disco.py); (2) the device-tensor builder
(models/dense_heads/disco_targets.py, plain torch: runs on any device) equals the oracle bit for bit -- instance labels, category
grid, positive flags and the covered-cell order -- on the golden cases, on random masks and on the empty cases.  The GPU twin
runs the same comparison with CUDA tensors (tests/test_solo_targets_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import solo_targets as ost
from oracle.make_golden_disco import CFG, case


def _same(want, got):
    for w_list, g_list in zip(want[:3], got[:3]):
        for w, g in zip(w_list, g_list):
            assert w.shape == g.shape and torch.equal(w, g.cpu())
    assert [list(x) for x in want[3]] == [x.cpu().tolist() for x in got[3]]


@pytest.mark.parametrize('seed', [0, 1, 2])
@pytest.mark.parametrize('best', [False, True])
def test_oracle_reproduces_reference_golden(golden, seed, best):
    g = golden('disco_targets')
    name = 'best' if best else 'gen'
    boxes, labels, masks, fsize = case(seed)
    ins, cate, ind, order = ost.disco_target_single(boxes, labels, masks, fsize, best=best, **CFG)
    for lvl in range(5):
        assert np.array_equal(cate[lvl].numpy(), g[f's{seed}_{name}_cate{lvl}'].astype(np.int64))
        assert np.array_equal(ind[lvl].numpy(), g[f's{seed}_{name}_ind{lvl}'])
        assert np.array_equal(np.asarray(order[lvl], dtype=np.int32), g[f's{seed}_{name}_order{lvl}'])
        shape = tuple(g[f's{seed}_{name}_insshape{lvl}'])
        assert tuple(ins[lvl].shape) == shape
        assert np.array_equal(np.unpackbits(g[f's{seed}_{name}_ins{lvl}'], axis=-1)[..., :shape[-1]], ins[lvl].numpy())


@pytest.mark.parametrize('seed', [0, 1, 2, 5, 6])
@pytest.mark.parametrize('best', [False, True])
def test_device_builder_equals_oracle(seed, best):
    from boxinstseg_b200.models.dense_heads.disco_targets import disco_target_single
    boxes, labels, masks, fsize = case(seed) if seed < 5 else case(seed, H=96, W=256, G=14)
    if seed == 6:                                                       # ragged random masks instead of rectangles
        gen = torch.Generator().manual_seed(9)
        masks = masks * (torch.rand(masks.shape, generator=gen) < 0.6).numpy().astype(np.uint8)
    want = ost.disco_target_single(boxes, labels, masks, fsize, best=best, **CFG)
    got = disco_target_single(boxes, labels, torch.from_numpy(masks), fsize, best=best, **CFG)
    _same(want, got)
    assert sum(len(x) for x in want[3]) > 0


@pytest.mark.parametrize('best', [False, True])
def test_no_ground_truth_and_all_masks_empty(best):
    from boxinstseg_b200.models.dense_heads.disco_targets import disco_target_single
    boxes, labels, masks, fsize = case(3)
    for b, l, m in ((boxes[:0], labels[:0], masks[:0]), (boxes, labels, masks * 0)):
        got = disco_target_single(b, l, torch.from_numpy(m), fsize, best=best, **CFG)
        if len(b):
            _same(ost.disco_target_single(b, l, m, fsize, best=best, **CFG), got)
        assert all(x.shape == (0, fsize[0], fsize[1]) for x in got[0]) and all(x.numel() == 0 for x in got[3])
        assert all((c == CFG['num_classes']).all() for c in got[1]) and not any(i.any() for i in got[2])


@pytest.mark.parametrize('best', [True, False])
def test_head_inputs_from_raw_outputs_equal_reference_loops(best):
    """DiscoBoxSOLOv2Head.corr_inputs (discobox_head.py:917-1003 / 1161-1260): targets of every image, kernels gathered by
    grid_order, one dynamic convolution per (level, image) -- against the oracle's loop form, with F.conv2d standing in for the
    wgmma kernel (the glue is plain torch; the kernel has its own GPU parity tests)."""
    import torch.nn.functional as F
    from boxinstseg_b200.models import build_head
    from oracle import corr as oc
    gen = torch.Generator().manual_seed(5)
    B, C = 3, 8
    cases = [case(s) for s in (0, 1, 2)]
    cases[1] = (cases[1][0][:0], cases[1][1][:0], cases[1][2][:0], cases[1][3])          # an image without ground truth
    fsize = cases[0][3]
    grids = CFG['seg_num_grids']
    kraw = [torch.randn(B, C, g, g, generator=gen) for g in grids]
    feat = torch.randn(B, C, fsize[0], fsize[1], generator=gen)
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=CFG['num_classes'], in_channels=C, scale_ranges=CFG['scale_ranges'],
                           strides=CFG['strides'], num_grids=grids, sigma=CFG['sigma']))
    conv = lambda f, k: F.conv2d(f[None], k.t()[:, :, None, None])[0]
    got = head.corr_inputs(kraw, None, feat, None, [c[0] for c in cases], [c[1] for c in cases],
                           [torch.from_numpy(c[2]) for c in cases], best=best, conv=conv)
    want = oc.corr_inputs(kraw, feat, [c[0] for c in cases], [c[1] for c in cases], [c[2] for c in cases], CFG['scale_ranges'],
                          CFG['strides'], grids, CFG['sigma'], CFG['num_classes'], best=best)
    s_list, t_list, img_list, ins_labels, klabels = got
    assert all(t is None for t in t_list)
    seen = 0
    for lv in range(len(grids)):
        assert torch.equal(ins_labels[lv], want[2][lv]) and torch.equal(klabels[lv], want[3][lv])
        if want[0][lv] is None:
            assert s_list[lv] is None and img_list[lv] is None
            continue
        assert torch.allclose(s_list[lv], want[0][lv], rtol=1e-5, atol=1e-5) and torch.equal(img_list[lv].float(), want[1][lv])
        assert s_list[lv].shape[0] == ins_labels[lv].shape[0] == klabels[lv].shape[0]
        seen += s_list[lv].shape[0]
    assert seen >= 8 and not (torch.cat([i for i in img_list if i is not None]) == 1).any()
