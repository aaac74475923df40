"""DiscoBoxSOLOv2Head.loss (discobox_head.py:1142-1360), CPU side: (1) the oracle (oracle/discobox_loss.py) reproduces the
golden vectors minted from the reference's own ``loss`` (oracle/make_golden_discobox_loss.py); (2) the host-side argument
checks of bxs_disco_cells_pack / bxs_disco_cells_unpack_grad; (3) the head builds with the reference's ``loss_cate`` and
raises outside the focal envelope.  The GPU twin of this file is tests/test_discobox_loss_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import discobox_loss as odl
from oracle.make_golden_discobox_loss import CASES, CFG, GRIDS, NUM_CLASSES, case

RUNS = [(seed, kw, ts, ind) for seed, kw, flags in CASES for ts, ind in flags]


def golden_run(seed, kw, ts, ind):
    """The oracle's losses and float64 gradients on a golden case."""
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = case(seed, **kw)
    leaves = [t.clone().requires_grad_(True) for t in cate + s_k + [s_in]]
    n = len(cate)
    out = odl.loss(leaves[:n], leaves[n:2 * n], t_k, leaves[2 * n], t_in, boxes, labels, masks, img, GRIDS, NUM_CLASSES,
                   use_loss_ts=ts, use_ind_teacher=ind, cfg=CFG)
    grads = torch.autograd.grad(sum(out.values()), leaves, allow_unused=True)
    grads = [torch.zeros_like(x) if g is None else g for x, g in zip(leaves, grads)]
    return out, grads


@pytest.mark.parametrize('seed,kw,ts,ind', RUNS, ids=[f's{r[0]}_ts{int(r[2])}_ind{int(r[3])}' for r in RUNS])
def test_oracle_reproduces_reference_golden(golden, seed, kw, ts, ind):
    g = golden('discobox_loss')
    tag = f's{seed}_ts{int(ts)}_ind{int(ind)}'
    out, grads = golden_run(seed, kw, ts, ind)
    for k in ('loss_ins', 'loss_ts', 'loss_cate', 'loss_corr'):
        assert np.allclose(out[k].detach().double().numpy(), g[f'{tag}_{k}'], rtol=1e-6, atol=1e-9), k
    n = len(GRIDS)
    for name, got in (('g_cate', torch.cat([t.reshape(-1) for t in grads[:n]])),
                      ('g_kern', torch.cat([t.reshape(-1) for t in grads[n:2 * n]])), ('g_ins', grads[2 * n])):
        want = torch.from_numpy(g[f's{seed}_g_cate' if name == 'g_cate' else f'{tag}_{name}']).double()
        assert torch.allclose(got.double().reshape(want.shape), want, rtol=1e-5, atol=1e-9 * float(want.abs().max())), name
    if not ts:
        assert float(out['loss_ts']) == 0.0


def test_golden_covers_the_empty_cases():
    """Two ground truths on the same cells, an image without any covered cell and a level without objects."""
    from oracle import solo_targets as ost
    for seed, kw, _ in CASES:
        cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = case(seed, **kw)
        tg = [ost.disco_target_single(b, l, m, tuple(s_in.shape[-2:]), CFG['scale_ranges'], CFG['strides'], GRIDS,
                                      CFG['sigma'], NUM_CLASSES) for b, l, m in zip(boxes, labels, masks)]
        orders = [[list(map(int, tg[b][3][lv])) for lv in range(len(GRIDS))] for b in range(len(tg))]
        assert any(len(o) != len(set(o)) for per_img in orders for o in per_img)                 # repeated cells
        assert all(not per_img[-1] for per_img in orders)                                        # the top level is empty
        if kw.get('empty_image') is not None:
            assert not any(orders[kw['empty_image']])


# ---------------------------------------------------------------------------------------------------------------- C ABI
def test_pack_plan_rejects_bad_arguments():
    from boxinstseg_b200 import _lib as L
    lib = L.lib()
    i64 = lambda *v: (ctypes.c_int64 * len(v))(*v)          # noqa: E731
    ptrs = lambda n: (ctypes.c_void_p * n)(*([256] * n))    # noqa: E731
    dummy = ctypes.c_void_p(256)

    def pack(grid, counts, n_cells, n_levels, B, C=32, I_pad=4, dtype=0, grids=None):
        return lib.bxs_disco_cells_pack(grids if grids is not None else ptrs(max(n_levels, 1)), grid, counts, dummy, n_cells,
                                        dummy, None, n_levels, B, C, I_pad, dtype, None)

    def unpack(grid, counts, n_cells, n_levels, B, C=32, I_pad=4, dtype=0):
        return lib.bxs_disco_cells_unpack_grad(dummy, grid, counts, dummy, n_cells, ptrs(max(n_levels, 1)), n_levels, B, C,
                                               I_pad, dtype, None)
    for fn in (pack, unpack):
        assert fn(i64(*[4] * 9), i64(*[0] * 18), 0, 9, 2) == -3                  # more than 8 levels
        assert fn(i64(4), i64(*[0] * 17), 0, 1, 17) == -3                         # more than 16 images
        assert fn(i64(65), i64(1, 1), 2, 1, 2) == -3                              # a grid above 64
        assert fn(i64(4, 4), i64(1, 2, 0, 1), 3, 2, 2) == -1                      # counts that do not sum to n_cells
        assert fn(i64(4, 4), i64(3, 2, 2, 1), 8, 2, 2, I_pad=4) == -1             # image 0 has 5 rows > I_pad
        assert fn(i64(4, 4), i64(1, 2, -1, 1), 3, 2, 2) == -1                     # a negative count
        assert fn(i64(4, 0), i64(1, 1, 1, 1), 4, 2, 2) == -1                      # a non-positive grid
        assert fn(i64(4), i64(1, 1), 2, 1, 2, dtype=3) == -1                      # an unknown dtype
        assert fn(i64(4), i64(1, 1), 2, 0, 2) == -1                               # no level
        assert fn(i64(4), i64(1, 1), 2, 1, 2, I_pad=4096) == -3                   # I_pad above 2048
    assert pack(i64(4, 4), i64(1, 1, 1, 1), 4, 2, 2, grids=(ctypes.c_void_p * 2)(256, None)) == -1   # a missing grid
    assert lib.bxs_disco_cells_pack(ptrs(1), i64(4), i64(1, 1), None, 2, dummy, None, 1, 2, 32, 4, 0, None) == -1  # no cells


def test_head_focal_envelope():
    from boxinstseg_b200.models import build_head
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256, num_grids=[40, 36, 24, 16, 12],
                           loss_cate=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)))
    assert head.focal == (2.0, 0.25, 1.0)
    odd = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256,
                          loss_cate=dict(type='FocalLoss', use_sigmoid=True, reduction='sum')))
    with pytest.raises(NotImplementedError, match='loss_cate FocalLoss'):
        odd.loss(None, None, None, torch.zeros(1), None, [], [], [], None, None)
