"""CondInstBoxHead.loss (condinst_head.py:364-476), CPU side: (1) the float64 oracle reproduces the golden vectors minted
from the reference's own code (oracle/make_golden_fcos_loss.py); (2) the HOST build of the kernel's own arithmetic
(csrc/fcos_loss_core.cuh through tests/host_harness/fcos_loss_host.cpp) against the oracle: points and centerness targets
bit for bit, element losses and gradients -- planted ties included -- within float32 rounding; (3) the C ABI's argument
checks; (4) the head builds from every BoxInst config and only defers or raises outside the loss envelope; (5) the one
all-reduce of the two loss denominators at world size 2 (gloo).  The GPU twin of this file is tests/test_fcos_loss_gpu.py."""
import ctypes
import os
import socket
import sys

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import fcos_loss as ofl
from oracle import fcos_targets as oft
from oracle.make_golden_fcos_loss import CASES, RANGES, STRIDES, case
from tests.helpers import host_twin

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


@pytest.mark.parametrize('seed,kw', CASES)
def test_oracle_reproduces_reference_golden(golden, seed, kw):
    g = golden('fcos_loss')
    cls, bbox, ctr, boxes, labels = case(seed, **kw)
    leaves = [t.clone().requires_grad_(True) for t in cls + bbox + ctr]
    n = len(cls)
    out = ofl.loss(leaves[:n], leaves[n:2 * n], leaves[2 * n:], boxes, labels, STRIDES, kw.get('C', 4))
    grads = torch.autograd.grad(sum(out[0].values()), leaves)
    for k in ('loss_cls', 'loss_bbox', 'loss_centerness'):
        assert np.array_equal(out[0][k].detach().numpy(), g[f's{seed}_{k}'])
    for j, name in enumerate(('cls', 'bbox', 'ctr')):
        assert np.array_equal(torch.cat([t.reshape(-1) for t in grads[j * n:(j + 1) * n]]).numpy(), g[f's{seed}_g_{name}'])
    assert np.array_equal(out[1].float().numpy(), g[f's{seed}_points'])
    for j, name in enumerate(('level_inds', 'img_inds', 'gt_inds')):
        assert out[2 + j].dtype == torch.int64
        assert np.array_equal(out[2 + j].numpy(), g[f's{seed}_{name}'].astype(np.int64))
    if kw.get('no_pos'):
        assert float(out[0]['loss_bbox'].detach()) == 0 and not grads[n].any()


def _positives(seed, kw):
    """float32 (points, preds, targets, centerness logits) of every positive of a golden case, in the flatten order."""
    cls, bbox, ctr, boxes, labels = case(seed, dtype=torch.float32, **kw)
    C = kw.get('C', 4)
    sizes = [tuple(c.shape[-2:]) for c in cls]
    pts = oft.grid_points(sizes, STRIDES)
    lab, tgt, _ = oft.get_targets(pts, boxes, labels, RANGES, STRIDES, C)
    B = cls[0].shape[0]
    f_lab = torch.cat(lab)
    pos = ((f_lab >= 0) & (f_lab < C)).nonzero().reshape(-1)
    f_pts = torch.cat([p.repeat(B, 1) for p in pts])[pos]
    f_pred = torch.cat([b.permute(0, 2, 3, 1).reshape(-1, 4) for b in bbox])[pos]
    f_ctr = torch.cat([c.permute(0, 2, 3, 1).reshape(-1) for c in ctr])[pos]
    return f_pts, f_pred, torch.cat(tgt)[pos], f_ctr


def _host_terms(pts, pred, tgt, ctr):
    lib = host_twin('fcos_loss_host')
    n = pts.shape[0]
    out = [torch.empty(n), torch.empty(n), torch.empty(n), torch.empty(n, 4), torch.empty(n)]
    lib.host_fcos_point_loss(ctypes.c_int64(n), *[_p(t.contiguous()) for t in (pts, pred, tgt, ctr)], *[_p(t) for t in out])
    return out


def _close(got, want, rel=2e-5):
    got, want = got.double(), want.double()
    scale = max(float(want.abs().max()), 1e-30)
    assert float((got - want).abs().max()) <= rel * scale, float((got - want).abs().max()) / scale


@pytest.mark.parametrize('seed,kw', [c for c in CASES if not c[1].get('no_pos')] + [(9, dict(B=2, H=320, W=416, G=(12, 20)))])
def test_kernel_core_on_host_equals_oracle(seed, kw):
    pts, pred, tgt, ctr = _positives(seed, kw)
    assert pts.shape[0] > 20
    ct, bbox, bce, g_pred, g_ctr = _host_terms(pts, pred, tgt, ctr)
    assert torch.equal(ct, ofl.centerness_target_rn(tgt))                               # bit for bit in float32
    w_ct, w_bbox, w_bce, w_gp, w_gc = ofl.element_terms(pts.double(), pred.double(), tgt.double(), ctr.double())
    for got, want in ((bbox, w_bbox), (bce, w_bce), (g_pred, w_gp), (g_ctr, w_gc)):
        _close(got, want)
    for got, want in ((bbox, w_bbox), (bce, w_bce)):                                     # elementwise, relative
        assert torch.allclose(got.double(), want, rtol=1e-5, atol=1e-6)
    assert torch.allclose(g_pred.double(), w_gp, rtol=1e-4, atol=1e-5 * float(w_gp.abs().max()))


def test_points_on_host_equal_grid_priors():
    lib = host_twin('fcos_loss_host')
    for s in STRIDES:
        idx = torch.arange(0, 4000, dtype=torch.int64)
        out = torch.empty(4000)
        lib.host_fcos_points(ctypes.c_int64(4000), _p(idx), ctypes.c_float(float(s)), _p(out))
        assert torch.equal(out, (torch.arange(4000) + 0.5) * s)


def test_planted_ties_follow_autograd():
    """One positive per tie kind, checked element by element: the gradient at a tie is autograd's (half to each side of
    an elementwise max / min, clamp(min=0) passing at 0), not a one-sided choice."""
    px, py = torch.tensor(52.), torch.tensor(36.)
    t = torch.tensor([3.25, 2.5, 4.0, 1.75])
    preds = torch.stack([t,                                                  # the prediction is its target
                         torch.tensor([3.25, 1.0, 2.0, 5.0]),                # a shared left edge
                         torch.tensor([0.0, 1.0, 0.0, 2.0]),                 # zero width
                         torch.tensor([4.25, 2.5, -3.25, 1.75]),             # touches the target's left edge
                         torch.tensor([3.25, 2.5, 4.0, 1.75]) * 2])          # encloses it, sharing the centre
    n = preds.shape[0]
    pts = torch.stack([px, py]).repeat(n, 1)
    tgt = t.repeat(n, 1)
    ctr = torch.tensor([0.3, -1.0, 2.0, 0.0, 5.0])
    ct, bbox, bce, g_pred, g_ctr = _host_terms(pts, preds, tgt, ctr)
    w_ct, w_bbox, w_bce, w_gp, w_gc = ofl.element_terms(pts.double(), preds.double(), tgt.double(), ctr.double())
    assert torch.allclose(bbox.double(), w_bbox, rtol=1e-6, atol=1e-7)
    assert torch.allclose(g_pred.double(), w_gp, rtol=1e-5, atol=1e-7)
    assert torch.allclose(g_ctr.double(), w_gc, rtol=1e-6, atol=1e-7)
    assert float(w_bbox[0]) == 0.0 and float(bbox[0]) == 0.0


# ---------------------------------------------------------------------------------------------------------------- C ABI
def _lib():
    from boxinstseg_b200 import _lib as L
    return L.lib()


def test_abi_argument_checks():
    lib = _lib()
    n = 2
    h = (ctypes.c_int64 * n)(4, 2)
    w = (ctypes.c_int64 * n)(6, 3)
    st = (ctypes.c_float * n)(8.0, 16.0)
    dummy = ctypes.c_void_p(256)
    ptrs = (ctypes.c_void_p * n)(256, 512)
    assert lib.bxs_fcos_loss_workspace_bytes(h, w, n, 2) > 0
    assert lib.bxs_fcos_loss_workspace_bytes(h, w, 9, 2) == 0
    assert lib.bxs_fcos_loss_workspace_bytes(None, w, n, 2) == 0
    assert lib.bxs_fcos_loss_workspace_bytes(h, w, n, 0) == 0
    stats = lambda *a: lib.bxs_fcos_loss_stats(*a, None)    # noqa: E731
    assert stats(ptrs, ptrs, h, w, st, None, dummy, n, 2, 80) == -1
    assert stats(None, ptrs, h, w, st, dummy, dummy, n, 2, 80) == -1
    assert stats(ptrs, ptrs, h, w, st, dummy, dummy, n, 2, 0) == -1
    assert stats(ptrs, ptrs, h, w, (ctypes.c_float * n)(8.0, 0.0), dummy, dummy, n, 2, 80) == -1
    assert stats(ptrs, ptrs, h, w, (ctypes.c_float * n)(8.0, float('nan')), dummy, dummy, n, 2, 80) == -1
    assert stats(ptrs, ptrs, (ctypes.c_int64 * n)(4, 0), w, st, dummy, dummy, n, 2, 80) == -1
    assert stats(ptrs, ptrs, h, w, st, dummy, dummy, 9, 2, 80) == -3
    assert stats(ptrs, ptrs, (ctypes.c_int64 * n)(1 << 16, 2), (ctypes.c_int64 * n)(1 << 15, 3), st, dummy, dummy, n, 2,
                 80) == -3
    assert stats(ptrs, ptrs, h, w, st, dummy, dummy, n, 2, 1 << 31) == -3
    fwd = lambda pred, g_pred, den, *rest: lib.bxs_fcos_loss_forward(pred, ptrs, ptrs, ptrs, g_pred, None, h, w, st, den,  # noqa: E731
                                                                     dummy, dummy, dummy, *rest, 1.0, 1.0, None)
    assert fwd(None, None, dummy, n, 2, 80) == -1
    assert fwd(ptrs, None, None, n, 2, 80) == -1
    assert fwd(ptrs, (ctypes.c_void_p * n)(256, None), dummy, n, 2, 80) == -1
    assert fwd(ptrs, None, dummy, 9, 2, 80) == -3
    bwd = lib.bxs_fcos_loss_backward
    assert bwd(None, 0, None, None, 0, None, None) == 0
    assert bwd(None, 4, dummy, None, 0, None, None) == -1
    assert bwd(dummy, -1, dummy, None, 0, None, None) == -1
    assert bwd(dummy, 4, None, None, 0, None, None) == -1
    cells = (ctypes.c_int64 * n)(24, 6)
    assert lib.bxs_sigmoid_focal_loss_cells_forward_workspace_bytes(cells, n, 2) > 0
    assert lib.bxs_sigmoid_focal_loss_cells_forward_workspace_bytes((ctypes.c_int64 * n)(24, 0), n, 2) == 0
    focal = lambda c, nl: lib.bxs_sigmoid_focal_loss_cells_forward(ptrs, ptrs, c, None, dummy, dummy, dummy, nl, 2, 80,  # noqa: E731
                                                                   2.0, 0.25, 1.0, None)
    assert focal((ctypes.c_int64 * n)(24, 0), n) == -1
    assert focal(None, n) == -1
    assert focal((ctypes.c_int64 * n)(24, (1 << 30) + 1), n) == -3
    assert focal(cells, 9) == -3
    grid = (ctypes.c_int64 * n)(5, 3)                          # the square-grid form keeps its statuses
    assert lib.bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(grid, n, 2) == \
        lib.bxs_sigmoid_focal_loss_cells_forward_workspace_bytes((ctypes.c_int64 * n)(25, 9), n, 2)
    levels = lambda g: lib.bxs_sigmoid_focal_loss_levels_forward(ptrs, ptrs, g, None, dummy, dummy, dummy, n, 2, 80,  # noqa: E731
                                                                 2.0, 0.25, 1.0, None)
    assert levels((ctypes.c_int64 * n)(5, 0)) == -1
    assert levels((ctypes.c_int64 * n)(5, (1 << 15) + 1)) == -3


# ----------------------------------------------------------------------------------------------------------------- head
def _boxinst_bbox_head(num_classes):
    """bbox_head of configs/boxinst/boxinst_{r50,r101}_fpn_{1x,3x}_{coco,voc}.py (80 classes for COCO, 20 for VOC)."""
    return dict(type='CondInstBoxHead', num_classes=num_classes, in_channels=256, center_sampling=True,
                center_sample_radius=1.5, norm_on_bbox=True, stacked_convs=4, feat_channels=256, strides=[8, 16, 32, 64, 128],
                loss_cls=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0),
                loss_bbox=dict(type='GIoULoss', loss_weight=1.0),
                loss_centerness=dict(type='CrossEntropyLoss', use_sigmoid=True, loss_weight=1.0))


@pytest.mark.parametrize('num_classes', [80, 20])
def test_every_boxinst_config_is_inside_the_envelope(num_classes):
    from boxinstseg_b200.models import build_head
    head = build_head(_boxinst_bbox_head(num_classes))
    assert head.box_losses == ((2.0, 0.25, 1.0), 1.0, 1.0)
    assert head.num_classes == num_classes and list(head.strides) == list(STRIDES)


@pytest.mark.parametrize('override', [dict(loss_bbox=dict(type='IoULoss', loss_weight=1.0)),
                                      dict(loss_cls=dict(type='FocalLoss', use_sigmoid=True, reduction='sum')),
                                      dict(loss_centerness=dict(type='CrossEntropyLoss', use_sigmoid=False)),
                                      dict(loss_bbox=dict(type='GIoULoss', eps=1e-7))])
def test_outside_the_envelope_builds_and_raises_in_loss(override):
    from boxinstseg_b200.models import build_head
    head = build_head({**_boxinst_bbox_head(80), **override})          # construction never raises
    assert isinstance(head.box_losses, str)
    with pytest.raises(NotImplementedError, match=next(iter(override))):
        head.loss([], [], [], [], [], [])
    # the reference's defaults (IoULoss) build too
    from boxinstseg_b200.models import build_head as bh
    assert isinstance(bh(dict(type='CondInstBoxHead', num_classes=80, in_channels=256)).box_losses, str)


# ------------------------------------------------------------------------------------------------------ world size 2
def _free_port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    sys.path.insert(0, ROOT)
    from boxinstseg_b200.models.dense_heads import condinst_box_head as m
    calls = []
    real = dist.all_reduce
    dist.all_reduce = lambda t, *a, **k: (calls.append(t.numel()), real(t, *a, **k))[1]
    # rank 0: 3 positives with ct sum 1e-7; rank 1: none.  The mean count 1.5 stays, the mean ct sum is clamped to 1e-6
    stats = torch.tensor([[3.0, 1e-7], [0.0, 0.0]])[rank]
    den = m.reduce_mean_clamped(stats)
    # rank 0: 0.5 positives in all -> clamped to 1
    den2 = m.reduce_mean_clamped(torch.tensor([[1.0, 0.75], [0.0, 0.5]])[rank])
    dist.all_reduce = real
    if rank == 0:
        out.put((den.tolist(), den2.tolist(), calls, stats.tolist()))
    dist.destroy_process_group()


def test_one_all_reduce_of_both_denominators_at_world_size_2():
    ctx = mp.get_context('spawn')
    q = ctx.SimpleQueue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in procs]
    [p.join(120) for p in procs]
    assert all(p.exitcode == 0 for p in procs)
    den, den2, calls, stats = q.get()
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))    # noqa: E731
    assert calls == [2, 2]                                                 # one all-reduce of both values per call
    assert den == [f32(1.5), f32(1e-6)]
    assert den2 == [1.0, f32(f32(0.75) / 2 + f32(0.5) / 2)]
    assert stats == [3.0, f32(1e-7)]                                       # the caller's tensor is left alone
