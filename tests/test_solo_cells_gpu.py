"""GPU parity of the positive-cell dynamic convolution (``ops.dynconv.solo_cells_conv``, bxs_dynconv1x1_cells_*) against
the reference's lines in float64: ``F.interpolate(F.conv2d(feature_pred, kernel cells, groups=B), (h_l, w_l))`` indexed by
the positive cells (box_solov2_head.py:204-216, 317-320).  The op resizes the operand instead of the result; the two
orders agree up to rounding, so the TF32 bar of the dense dynconv tests holds (1e-3 of the output's scale)."""
import pytest
import torch
import torch.nn.functional as F

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GRIDS = (40, 36, 24, 16, 12)


def _sizes(h, w):
    return [(h, w), (h, w), (h // 2, w // 2), (h // 4, w // 4), (h // 4, w // 4)]


def _cells(B, grids, gen, counts=None):
    """per level, per image: ascending random cells; counts[l][b] overrides the random count."""
    out = []
    for l, S in enumerate(grids):
        lvl = []
        for b in range(B):
            n = counts[l][b] if counts is not None else int(torch.randint(0, 3 * S, (1,), generator=gen))
            lvl.append(torch.randperm(S * S, generator=gen)[:n].sort().values.to(DEV))
        out.append(lvl)
    return out


def _reference(feat, kerns, cells, sizes):
    """float64, the reference's order: convolve, resize, keep the positive rows (image-major, cells ascending)."""
    outs = []
    for k, lvl, size in zip(kerns, cells, sizes):
        B, C = k.shape[:2]
        rows = []
        for b in range(B):
            kb = k[b].reshape(C, -1)[:, lvl[b]].t()                       # [n, C]
            conv = torch.einsum('nc,chw->nhw', kb, feat[b])[None]         # conv2d(groups=B) rows of image b
            if kb.shape[0] == 0:                                          # interpolate rejects zero channels
                rows.append(conv.new_zeros((0,) + tuple(size)) + 0 * conv.sum())
                continue
            rows.append(F.interpolate(conv, size, mode='bilinear', align_corners=False)[0])
        outs.append(torch.cat(rows, 0))
    return outs


def _check(B, C, h, w, grids, sizes, cells, seed):
    from boxinstseg_b200.ops.dynconv import solo_cells_conv
    gen = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, C, h, w, generator=gen).to(DEV)
    kerns = [(torch.randn(B, C, S, S, generator=gen) * 0.05).to(DEV) for S in grids]
    f = feat.clone().requires_grad_(True)
    ks = [k.clone().requires_grad_(True) for k in kerns]
    outs = solo_cells_conv(f, ks, cells, sizes)
    gouts = [torch.randn(o.shape, generator=gen).to(DEV) for o in outs]
    gf, *gk = torch.autograd.grad(sum((o * g).sum() for o, g in zip(outs, gouts)), [f, *ks], allow_unused=True)
    # run to run: bit-identical
    outs2 = solo_cells_conv(f, ks, cells, sizes)
    gf2, *gk2 = torch.autograd.grad(sum((o * g).sum() for o, g in zip(outs2, gouts)), [f, *ks], allow_unused=True)
    assert all(torch.equal(a, b) for a, b in zip(outs, outs2))
    assert torch.equal(gf, gf2) and all(torch.equal(a, b) for a, b in zip(gk, gk2))

    f64 = feat.double().requires_grad_(True)
    k64 = [k.double().requires_grad_(True) for k in kerns]
    refs = _reference(f64, k64, cells, sizes)
    rgf, *rgk = torch.autograd.grad(sum((r * g.double()).sum() for r, g in zip(refs, gouts)), [f64, *k64],
                                    allow_unused=True)
    for o, r in zip(outs, refs):
        assert o.shape == r.shape and o.dtype == torch.float32
        if r.numel():
            assert rel_err(o, r) < 1e-3, rel_err(o, r)
    assert rel_err(gf, rgf) < 1e-3, rel_err(gf, rgf)
    for l, (g, r) in enumerate(zip(gk, rgk)):
        if r is None:
            r = torch.zeros_like(g, dtype=torch.float64)
        assert g.shape == ks[l].shape
        S2 = g.shape[2] * g.shape[3]
        pos = torch.zeros(B, S2, dtype=torch.bool, device=DEV)
        for b in range(B):
            pos[b, cells[l][b]] = True
        neg = ~pos[:, None, :].expand(B, C, S2)
        assert torch.all(g.flatten(2)[neg] == 0)                    # non-positive cells: exactly zero
        if pos.any():
            assert rel_err(g, r) < 1e-3, (l, rel_err(g, r))
    return outs


@pytest.mark.parametrize('h,w', [(200, 256), (200, 336)])
def test_cells_config_d_shapes(h, w):
    """config D's feature map (and a 1344x800 pad's), ragged counts, an image without positives in one level, a level
    without any."""
    gen = torch.Generator().manual_seed(h + w)
    counts = [[37, 0], [12, 90], [0, 0], [5, 1], [17, 130]]
    cells = _cells(2, GRIDS, gen, counts)
    _check(2, 256, h, w, GRIDS, _sizes(h, w), cells, seed=w)


@pytest.mark.parametrize('B', [1, 8])
def test_cells_batch_sizes(B):
    gen = torch.Generator().manual_seed(B)
    h, w = 64, 80
    cells = _cells(B, GRIDS, gen)
    _check(B, 256, h, w, GRIDS, _sizes(h, w), cells, seed=10 + B)


def test_cells_every_cell_positive():
    """all 1600 cells of a 40x40 level (13 kernel chunks of 128; d/d operand beyond 256 kernels goes through cuBLAS) and
    the 128 / 256 boundaries of the native d/d operand on the other image and level."""
    gen = torch.Generator().manual_seed(7)
    grids, h, w = (40, 24), 48, 64
    counts = [[1600, 129], [256, 128]]
    cells = _cells(2, grids, gen, counts)
    _check(2, 256, h, w, grids, [(h, w), (h // 2, w // 2)], cells, seed=7)
    counts = [[129, 200], [0, 0]]                 # native d/d operand with 129..200 kernels per problem, C = 64
    _check(2, 64, h, w, grids, [(h, w), (h // 2, w // 2)], _cells(2, grids, gen, counts), seed=8)


def test_cells_no_positive_at_all():
    from boxinstseg_b200.ops.dynconv import solo_cells_conv
    f = torch.randn(2, 32, 16, 20, device=DEV, requires_grad=True)
    k = torch.randn(2, 32, 4, 4, device=DEV, requires_grad=True)
    empty = [torch.zeros(0, dtype=torch.long, device=DEV)] * 2
    out, = solo_cells_conv(f, [k], [empty], [(16, 20)])
    assert out.shape == (0, 16, 20)
    gf, gk = torch.autograd.grad(out.sum(), [f, k])
    assert gf.shape == f.shape and gk.shape == k.shape
    assert torch.all(gf == 0) and torch.all(gk == 0)


def test_cells_operand_grad_isolated_between_images():
    """d/d operand reads a level's gradient rows in blocks of 32: the rows of the next image in a block must not reach
    this image's gradient, not even as 0 * Inf."""
    from boxinstseg_b200.ops.dynconv import solo_cells_conv
    gen = torch.Generator().manual_seed(5)
    f = torch.randn(2, 64, 16, 20, generator=gen).to(DEV).requires_grad_(True)
    k = (torch.randn(2, 64, 8, 8, generator=gen) * 0.05).to(DEV).requires_grad_(True)
    cells = [[torch.arange(5, device=DEV), torch.arange(3, 40, device=DEV)]]
    out, = solo_cells_conv(f, [k], cells, [(16, 20)])
    g = torch.randn(out.shape, generator=gen).to(DEV)
    g[5:] = float('inf')                                  # every row of image 1
    gf, = torch.autograd.grad(out, [f], g)
    ref = torch.einsum('cn,nhw->chw', k[0].detach().double().reshape(64, -1)[:, :5], g[:5].double())
    assert torch.isfinite(gf[0]).all()
    assert rel_err(gf[0], ref) < 1e-3


def test_dynamic_conv_cells_matches_dense():
    """BoxSOLOv2Head.dynamic_conv(cells=...) returns the dense path's rows of the given cells."""
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import BoxSOLOv2Head
    gen = torch.Generator().manual_seed(3)
    head = BoxSOLOv2Head()
    feat = torch.randn(2, 256, 40, 48, generator=gen).to(DEV)
    kp = (torch.randn(2, 256, 12, 12, generator=gen) * 0.05).to(DEV)
    cells = [torch.tensor([3, 17, 100], device=DEV), torch.tensor([0, 143], device=DEV)]
    dense = head.dynamic_conv(feat, kp, out_size=(20, 24))
    rows = head.dynamic_conv(feat, kp, out_size=(20, 24), cells=cells)
    for b in range(2):
        assert rel_err(rows[b], dense[b, cells[b]].double()) < 1e-3


def test_cells_c_abi_limits():
    import ctypes
    from boxinstseg_b200 import _lib as L
    i64 = lambda v: (ctypes.c_int64 * len(v))(*v)    # noqa: E731
    lib = L.lib()
    f = torch.zeros(1, 32, 4, 4, device=DEV)
    ptrs = (ctypes.c_void_p * 9)(*([f.data_ptr()] * 9))
    cells = torch.zeros(1, dtype=torch.int32, device=DEV)
    ws = torch.empty(1 << 20, dtype=torch.uint8, device=DEV)
    # nine levels: beyond the limit
    rc = lib.bxs_dynconv1x1_cells_forward(ptrs, i64([16]), ptrs, i64([2] * 9), i64([0] * 9), i64([0] * 9), L.ptr(cells),
                                          ptrs, L.ptr(ws), 9, 1, 1, 32, L.stream())
    assert rc == -3
    # C not a multiple of 32
    rc = lib.bxs_dynconv1x1_cells_forward(ptrs, i64([16]), ptrs, i64([2]), i64([0]), i64([1]), L.ptr(cells), ptrs,
                                          L.ptr(ws), 1, 1, 1, 48, L.stream())
    assert rc == -3
    # a level_op that skips an operand; a count above S^2
    rc = lib.bxs_dynconv1x1_cells_forward(ptrs, i64([16, 16]), ptrs, i64([2, 2]), i64([0, 2]), i64([1, 1]), L.ptr(cells),
                                          ptrs, L.ptr(ws), 2, 2, 1, 32, L.stream())
    assert rc == -1
    rc = lib.bxs_dynconv1x1_cells_forward(ptrs, i64([16]), ptrs, i64([2]), i64([0]), i64([5]), L.ptr(cells), ptrs,
                                          L.ptr(ws), 1, 1, 1, 32, L.stream())
    assert rc == -1
    # the first level must take operand 0
    rc = lib.bxs_dynconv1x1_cells_forward(ptrs, i64([16]), ptrs, i64([2]), i64([1]), i64([1]), L.ptr(cells), ptrs,
                                          L.ptr(ws), 1, 1, 1, 32, L.stream())
    assert rc == -1
