"""GPU parity of the positive-cell dynamic convolution (``ops.dynconv.solo_cells_conv``: the cell pack and ``dynconv1x1``)
against the reference's lines in float64: ``F.interpolate(F.conv2d(feature_pred, kernel cells, groups=B), (h_l, w_l))``
indexed by the positive cells (box_solov2_head.py:204-216, 317-320).  The op resizes the operand instead of the result.

Every case runs twice:
  * random data, judged element-wise (``scaled_err``, tests/helpers.py) against the float64 reference.  The op's
    operands are TF32 (10-bit mantissa) and it resizes before it convolves, so its rounding differs from the reference's;
    the bars below sit above the largest value observed on an H100 80GB HBM3 (SXM, 700 W power limit), given next to
    each;
  * an exactness probe: features and kernel grids drawn from {-2..2}, output gradients from {-1, 0, 1}, every level the
    feature map's size or exactly 1/2 or 1/4 of each side.  A bilinear resize by exactly 1/2 or 1/4 (align_corners=False)
    averages 2x2 pixels, so every resized operand, output row, d/d feature and d/d kernel is a multiple of 1/4 far below
    2^20: exact as a TF32 operand, in every FP32 partial sum and whatever the order of the sums.  The op must then equal
    the float64 reference bit for bit, so one misplaced, dropped or stale element fails the case.
Row order, determinism (bit-identical reruns) and exact zeros at the non-positive cells of d/d kernel are checked too."""
import pytest
import torch
import torch.nn.functional as F

from tests.helpers import scaled_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GRIDS = (40, 36, 24, 16, 12)
# element-wise bars (scaled_err) for random data; the largest value observed over all cases in the comments
TOL_OUT = 5e-2             # level rows                                     2.9e-2
TOL_GFEAT = 5e-2           # d / d feature_pred                             2.7e-2
TOL_GKERN = 5e-2           # d / d kernel grids                             2.7e-2


def _sizes(h, w):
    return [(h, w), (h, w), (h // 2, w // 2), (h // 4, w // 4), (h // 4, w // 4)]


def _sizes8(h, w):
    """8 levels over 4 operands (consecutive levels of one size share an operand)."""
    f, half, quarter = (h, w), (h // 2, w // 2), (h // 4, w // 4)
    return [f, f, half, half, quarter, quarter, f, f]


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


def _run(feat, kerns, gouts, cells, sizes):
    """The op's level rows and gradients (d/d feature, d/d every grid); a second run must give the same bits."""
    from boxinstseg_b200.ops.dynconv import solo_cells_conv
    runs = []
    for _ in range(2):
        f = feat.clone().requires_grad_(True)
        ks = [k.clone().requires_grad_(True) for k in kerns]
        outs = solo_cells_conv(f, ks, cells, sizes)
        gf, *gk = torch.autograd.grad(sum((o * g).sum() for o, g in zip(outs, gouts)), [f, *ks], allow_unused=True)
        runs.append((outs, gf, [torch.zeros_like(k) if g is None else g for k, g in zip(ks, gk)]))
    (outs, gf, gk), (outs2, gf2, gk2) = runs
    assert all(torch.equal(a, b) for a, b in zip(outs, outs2))
    assert torch.equal(gf, gf2) and all(torch.equal(a, b) for a, b in zip(gk, gk2))
    return outs, gf, gk


def _reference_grads(feat, kerns, gouts, cells, sizes):
    f64 = feat.double().requires_grad_(True)
    k64 = [k.double().requires_grad_(True) for k in kerns]
    refs = _reference(f64, k64, cells, sizes)
    rgf, *rgk = torch.autograd.grad(sum((r * g.double()).sum() for r, g in zip(refs, gouts)), [f64, *k64],
                                    allow_unused=True)
    return [r.detach() for r in refs], rgf, [torch.zeros_like(k) if g is None else g for k, g in zip(k64, rgk)]


def _check_zero_cells(gk, cells):
    """d/d kernel is exactly zero at every cell that is not positive."""
    for l, g in enumerate(gk):
        B, C = g.shape[:2]
        S2 = g.shape[2] * g.shape[3]
        pos = torch.zeros(B, S2, dtype=torch.bool, device=DEV)
        for b in range(B):
            pos[b, cells[l][b]] = True
        assert torch.all(g.flatten(2)[~pos[:, None, :].expand(B, C, S2)] == 0), l


def _elementwise(name, got, ref, tol):
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = scaled_err(got, ref)
    print(f'[elementwise] {name}: {err:.3e} (bar {tol:.0e})')
    assert err <= tol, (name, err)


def _check(B, C, h, w, grids, sizes, cells, seed):
    """Random data against the element-wise bars, then the exactness probe; returns the random run's rows."""
    gen = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, C, h, w, generator=gen).to(DEV)
    kerns = [(torch.randn(B, C, S, S, generator=gen) * 0.05).to(DEV) for S in grids]
    n = [sum(int(c.numel()) for c in lvl) for lvl in cells]
    gouts = [torch.randn((m,) + tuple(s), generator=gen).to(DEV) for m, s in zip(n, sizes)]
    outs, gf, gk = _run(feat, kerns, gouts, cells, sizes)
    refs, rgf, rgk = _reference_grads(feat, kerns, gouts, cells, sizes)
    for l, (o, r) in enumerate(zip(outs, refs)):
        assert o.shape == r.shape and o.dtype == torch.float32
        _elementwise(f'rows {l}', o, r, TOL_OUT)
    _elementwise('d/d feature', gf, rgf, TOL_GFEAT)
    for l, (g, r) in enumerate(zip(gk, rgk)):
        assert g.shape == kerns[l].shape
        _elementwise(f'd/d kernel {l}', g, r, TOL_GKERN)
    _check_zero_cells(gk, cells)
    _probe(B, C, h, w, grids, sizes, cells, gen)
    return outs


def _probe(B, C, h, w, grids, sizes, cells, gen):
    for s in sizes:
        assert s in ((h, w), (h // 2, w // 2), (h // 4, w // 4)) and (h // 4) * 4 == h and (w // 4) * 4 == w
        assert s[0] * s[1] % 4 == 0
    feat = torch.randint(-2, 3, (B, C, h, w), generator=gen).float().to(DEV)
    kerns = [torch.randint(-2, 3, (B, C, S, S), generator=gen).float().to(DEV) for S in grids]
    n = [sum(int(c.numel()) for c in lvl) for lvl in cells]
    gouts = [(torch.randint(-1, 2, (m,) + tuple(s), generator=gen) * (torch.rand((m,) + tuple(s), generator=gen) < 0.5))
             .float().to(DEV) for m, s in zip(n, sizes)]
    refs, rgf, rgk = _reference_grads(feat, kerns, gouts, cells, sizes)
    # the probe's precondition: every reference value a multiple of 1/4 below 2^20, and every partial sum of the op
    # bounded by a sum of absolute values below 2^20 (|kernel * operand| <= 4 over C channels; |g * operand| <= 2 over the
    # pixels of an operand or the kernels of an image)
    for r in refs + [rgf] + rgk:
        assert torch.equal(r * 4, (r * 4).round()) and bool((r.abs() < 2 ** 20).all())
    assert 4 * C < 2 ** 20 and 2 * h * w < 2 ** 20 and 2 * sum(n) < 2 ** 20
    outs, gf, gk = _run(feat, kerns, gouts, cells, sizes)
    for l, (o, r) in enumerate(zip(outs, refs)):
        assert o.shape == r.shape
        assert torch.equal(o.double(), r), ('rows', l, (o.double() - r).abs().max().item())
    assert torch.equal(gf.double(), rgf), ('d/d feature', (gf.double() - rgf).abs().max().item())
    for l, (g, r) in enumerate(zip(gk, rgk)):
        assert torch.equal(g.double(), r), ('d/d kernel', l, (g.double() - r).abs().max().item())


@pytest.mark.parametrize('h,w', [(200, 256), (200, 336)])
def test_cells_config_d_shapes(h, w):
    """config D's feature map (and a 1344x800 pad's), ragged counts, an image without positives in one level, a level
    without any."""
    gen = torch.Generator().manual_seed(h + w)
    counts = [[37, 0], [12, 90], [0, 0], [5, 1], [17, 130]]
    cells = _cells(2, GRIDS, gen, counts)
    _check(2, 256, h, w, GRIDS, _sizes(h, w), cells, seed=w)


@pytest.mark.parametrize('B', [1, 8, 16, 17, 33])
def test_cells_batch_sizes(B):
    """8 levels over 4 operands with random counts; 16 images fill one pack call's table, 17 and 33 take two and three."""
    gen = torch.Generator().manual_seed(B)
    h, w = 64, 80
    grids = (40, 36, 24, 16, 12, 12, 40, 36)
    counts = [[int(torch.randint(0, S, (1,), generator=gen)) for _ in range(B)] for S in grids]
    if B > 2:
        for lvl in counts:
            lvl[B // 2] = 0                         # an image without positives between images with some
    _check(B, 256, h, w, grids, _sizes8(h, w), _cells(B, grids, gen, counts), seed=10 + B)


# per level (8 levels, operands: levels 0-1 full size, 2-3 half, 4-5 quarter, 6-7 full again), per image (3: the middle one
# without any positive); per (level, image) segment and per (operand, image) problem the kernel counts 0, 1, 31, 32, 33,
# 127, 128 and 129 -- the edges of the 32-row K-blocks of d/d operand, the 128-row chunks of d/d kernel and the forward's
# kernel chunks.  'native': the widest problem holds exactly 256 kernels (operand 0, image 2: 128 + 128), the most the
# d/d operand kernel takes; 'fallback': operand 0, image 0 holds 129 + 128 > 256, d/d operand through cuBLAS.
EDGE_GRIDS = (12, 16, 12, 12, 12, 12, 16, 12)
EDGE_COUNTS = {
    'native': [[31, 0, 128], [1, 0, 128], [33, 0, 127], [0, 0, 0], [32, 0, 129], [0, 0, 1], [127, 0, 33], [0, 0, 31]],
    'fallback': [[129, 0, 1], [128, 0, 0], [31, 0, 0], [0, 0, 0], [0, 0, 128], [0, 0, 1], [1, 0, 127], [127, 0, 1]],
}
# feature maps whose quarter-size operand has a pixel tail: 11x12 = 132 = 128 + 4, 14x18 = 252 = 128 + 124
EDGE_MAPS = {'native': (44, 48), 'fallback': (56, 72)}


@pytest.mark.parametrize('table', ['native', 'fallback'])
@pytest.mark.parametrize('C', [32, 96, 160, 224, 256])
def test_cells_envelope_edges_per_image(C, table):
    counts = EDGE_COUNTS[table]
    level_op = [0, 0, 1, 1, 2, 2, 3, 3]
    widest = max(sum(n[b] for n, lo in zip(counts, level_op) if lo == o) for o in range(4) for b in range(3))
    assert widest == 256 if table == 'native' else widest > 256
    gen = torch.Generator().manual_seed(C)
    h, w = EDGE_MAPS[table]
    _check(3, C, h, w, EDGE_GRIDS, _sizes8(h, w), _cells(3, EDGE_GRIDS, gen, counts), seed=C + len(table))


def test_cells_four_pixel_operand():
    """an 8x8 feature map: operands of 64, 16 and 4 pixels (one 128-pixel tile, almost all of it tail)."""
    gen = torch.Generator().manual_seed(4)
    grids, h, w = (12, 8, 6, 6), 8, 8
    counts = [[33, 1, 0], [0, 64, 2], [36, 0, 35], [1, 1, 1]]
    _check(3, 160, h, w, grids, [(8, 8), (4, 4), (2, 2), (2, 2)], _cells(3, grids, gen, counts), seed=4)


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


def test_cells_rows_beyond_one_pack():
    """every cell of a 40x40 and a 36x36 level of one operand on image 0: 2896 rows, more than the 2048 of one pack call,
    so they take two and level 1's rows of that image straddle them; image 1's 1600 rows fit the first."""
    gen = torch.Generator().manual_seed(9)
    grids, h, w = (40, 36), 32, 40
    counts = [[1600, 700], [1296, 900]]
    _check(2, 64, h, w, grids, [(h, w), (h, w)], _cells(2, grids, gen, counts), seed=9)


def test_cells_grid_beyond_64_raises():
    """the pack takes grids of at most 64 x 64 cells: a larger one is an error, never wrong rows."""
    from boxinstseg_b200.ops.dynconv import solo_cells_conv
    f = torch.randn(1, 32, 8, 8, device=DEV)
    k = torch.randn(1, 32, 65, 65, device=DEV)
    with pytest.raises(NotImplementedError, match='64 x 64'):
        solo_cells_conv(f, [k], [[torch.arange(3, device=DEV)]], [(8, 8)])


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
    _elementwise('d/d feature, image 0', gf[0], ref, TOL_GFEAT)


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
        _elementwise(f'rows of image {b} against the dense path', rows[b], dense[b, cells[b]], TOL_OUT)
