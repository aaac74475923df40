"""Exact arg-max ties in the projection term, and the single-pass BoxInst loss across its whole envelope.

Every projection path sends the gradient of a row / column maximum to ONE element: the first index on exact ties, like
torch.max(dim), with -0 equal to +0; the BoxInst paths choose it on the logits (DESIGN section 4, note (i)).  Real inputs
tie: the CondInst head's x2 aligned upsample makes rows 0/1 and columns 0/1 bit-identical, and 16-bit masks tie all the
time.  The generators below plant ties wherever a kernel merges partial maxima: inside and across float4 groups and
128-column chunks (row maxima), inside and across 4-row groups, 24-row stream items and the finalize's 12-item batches
(single pass), across strips (two-call) and 8-row segments (dense).  Everything is judged element-wise against the
float64 oracle: oracle.boxinst.projection_losses_logit_argmax plus the pairwise term of oracle.boxinst.pairwise_nlog.
"""
import functools

import pytest
import torch

from oracle import boxinst as ob

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
UPSTREAM = [(1.0, 1.0), (0.75, 2.5), (1.0, 0.0), (0.0, 1.0)]      # (g_prj, g_pair)


# ------------------------------------------------------------------ problems: logits, boxes, edge bits, oracle
def _rect_set(H, W):
    """(j0, j1, i0, i1), inclusive: the whole map, one pixel, boxes touching each border, an empty rect."""
    h2, w2 = H // 2, W // 2
    return [(0, H - 1, 0, W - 1), (h2, h2, w2, w2), (0, h2, w2 // 2, w2), (h2, H - 1, 0, w2), (h2 // 2, h2, 0, W // 3),
            (0, H // 3, w2, W - 1), (h2, h2 - 1, 1, 0)]


def _edge_bits(H, W, dil, gen):
    """uint8 [1,H,W]: bit c set with probability 0.7 where neighbour c (neighbour_offsets order) is inside the map."""
    bits = torch.zeros(H, W, dtype=torch.int32)
    for c, (dy, dx) in enumerate(ob.neighbour_offsets(3, dil)):
        inside = ob._inside(H, W, dy, dx, torch.zeros(1)) > 0
        bits |= ((torch.rand(H, W, generator=gen) < 0.7) & inside).to(torch.int32) << c
    return bits.to(torch.uint8)[None]


class Problem:
    """One image's edge bits, the rect set, instance n -> rect n % 7; warm-up factor 1."""

    def __init__(self, logits, dil, seed):
        N, _, H, W = logits.shape
        self.x, self.dil = logits.float().contiguous(), dil
        self.rects = torch.tensor(_rect_set(H, W), dtype=torch.int32)
        self.inst_gt = torch.arange(N, dtype=torch.int32) % self.rects.shape[0]
        self.bits = _edge_bits(H, W, dil, torch.Generator().manual_seed(seed))
        self._oracle = None

    def targets(self):
        from boxinstseg_b200.ops.boxinst import BoxInstTargets
        G = self.rects.shape[0]
        return BoxInstTargets(self.bits.to(DEV), None, self.rects.to(DEV), torch.zeros(G, dtype=torch.int32, device=DEV),
                              [G], None, None)

    def box_masks(self):
        _, _, H, W = self.x.shape
        j0, j1, i0, i1 = (self.rects[self.inst_gt.long(), k].view(-1, 1, 1) for k in range(4))
        ys, xs = torch.arange(H).view(1, H, 1), torch.arange(W).view(1, 1, W)
        return ((ys >= j0) & (ys <= j1) & (xs >= i0) & (xs <= i1))[:, None].double()

    def oracle(self):
        """(loss_prj, loss_pair, d loss_prj / d x, d loss_pair / d x) in float64."""
        if self._oracle is None:
            x64 = self.x.double().requires_grad_(True)
            bm = self.box_masks()
            prj = ob.projection_losses_logit_argmax(x64, bm).mean()
            wc = torch.stack([(self.bits[0].long() >> c) & 1 for c in range(8)]).double()
            w = wc[None] * bm
            pair = (ob.pairwise_nlog(x64, 3, self.dil) * w).sum() / w.sum().clamp(min=1.0)
            (g_prj,) = torch.autograd.grad(prj, x64)
            (g_pair,) = torch.autograd.grad(pair, x64)
            self._oracle = (prj.item(), pair.item(), g_prj, g_pair)
        return self._oracle


def _iters():
    return torch.tensor([10000.0], device=DEV)


def _single_pass(p, gp, gq):
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss
    x = p.x.to(DEV).requires_grad_(True)
    prj, pair = boxinst_mask_loss(x, p.targets(), p.inst_gt.to(DEV), _iters(), pairwise_dilation=p.dil)
    (g,) = torch.autograd.grad(prj * gp + pair * gq, x)
    return prj.item(), pair.item(), g


def _second_backward(p, gp, gq):
    """retain_graph: the second backward through the same node recomputes with the two-call kernels."""
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss
    x = p.x.to(DEV).requires_grad_(True)
    prj, pair = boxinst_mask_loss(x, p.targets(), p.inst_gt.to(DEV), _iters(), pairwise_dilation=p.dil)
    torch.autograd.grad(prj + pair, x, retain_graph=True)
    (g,) = torch.autograd.grad(prj * gp + pair * gq, x)
    return prj.item(), pair.item(), g


def _two_call(p, gp, gq):
    from tests.test_boxinst_gpu import _two_call as two_call
    out, g = two_call(dict(logits=p.x, gt_inds=p.inst_gt), p.targets(), DEV, p.dil, gp, gq)
    return out[0].item(), out[1].item(), g


def _no_grad(p):
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss
    with torch.no_grad():
        prj, pair = boxinst_mask_loss(p.x.to(DEV), p.targets(), p.inst_gt.to(DEV), _iters(), pairwise_dilation=p.dil)
    return prj.item(), pair.item()


def _check_losses(p, prj, pair):
    prj64, pair64, _, _ = p.oracle()
    assert abs(prj - prj64) <= 1e-4 * abs(prj64) + 1e-7, (prj, prj64)
    assert abs(pair - pair64) <= 1e-4 * abs(pair64) + 1e-7, (pair, pair64)


def _check(p, result, gp, gq, exact_support=True):
    """Losses, every gradient element, and at (1, 0) the support: exactly the oracle's nonzero elements, which are
    first row / column arg-max positions of the logits."""
    prj, pair, g = result
    _check_losses(p, prj, pair)
    _, _, g_prj, g_pair = p.oracle()
    ref = gp * g_prj + gq * g_pair
    g = g.cpu()
    bad = ~torch.isclose(g.double(), ref, rtol=1e-4, atol=1e-6 * ref.abs().max().item() + 1e-9)
    assert not bad.any(), (bad.nonzero()[:8].tolist(), g[bad][:8].tolist(), ref[bad][:8].tolist())
    if gq == 0.0:
        assert not ((g != 0) & ~ob.logit_argmax_mask(p.x)).any(), (g != 0).logical_and(~ob.logit_argmax_mask(p.x)).nonzero()[:8]
        if exact_support:
            assert torch.equal(g != 0, ref != 0), ((g != 0) ^ (ref != 0)).nonzero()[:8].tolist()


# ------------------------------------------------------------------ tied logits (seeded)
def _planted(N, H, W, gen):
    """Ties on every structural boundary.  Base <= 2; column ties at 7 (distinct columns), row ties at 5 (rows without a
    7), and a 9 that is both a row and a column arg-max at an interior position, tied later in its row and column."""
    x = torch.randn(N, 1, H, W, generator=gen).clamp(max=2.0)
    col_ties = [((1, 2), 5), ((0, 3), 9), ((3, 6), 14),          # inside a 4-row group / across groups
                ((23, 24), 21), ((22, 27), 30),                  # across 24-row stream items
                ((287, 288), 38), ((283, 290), 45)]              # across the finalize's 12-item batches
    row_ties = [(10, (1, 2)), (12, (2, 5)), (15, (3, 4)),        # inside a float4 group / across groups
                (17, (100, 140)), (40, (0, 129)), (41, (127, 128))]     # across 128-column chunks
    for (r1, r2), c in col_ties:
        if r2 < H and c < W:
            x[:, 0, r1, c] = x[:, 0, r2, c] = 7.0
    for r, (c1, c2) in row_ties:
        if r < H and c2 < W:
            x[:, 0, r, c1] = x[:, 0, r, c2] = 5.0
    yc, xc = min(50, H - 3), min(60, W - 4)
    x[:, 0, yc, xc] = x[:, 0, yc, xc + 3] = x[:, 0, yc + 2, xc] = 9.0
    return x


def _signed_zero(N, H, W, gen):
    """All logits negative except planted zeros, -0.0 first: columns across 8-row segments, strips, 24-row items and
    inside a 4-row group; rows across float4 groups and 128-column chunks."""
    x = -(torch.randn(N, 1, H, W, generator=gen).abs() + 0.5)
    for r1, r2, c in [(0, 8, 3), (2, 26, 7), (5, H - 1, 11), (23, 24, 13), (1, 3, 17)]:
        x[:, 0, r1, c], x[:, 0, r2, c] = -0.0, 0.0
    for r, c1, c2 in [(10, 1, 2), (12, 2, min(130, W - 1)), (15, 0, W - 1)]:
        x[:, 0, r, c1], x[:, 0, r, c2] = -0.0, 0.0
    return x


def _head_logits(N, H, W, gen):
    """Logits of CondInstMaskHead.forward (x2 aligned upsample of an (H/2) x (W/2) map): rows 0/1, columns 0/1 tie."""
    from boxinstseg_b200.models import build_head
    head = build_head(dict(type='CondInstMaskHead', in_channels=16, in_stride=8, out_stride=4, topk_per_img=64,
                           max_proposals=-1, boxinst_enabled=True)).to(DEV)
    h, w = H // 2, W // 2
    feat = torch.randn(1, 16, h, w, generator=gen).to(DEV)
    params = (torch.randn(N, 233, generator=gen) * 0.3).to(DEV)
    coors = (torch.rand(N, 2, generator=gen) * torch.tensor([w * 8.0, h * 8.0])).to(DEV)
    levels = torch.randint(0, 5, (N,), generator=gen).to(DEV)
    with torch.no_grad():
        x = head(feat, params, coors, levels, torch.zeros(N, dtype=torch.long, device=DEV)).float().cpu()
    assert x.shape == (N, 1, H, W)
    assert torch.equal(x[:, :, 0], x[:, :, 1]) and torch.equal(x[..., 0], x[..., 1])
    return x


def _tied_logits(kind, N, H, W, gen):
    if kind == 'upsample':
        return ob.aligned_bilinear(torch.randn(N, 1, H // 2, W // 2, generator=gen) * 3, 2)
    if kind == 'head':
        return _head_logits(N, H, W, gen)
    if kind == 'fp16':
        return (torch.randn(N, 1, H, W, generator=gen) * 3).half().float()
    if kind == 'bf16':
        return (torch.randn(N, 1, H, W, generator=gen) * 3).bfloat16().float()
    if kind == 'quarter':
        return torch.round(4 * torch.randn(N, 1, H, W, generator=gen) * 2) / 4
    if kind == 'constant':
        return torch.randn(N, 1, 1, 1, generator=gen).expand(N, 1, H, W).contiguous()
    if kind == 'saturated':              # even instances: +-30 only (ties at 30); odd: |x| in [20, 40), distinct
        sign = torch.where(torch.rand(N, 1, H, W, generator=gen) < 0.5, -1.0, 1.0)
        mag = torch.where(torch.arange(N).view(N, 1, 1, 1) % 2 == 0, torch.tensor(30.0),
                          20 + 20 * torch.rand(N, 1, H, W, generator=gen))
        return sign * mag
    if kind == 'planted':
        return _planted(N, H, W, gen)
    if kind == 'signed_zero':
        return _signed_zero(N, H, W, gen)
    raise ValueError(kind)


KINDS = ['upsample', 'head', 'fp16', 'bf16', 'quarter', 'constant', 'saturated', 'planted', 'signed_zero']
SHAPES = [(7, 296, 160, 2),            # S = 13 stream items: two finalize batches; W > 128, not a multiple of 128
          (6, 48, 256, 3)]             # two full 128-column chunks


@functools.lru_cache(maxsize=None)
def _tie_problem(kind, shape):
    N, H, W, dil = shape
    seed = 100 * KINDS.index(kind) + SHAPES.index(shape)
    return Problem(_tied_logits(kind, N, H, W, torch.Generator().manual_seed(seed)), dil, seed)


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('kind', KINDS)
def test_single_pass_ties(kind, shape):
    from boxinstseg_b200 import _lib as L
    p = _tie_problem(kind, shape)
    N, _, H, W = p.x.shape
    assert L.lib().bxs_boxinst_loss_fused_supported(N, H, W, p.dil) == 1
    for gp, gq in UPSTREAM:
        r1 = _single_pass(p, gp, gq)
        _check(p, r1, gp, gq, exact_support=kind != 'saturated')
        r2 = _single_pass(p, gp, gq)
        assert r1[:2] == r2[:2] and torch.equal(r1[2], r2[2])          # bitwise run to run


@pytest.mark.parametrize('shape', SHAPES)
@pytest.mark.parametrize('kind', KINDS)
def test_two_call_no_grad_and_second_backward_ties(kind, shape):
    p = _tie_problem(kind, shape)
    _check_losses(p, *_no_grad(p))
    for gp, gq in UPSTREAM:
        r1 = _two_call(p, gp, gq)
        _check(p, r1, gp, gq, exact_support=kind != 'saturated')
        r2 = _two_call(p, gp, gq)
        assert r1[:2] == r2[:2] and torch.equal(r1[2], r2[2])
        r3 = _second_backward(p, gp, gq)
        _check(p, r3, gp, gq, exact_support=kind != 'saturated')
        r4 = _second_backward(p, gp, gq)
        assert torch.equal(r3[2], r4[2])


@pytest.mark.parametrize('kind', KINDS)
def test_dense_projection_ties(kind):
    """projection_losses / BoxProjectionLoss / mil_loss choose positions on the SCORES: judged by the float64 score
    oracle on the tied maps themselves and on their fp16 / bf16-quantised sigmoids."""
    from boxinstseg_b200.models.losses import BoxProjectionLoss, mil_loss, projection_losses
    p = _tie_problem(kind, SHAPES[0])
    bm = p.box_masks().float()
    N = bm.shape[0]
    gl = torch.arange(1, N + 1, dtype=torch.float64)
    variants = [('projection_losses', lambda s, t: projection_losses(s, t), 1e-5, 1.0),
                ('BoxProjectionLoss', BoxProjectionLoss(loss_weight=2.5), 1e-5, 2.5),
                ('mil_loss', lambda s, t: mil_loss(None, s[:, 0], None, t[:, 0]), 2e-3, 1.0)]
    for scores in (p.x, p.x.sigmoid().half().float(), p.x.sigmoid().bfloat16().float()):
        for name, fn, eps, lw in variants:
            s64 = scores.double().requires_grad_(True)
            ref = lw * ob.projection_losses(s64, bm.double(), eps)
            (gref,) = torch.autograd.grad((ref * gl).sum(), s64)
            sg = scores.to(DEV).requires_grad_(True)
            out = fn(sg, bm.to(DEV))
            (gs,) = torch.autograd.grad((out * gl.float().to(DEV)).sum(), sg)
            gs = gs.cpu().reshape(gref.shape)
            assert torch.allclose(out.cpu().double(), ref.detach(), rtol=1e-5, atol=1e-6), name
            # support: nothing off the oracle's first-index arg-max positions, and every one of them that float32 can
            # resolve.  (Where the scores saturate to 1.0 under a whole-map box, d dice / d s = -2 eps / U^2 ~ 1e-10:
            # eps is below float32 resolution in U = |s|^2 + |t|^2 + eps, so the kernel's coefficient is exactly 0.)
            off = (gs != 0) & (gref == 0)
            missing = (gs == 0) & (gref.abs() > 1e-6 * gref.abs().max())
            assert not off.any() and not missing.any(), (name, off.nonzero()[:8].tolist(), missing.nonzero()[:8].tolist())
            assert torch.allclose(gs.double(), gref, rtol=1e-4, atol=1e-7), name


# ------------------------------------------------------------------ the single-pass envelope
ENVELOPE = ([(N, 8, 8) for N in (1, 1025, 2048)] +                               # N > 1024: plan scan, 16-bit arrivals
            [(7, H, 20) for H in (1, 3, 4, 23, 24, 25, 289, 312, 512)] +         # S = 1 .. 22 stream items
            [(7, 26, W) for W in (4, 8, 124, 128, 132, 512)])


@pytest.mark.parametrize('dil', [1, 2, 3, 4])
@pytest.mark.parametrize('N,H,W', ENVELOPE)
def test_single_pass_envelope(N, H, W, dil):
    """fp16-valued logits (ties included): the single pass against the two-call kernels and the float64 oracle."""
    from boxinstseg_b200 import _lib as L
    assert L.lib().bxs_boxinst_loss_fused_supported(N, H, W, dil) == 1
    seed = N * 7919 + H * 131 + W * 7 + dil
    x = (torch.randn(N, 1, H, W, generator=torch.Generator().manual_seed(seed)) * 3).half().float()
    p = Problem(x, dil, seed)
    for gp, gq in [(1.0, 1.0), (0.75, 2.5)]:
        prj, pair, g = _single_pass(p, gp, gq)
        prj2, pair2, g2 = _two_call(p, gp, gq)
        assert abs(prj - prj2) <= 1e-5 * abs(prj2) and abs(pair - pair2) <= 1e-5 * abs(pair2) + 1e-9
        assert torch.allclose(g, g2, rtol=1e-4, atol=1e-9)
        _check(p, (prj, pair, g), gp, gq)


@pytest.mark.parametrize('N,H,W', [(2049, 8, 8), (3, 513, 8), (3, 8, 516), (3, 8, 510)])
def test_just_outside_the_envelope_is_the_two_call_path(N, H, W):
    from boxinstseg_b200 import _lib as L
    assert L.lib().bxs_boxinst_loss_fused_supported(N, H, W, 2) == 0
    x = (torch.randn(N, 1, H, W, generator=torch.Generator().manual_seed(N + H + W)) * 3).half().float()
    p = Problem(x, 2, 5)
    prj, pair, g = _single_pass(p, 0.75, 2.5)
    prj2, pair2, g2 = _two_call(p, 0.75, 2.5)
    assert prj == prj2 and pair == pair2 and torch.equal(g, g2)
