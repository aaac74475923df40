"""The registry losses of ``models/losses`` across their envelopes, every output judged element-wise against float64
autograd of the oracle.

  * level-set energy (fused_assembly.cu, ``lsf_forward_kernel`` / ``lsf_backward_kernel``): one cluster of 8 CTAs of 512
    threads per instance, so one pass over a map strides 4096 pixels; channel loops unrolled to MC = 4 for C <= 4 and to
    LS_MAXC = 8 above.  Mode 1 is ``levelset_assembly`` (sigmoid, cat(s, 1 - s) * box, T * box, clamp(sum box, 1) inside
    the kernel), mode 0 is the dense ``LevelsetLoss`` / ``region_levelset``.  Every batch mixes instances in every clamp
    regime of the means (see ``ls_batch``);
  * dense box projection (projection_levelset.cu, ``prj_*_kernel``): column maxima over row segments whose count follows
    from n * w and the SM count;
  * length regulariser (``length_*_kernel``): per-instance partial sums over an SM-derived chunk count capped at 64.
The SM-derived counts are restated here and every case asserts the side it lands on; the SM count is read from the
library, so the cases keep their meaning on any H100 variant.  Every case runs twice and must repeat bit for bit.

Element-wise bars: ``scaled_err`` = max |got - ref| / (|ref| + 1e-2 max |ref|) over all elements of one output.  The
largest value observed over all cases on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit) is given next to each bar.
"""
import functools

import pytest
import torch

from oracle import boxinst as ob
from oracle import levelset as ol
from tests.helpers import scaled_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

# element-wise bars (scaled_err) and, in the comments, the largest value observed over all cases (H100, see above)
TOL_LS_LOSS = 1e-5         # level-set loss per instance                             1.6e-6 (n = 65536, 2x3)
TOL_LS_GLOGIT = 5e-5       # d / d logits (mode 1)                                   1.7e-5 (n = 37, C = 1, 33x47)
TOL_LS_GSCORE = 2e-6       # d / d scores2 (mode 0)                                  3.2e-7 (n = 65536, 2x3)
TOL_LS_GT = 2e-5           # d / d T (both modes)                                    5.3e-6 (mode 1, 1x1)
TOL_PRJ_LOSS = 1e-5        # projection loss per instance                            3.3e-6 (n = 3, 200x256)
TOL_PRJ_GRAD = 1e-5        # projection d / d scores                                 3.8e-6 (n = 4096, 9x257)
TOL_LEN_LOSS = 3e-7        # length regulariser per instance                         8.7e-8 (n = 4, C = 3, 300x1)
TOL_LEN_GRAD = 3e-7        # length regulariser d / d scores                         5.9e-8 (n = 1024, C = 2, 16x20)


@functools.lru_cache(maxsize=None)
def sms():
    from boxinstseg_b200 import _lib as L
    n = L.lib().bxs_device_sm_count()
    assert n > 0
    return n


def check_close(name, got, ref, tol, floor=None):
    """scaled_err; ``floor`` [n], one value per instance (leading dimension), is added to the denominator where the
    reference is only rounding noise (see check_levelset)."""
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    if floor is not None:
        got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
        floor = floor.double().view((-1,) + (1,) * (ref.dim() - 1))
        err = ((got - ref).abs() / (ref.abs() + 1e-2 * ref.abs().max() + floor)).max().item()
    else:
        err = scaled_err(got, ref)
    print(f'[elementwise] {name}: {err:.3e} (bar {tol:.0e})')
    assert err <= tol, (name, err)


def twice(fn):
    """fn() run twice; the two results must be bit-identical."""
    first, second = fn(), fn()
    assert len(first) == len(second)
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    return second


def upstream(n, gen):
    """Per-instance upstream gradient in [0.5, 1.5) with an exact zero on every fourth instance (3, 7, ...)."""
    g = torch.rand(n, generator=gen) + 0.5
    g[3::4] = 0
    return g


# ================================================================== level-set energy
LS_REGIMES = 9


def ls_batch(n, C, h, w, seed, soft):
    """(logits [n,h,w], box [n,h,w], T [n,C,h,w]); instance i is in regime i % 9:
       0 a box over at least half of each side (soft values in [0, 1) when ``soft``), logits N(0, 2)
       1 an empty box: sum a = sum b = 0, both means clamped, clamp(sum box, 1) = 1
       2 a one-pixel box
       3 the whole map
       4 / 5 logits +30 / -30 in a random box: sigmoid is 1 / 1e-13, so one of sum a, sum b falls below 1e-5, the other not
       6 / 7 logits +100 / -100: the same with sigmoid exactly 1 / 0
       8 a random box, logits N(0, 2).
    T is N(0, 1) plus +-2 (alternating over the channels) where the logit is positive."""
    gen = torch.Generator().manual_seed(seed)
    reg = torch.arange(n) % LS_REGIMES
    logits = torch.randn(n, h, w, generator=gen) * 2
    for r, v in ((4, 30.0), (5, -30.0), (6, 100.0), (7, -100.0)):
        logits[reg == r] = v
    # features that differ inside and outside the mask, as image colours and tree-filtered features do: the means m0, m1
    # then differ by O(1), and d/d logits ~ (T - m0)^2 - (T - m1)^2 is not a near-cancellation of two equal squares
    sign = torch.tensor([(-1.0) ** c for c in range(C)]).view(1, C, 1, 1)
    T = torch.randn(n, C, h, w, generator=gen) + 2 * sign * (logits > 0).float().unsqueeze(1)

    def span(size, large):
        """[lo, hi) per instance: any non-empty range, or one that leaves at most a quarter of each end uncovered."""
        if large:
            return (torch.randint(0, max(size // 4, 1), (n,), generator=gen),
                    size - torch.randint(0, max(size // 4, 1), (n,), generator=gen))
        a = torch.randint(0, size, (n,), generator=gen)
        b = torch.randint(0, size, (n,), generator=gen)
        return torch.minimum(a, b), torch.maximum(a, b) + 1
    y0, y1 = span(h, False)
    x0, x1 = span(w, False)
    ly0, ly1 = span(h, True)
    lx0, lx1 = span(w, True)
    big = reg == 0
    y0, y1 = torch.where(big, ly0, y0), torch.where(big, ly1, y1)
    x0, x1 = torch.where(big, lx0, x0), torch.where(big, lx1, x1)
    one = reg == 2
    y1, x1 = torch.where(one, y0 + 1, y1), torch.where(one, x0 + 1, x1)
    full = reg == 3
    y0, y1 = torch.where(full, 0, y0), torch.where(full, h, y1)
    x0, x1 = torch.where(full, 0, x0), torch.where(full, w, x1)
    ys, xs = torch.arange(h).view(1, h, 1), torch.arange(w).view(1, 1, w)
    box = ((ys >= y0.view(n, 1, 1)) & (ys < y1.view(n, 1, 1)) & (xs >= x0.view(n, 1, 1)) & (xs < x1.view(n, 1, 1))).float()
    box[reg == 1] = 0
    if soft:
        box[big] *= torch.rand(int(big.sum()), h, w, generator=gen)
    return logits, box, T


def ls_dense_inputs(logits, box, T, seed):
    """mode-0 inputs from a mode-1 batch: scores2 = cat(s, 1 - s) * box in float32, T * box, and a pixel_num that is the
    box area on even instances and an unrelated positive number on odd ones."""
    gen = torch.Generator().manual_seed(seed + 1)
    s = torch.sigmoid(logits).unsqueeze(1)
    b = box.unsqueeze(1)
    scores2 = torch.cat((s, 1 - s), 1) * b
    pix = b.sum((1, 2, 3)).clamp(min=1)
    odd = torch.arange(pix.numel()) % 2 == 1
    pix[odd] = torch.rand(int(odd.sum()), generator=gen) * 50 + 0.25
    return scores2, T * b, pix


def check_levelset(entry, n, C, h, w, grads='xT', seed=0):
    """entry: 'assembly' (mode 1, levelset_assembly, loss_weight 1.5), 'LevelsetLoss' (mode 0, loss_weight 0.7) or
    'region_levelset' (mode 0, energy alone).  grads: which of x (logits / scores2) and T require a gradient."""
    from boxinstseg_b200.models.losses import LevelsetLoss, levelset_assembly, region_levelset
    logits, box, T = ls_batch(n, C, h, w, seed=seed or n * 7 + C * 131 + h * 3 + w, soft=entry == 'assembly')
    gen = torch.Generator().manual_seed(seed + 5)
    gup = upstream(n, gen)
    if entry == 'assembly':
        lw = 1.5
        x, tt = logits, T
    else:
        lw = 0.7 if entry == 'LevelsetLoss' else 1.0
        x, tt, pix = ls_dense_inputs(logits, box, T, seed)
    # float64 reference
    x64 = x.double().requires_grad_(True)
    t64 = tt.double().requires_grad_(True)
    if entry == 'assembly':
        s = torch.sigmoid(x64.unsqueeze(1))
        b = box.double().unsqueeze(1)
        phi, t_in, p_in = torch.cat((s, 1 - s), 1) * b, t64 * b, b.sum((1, 2, 3)).clamp(min=1)
    else:
        phi, t_in, p_in = x64, t64, pix.double() if entry == 'LevelsetLoss' else torch.ones(n, dtype=torch.float64)
    ref = ol.levelset_loss(phi, t_in, p_in, lw)
    gx_ref, gt_ref = torch.autograd.grad((ref * gup.double()).sum(), [x64, t64])
    # Where the means sit on T (every instance of a one-pixel map) the energy and both gradients are 0 but for fp32
    # rounding of T - m_k, in any implementation, and the reference holds only rounding noise.  Each output is therefore
    # also judged against 1e-6 of its instance's size with both means at zero: lw sum T^2 (S_0 + S_1) / (C pix) for the
    # loss, g lw / pix times max T^2 for d/dx and times max |T| for d/dT.
    with torch.no_grad():
        mag = lw * ((t_in * t_in) * phi.sum(1, keepdim=True)).sum((1, 2, 3)) / (C * p_in)
        gscale = (lw * gup.double() / p_in).abs()
        tmax = tt.abs().max().item()

    def once():
        xg = x.to(DEV).requires_grad_('x' in grads)
        tg = tt.to(DEV).requires_grad_('T' in grads)
        if entry == 'assembly':
            out = levelset_assembly(xg, box.to(DEV), tg, loss_weight=lw)
        elif entry == 'LevelsetLoss':
            out = LevelsetLoss(lw)(xg, tg, pix.to(DEV))
        else:
            out = region_levelset()(xg, tg)
        wrt = [v for k, v in (('x', xg), ('T', tg)) if k in grads]
        return (out.detach(),) + torch.autograd.grad((out * gup.to(DEV)).sum(), wrt)
    got = twice(once)
    tag = f'{entry} n={n} C={C} {h}x{w} grads={grads}'
    check_close(f'{tag} loss', got[0], ref.detach(), TOL_LS_LOSS, floor=1e-6 * mag.abs())
    rest = list(got[1:])
    if 'x' in grads:
        check_close(f'{tag} d/dx', rest.pop(0), gx_ref, TOL_LS_GLOGIT if entry == 'assembly' else TOL_LS_GSCORE,
                    floor=1e-6 * gscale * tmax * tmax)
    if 'T' in grads:
        check_close(f'{tag} d/dT', rest.pop(0), gt_ref, TOL_LS_GT, floor=1e-6 * gscale * tmax)


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 7, 8])
@pytest.mark.parametrize('entry', ['assembly', 'LevelsetLoss'])
def test_levelset_channels(entry, C):
    """Both sides of the MC = 4 switch (C = 4: every unrolled slot live; C = 5: the first LS_MAXC instantiation) and the
    cap C = 8; 37 instances of 1551 pixels (four CTAs of each cluster hold pixels)."""
    check_levelset(entry, 37, C, 33, 47)


LS_MAPS = [
    (9, 3, 1, 1), (9, 2, 1, 300), (9, 3, 300, 1), (9, 5, 9, 7),           # fewer pixels than one CTA's 512
    (9, 3, 63, 65), (9, 2, 64, 64), (9, 4, 17, 241),                      # 4095, 4096, 4097: the cluster's stride
    (18, 3, 200, 256), (9, 2, 256, 256),                                  # the heads' maps (config D, Box2Mask)
    (1, 3, 1024, 1024),                                                   # fp32 sums over a large map
    (2048, 2, 12, 20),
]


@pytest.mark.parametrize('n,C,h,w', LS_MAPS)
@pytest.mark.parametrize('entry', ['assembly', 'LevelsetLoss'])
def test_levelset_map_sizes(entry, n, C, h, w):
    check_levelset(entry, n, C, h, w)


@pytest.mark.parametrize('n', [8191, 8192, 65536, 70001])
@pytest.mark.parametrize('entry', ['assembly', 'LevelsetLoss'])
def test_levelset_many_instances(entry, n):
    """The forward grid is n clusters of 8 CTAs in x; the backward puts the instance in y and so must be split into
    launches of at most 65535 instances.  Neither limit may reach the caller."""
    check_levelset(entry, n, 1, 2, 3)


@pytest.mark.parametrize('grads', ['x', 'T', 'xT'])
@pytest.mark.parametrize('entry', ['assembly', 'LevelsetLoss', 'region_levelset'])
def test_levelset_backward_variants(entry, grads):
    """Only one of the inputs requiring a gradient makes the backward run with g_x or g_T null."""
    check_levelset(entry, 37, 5, 64, 64, grads=grads)


# ================================================================== dense box projection
def prj_segments(n, h, w):
    """bxs_projection_loss_forward: (rows_per_seg, segs) of prj_cols_kernel."""
    segs = min(-(-h // 8), max(1, -(-(sms() * 8 * 256) // (n * w))))
    rows = -(-h // segs)
    return rows, -(-h // rows)


PRJ_CASES = [(3, h, w, 'many' if h > 8 else 'one') for h in (1, 7, 8, 9, 200) for w in (1, 255, 256, 257, 1300)]
PRJ_CASES += [(1, 1, 1, 'one'), (1, 9, 257, 'many'), (1, 200, 1300, 'many'),
              (4096, 7, 255, 'one'), (4096, 8, 256, 'one'), (4096, 9, 257, 'one'), (4096, 200, 1, 'many')]


@pytest.mark.parametrize('n,h,w,side', PRJ_CASES)
def test_projection_envelope(n, h, w, side):
    """Column maxima over one or several row segments (prj_cols_kernel), one or several 256-column x-blocks; soft,
    binary and all-zero targets; the registry class (eps 1e-5) on odd cases, projection_losses with DiscoBox's eps on
    even ones.  Scores stay below 0.8: a profile equal to its target is the dice's optimum, where the gradient
    (2 / U) (2 s I / U - t) cancels and fp32 rounding of I / U, in any implementation, would be all the comparison sees."""
    from boxinstseg_b200.models.losses import BoxProjectionLoss, projection_losses
    rows, segs = prj_segments(n, h, w)
    assert (segs > 1) == (side == 'many'), (n, h, w, rows, segs)
    if h == 9 and side == 'many':
        assert h % rows != 0                                       # a short last segment
    gen = torch.Generator().manual_seed(n * 7 + h * 13 + w)
    s = torch.rand(n, 1, h, w, generator=gen) * 0.8
    t = (torch.rand(n, 1, h, w, generator=gen) > 0.6).float()
    kind = torch.arange(n) % 4                                     # 0, 3 binary, 1 all zero, 2 soft
    t[kind == 1] = 0
    t[kind == 2] *= torch.rand(int((kind == 2).sum()), 1, h, w, generator=gen)
    gup = upstream(n, gen)
    use_class = (n + h + w) % 2 == 1
    eps, lw = (1e-5, 2.0) if use_class else (2e-3, 0.6)
    s64 = s.double().requires_grad_(True)
    ref = lw * ob.projection_losses(s64, t.double(), eps)
    (gref,) = torch.autograd.grad((ref * gup.double()).sum(), s64)

    def once():
        sg = s.to(DEV).requires_grad_(True)
        out = BoxProjectionLoss(lw)(sg, t.to(DEV)) if use_class else projection_losses(sg, t.to(DEV), eps, lw)
        (gs,) = torch.autograd.grad((out * gup.to(DEV)).sum(), sg)
        return out.detach(), gs
    out, gs = twice(once)
    tag = f'projection n={n} {h}x{w} segs={segs} rows={rows}'
    check_close(f'{tag} loss', out, ref.detach(), TOL_PRJ_LOSS)
    check_close(f'{tag} d/ds', gs, gref, TOL_PRJ_GRAD)


# ================================================================== length regulariser
def length_chunks(n, work_items):
    """pick_chunks of projection_levelset.cu: partial sums per instance of bxs_length_reg_forward."""
    want = -(-(sms() * 4) // n)
    c = min(want, -(-work_items // 256))
    return max(1, min(64, c))


@pytest.mark.parametrize('n,C,h,w,side,equal', [
    (1, 2, 100, 128, 'cap', False), (2, 3, 200, 256, 'cap', True),
    (1024, 2, 16, 20, 'one', True), (3, 1, 8, 16, 'one', False), (5, 1, 1, 1, 'one', False),
    (4, 3, 1, 300, 'some', True), (4, 3, 300, 1, 'some', False), (7, 4, 33, 47, 'some', True),
])
def test_length_envelope(n, C, h, w, side, equal):
    """sum |dy| + sum |dx| per instance over all channels.  ``equal``: values in {0, 1/4, 1/2, 3/4}, so that many
    neighbours are equal and abs'(0) = 0 of the reference must give them no gradient."""
    from boxinstseg_b200.models.losses import length_regularization
    chunks = length_chunks(n, C * h * w)
    assert {'one': chunks == 1, 'cap': chunks == 64, 'some': 1 < chunks < 64}[side], (n, C, h, w, chunks)
    gen = torch.Generator().manual_seed(n + C * 3 + h * 5 + w)
    s = torch.rand(n, C, h, w, generator=gen)
    if equal:
        s = (s * 4).floor() / 4
    gup = upstream(n, gen)
    s64 = s.double().requires_grad_(True)
    ref = ol.length_regularization(s64)
    (gref,) = torch.autograd.grad((ref * gup.double()).sum(), s64)

    def once():
        sg = s.to(DEV).requires_grad_(True)
        out = length_regularization()(sg)
        (gs,) = torch.autograd.grad((out * gup.to(DEV)).sum(), sg)
        return out.detach(), gs
    out, gs = twice(once)
    tag = f'length n={n} C={C} {h}x{w} chunks={chunks}'
    check_close(f'{tag} loss', out, ref.detach(), TOL_LEN_LOSS)
    check_close(f'{tag} d/ds', gs, gref, TOL_LEN_GRAD)
