"""The DiscoBox mask loss on float16 / bfloat16 logits (csrc/discobox_loss.cu: ``db_forward_kernel``,
``db_finalize_kernel``, ``db_total_kernel``, ``db_backward_kernel``; the pseudo-label of ``bxs_meanfield_forward_logits``)
across its envelope, every gradient element judged in units of its own type.

The kernel's contract (discobox_loss.cu, header): s = round_T(sigmoid(x)) as torch computes it, every sum in float32 in a
fixed order, and g_x = round_T(g_s (1 - s) s) rounded once.  So each element of g_x is the float64 value of
tests/discobox_half_oracle.py (computed from the same rounded s) rounded to T, up to the float32 error of g_s:

    |got - ref| <= ulp_T(ref) + ALLOW 2^-24 M,

ulp_T the spacing of T at |ref| (floored at T's smallest subnormal spacing).  One ulp covers the final rounding, also
when the float32 value sits across a binade boundary from ref.  M is the element's term magnitude before cancellation,
restated here in float64: (|g_ins| (m_row + m_col) + |g_ts| enl (|ca| p + |cb| s)) s (1 - s), where m_row / m_col are
|2 l / U| + |4 I r / U^2| of the row / column dice at the row's / column's first arg-max and zero elsewhere, and
ca = -2 / U_ts, cb = 4 I_ts / U_ts^2 are the teacher-student coefficients.  An element no term touches (M = 0) must be
exactly zero, and so must every element of an all-zero target (keep weight 0) and every element whose s is 0 or 1.

The kernel's partitioning is where it can go wrong, so the cases sit on it: strips of 16 rows (the enlarged target band
is seeded per strip from row y0 - 1, column maxima merge across strips), tiles of 256 columns (the 3x3 pool reads
col +- 1 across the tile edge, row maxima and their first arg-max merge across tiles), partial warps (w % 32 != 0,
w < 32, a last tile past w), and targets whose edges lie on rows 15 / 16 / 31 / 32 and columns 255 / 256 / 511 / 512.
Every case runs twice and must repeat bit for bit; the pseudo-label must equal MeanField.forward bit for bit, on the
side of the per-object / grid-wide schedule switch of meanfield.cu that each case asserts.

Bars (largest value observed over all cases on an H100 80GB HBM3, SXM, 132 SMs, 700 W power limit, in the comments).
"""
import functools

import pytest
import torch
import torch.nn.functional as F

from tests.discobox_half_oracle import disco_half_loss
from tests.helpers import tied_logits, ulp_half
from tests.test_discobox_half_gpu import _mean_field, _pseudo_ref

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
DTYPES = [torch.float16, torch.bfloat16]
EPS = 1e-3                      # dice eps of the mask loss
FUSED_SMEM = 200 * 1024         # kMaxFusedSmem of meanfield.cu
U32 = 2.0 ** -24

# element-wise and sum bars, and in the comments the largest value observed over all cases (H100, see above).
# ALLOW: the float32 sums behind g_s run about 16 rows per thread, a 256-thread tree, the parts of an instance and another
# tree deep, and each coefficient divides by one of them and multiplies by another; 64 u of the magnitude covers that.
ALLOW = 64                      # float32 allowance of g_x, in units of 2^-24 M         0 used: every element was within
                                #                          0.54 ulp_T (bf16, n=18 17x769, independent teacher)
TOL_INEXACT = 1e-2              # share of elements != round_T(ref)                     1.7e-3 (fp16, n=18 1x32: 1 of 576)
TOL_NUM_INS = 5e-7              # |num_ins - ref| / sum of its dice terms' magnitudes   4.5e-8 (fp16, config C 32x200x256)
TOL_NUM_TS = 5e-7               # |num_ts - ref| / sum of its dice terms' magnitudes    6.0e-8 (fp16, n=18 33x513)

SEAM_ROWS = (15, 16, 31, 32)
SEAM_COLS = (255, 256, 511, 512)
# target of instance i: KINDS[i % len(KINDS)]; all-zero targets between kept ones
KINDS = ('random', 'zero', 'seam_br0', 'seam_tl0', 'full', 'seam_br1', 'seam_tl1', 'zero', 'corner_tl', 'seam_br2',
         'seam_tl2', 'pixel', 'corner_br', 'seam_br3', 'seam_tl3', 'last_row', 'last_col', 'zero')


@functools.lru_cache(maxsize=None)
def sms():
    from boxinstseg_b200 import _lib as L
    n = L.lib().bxs_device_sm_count()
    assert n > 0
    return n


def mf_per_object(n, h, w):
    """meanfield.cu's schedule for bxs_meanfield_forward_logits with a workspace (the op always passes one): one CTA per
    object iff both bit maps (2 h w bytes, rounded up to 16 each) fit 200 KB of shared memory and n >= 2 * SMs,
    grid-wide rounds otherwise."""
    return 2 * ((h * w + 15) // 16) * 16 <= FUSED_SMEM and n >= 2 * sms()


def seam_targets(n, h, w, gen):
    """uint8 [n,h,w] targets, instance i of kind KINDS[i % len(KINDS)]:
       random       a box with a notch and a hole
       zero         all zero (keep weight 0)
       seam_brK     a box whose last row is SEAM_ROWS[K] and last column SEAM_COLS[K] (clipped to the map)
       seam_tlK     a box whose first row is SEAM_ROWS[K] and first column SEAM_COLS[K] (clipped to the map)
       full         the whole map: touches all four borders
       corner_tl / corner_br   a box touching the top and left / bottom and right borders
       pixel        one pixel
       last_row / last_col     a run of pixels in the last row / column only"""
    t = torch.zeros(n, h, w, dtype=torch.uint8)

    def rnd(lo, hi):                                               # an int in [lo, hi]
        return lo + int(torch.randint(0, max(hi - lo + 1, 1), (1,), generator=gen))
    for i in range(n):
        kind = KINDS[i % len(KINDS)]
        if kind == 'zero':
            continue
        if kind == 'random':
            y0, x0 = rnd(0, (h - 1) // 2), rnd(0, (w - 1) // 2)
            y1, x1 = rnd(y0 + 1, h), rnd(x0 + 1, w)
            t[i, y0:y1, x0:x1] = 1
            if y1 - y0 > 2 and x1 - x0 > 2:
                t[i, y0, x0] = 0
                t[i, (y0 + y1) // 2, (x0 + x1) // 2] = 0
        elif kind.startswith('seam_br'):
            k = int(kind[-1])
            y1, x1 = min(SEAM_ROWS[k] + 1, h), min(SEAM_COLS[k] + 1, w)
            t[i, rnd(max(y1 - 40, 0), y1 - 1):y1, rnd(max(x1 - 300, 0), x1 - 1):x1] = 1
        elif kind.startswith('seam_tl'):
            k = int(kind[-1])
            y0, x0 = min(SEAM_ROWS[k], h - 1), min(SEAM_COLS[k], w - 1)
            t[i, y0:rnd(y0 + 1, min(y0 + 40, h)), x0:rnd(x0 + 1, min(x0 + 300, w))] = 1
        elif kind == 'full':
            t[i] = 1
        elif kind == 'corner_tl':
            t[i, :rnd(1, h), :rnd(1, w)] = 1
        elif kind == 'corner_br':
            t[i, rnd(0, h - 1):, rnd(0, w - 1):] = 1
        elif kind == 'pixel':
            t[i, rnd(0, h - 1), rnd(0, w - 1)] = 1
        elif kind == 'last_row':
            x0 = rnd(0, w - 1)
            t[i, h - 1, x0:rnd(x0 + 1, w)] = 1
        elif kind == 'last_col':
            y0 = rnd(0, h - 1)
            t[i, y0:rnd(y0 + 1, h), w - 1] = 1
    return t


def make_logits(n, h, w, dt, kind, gen):
    """'random': N(0, 9); 'saturated': N(0, 9) with every fourth row at +16 (s rounds to 1 in both types), every third
    pixel of the next rows at -100 (s = 0) and at -16 (s subnormal in float16, tiny in bfloat16); otherwise a kind of
    tests.helpers.tied_logits."""
    if kind == 'random':
        return (torch.randn(n, h, w, generator=gen) * 3).to(dt)
    if kind == 'saturated':
        x = torch.randn(n, h, w, generator=gen) * 3
        x[:, 0::4] = 16.0
        x[:, 1::4, ::3] = -100.0
        x[:, 2::4, 1::3] = -16.0
        return x.to(dt)
    return tied_logits(n, h, w, dt, kind, gen)


def restated_terms(s, tg, pseudo, g_ins, g_ts):
    """float64 (M [n,h,w], arg-max support [n,h,w] bool, magnitude of num_ins, magnitude of num_ts): the gradient's
    term magnitudes before cancellation (see the module docstring) and, for the sums, sum over kept instances of
    1 + 2 I / U per dice."""
    s = s.double()
    t = (tg != 0).double()
    n, h, w = s.shape
    keep = (t.flatten(1).sum(1) > 0).double()
    M = torch.zeros(n, h, w, dtype=torch.float64)
    support = torch.zeros(n, h, w, dtype=torch.float64)
    mag_ins = torch.zeros((), dtype=torch.float64)
    for dim in (2, 1):                                             # rows (max over columns), columns (max over rows)
        a = torch.argmax(s, dim=dim, keepdim=True)                 # first index of the maximum
        r = s.gather(dim, a)
        lab = t.amax(dim, keepdim=True)
        inter = (r * lab).sum((1, 2), keepdim=True)
        u = ((r * r).sum((1, 2), keepdim=True) + EPS) + ((lab * lab).sum((1, 2), keepdim=True) + EPS)
        M.scatter_add_(dim, a, abs(g_ins) * (2 * lab / u + 4 * inter * r / (u * u)))
        support.scatter_(dim, a, 1.0)
        mag_ins = mag_ins + ((1 + 2 * inter / u).flatten() * keep).sum()
    mag_ts = torch.zeros((), dtype=torch.float64)
    if pseudo is not None:
        enl = F.max_pool2d(t.unsqueeze(1), 3, 1, 1).squeeze(1)
        p = pseudo.double()
        xts = s * enl
        inter = (xts * p).sum((1, 2), keepdim=True)
        u = ((xts * xts).sum((1, 2), keepdim=True) + EPS) + ((p * p).sum((1, 2), keepdim=True) + EPS)
        M += abs(g_ts) * enl * (2 / u * p + 4 * inter / (u * u) * s)
        mag_ts = ((1 + 2 * inter / u).flatten() * keep).sum()
    kv = keep.view(n, 1, 1)
    return M * kv * s * (1 - s), (support * kv) > 0, mag_ins, mag_ts


def run_case(dt, n, h, w, logits='random', teacher='shared', g_up=(0.7, 1.3), seed=0):
    """One case: the op twice (bit-identical), the pseudo-label against MeanField.forward, the sums and every gradient
    element against the float64 oracle.  teacher: 'none' (no teacher-student term), 'shared' (the student is its own
    teacher) or 'independent' (separate teacher logits).  Returns the side of the mean-field schedule, or None."""
    from boxinstseg_b200.ops.discobox import _pseudo_label, discobox_mask_loss
    gen = torch.Generator().manual_seed(seed or n * 7919 + h * 131 + w * 7 + (dt == torch.bfloat16))
    x = make_logits(n, h, w, dt, logits, gen)
    xt = (torch.randn(n, h, w, generator=gen) * 3).to(dt) if teacher == 'independent' else None
    tg = seam_targets(n, h, w, gen)
    ii = (torch.arange(n) % 2).to(torch.int32)
    use_ts = teacher != 'none'
    mf = _mean_field(2, h, w, seed=h + w) if use_ts else None
    xd, tgd, iid = x.to(DEV), tg.to(DEV), ii.to(DEV)
    xtd = None if xt is None else xt.to(DEV)

    def once():
        leaf = xd.detach().requires_grad_(True)                   # a fresh leaf per call
        ni, nt, cnt = discobox_mask_loss(leaf, tgd, iid, mf, xtd, use_ts)
        (g,) = torch.autograd.grad(g_up[0] * ni + g_up[1] * nt, leaf)
        return torch.stack((ni, nt, cnt)).detach(), g
    first, second = once(), once()
    assert torch.equal(first[0], second[0]) and torch.equal(first[1], second[1]), 'not deterministic'
    sums, g = second[0].cpu().double(), second[1].cpu()
    assert g.dtype == dt and g.shape == x.shape

    side, pseudo = None, None
    if use_ts:
        side = 'per-object' if mf_per_object(n, h, w) else 'grid'
        pseudo = _pseudo_ref(x, xt, tg, ii, mf)
        assert torch.equal(_pseudo_label(mf, xd, xtd, tgd, iid), pseudo), 'pseudo-label differs from MeanField.forward'
        pseudo = pseudo.cpu()
    s = torch.sigmoid(xd).cpu()
    o_ins, o_ts, o_cnt, ref = disco_half_loss(s, tg, pseudo, *g_up)
    M, support, mag_ins, mag_ts = restated_terms(s, tg, pseudo, *g_up)

    tag = f'{dt} n={n} {h}x{w} logits={logits} teacher={teacher} g={g_up}'
    assert float(sums[2]) == float(o_cnt), (tag, 'count', float(sums[2]), float(o_cnt))
    e_ins = abs(float(sums[0]) - float(o_ins)) / max(float(mag_ins), 1e-30)
    e_ts = abs(float(sums[1]) - float(o_ts)) / max(float(mag_ts), 1e-30)
    if not use_ts:
        assert float(sums[1]) == 0.0, tag

    got = g.double()
    ulp = ulp_half(ref, dt)
    diff = (got - ref).abs()
    err = diff / ulp
    excess = ((diff - ulp).clamp(min=0) / (U32 * M)).nan_to_num(nan=0.0, posinf=float('inf'))
    inexact = float((g != ref.to(dt)).double().mean())
    kappa = float(excess.max()) if excess.numel() else 0.0
    print(f'[half-envelope] {tag} side={side}: max err {float(err.max()):.2f} ulp, allowance used {kappa:.1f} '
          f'(bar {ALLOW}), not round_T(ref) {inexact:.2e}, num_ins {e_ins:.1e}, num_ts {e_ts:.1e}')
    assert e_ins <= TOL_NUM_INS, (tag, 'num_ins', e_ins)
    assert e_ts <= TOL_NUM_TS, (tag, 'num_ts', e_ts)
    assert inexact <= TOL_INEXACT, (tag, 'share not round_T(ref)', inexact)
    bad = err > 1 + ALLOW * U32 * M / ulp
    assert not bad.any(), (tag, 'elements off', int(bad.sum()), bad.nonzero()[:5].tolist(),
                           got[bad][:5].tolist(), ref[bad][:5].tolist())
    zero = (M == 0) | (s.double() == 0) | (s.double() == 1)
    assert not (got[zero] != 0).any(), (tag, 'nonzero where no term reaches', int((got[zero] != 0).sum()))
    if g_up[1] == 0 or not use_ts:
        # MIL term alone: the support is exactly the first-arg-max positions whose value does not round to zero
        assert torch.equal(g != 0, support & (ref.to(dt) != 0)), tag
    return side


# ------------------------------------------------------------------ map sizes
H_SWEEP = [(h, w) for w in (31, 257) for h in (1, 15, 16, 17, 33, 200, 257)]
W_SWEEP = [(h, w) for h in (1, 17, 33) for w in (1, 31, 32, 255, 256, 257, 512, 513, 769) if (h, w) not in H_SWEEP]
MAPS = H_SWEEP + W_SWEEP


@pytest.mark.parametrize('dt', DTYPES, ids=['fp16', 'bf16'])
@pytest.mark.parametrize('h,w', MAPS)
def test_map_sizes(h, w, dt):
    """18 instances (every target kind of KINDS, three all-zero) per map; both teacher forms, alternating over the maps,
    with upstream gradients (0.7, 1.3)."""
    teacher = 'shared' if MAPS.index((h, w)) % 2 == 0 else 'independent'
    run_case(dt, len(KINDS), h, w, teacher=teacher)


# ------------------------------------------------------------------ every term configuration
@pytest.mark.parametrize('dt', DTYPES, ids=['fp16', 'bf16'])
@pytest.mark.parametrize('teacher', ['none', 'shared', 'independent'])
@pytest.mark.parametrize('g_up', [(1.0, 1.0), (0.7, 1.3), (1.0, 0.0), (0.0, 1.0)], ids=str)
def test_term_configurations(g_up, teacher, dt):
    """40 x 300: three strips, two tiles, a partial last tile; at (1, 0) and without the teacher term the support must be
    exactly the first arg-max positions."""
    run_case(dt, len(KINDS), 40, 300, teacher=teacher, g_up=g_up)


# ------------------------------------------------------------------ instance counts and the mean-field schedules
@pytest.mark.parametrize('dt', DTYPES, ids=['fp16', 'bf16'])
@pytest.mark.parametrize('n,h,w,teacher,side', [
    (1, 48, 300, 'shared', 'grid'), (2, 48, 300, 'independent', 'grid'), (33, 48, 300, 'shared', 'grid'),
    (32, 200, 256, 'shared', 'grid'),                                      # config C's level
    (512, 64, 80, 'shared', 'per-object'), (512, 64, 80, 'independent', 'per-object'),
])
def test_instance_counts(n, h, w, teacher, side, dt):
    """One instance up to 512: a 1-D grid of n * strips * tiles CTAs, one finalize CTA per instance, and db_total_kernel
    reducing 512 instance records over its 256 threads.  512 objects fill the SMs twice, so their pseudo-label runs one
    CTA per object; the others run grid-wide rounds."""
    assert run_case(dt, n, h, w, teacher=teacher) == side


# ------------------------------------------------------------------ logits that stress the arithmetic
@pytest.mark.parametrize('dt', DTYPES, ids=['fp16', 'bf16'])
@pytest.mark.parametrize('logits', ['saturated', 'quantised', 'constant', 'boundaries'])
def test_stress_logits(logits, dt):
    """70 x 530 (five strips, three tiles): saturated scores whose gradient is exactly 0, and maps of many tied s with
    ties planted on both sides of every strip and tile boundary (the first arg-max must win)."""
    run_case(dt, len(KINDS), 70, 530, logits=logits, teacher='shared', g_up=(1.0, 1.0))
    run_case(dt, len(KINDS), 70, 530, logits=logits, teacher='none', g_up=(1.0, 0.0))
