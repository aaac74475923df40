"""The heads' classification and box-regression losses across their envelopes, every output judged element-wise against a
float64 reference in units of the rounding each element can carry.

  * sigmoid focal loss (focal_loss.cu, ``focal_levels_kernel``): a CTA owns FL_TILE = 64 cells of one (level, image) and
    walks the class planes FL_GROUPS = 4 at a time; at most 8 levels.  Both entry points: the cells form through
    ``ops.focal.sigmoid_focal_loss_levels`` and the square-grid form ``bxs_sigmoid_focal_loss_levels_forward``, which
    must agree bit for bit.  Neither branch of ``focal_element`` cancels (``q - g p log p`` and ``g q log(1-p) - p`` add
    terms of one sign), so each element is judged relative to itself:
        |g - ref| <= k 2^-24 (1 + (1 + gamma) |x|) |ref| + 2^-126 |scale|,
    with (1 + (1 + gamma) |x|) the conditioning of p = exp(log_sigmoid(x)) and of its power (an error of ulp(x) in the
    exponent is a relative error of |x| 2^-24 in p), and 2^-126 |scale| the float32 underflow of terms below the normal
    range (logits of +-88 and +-104).  The loss is judged against the sum of its terms' magnitudes, weighted the same way.
  * softmax cross-entropy over decoder layers (cross_entropy.cu, ``ce_layers_kernel``, ``ce_scale_kernel``): CE_ROWS = 32
    query rows per CTA, one warp per row striding K; at most 16 layers.  With m the row maximum, d_k = x_k - m,
    s = sum_k exp(d_k) and p_k the softmax, each gradient element is judged in units of its terms before the p_y - 1
    cancellation,
        |g - ref| <= k 2^-24 w_y scale |g_up| ((1 + |log p_k| + ceil(K / 32)) p_k + [k == y]),
    |log p_k| being the float32 conditioning of exp(d_k - log s) and ceil(K / 32) that of s, which each lane sums over
    its ceil(K / 32) logits.  Each layer's loss is judged against sum_rows w_y scale (1 + log s + |d_y|): s >= 1 is
    summed in float32, so log s carries an absolute error of order 2^-24 however small it is.  The row offsets reach
    |m| = 1000, where a loss or softmax formed through lse = m + log s is rounded to ulp(m).  Rows whose weight or
    upstream gradient is 0 must have an exactly zero gradient.
  * FCOS GIoU and centerness losses (fcos_loss.cu, ``fcos_loss_kernel``, ``fcos_scale_kernel``): FC_NT = 256 points per
    CTA; at most 8 levels.  Every positive's d / d bbox_pred equals, bit for bit, the host build of the kernel's own
    per-point arithmetic (tests/host_harness/fcos_loss_host.cpp) times the same float32 scale; d / d centerness =
    sigmoid(x) - ct differs from it only by expf of the device against that of the host library, judged in units of
    2^-24 (sigmoid(x) + ct) scale; every other point is exactly zero.  Against the float64 oracle the elements carry
    the float32 decoding of the boxes around the points (scaled_err of tests/helpers.py); points where that decoding
    makes a tie of the two boxes that float64 does not, and boxes of 1e-4 around points in the hundreds, are left to
    the host twin.

The SM-derived grids of ``ce_scale_kernel`` and ``fcos_scale_kernel`` are restated here and every case asserts the side
it lands on; the SM count is read from the library.  Every case runs twice and must repeat bit for bit.

Bars: the largest value observed over all cases on an H100 80GB HBM3 (SXM, 132 SMs, 700 W power limit) is given next
to each bar.
"""
import ctypes
import functools

import pytest
import torch
import torch.nn.functional as F

from oracle import fcos_loss as ofl
from tests.helpers import host_twin, scaled_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
U = 2.0 ** -24
TINY = 2.0 ** -126
FLT_EPS = float(torch.finfo(torch.float32).eps)

# bars and, in the comments, the largest value observed over all cases (H100, see above)
TOL_FL_GRAD = 32.0         # focal d / dx, units of 2^-24 (1 + (1 + gamma)|x|) |ref|     11.3 (C=7, gamma=4, g=-2.5)
TOL_FL_LOSS = 0.04         # focal loss, units of 2^-24 sum (1 + (1 + gamma)|x|) |terms|  1.3e-2 (C=7, gamma=1.5, alpha=1)
TOL_CE_GRAD = 6.0          # cross-entropy d / dx, units as above                       2.4 (L=16, B*Q=800, K=1000)
TOL_CE_LOSS = 4.0          # cross-entropy loss per layer, units as above               1.6 (L=2, B*Q=65, K=134)
TOL_FC_CTR = 12.0          # FCOS d / d centerness against the host twin, units above   4.6 (B=3, 100x128 + 2 levels)
TOL_FC_BBOX64 = 6e-4       # FCOS d / d bbox_pred against float64, scaled_err          2.1e-4 (B=3, 100x128 + 2 levels)
TOL_FC_CTR64 = 2e-5        # FCOS d / d centerness against float64, scaled_err         7.3e-6 (B=3, 100x128 + 2, C=1)
TOL_FC_LOSS = 2e-6         # FCOS losses against float64, relative to the sum of |terms| 5.5e-7 (B=1, 1x1)


@functools.lru_cache(maxsize=None)
def sms():
    from boxinstseg_b200 import _lib as L
    n = L.lib().bxs_device_sm_count()
    assert n > 0
    return n


def twice(fn):
    """fn() run twice; the two results must be bit-identical."""
    first, second = fn(), fn()
    assert len(first) == len(second)
    for a, b in zip(first, second):
        assert a.shape == b.shape and torch.equal(a, b)
    return second


def ratio(name, got, ref, unit, tol, case):
    """max |got - ref| / unit over the elements; where unit is 0 the result must be exactly 0."""
    got = got.detach().double().cpu().reshape(-1)
    ref, unit = ref.detach().double().cpu().reshape(-1), unit.detach().double().cpu().reshape(-1)
    d = (got - ref).abs()
    live = unit > 0
    assert not (got[~live] != 0).any(), (name, case, 'a nonzero value where the reference is exactly 0')
    err = (d[live] / unit[live]).max().item() if live.any() else 0.0
    print(f'[envelope] {name}: {err:.3e} (bar {tol:g}) {case}')
    assert err <= tol, (name, case, err)
    return err


# ================================================================== sigmoid focal loss
FL_TILE = 64
LOGIT_VALUES = [0.0, 2.0, -2.0, 15.0, -15.0, 30.0, -30.0, 88.0, -88.0, 104.0, -104.0, 1e4, -1e4]


def focal_inputs(levels, B, C, seed):
    """Per level float32 logits [B,C,H,W] and int64 labels [B,H*W].  A third of the logits come from LOGIT_VALUES, the
    rest are N(0, 3).  Labels mix the background C with -1, C + 1, 2^40 (all negative), 0, C - 1 and other classes;
    the first and the last cell of every 64-cell tile are positives.  With B > 1 the last image is all background; with
    more than one level the last level is all positive."""
    gen = torch.Generator().manual_seed(seed)
    xs, labs = [], []
    vals = torch.tensor(LOGIT_VALUES)
    for li, (h, w) in enumerate(levels):
        n = h * w
        x = torch.randn(B, C, h, w, generator=gen) * 3
        pick = torch.rand(B, C, h, w, generator=gen) < 0.35
        x = torch.where(pick, vals[torch.randint(len(LOGIT_VALUES), (B, C, h, w), generator=gen)], x)
        kinds = torch.tensor([-1, C, C + 1, 2 ** 40, 0, C - 1, C, C])
        lab = kinds[torch.randint(len(kinds), (B, n), generator=gen)]
        rnd = torch.randint(0, C, (B, n), generator=gen)
        lab = torch.where(torch.rand(B, n, generator=gen) < 0.15, rnd, lab)
        for c0 in range(0, n, FL_TILE):
            lab[:, c0] = (c0 // FL_TILE) % C
            lab[:, min(c0 + FL_TILE - 1, n - 1)] = C - 1 - (c0 // FL_TILE) % C
        if len(levels) > 1 and li == len(levels) - 1:
            lab = rnd
        if B > 1:
            lab[-1] = kinds[torch.randint(4, (n,), generator=gen)]
        xs.append(x)
        labs.append(lab)
    return xs, labs


def focal_ref(x, lab, gamma, alpha):
    """float64 (loss, d loss / dx) of every element of one level in the stable form: log p and log(1 - p) from
    log_sigmoid, so that (1 - p)^gamma stays accurate where it underflows in 1 - sigmoid(x)."""
    B, C = x.shape[:2]
    x = x.double()
    pos = lab.view(B, 1, *x.shape[2:]) == torch.arange(C).view(1, C, 1, 1)
    lp, lm = F.logsigmoid(x), F.logsigmoid(-x)
    p, q = lp.exp(), lm.exp()
    wp, wn = alpha * q.pow(gamma), (1 - alpha) * p.pow(gamma)
    loss = torch.where(pos, -wp * lp, -wn * lm)
    dx = torch.where(pos, -wp * (q - gamma * p * lp), -wn * (gamma * q * lm - p))
    return loss, dx


def focal_grid(xs, labs, avg_t, gamma, alpha, lw):
    """The square-grid entry point through ctypes: (loss, per-level d loss / dx)."""
    from boxinstseg_b200 import _lib as L
    n, B, C = len(xs), xs[0].shape[0], xs[0].shape[1]
    grid = (ctypes.c_int64 * n)(*[x.shape[2] for x in xs])
    ptrs = lambda ts: (ctypes.c_void_p * n)(*[t.data_ptr() for t in ts])    # noqa: E731
    grads = [torch.empty_like(x) for x in xs]
    loss = torch.empty((), device=DEV)
    lib = L.lib()
    ws = torch.empty(lib.bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(grid, n, B), dtype=torch.uint8, device=DEV)
    L.check(lib.bxs_sigmoid_focal_loss_levels_forward(ptrs(xs), ptrs(labs), grid, ptrs(grads), L.ptr(avg_t), L.ptr(loss),
                                                      L.ptr(ws), n, B, C, gamma, alpha, lw, L.stream()),
            'sigmoid_focal_loss_levels_forward')
    return loss, grads


def check_focal(levels, B, C, gamma=2.0, alpha=0.25, avg=9.0, avg_tensor=False, lw=1.5, gup=1.0, seed=0):
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    xs, labs = focal_inputs(levels, B, C, seed or B * 1000 + C * 10 + len(levels))
    scale = lw / (float(torch.tensor(avg, dtype=torch.float32)) + FLT_EPS)
    refs = [focal_ref(x, l, gamma, alpha) for x, l in zip(xs, labs)]
    square = all(h == w for h, w in levels)

    def once():
        xg = [x.to(DEV).requires_grad_(True) for x in xs]
        dl = [l.to(DEV) for l in labs]
        avg_arg = torch.tensor(avg, device=DEV) if avg_tensor else avg
        loss = sigmoid_focal_loss_levels(xg, dl, avg_arg, gamma, alpha, lw)
        gs = torch.autograd.grad(loss, xg, grad_outputs=torch.tensor(gup, device=DEV))
        fwd = sigmoid_focal_loss_levels([x.detach() for x in xg], dl, avg_arg, gamma, alpha, lw)   # no gradient written
        out = [loss.detach(), fwd] + list(gs)
        if square:
            g_loss, g_grads = focal_grid([x.detach() for x in xg], dl, torch.tensor(float(avg), device=DEV), gamma, alpha,
                                         lw)
            out += [g_loss] + g_grads
        return out
    got = twice(once)
    n = len(levels)
    loss, fwd, grads = got[0], got[1], got[2:2 + n]
    case = f'levels={levels} B={B} C={C} gamma={gamma} alpha={alpha} avg={avg}{"(t)" if avg_tensor else ""} lw={lw} g={gup}'
    assert torch.equal(fwd, loss), case                        # the forward alone computes the same loss
    if square:                                                 # the square-grid form is the same kernel
        assert torch.equal(got[2 + n], loss), case
        for a, b in zip(got[3 + n:], grads):
            assert torch.equal(a * gup, b), case
    cond = [1 + (1 + gamma) * x.double().abs() for x in xs]
    g_ref = torch.cat([(dx * scale * gup).reshape(-1) for _, dx in refs])
    g_unit = torch.cat([(k * U * (dx * scale * gup).abs() + TINY * abs(scale * gup)).reshape(-1)
                        for k, (_, dx) in zip(cond, refs)])
    ratio('focal d/dx', torch.cat([g.reshape(-1) for g in grads]), g_ref, g_unit, TOL_FL_GRAD, case)
    l_ref = scale * sum(float(t.sum()) for t, _ in refs)
    l_unit = abs(scale) * (U * sum(float((k * t.abs()).sum()) for k, (t, _) in zip(cond, refs))
                           + TINY * sum(t.numel() for t, _ in refs))
    ratio('focal loss', loss.reshape(1), torch.tensor([l_ref], dtype=torch.float64),
          torch.tensor([l_unit], dtype=torch.float64), TOL_FL_LOSS, case)


TILE_LEVELS = [(1, 1), (7, 9), (8, 8), (5, 13), (127, 1), (1, 128), (3, 43), (17, 241)]    # 1 .. 4097 cells


@pytest.mark.parametrize('levels', [TILE_LEVELS, [(1, 1)], [(1, 64)], [(65, 1)], [(64, 64)], [(1, 1), (12, 12)],
                                    [(40, 40), (36, 36), (24, 24), (16, 16), (12, 12), (8, 8), (5, 5), (1, 1)]])
@pytest.mark.parametrize('B', [1, 2, 17])
def test_focal_tiles_and_levels(levels, B):
    """Cells per level on both sides of every multiple of the 64-cell tile, 1xW and Hx1 levels, 1 and 8 levels; the
    all-square sets also run the square-grid entry point."""
    check_focal(levels, B, 80 if B < 17 else 9)


@pytest.mark.parametrize('C', [1, 2, 3, 4, 5, 7, 8, 9, 80])
def test_focal_classes(C):
    """Class planes on both sides of FL_GROUPS = 4 in flight, and of the planes a group's last pass holds."""
    check_focal([(9, 9), (1, 70), (4, 4)], (1, 2, 17)[C % 3], C, gup=(1.0, 0.0, -2.5)[C % 3])
    check_focal([(9, 9), (3, 3)], 2, C, gup=-2.5)


@pytest.mark.parametrize('gamma', [0.0, 0.5, 1.0, 1.5, 2.0, 4.0])
@pytest.mark.parametrize('alpha', [0.0, 0.25, 1.0])
def test_focal_parameters(gamma, alpha):
    """Integer and non-integer powers (powf), and alpha at both ends (one branch weighted 0)."""
    check_focal([(8, 8), (1, 65)], 2, 7, gamma=gamma, alpha=alpha, gup=-2.5 if gamma > 1 else 1.0)


@pytest.mark.parametrize('avg', [0.0, 0.5, 1.0, 1e6])
@pytest.mark.parametrize('avg_tensor', [False, True])
def test_focal_scaling(avg, avg_tensor):
    """avg_factor as a number and as a device tensor, down to 0 (the loss divides by FLT_EPSILON), with loss_weight 0.3."""
    check_focal([(13, 13), (2, 50)], 2, 80, avg=avg, avg_tensor=avg_tensor, lw=0.3, gup=(1.0, 0.0, -2.5)[int(avg) % 3])


def test_focal_rejects_nine_levels():
    from boxinstseg_b200 import _lib as L
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    xs = [torch.zeros(1, 3, 2, 2, device=DEV) for _ in range(9)]
    labs = [torch.zeros(1, 4, dtype=torch.int64, device=DEV) for _ in range(9)]
    with pytest.raises(L.BoxSegError, match='unsupported'):
        sigmoid_focal_loss_levels(xs, labs, 1.0)


# ================================================================== softmax cross-entropy over layers
CE_ROWS = 32
CE_WARP = 32
CE_BWD_NT = 256
MARGINS = (2.0, 6.0, 10.0, 20.0)
UPSTREAM = (1.0, 0.0, 0.5, -3.0)


def ce_per_layer(L, N, K):
    """bxs_softmax_cross_entropy_layers_backward: CTAs of ce_scale_kernel per layer."""
    return min(-(-(N * K) // CE_BWD_NT), max(1, 4 * sms() // L))


def ce_inputs(L, N, K, shift, seed, weights):
    """([L] float32 [N,K] scores, int64 labels [L,N], class weights [K] or None).  Row r: its top entry sits at the label
    (at a random class for an out-of-range label, at another class on every seventh row) MARGINS[r % 4] above the other
    entries, which spread over 8 more; every sixth row has tied maxima and every eleventh is constant; each row is
    offset by shift + U(0, 1).  Labels: K - 1 (no object) mostly, other classes, -1, K and 10^6; with L > 1 the last
    layer's labels are all out of range (avg_factor 0)."""
    gen = torch.Generator().manual_seed(seed)
    xs, ys = [], []
    r = torch.arange(N)
    for layer in range(L):
        y = torch.full((N,), K - 1, dtype=torch.int64)
        u = torch.rand(N, generator=gen)
        y = torch.where(u < 0.25, torch.randint(0, K, (N,), generator=gen), y)
        bad = torch.tensor([-1, K, 10 ** 6])[torch.randint(3, (N,), generator=gen)]
        y = torch.where(u > 0.9, bad, y)
        if L > 1 and layer == L - 1:
            y = bad
        top = torch.where((y >= 0) & (y < K), y, torch.randint(0, K, (N,), generator=gen))
        top = torch.where((r % 7 == 3) & (K > 1), (top + 1 + torch.randint(0, max(K - 1, 1), (N,), generator=gen)) % K, top)
        margin = torch.tensor(MARGINS)[r % 4].view(N, 1)
        x = -(torch.rand(N, K, generator=gen) * 8 + margin).double()
        x[r, top] = 0.0
        tie = (r % 6 == 5) & (K > 1)
        x[r[tie], ((top + 1) % K)[tie]] = 0.0
        x[r % 11 == 10] = 0.0
        xs.append((x + shift + torch.rand(N, 1, generator=gen).double()).float())
        ys.append(y)
    cw = None
    if weights:
        cw = torch.rand(K, generator=gen) + 0.5
        cw[::5] = 0.0
        cw[-1] = 0.1
    return xs, torch.stack(ys), cw


def ce_reference(x, y, cw, lw):
    """float64 (loss, d loss / dx, gradient unit, loss unit) of one layer: F.cross_entropy(weight=w, reduction='none')
    plus weight_reduce_loss(avg_factor=w[y].sum()), labels outside [0, K) dropped; the units are those of the module
    docstring for an upstream gradient of 1."""
    x = x.double()
    N, K = x.shape
    w = torch.ones(K, dtype=torch.float64) if cw is None else cw.double()
    keep = (y >= 0) & (y < K)
    yk = y.clamp(0, K - 1)
    wr = torch.where(keep, w[yk], torch.zeros(N, dtype=torch.float64))
    scale = lw / (float(torch.tensor(float(wr.sum()), dtype=torch.float32)) + FLT_EPS)
    rows = torch.zeros(N, dtype=torch.float64)
    rows[keep] = F.cross_entropy(x[keep], y[keep], weight=w, reduction='none')
    logp = torch.log_softmax(x, 1)
    p = logp.exp()
    onehot = F.one_hot(yk, K).double()
    g = (wr * scale).view(N, 1) * (p - onehot)
    g_unit = U * (wr * scale).view(N, 1) * ((1 + logp.abs() + -(-K // CE_WARP)) * p + onehot)
    d = x - x.max(1, keepdim=True).values
    ls = d.exp().sum(1).log()
    l_unit = U * scale * float((wr * (1 + ls + d.gather(1, yk.view(N, 1)).view(N).abs())).sum())
    return scale * float(rows.sum()), g, g_unit, l_unit


def check_ce(L, B, Q, K, shift=0.0, weights=True, lw=2.0, seed=0, side=None):
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    N = B * Q
    if side is not None:
        per = ce_per_layer(L, N, K)
        assert (per == 1) == (side == 'one'), (L, N, K, per)
    xs, ys, cw = ce_inputs(L, N, K, shift, seed or L * 7 + N * 13 + K + int(abs(shift)) * 3 + (shift < 0), weights)
    gup = torch.tensor([UPSTREAM[i % 4] for i in range(L)])
    refs = [ce_reference(x, y, cw, lw) for x, y in zip(xs, ys)]

    def once():
        xg = [x.view(B, Q, K).to(DEV).requires_grad_(True) for x in xs]
        loss = softmax_cross_entropy_layers(xg, ys.view(L, B, Q).to(DEV), None if cw is None else cw.to(DEV), lw)
        return [loss.detach()] + list(torch.autograd.grad(loss, xg, grad_outputs=gup.to(DEV)))
    got = twice(once)
    case = f'L={L} B*Q={N} K={K} shift={shift} cw={"w" if weights else None}'
    for i, (loss_ref, g, g_unit, l_unit) in enumerate(refs):
        gi = float(gup[i])
        ratio(f'ce d/dx layer {i} (g={gi})', got[1 + i], g * gi, g_unit * abs(gi), TOL_CE_GRAD, case)
        ratio(f'ce loss layer {i}', got[0][i:i + 1], torch.tensor([loss_ref], dtype=torch.float64),
              torch.tensor([l_unit], dtype=torch.float64), TOL_CE_LOSS, case)
    return xs, ys, cw


@pytest.mark.parametrize('K', [1, 2, 31, 32, 33, 64, 65, 81, 134, 1000])
def test_ce_classes(K):
    """K on both sides of the warp width a row is strided over."""
    check_ce(2, 1, 65, K, weights=K % 2 == 1, side='one' if 65 * K <= CE_BWD_NT else 'many')


@pytest.mark.parametrize('B,Q', [(1, 1), (1, 31), (1, 32), (1, 33), (3, 21), (2, 32), (5, 13), (1, 100), (8, 100)])
def test_ce_rows(B, Q):
    """B*Q on both sides of CE_ROWS = 32 rows per CTA; a single row leaves one scale CTA per layer."""
    check_ce(4, B, Q, 81, weights=Q % 2 == 0, side='one' if B * Q == 1 else 'many')


@pytest.mark.parametrize('L', [1, 2, 10, 16])
def test_ce_layers(L):
    check_ce(L, 2, 50, 134, side='many')


@pytest.mark.parametrize('shift', [0.0, 16.0, -16.0, 64.0, -64.0, 1000.0, -1000.0])
def test_ce_row_offsets(shift):
    """Rows far from zero: a loss or softmax formed through m + log s would round to ulp(m)."""
    check_ce(3, 8, 100, 81, shift=shift)
    check_ce(2, 1, 40, 1000, shift=shift, weights=False)


def test_ce_large_scale_grid():
    """Every layer's gradient larger than the scale grid: ce_scale_kernel strides it several times."""
    L, B, Q, K = 16, 8, 100, 1000
    per = ce_per_layer(L, B * Q, K)
    assert per * CE_BWD_NT * 2 < B * Q * K, per
    check_ce(L, B, Q, K, side='many')


def test_ce_rejects_seventeen_layers():
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    xs = [torch.zeros(1, 2, 3, device=DEV) for _ in range(17)]
    with pytest.raises(ValueError, match='at most 16'):
        softmax_cross_entropy_layers(xs, torch.zeros(17, 1, 2, dtype=torch.int64, device=DEV))


def test_ce_second_backward():
    """retain_graph: a second backward recomputes the spent in-place gradients and scales them by its own upstream."""
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    L, B, Q, K = 3, 2, 40, 81
    xs, ys, cw = ce_inputs(L, B * Q, K, 16.0, 5, True)
    xg = [x.view(B, Q, K).to(DEV).requires_grad_(True) for x in xs]
    loss = softmax_cross_entropy_layers(xg, ys.view(L, B, Q).to(DEV), cw.to(DEV), 2.0)
    g1 = torch.autograd.grad(loss, xg, grad_outputs=torch.tensor([1.0, 0.5, -3.0], device=DEV), retain_graph=True)
    g2 = torch.autograd.grad(loss, xg, grad_outputs=torch.tensor([1.0, 1.0, 1.0], device=DEV))
    assert torch.equal(g1[0], g2[0])
    for a, b, s in zip(g1[1:], g2[1:], (0.5, -3.0)):
        assert torch.equal(a, b * s)
    for i, (x, y) in enumerate(zip(xs, ys)):
        _, g, g_unit, _ = ce_reference(x, y, cw, 2.0)
        ratio(f'ce d/dx second backward layer {i}', g2[i], g, g_unit, TOL_CE_GRAD, 'retain_graph')


# ================================================================== FCOS GIoU and centerness losses
FC_NT = 256
FC_BWD_NT = 256
STRIDES = (8.0, 16.0, 32.0, 64.0, 128.0, 4.0, 2.0, 1.0)
N_KINDS = 12
TINY_KIND = 7


def fc_scale_ctas(n):
    """bxs_fcos_loss_backward: CTAs of fcos_scale_kernel for the larger of the two gradients."""
    return min(-(-n // FC_BWD_NT), 4 * sms())


def planted(kind, gen):
    """(target l, t, r, b, prediction l, t, r, b) of a positive of GIoU kind ``kind``:
       0 generic, 1 the prediction is its target (ties on every side of dmax_first / dmin_first),
       2-5 one shared side (a tie in one coordinate), 6 a zero-width prediction, 7 a zero-size prediction and a target
       of area 4e-8 (union and enclosing area below eps), 8 an inverted prediction (the clamp0 branches), 9 a tiny
       centerness target (l / r = 1e-16), 10 the prediction touching the target's left edge (an overlap width of
       exactly 0), 11 a prediction enclosing the target."""
    t = torch.rand(4, generator=gen) * 40 + 0.5
    d = t * (torch.rand(4, generator=gen) + 0.5)
    if kind == 1:
        d = t.clone()
    elif 2 <= kind <= 5:
        d[kind - 2] = t[kind - 2]
    elif kind == 6:
        d[2] = -d[0]
    elif kind == TINY_KIND:
        t = torch.full((4,), 1e-4)
        d = torch.tensor([0.0, 0.0, -0.0, 0.0])
    elif kind == 8:
        d[0], d[2] = -d[0] - 1.0, d[0] * 0.25
    elif kind == 9:
        t[0] = t[2] * 1e-16
    elif kind == 10:
        d[2] = -t[0]
    elif kind == 11:
        d = t * 2
    return t, d


def fcos_inputs(levels, B, C, seed, tiny_only=False):
    """Per level: bbox_pred [B,4,H,W], centerness [B,1,H,W], labels [B*H*W], targets [B*H*W,4], and the planted kind of
    every positive (-1 elsewhere).  Positives: the first and last point of every level, of every image of a level and of
    every 256-point CTA, and a random 30 % of the rest; negatives carry C, -1 or C + 7 and random targets."""
    gen = torch.Generator().manual_seed(seed)
    total = sum(B * h * w for h, w in levels)
    g = torch.arange(total)
    pos = torch.rand(total, generator=gen) < 0.3
    pos[(g % FC_NT == 0) | (g % FC_NT == FC_NT - 1) | (g == total - 1)] = True
    first = 0
    out = []
    n_kind = 0
    for h, w in levels:
        P = h * w
        n = B * P
        p_l = pos[first:first + n].clone()
        p_l[0] = p_l[n - 1] = True
        p_l[::P] = True
        p_l[P - 1::P] = True
        first += n
        bbox = torch.randn(B, 4, h, w, generator=gen).abs() * 10
        ctr = torch.randn(B, 1, h, w, generator=gen) * 2
        pick = torch.rand(B, 1, h, w, generator=gen) < 0.3
        ctr = torch.where(pick, torch.tensor([0.0, 30.0, -30.0, 100.0, -100.0])[torch.randint(5, (B, 1, h, w),
                                                                                               generator=gen)], ctr)
        lab = torch.tensor([C, -1, C + 7])[torch.randint(3, (n,), generator=gen)]
        tgt = torch.rand(n, 4, generator=gen) * 20 + 0.5
        kinds = torch.full((n,), -1, dtype=torch.int64)
        for i in p_l.nonzero().reshape(-1).tolist():
            kind = 9 if tiny_only else n_kind % N_KINDS
            n_kind += 1
            t, d = planted(kind, gen)
            b, q = divmod(i, P)
            tgt[i] = t
            bbox[b, :, q // w, q % w] = d
            lab[i] = int(torch.randint(C, (1,), generator=gen))
            kinds[i] = kind
        out.append((bbox, ctr, lab, tgt, kinds))
    return out


def fcos_host(levels, B, inputs):
    """The host twin on every positive, in level / image / point order: (kind, level, flat index into the level's
    [B,H,W], ct, bbox, bce, g_pred [n,4], g_ctr, point xy, pred, target, ctr logit)."""
    lib = host_twin('fcos_loss_host')
    rows = []
    for li, ((h, w), (bbox, ctr, lab, tgt, kinds)) in enumerate(zip(levels, inputs)):
        idx = kinds.ge(0).nonzero().reshape(-1)
        P = h * w
        b, q = idx // P, idx % P
        xy = torch.stack([((q % w).float() + 0.5) * STRIDES[li], ((q // w).float() + 0.5) * STRIDES[li]], 1)
        pred = bbox.permute(0, 2, 3, 1).reshape(-1, 4)[idx].contiguous()
        c = ctr.reshape(-1)[idx].contiguous()
        t = tgt[idx].contiguous()
        n = idx.numel()
        res = [torch.empty(n), torch.empty(n), torch.empty(n), torch.empty(n, 4), torch.empty(n)]
        p = lambda v: ctypes.c_void_p(v.data_ptr())    # noqa: E731
        lib.host_fcos_point_loss(ctypes.c_int64(n), p(xy.contiguous()), p(pred), p(t), p(c), *[p(r) for r in res])
        rows.append(dict(kind=kinds[idx], level=li, idx=idx, ct=res[0], bbox=res[1], bce=res[2], g_pred=res[3],
                         g_ctr=res[4], xy=xy, pred=pred, tgt=t, ctr=c))
    return rows


def decoding_ties(xy, pred, tgt):
    """[n] bool: points whose predicted and target box share a coordinate in float32 (x - l, y - t, x + r, y + b) but
    not in float64.  The gradient of an elementwise max / min jumps at a tie, so there float32 decoding -- the
    reference's own precision -- and the float64 oracle sit on different sides of the jump."""
    s = torch.tensor([-1.0, -1.0, 1.0, 1.0])
    c = torch.cat([xy, xy], 1)
    f32 = (c + s * pred) == (c + s * tgt)
    f64 = (c.double() + s.double() * pred.double()) == (c.double() + s.double() * tgt.double())
    return (f32 & ~f64).any(1)


def check_fcos(levels, B, C, ups=(1.0, 1.0), need=(True, True), lw=(1.0, 1.0), seed=0, tiny_only=False, side=None):
    from boxinstseg_b200.ops.fcos import fcos_box_losses
    inputs = fcos_inputs(levels, B, C, seed or B * 100 + C + len(levels), tiny_only)
    host = fcos_host(levels, B, inputs)
    n_pos = sum(int(r['idx'].numel()) for r in host)
    ct_sum = sum(float(r['ct'].double().sum()) for r in host)
    den = torch.tensor([max(float(n_pos), 1.0), max(ct_sum, 1e-6)], dtype=torch.float32)
    if tiny_only:
        assert float(den[1]) == float(torch.tensor(1e-6, dtype=torch.float32)), den
    if side is not None:
        n = max(B * 4 * sum(h * w for h, w in levels), B * sum(h * w for h, w in levels))
        assert (fc_scale_ctas(n) * FC_BWD_NT < n) == (side == 'strided'), (n, fc_scale_ctas(n))
    sb = torch.tensor(lw[0], dtype=torch.float32) / (den[1] + torch.tensor(FLT_EPS, dtype=torch.float32))
    sc = torch.tensor(lw[1], dtype=torch.float32) / (den[0] + torch.tensor(FLT_EPS, dtype=torch.float32))

    def once():
        bb = [i[0].to(DEV).requires_grad_(need[0]) for i in inputs]
        cc = [i[1].to(DEV).requires_grad_(need[1]) for i in inputs]
        lb, lc = fcos_box_losses(bb, cc, [i[2].to(DEV) for i in inputs], [i[3].to(DEV) for i in inputs], den.to(DEV),
                                 STRIDES[:len(levels)], C, lw[0], lw[1])
        wrt = (bb if need[0] else []) + (cc if need[1] else [])
        gs = torch.autograd.grad([lb, lc], wrt, grad_outputs=[torch.tensor(ups[0], device=DEV),
                                                              torch.tensor(ups[1], device=DEV)])
        return [lb.detach().reshape(1), lc.detach().reshape(1)] + [g.cpu() for g in gs]
    got = twice(once)
    case = f'levels={levels} B={B} C={C} up={ups} grads={need} lw={lw}'
    n = len(levels)
    g_bb = got[2:2 + n] if need[0] else None
    g_cc = got[2 + n * need[0]:] if need[1] else None
    ref_gp, ref_gc, got_gp, ref_b, ref_c, abs_b, abs_c = [], [], [], 0.0, 0.0, 0.0, 0.0
    for r in host:
        li, idx = r['level'], r['idx']
        h, w = levels[li]
        P = h * w
        if g_bb is not None:                   # bit for bit: the host twin's gradient times the same float32 scale
            gk = g_bb[li].permute(0, 2, 3, 1).reshape(-1, 4)
            want = r['g_pred'] * sb
            if ups[0] != 1.0:
                want = want * torch.tensor(ups[0], dtype=torch.float32)
            assert torch.equal(gk[idx], want), (case, li, (gk[idx] != want).nonzero()[:4], r['kind'])
            mask = torch.ones(B * P, dtype=torch.bool)
            mask[idx] = False
            assert not gk[mask].any(), (case, li, 'a nonzero d/d bbox_pred at a non-positive')
        if g_cc is not None:
            gk = g_cc[li].reshape(-1)
            want = r['g_ctr'] * sc * torch.tensor(ups[1], dtype=torch.float32)
            # sigmoid(x) - ct cancels: judged in units of its two terms, sigmoid(x) = g_ctr + ct taken from the host twin
            unit = U * ((r['g_ctr'] + r['ct']).double().abs() + r['ct'].double()) * float(sc) * abs(ups[1])
            ratio('fcos d/d centerness against the host twin', gk[idx], want, unit, TOL_FC_CTR, case)
            mask = torch.ones(B * P, dtype=torch.bool)
            mask[idx] = False
            assert not gk[mask].any(), (case, li, 'a nonzero d/d centerness at a non-positive')
        # float64 oracle of the reference's lines on the same float32 inputs
        w_ct, w_bbox, w_bce, w_gp, w_gc = ofl.element_terms(r['xy'].double(), r['pred'].double(), r['tgt'].double(),
                                                            r['ctr'].double())
        keep = (r['kind'] != TINY_KIND) & ~decoding_ties(r['xy'], r['pred'], r['tgt'])
        ref_b += float(w_bbox[keep].sum())
        abs_b += float(w_bbox[keep].abs().sum())
        ref_c += float(w_bce.sum())
        abs_c += float(w_bce.abs().sum())
        if g_bb is not None:
            ref_gp.append(w_gp[keep] * float(sb) * ups[0])
            got_gp.append(g_bb[li].permute(0, 2, 3, 1).reshape(-1, 4)[idx][keep])
        if g_cc is not None:
            ref_gc.append((w_gc * float(sc) * ups[1], g_cc[li].reshape(-1)[idx]))
    if g_bb is not None and ref_gp:
        e = scaled_err(torch.cat(got_gp), torch.cat(ref_gp))
        print(f'[envelope] fcos d/d bbox_pred against float64: {e:.3e} (bar {TOL_FC_BBOX64:g}) {case}')
        assert e <= TOL_FC_BBOX64, (case, e)
    if g_cc is not None and ref_gc:
        e = scaled_err(torch.cat([b for _, b in ref_gc]), torch.cat([a for a, _ in ref_gc]))
        print(f'[envelope] fcos d/d centerness against float64: {e:.3e} (bar {TOL_FC_CTR64:g}) {case}')
        assert e <= TOL_FC_CTR64, (case, e)
    # the losses against the oracle's sums; the positives left out above are taken from the host twin
    tiny_b = sum(float(r['bbox'][(r['kind'] == TINY_KIND) | decoding_ties(r['xy'], r['pred'], r['tgt'])].double().sum())
                 for r in host)
    want_b = lw[0] * (ref_b + tiny_b) / (float(den[1]) + FLT_EPS)
    want_c = lw[1] * ref_c / (float(den[0]) + FLT_EPS)
    for name, g, want, mag in (('loss_bbox', got[0], want_b, lw[0] * (abs_b + abs(tiny_b)) / (float(den[1]) + FLT_EPS)),
                               ('loss_centerness', got[1], want_c, lw[1] * abs_c / (float(den[0]) + FLT_EPS))):
        e = abs(float(g) - want) / mag if mag > 0 else abs(float(g))
        print(f'[envelope] fcos {name} / sum |terms|: {e:.3e} (bar {TOL_FC_LOSS:g}) {case}')
        assert e <= TOL_FC_LOSS, (case, name, e)


FC_SHAPES = [
    ([(15, 17)], 1, 'one'), ([(16, 16)], 1, 'one'), ([(257, 1)], 1, 'one'),           # B*H*W = 255, 256, 257
    ([(5, 17)], 3, 'one'), ([(8, 16)], 2, 'one'), ([(1, 1)], 1, 'one'), ([(1, 300)], 2, 'one'),
    ([(20, 24), (10, 12), (5, 6), (3, 3), (1, 1), (1, 7), (9, 1), (2, 2)], 2, 'one'),  # 8 levels
    ([(100, 128), (50, 64), (25, 32)], 3, 'strided'),                                 # the scale grid strides
]


@pytest.mark.parametrize('C', [1, 80])
@pytest.mark.parametrize('levels,B,side', FC_SHAPES)
def test_fcos_shapes(levels, B, side, C):
    check_fcos(levels, B, C, ups=(0.7, 1.3), side=side)


@pytest.mark.parametrize('ups', [(1.0, 1.0), (0.7, 1.3), (0.0, 1.0), (1.0, 0.0)])
@pytest.mark.parametrize('need', [(True, True), (True, False), (False, True)])
def test_fcos_upstream(ups, need):
    """Upstream gradients of exactly 1 (nothing to scale), 0 and others, and only one input requiring a gradient."""
    check_fcos([(20, 24), (10, 12), (1, 5)], 2, 80, ups=ups, need=need, lw=(2.0, 0.5))


def test_fcos_denominator_floor():
    """Only tiny centerness targets: their sum is below 1e-6 and the GIoU loss divides by the floor."""
    check_fcos([(3, 4)], 1, 80, ups=(0.7, 1.3), tiny_only=True)


def test_fcos_rejects_nine_levels():
    from boxinstseg_b200.ops.fcos import fcos_box_losses
    z = [torch.zeros(1, 4, 1, 1, device=DEV) for _ in range(9)]
    with pytest.raises(ValueError, match='1 to 8 levels'):
        fcos_box_losses(z, [t[:, :1] for t in z], [torch.zeros(1, dtype=torch.int64)] * 9, [torch.ones(1, 4)] * 9,
                        torch.ones(2, device=DEV), [8.0] * 9, 80)
