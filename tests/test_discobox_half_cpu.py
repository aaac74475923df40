"""CPU: the float64 restatement of the 16-bit DiscoBox mask loss (tests/discobox_half_oracle.py) against the reference's
composition run by autograd in float16 / bfloat16 on CPU torch (oracle.levelset.disco_mil_loss / disco_dice_loss /
meanfield_forward), and the argument validation of the new C entry points, which runs before any device call."""
import ctypes
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import levelset as ol
from tests.discobox_half_oracle import disco_half_loss, pseudo_label

F16, BF16 = 0, 1
TOL_G = {torch.float16: 1e-3, torch.bfloat16: 8e-3}


def _boxes(n, h, w, gen):
    t = torch.zeros(n, h, w)
    for i in range(n):
        y0, x0 = int(torch.randint(0, h // 2, (1,), generator=gen)), int(torch.randint(0, w // 2, (1,), generator=gen))
        y1, x1 = y0 + int(torch.randint(2, h - y0, (1,), generator=gen)), x0 + int(torch.randint(2, w - x0, (1,), generator=gen))
        t[i, y0:y1, x0:x1] = 1
        t[i, y0, x0] = 0                                       # not a rectangle
    return t


def _composition(x, t_logits, tg, kernels, img_inds, use_loss_ts):
    """DiscoBoxSOLOv2Head.loss's mask terms on 16-bit logits as the reference computes them under autocast, with the
    all-zero targets kept at weight 0: per-level sums (num_ins, num_ts, count)."""
    s = torch.sigmoid(x)
    t = s if t_logits is None else torch.sigmoid(t_logits)
    tgf = tg.float()
    keep = (tgf.flatten(1).sum(1) > 0).float()
    num_ins = (ol.disco_mil_loss(s, tgf) * keep).sum()
    num_ts = torch.zeros(())
    if use_loss_ts:
        enl = F.max_pool2d(tgf.unsqueeze(1), 3, 1, 1).squeeze(1)
        m = ((t + s) / 2).detach().float()
        pseudo = torch.zeros_like(tgf)
        for b, k in enumerate(kernels):
            sel = img_inds == b
            p, _ = ol.meanfield_forward(k, m[sel].unsqueeze(1), tgf[sel].unsqueeze(1), 3, 10, 0.1)
            pseudo[sel] = p[:, 0]
        num_ts = (ol.disco_dice_loss(s * enl, pseudo) * keep).sum()
    return num_ins, num_ts, keep.sum()


def _rel(a, b):
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


@pytest.mark.parametrize('dt', [torch.float16, torch.bfloat16])
@pytest.mark.parametrize('teacher,use_ts', [(False, True), (True, True), (False, False)])
def test_oracle_matches_autocast_composition(dt, teacher, use_ts):
    gen = torch.Generator().manual_seed(11)
    n, h, w = 5, 24, 29
    color = F.interpolate(torch.randn(2, 3, 5, 6, generator=gen), size=(h, w), mode='bilinear', align_corners=True)
    kernels = [ol.meanfield_kernel(color[b:b + 1], 3, 0.5, 30.0, 2.0) for b in range(2)]
    img_inds = torch.tensor([0, 0, 1, 1, 1])
    tg = _boxes(n, h, w, gen)
    tg[3] = 0
    x = (torch.randn(n, h, w, generator=gen) * 3).to(dt).requires_grad_(True)
    xt = (torch.randn(n, h, w, generator=gen) * 3).to(dt) if teacher else None
    ni, nt, cnt = _composition(x, xt, tg, kernels, img_inds, use_ts)
    (g_ref,) = torch.autograd.grad(ni + nt, x)

    s = torch.sigmoid(x.detach())
    t = torch.sigmoid(xt) if teacher else None
    pseudo = pseudo_label(s, tg, kernels, img_inds, t=t) if use_ts else None
    oi, ot, oc, g = disco_half_loss(s, tg, pseudo)
    ni, nt = float(ni.detach()), float(nt.detach())
    assert abs(float(oi) - ni) <= 1e-4 * abs(ni)
    assert abs(float(ot) - nt) <= 1e-4 * max(abs(nt), 1e-30)
    assert float(oc) == float(cnt) == 4.0
    assert _rel(g.to(dt).double(), g_ref.double()) <= TOL_G[dt]
    assert float(g[3].abs().max()) == 0.0


def test_oracle_first_index_on_ties():
    """A constant map ties every row and column: the gradient of the MIL term lands on the first column / row."""
    s = torch.full((1, 3, 4), 0.75).half()
    tg = torch.ones(1, 3, 4)
    *_, g_s = disco_half_loss(s, tg)
    support = g_s[0] != 0
    expect = torch.zeros(3, 4, dtype=torch.bool)
    expect[:, 0] = True                                               # row maxima: column 0
    expect[0, :] = True                                               # column maxima: row 0
    assert torch.equal(support, expect)


# ----------------------------------------------------------------------------------------------- C ABI, no device
@pytest.fixture(scope='module')
def lib():
    from boxinstseg_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.lib()


_BUF = ctypes.create_string_buffer(256)


@pytest.fixture(scope='module')
def p():
    return ctypes.c_void_p((ctypes.addressof(_BUF) + 15) & ~15)


@pytest.mark.parametrize('dt', [F16, BF16])
def test_loss_forward_validation(lib, p, dt):
    fwd = lib.bxs_discobox_loss_forward
    assert fwd(None, p, p, dt, p, p, 1, 4, 4, None) == -1
    assert fwd(p, None, p, dt, p, p, 1, 4, 4, None) == -1
    assert fwd(p, p, p, dt, None, p, 1, 4, 4, None) == -1             # no workspace
    assert fwd(p, p, p, dt, p, None, 1, 4, 4, None) == -1             # no output
    assert fwd(p, p, p, dt, p, p, -1, 4, 4, None) == -1
    assert fwd(p, p, p, dt, p, p, 1, 0, 4, None) == -1
    assert fwd(p, p, p, dt, p, p, 1, 4, -4, None) == -1
    assert fwd(p, p, p, 2, p, p, 1, 4, 4, None) == -1                 # unknown dtype
    assert fwd(p, p, p, dt, p, p, 1, 1 << 31, 4, None) == -3           # h above INT32_MAX
    assert fwd(p, p, p, dt, p, p, 1 << 40, 1 << 20, 1 << 10, None) == -3   # more than INT32_MAX CTAs


@pytest.mark.parametrize('dt', [F16, BF16])
def test_loss_backward_validation(lib, p, dt):
    bwd = lib.bxs_discobox_loss_backward
    assert bwd(None, p, p, dt, p, p, p, 1, 4, 4, None) == -1
    assert bwd(p, None, p, dt, p, p, p, 1, 4, 4, None) == -1
    assert bwd(p, p, p, dt, None, p, p, 1, 4, 4, None) == -1
    assert bwd(p, p, p, dt, p, None, p, 1, 4, 4, None) == -1           # no upstream gradients
    assert bwd(p, p, p, dt, p, p, None, 1, 4, 4, None) == -1
    assert bwd(p, p, p, -1, p, p, p, 1, 4, 4, None) == -1
    assert bwd(p, p, p, dt, p, p, p, 1, 4, 0, None) == -1
    assert bwd(p, p, p, dt, p, p, p, 1, 4, 1 << 31, None) == -3
    assert bwd(None, None, None, dt, None, None, None, 0, 4, 4, None) == 0   # n == 0: nothing to do


def test_loss_workspace_query(lib):
    ws = lib.bxs_discobox_loss_workspace_bytes
    assert ws(32, 200, 256) > 32 * 13 * 256 * 8                       # at least the column partials
    assert ws(0, 200, 256) == 0 and ws(-1, 4, 4) == 0 and ws(1, 0, 4) == 0 and ws(1, 4, 0) == 0


@pytest.mark.parametrize('dt', [F16, BF16])
def test_meanfield_logits_validation(lib, p, dt):
    mf = lib.bxs_meanfield_forward_logits
    args = lambda **kw: [kw.get(k, v) for k, v in dict(  # noqa: E731
        K=p, obj=None, s=p, t=None, tg=p, dt=dt, neg=p, out=p, ws=p, n=2, h=8, w=8, ks=3, it=10, st=None).items()]
    for key in ('K', 's', 'tg', 'neg', 'out'):
        assert mf(*args(**{key: None})) == -1, key
    assert mf(*args(n=-1)) == -1
    assert mf(*args(h=0)) == -1
    assert mf(*args(ks=2)) == -1                                        # even kernel size
    assert mf(*args(it=-1)) == -1
    assert mf(*args(dt=5)) == -1
    assert mf(*args(ws=None, h=512, w=512)) == -1                       # too large for the per-object schedule
    assert mf(*args(h=1 << 15, w=1 << 15)) == -3                        # h*w >= 2^30
    assert mf(*args(K=None, s=None, tg=None, neg=None, out=None, n=0)) == 0   # n == 0: nothing to do
