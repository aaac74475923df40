"""GPU parity of the registry loss classes (a6 dense, a9, a10) against golden vectors minted from the
reference's own BoxProjectionLoss / LevelsetLoss / mil_loss and against the float64 oracle."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
T = torch.from_numpy
DEV = 'cuda:0'


def test_projection_golden(golden):
    from boxinstseg_b200.models import build_loss
    from boxinstseg_b200.models.losses import mil_loss
    g = golden('projection')
    s, t, soft = (T(g[k]).to(DEV) for k in ('scores', 'targets', 'soft'))
    loss = build_loss(dict(type='BoxProjectionLoss', loss_weight=3.0))
    assert torch.allclose(loss(s, t).cpu(), T(g['loss_w3']), rtol=1e-5, atol=1e-6)
    assert torch.allclose(loss(s, soft).cpu(), T(g['loss_w3_soft']), rtol=1e-5, atol=1e-6)
    assert torch.allclose(mil_loss(None, s[:, 0], None, t[:, 0]).cpu(), T(g['disco_mil']), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('shape', [(5, 1, 50, 64), (3, 1, 37, 301), (2, 1, 200, 256), (1, 1, 3, 2)])
def test_projection_vs_oracle(shape):
    from boxinstseg_b200.models.losses import projection_losses
    from oracle.boxinst import projection_losses as oracle_prj
    gen = torch.Generator().manual_seed(3)
    s = torch.rand(shape, generator=gen)
    t = (torch.rand(shape, generator=gen) > 0.7).float() * torch.rand(shape, generator=gen)
    t[0] = 0                                                     # empty target
    gl = torch.rand(shape[0], generator=gen)
    s64 = s.double().requires_grad_(True)
    ref = 2.5 * oracle_prj(s64, t.double())
    (gref,) = torch.autograd.grad((ref * gl.double()).sum(), s64)
    sg = s.to(DEV).requires_grad_(True)
    out = projection_losses(sg, t.to(DEV), 1e-5, 2.5)
    (gs,) = torch.autograd.grad((out * gl.to(DEV)).sum(), sg)
    assert torch.allclose(out.cpu().double(), ref.detach(), rtol=1e-5, atol=1e-6)
    assert torch.allclose(gs.cpu().double(), gref, rtol=1e-4, atol=1e-7)


def test_projection_tie_goes_to_first_index():
    from boxinstseg_b200.models.losses import projection_losses
    s = torch.full((1, 1, 4, 6), 0.25, device=DEV)
    s[0, 0, 2, 3] = 0.75
    s[0, 0, 2, 5] = 0.75
    s.requires_grad_(True)
    t = torch.zeros(1, 1, 4, 6, device=DEV)
    t[0, 0, 1:3, 2:5] = 1
    (g,) = torch.autograd.grad(projection_losses(s, t).sum(), s)
    sc = s.detach().cpu().requires_grad_(True)
    from oracle.boxinst import projection_losses as oracle_prj
    (gc,) = torch.autograd.grad(oracle_prj(sc, t.cpu()).sum(), sc)
    assert torch.allclose(g.cpu(), gc, rtol=1e-5, atol=1e-7)     # torch.max(dim): first maximal index


def test_levelset_golden(golden):
    from boxinstseg_b200.models import build_loss
    g = golden('levelset')
    sc = T(g['scores']).to(DEV).requires_grad_(True)
    tg = T(g['target']).to(DEV).requires_grad_(True)
    m = T(g['mask']).to(DEV)
    phi = torch.cat([sc, 1 - sc], 1) * m
    loss = build_loss(dict(type='LevelsetLoss', loss_weight=1.0))(phi, tg * m, T(g['pixel_num']).to(DEV))
    assert torch.allclose(loss.cpu(), T(g['loss']), rtol=1e-5, atol=1e-7)
    gs, gt = torch.autograd.grad((loss * T(g['g_loss']).to(DEV)).sum(), [sc, tg])
    assert torch.allclose(gs.cpu(), T(g['g_scores']), rtol=1e-3, atol=1e-6)
    assert torch.allclose(gt.cpu(), T(g['g_target']), rtol=1e-3, atol=1e-6)
    from boxinstseg_b200.models.losses import length_regularization
    assert torch.allclose(length_regularization()(sc.detach()).cpu(), T(g['length']), rtol=1e-5)


@pytest.mark.parametrize('n,C,h,w', [(4, 3, 50, 64), (3, 2, 33, 47), (2, 5, 100, 128), (16, 3, 200, 256)])
def test_levelset_vs_oracle(n, C, h, w):
    from boxinstseg_b200.models.losses import LevelsetLoss
    from oracle.levelset import levelset_loss as oracle_ls
    gen = torch.Generator().manual_seed(21)
    s = torch.rand(n, 1, h, w, generator=gen)
    m = torch.zeros(n, 1, h, w)
    for i in range(n):
        m[i, 0, h // 5: h // 5 + 2 + i * 3, w // 6: w // 2 + i] = 1
    m[-1] = 0                                                    # empty box: clamp(min=1e-5) is active
    t = torch.randn(n, C, h, w, generator=gen)
    gl = torch.rand(n, generator=gen)
    pix = m.sum((1, 2, 3)).clamp(min=1)
    s64 = s.double().requires_grad_(True)
    t64 = t.double().requires_grad_(True)
    ref = oracle_ls(torch.cat([s64, 1 - s64], 1) * m.double(), t64 * m.double(), pix.double(), 0.7)
    rs, rt = torch.autograd.grad((ref * gl.double()).sum(), [s64, t64])
    sg = s.to(DEV).requires_grad_(True)
    tg = t.to(DEV).requires_grad_(True)
    md = m.to(DEV)
    out = LevelsetLoss(0.7)(torch.cat([sg, 1 - sg], 1) * md, tg * md, pix.to(DEV))
    gs, gt = torch.autograd.grad((out * gl.to(DEV)).sum(), [sg, tg])
    assert torch.allclose(out.cpu().double(), ref.detach(), rtol=1e-4, atol=1e-7)
    assert rel_err(gs.cpu(), rs) < 1e-4 and rel_err(gt.cpu(), rt) < 1e-4
    # region_levelset: the energy alone (pixel_num = 1, loss_weight = 1)
    from boxinstseg_b200.models.losses import region_levelset
    from oracle.levelset import region_levelset as oracle_region
    ref = oracle_region(torch.cat([s64, 1 - s64], 1) * m.double(), t64 * m.double())
    rs, rt = torch.autograd.grad((ref * gl.double()).sum(), [s64, t64])
    out = region_levelset()(torch.cat([sg, 1 - sg], 1) * md, tg * md)
    gs, gt = torch.autograd.grad((out * gl.to(DEV)).sum(), [sg, tg])
    assert torch.allclose(out.cpu().double(), ref.detach(), rtol=1e-4, atol=1e-7)
    assert rel_err(gs.cpu(), rs) < 1e-4 and rel_err(gt.cpu(), rt) < 1e-4


def test_levelset_more_than_eight_channels_is_unsupported():
    """The level-set kernels unroll at most 8 target channels: more is an error, never a silent fallback."""
    from boxinstseg_b200._lib import BoxSegError
    from boxinstseg_b200.models.losses import LevelsetLoss, region_levelset
    s, t = torch.rand(2, 2, 8, 8, device=DEV), torch.rand(2, 9, 8, 8, device=DEV)
    with pytest.raises(BoxSegError, match='unsupported shape'):
        LevelsetLoss()(s, t, torch.ones(2, device=DEV))
    with pytest.raises(BoxSegError, match='unsupported shape'):
        region_levelset()(s, t)


def test_length_regularization_grad():
    from boxinstseg_b200.models.losses import length_regularization
    from oracle.levelset import length_regularization as oracle_len
    gen = torch.Generator().manual_seed(2)
    s = torch.rand(3, 2, 17, 23, generator=gen)
    s64 = s.double().requires_grad_(True)
    (gref,) = torch.autograd.grad(oracle_len(s64).sum(), s64)
    sg = s.to(DEV).requires_grad_(True)
    out = length_regularization()(sg)
    (g,) = torch.autograd.grad(out.sum(), sg)
    assert torch.allclose(out.cpu().double(), oracle_len(s.double()), rtol=1e-5)
    assert torch.allclose(g.cpu().double(), gref, atol=1e-6)


# ------------------------------------------------------------------ a11 LCM
def test_lcm_golden(golden):
    from boxinstseg_b200.models.losses import LCM
    g = golden('lcm')
    phis = T(g['phis']).to(DEV).requires_grad_(True)
    loss = LCM(T(g['imgs']).to(DEV), phis, T(g['box']).to(DEV))
    assert abs(loss.item() - float(g['loss'])) <= 1e-4 * abs(float(g['loss']))
    (gp,) = torch.autograd.grad(loss, phis)
    assert torch.allclose(gp.cpu(), T(g['g_phis']), rtol=1e-3, atol=1e-7)


@pytest.mark.parametrize('n,h,w', [(3, 96, 96), (2, 17, 23), (2, 5, 4), (1, 200, 256)])
def test_lcm_vs_oracle(n, h, w):
    from boxinstseg_b200.models.losses import LCM
    from oracle.levelset import lcm_loss
    gen = torch.Generator().manual_seed(8)
    imgs = torch.rand(n, 3, h, w, generator=gen)
    phis = torch.rand(n, 1, h, w, generator=gen)
    box = (torch.rand(n, 1, h, w, generator=gen) > 0.4).float() * torch.rand(n, 1, h, w, generator=gen)
    p64 = phis.double().requires_grad_(True)
    ref = lcm_loss(imgs.double(), p64, box.double())
    (gref,) = torch.autograd.grad(ref * 1.7, p64)
    pg = phis.to(DEV).requires_grad_(True)
    out = LCM(imgs.to(DEV), pg, box.to(DEV))
    (gp,) = torch.autograd.grad(out * 1.7, pg)
    assert abs(out.item() - ref.item()) <= 1e-4 * abs(ref.item())
    assert rel_err(gp.cpu(), gref) < 1e-3
    (gp2,) = torch.autograd.grad(LCM(imgs.to(DEV), pg, box.to(DEV)) * 1.7, pg)
    assert torch.equal(gp, gp2)


def test_local_consistency_module_forward():
    """LocalConsistencyModule.forward (levelset_loss.py:121-126): the refined masks themselves."""
    from boxinstseg_b200.models.losses import LocalConsistencyModule
    from oracle.levelset import lcm_refine
    gen = torch.Generator().manual_seed(8)
    imgs = torch.rand(3, 3, 96, 96, generator=gen)
    phis = torch.rand(3, 1, 96, 96, generator=gen)
    out = LocalConsistencyModule(dilations=[2], num_iter=10)(imgs.to(DEV), phis.to(DEV))
    ref = lcm_refine(imgs.double(), phis.double(), 10, 2)
    assert out.shape == phis.shape and rel_err(out.cpu(), ref) <= 1e-5


# ------------------------------------------------------------------ a16 mean field
def test_meanfield_golden(golden):
    from boxinstseg_b200.models.dense_heads import MeanField
    g = golden('meanfield')
    mf = MeanField(T(g['feature']).to(DEV), kernel_size=3, theta0=0.5, theta1=30, theta2=10, alpha0=2, iter=10, base=0.1)
    assert torch.allclose(mf.kernel[0].flatten(1).cpu(), T(g['kernel'])[0], rtol=1e-5, atol=1e-9)
    ps, va = mf(T(g['x']).to(DEV), T(g['targets']).to(DEV))
    assert torch.equal(ps.cpu(), T(g['pseudo'])) and torch.equal(va.cpu(), T(g['valid']))     # binary output: exact


@pytest.mark.parametrize('seed,gamma', [(0, 0.01), (1, 0.5), (2, 2.0)])
def test_meanfield_inter_image_term_golden(golden, seed, gamma):
    """MeanField.forward(x, targets, inter_img_mask) as corr_loss calls it (discobox_head.py:616,643-644): binary output,
    bit-exact against the golden vectors of the reference's own class; both kernel paths (per-object CTAs / grid-wide rounds)."""
    import numpy as np
    from boxinstseg_b200.models.dense_heads import MeanField
    from oracle.make_golden_meanfield_inter import CFG, case
    g = golden('meanfield_inter')
    fm, x, t, iiu = case(seed)
    mf = MeanField(fm.to(DEV), gamma=gamma, **CFG)
    ps, va = mf(x.to(DEV), t.to(DEV), iiu.to(DEV))
    want = np.unpackbits(g[f's{seed}_pseudo'], axis=-1)[..., :ps.shape[-1]]
    assert np.array_equal(ps.cpu().numpy().astype(np.uint8), want) and np.array_equal(va.cpu().numpy(), g[f's{seed}_valid'])
    if int(g[f's{seed}_flips']):
        plain, _ = mf(x.to(DEV), t.to(DEV))
        assert int((plain != ps).sum()) == int(g[f's{seed}_flips'])
    # the per-object shared-memory path (chosen for >= 2 objects per SM, or without a workspace): same bits
    from boxinstseg_b200 import _lib as L
    xs, tg, ii = x.to(DEV).contiguous(), t.to(DEV).contiguous(), iiu.to(DEV).contiguous()
    ret, valid = torch.empty_like(xs), torch.empty(xs.shape[0], device=DEV)
    L.check(L.lib().bxs_meanfield_forward_inter(L.ptr(mf.kernel), None, L.ptr(xs), L.ptr(tg), L.ptr(ii), float(np.float32(gamma)),
                                                mf._neglog.ctypes.data, L.ptr(ret), L.ptr(valid), None, xs.shape[0],
                                                xs.shape[2], xs.shape[3], 3, 10, L.stream()), 'meanfield_forward_inter')
    assert torch.equal(ret, ps) and torch.equal(valid, va)


@pytest.mark.parametrize('n,h,w,big', [(6, 50, 64, False), (3, 200, 256, False), (2, 330, 340, True)])
def test_meanfield_vs_oracle(n, h, w, big):
    from boxinstseg_b200.models.dense_heads import MeanField
    from oracle.levelset import meanfield_forward, meanfield_kernel
    import torch.nn.functional as F
    gen = torch.Generator().manual_seed(4)
    fm = F.interpolate(torch.randn(1, 3, max(h // 8, 2), max(w // 8, 2), generator=gen), size=(h, w), mode='bilinear')
    fm = fm + torch.randn(1, 3, h, w, generator=gen) * 0.1
    x = torch.rand(n, 1, h, w, generator=gen)
    t = torch.zeros(n, 1, h, w)
    for i in range(n):
        t[i, 0, h // 6: h // 6 + h // 3 + i, w // 5: w // 5 + w // 2] = 1
    k = meanfield_kernel(fm, 3, 0.5, 30.0, 2.0)
    ps, va = meanfield_forward(k, x, t, 3, 10, 0.1)
    mf = MeanField(fm.to(DEV), kernel_size=3, theta0=0.5, theta1=30, theta2=10, alpha0=2, iter=10, base=0.1)
    gps, gva = mf(x.to(DEV), t.to(DEV))
    mism = (gps.cpu() != ps).float().mean().item()
    assert mism <= 2e-5, mism          # expf differs from the CPU libm by <= 2 ulp: exact ties may flip
    assert torch.equal(gva.cpu(), va)
