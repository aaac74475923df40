"""GPU parity of the wgmma dynamic 1x1 convolution (a2/a3/a4) against a float64 reference.
Tolerance 1e-3 of the output's scale: TF32 operands (10-bit mantissa), FP32 accumulation -> ~3e-4 at K = 256 (forward,
d/d feat) and at K = 51 200 pixels (d/d kernel; the rounding errors are independent, the sum grows like sqrt(K) as
the result does); the reference's own cuDNN conv2d runs in TF32 by default on Ampere and later GPUs.  Inputs that
are exactly representable in TF32 must come out exact up to FP32 accumulation (the "exactness probes")."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _ref(feat, kern):
    return torch.einsum('bic,bchw->bihw', kern.double(), feat.double())


@pytest.mark.parametrize('B,C,h,w,I', [(1, 256, 16, 32, 16), (2, 256, 50, 64, 100), (1, 256, 200, 256, 37),
                                       (2, 128, 25, 36, 130), (1, 256, 96, 96, 300), (1, 32, 8, 4, 5)])
def test_dynconv_forward(B, C, h, w, I):
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    gen = torch.Generator().manual_seed(I)
    feat = torch.randn(B, C, h, w, generator=gen)
    kern = torch.randn(B, I, C, generator=gen) * 0.05
    out = dynconv1x1(feat.to(DEV), kern.to(DEV))
    torch.cuda.synchronize()
    ref = _ref(feat, kern)
    assert out.shape == ref.shape
    assert rel_err(out.cpu(), ref) < 1e-3
    # exactness probe: inputs representable in TF32 -> only fp32 accumulation error remains
    f2 = (torch.randint(-8, 9, (B, C, h, w), generator=gen).float() / 8)
    k2 = (torch.randint(-8, 9, (B, I, C), generator=gen).float() / 16)
    out2 = dynconv1x1(f2.to(DEV), k2.to(DEV))
    assert torch.allclose(out2.cpu().double(), _ref(f2, k2), rtol=1e-5, atol=1e-4)


def test_dynconv_backward_and_call_sites():
    from boxinstseg_b200.ops.dynconv import box2mask_mask_pred, dynconv1x1, solo_dynamic_conv
    gen = torch.Generator().manual_seed(0)
    feat = torch.randn(2, 256, 20, 24, generator=gen).to(DEV).requires_grad_(True)
    kern = (torch.randn(2, 48, 256, generator=gen) * 0.05).to(DEV).requires_grad_(True)
    gout = torch.randn(2, 48, 20, 24, generator=gen).to(DEV)
    out = dynconv1x1(feat, kern)
    gf, gk = torch.autograd.grad((out * gout).sum(), [feat, kern])
    f64, k64 = feat.detach().double().requires_grad_(True), kern.detach().double().requires_grad_(True)
    rf, rk = torch.autograd.grad((torch.einsum('bic,bchw->bihw', k64, f64) * gout.double()).sum(), [f64, k64])
    assert rel_err(gf, rf) < 1e-3 and rel_err(gk, rk) < 1e-3
    # SOLO order: cell s = gy*S + gx
    kp = torch.randn(2, 256, 4, 4, generator=gen).to(DEV) * 0.05
    solo = solo_dynamic_conv(feat.detach(), kp)
    ref = torch.nn.functional.conv2d(feat.detach().reshape(1, 512, 20, 24).double(),
                                     kp.permute(0, 2, 3, 1).reshape(-1, 256, 1, 1).double(), groups=2).view(2, 16, 20, 24)
    assert rel_err(solo, ref) < 1e-3
    assert rel_err(box2mask_mask_pred(kern.detach(), feat.detach()), out.detach().double()) < 1e-6


@pytest.mark.parametrize('B,C,h,w,I', [(1, 256, 16, 32, 16), (2, 256, 50, 64, 100), (1, 256, 200, 256, 37),
                                       (2, 128, 25, 36, 130), (1, 256, 96, 96, 300), (1, 32, 8, 4, 5),
                                       (3, 64, 10, 14, 256), (2, 256, 40, 52, 129)])
def test_dynconv_backward_kernels(B, C, h, w, I):
    """d/d feat (forward kernel, swapped roles, zero-filled instance tail) and d/d kernel (split-K over pixels, pixel
    tail zero-filled by the tensor map, I > 128 in row chunks); I > 256: d/d feat through cuBLAS."""
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    gen = torch.Generator().manual_seed(100 + I)
    for exact in (False, True):
        if exact:
            feat = torch.randint(-8, 9, (B, C, h, w), generator=gen).float() / 8
            kern = torch.randint(-8, 9, (B, I, C), generator=gen).float() / 16
            gout = torch.randint(-4, 5, (B, I, h, w), generator=gen).float() / 4
        else:
            feat = torch.randn(B, C, h, w, generator=gen)
            kern = torch.randn(B, I, C, generator=gen) * 0.05
            gout = torch.randn(B, I, h, w, generator=gen)
        f = feat.to(DEV).requires_grad_(True)
        k = kern.to(DEV).requires_grad_(True)
        gf, gk = torch.autograd.grad(dynconv1x1(f, k), [f, k], gout.to(DEV))
        gf1, = torch.autograd.grad(dynconv1x1(f, k.detach()), [f], gout.to(DEV))          # only one of the two needed
        gk1, = torch.autograd.grad(dynconv1x1(f.detach(), k), [k], gout.to(DEV))
        torch.cuda.synchronize()
        rf = torch.einsum('bic,bihw->bchw', kern.double(), gout.double())
        rk = torch.einsum('bihw,bchw->bic', gout.double(), feat.double())
        assert torch.equal(gf, gf1) and torch.equal(gk, gk1)                               # deterministic
        if exact:
            assert torch.allclose(gf.cpu().double(), rf, rtol=1e-5, atol=1e-4)
            assert torch.allclose(gk.cpu().double(), rk, rtol=1e-5, atol=1e-4 * (h * w) ** 0.5)
        else:
            assert rel_err(gf.cpu(), rf) < 1e-3, rel_err(gf.cpu(), rf)
            assert rel_err(gk.cpu(), rk) < 1e-3, rel_err(gk.cpu(), rk)


def test_dynconv_backward_c_abi_errors():
    from boxinstseg_b200 import _lib as L
    f = torch.zeros(1, 32, 8, 4, device=DEV)
    k = torch.zeros(1, 300, 32, device=DEV)
    g = torch.zeros(1, 300, 8, 4, device=DEV)
    ws = torch.empty(L.lib().bxs_dynconv1x1_backward_workspace_bytes(1, 32, 32, 300), dtype=torch.uint8, device=DEV)
    gf, gk = torch.empty_like(f), torch.empty_like(k)
    args = (1, 32, 32, 300, L.stream())
    assert L.lib().bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), L.ptr(gf), L.ptr(gk), L.ptr(ws), *args) == -3
    assert L.lib().bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), None, L.ptr(gk), L.ptr(ws), *args) == 0
    assert L.lib().bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), None, None, L.ptr(ws), *args) == -1
    assert L.lib().bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), L.ptr(gf), L.ptr(gk), None, *args) == -1
