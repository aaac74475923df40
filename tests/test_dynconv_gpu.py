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


# channel counts 96..224 (a half-filled or partial last K-block, BN = 128 / 256 in the d/d kernel body) and kernel
# counts at the 32 / 64 / 128 / 256 chunk edges, past the native d/d feat limit (257) and at DiscoBox's I_pad limit (2048)
EDGE_SHAPES = [(1, 96, 20, 24, 1), (2, 160, 10, 14, 33), (1, 192, 24, 28, 65), (1, 224, 12, 20, 127), (2, 96, 16, 18, 255),
               (1, 224, 8, 12, 128), (2, 192, 8, 12, 256), (1, 160, 30, 36, 257), (1, 192, 16, 20, 2048)]


@pytest.mark.parametrize('B,C,h,w,I', [(1, 256, 16, 32, 16), (2, 256, 50, 64, 100), (1, 256, 200, 256, 37),
                                       (2, 128, 25, 36, 130), (1, 256, 96, 96, 300), (1, 32, 8, 4, 5)] + EDGE_SHAPES)
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
    # exactness probe: operands exact in TF32 (multiples of 1/8 and 1/16 below 1), products multiples of 2^-7 whose
    # partial sums stay below 2^7 * C / 256: every FP32 sum is exact, so the result must equal the float64 reference
    f2 = (torch.randint(-8, 9, (B, C, h, w), generator=gen).float() / 8)
    k2 = (torch.randint(-8, 9, (B, I, C), generator=gen).float() / 16)
    out2 = dynconv1x1(f2.to(DEV), k2.to(DEV))
    r2 = _ref(f2, k2)
    assert torch.equal(out2.cpu().double(), r2), (out2.cpu().double() - r2).abs().max().item()


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
                                       (3, 64, 10, 14, 256), (2, 256, 40, 52, 129)] + EDGE_SHAPES)
def test_dynconv_backward_kernels(B, C, h, w, I):
    """d/d feat (forward kernel, swapped roles, zero-filled instance tail) and d/d kernel (split-K over pixels, pixel
    tail zero-filled by the tensor map, I > 128 in row chunks); I > 256: d/d feat through cuBLAS.  The exact inputs are
    multiples of 1/8, 1/16 and 1/4: every product is a multiple of 2^-6 (d/d feat) or 2^-5 (d/d kernel) and every partial
    sum stays below 2^11 (at most 2048 kernels of |k g| <= 1/2) or 2^16 (at most 51 200 pixels of |g f| <= 1): exact in
    FP32, so both gradients must equal the float64 reference."""
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
            assert h * w <= 51200 and I <= 2048                                             # the probe's precondition
            assert torch.equal(gf.cpu().double(), rf), (gf.cpu().double() - rf).abs().max().item()
            assert torch.equal(gk.cpu().double(), rk), (gk.cpu().double() - rk).abs().max().item()
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
