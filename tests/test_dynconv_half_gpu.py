"""GPU: the 16-bit (FP16 / BF16) dynamic 1x1 convolution -- forward, d/d feat and d/d kernel on the tensor cores with FP32
accumulation, and the dtype contract of ``dynconv1x1`` (16-bit in, 16-bit out; autocast casts first; envelope fallback).

Parity is measured against a float64 einsum of the SAME 16-bit operands, so only the accumulation order and the one
rounding of each result to the operand dtype remain: rel_err <= 1e-3 for FP16 (11-bit significand), <= 8e-3 for BF16
(8-bit).  The exactness probes use small integer operands whose results are integers below 2^11 (FP16) or 2^8 (BF16):
every product and partial sum is then exact in FP32 and so is the final rounding, so any error in the MN-major operand
layout, the channel / pixel order of the epilogue or the split-K reduction shows up as a wrong integer."""
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
DTYPES = [pytest.param(torch.float16, 1e-3, 2 ** 11, id='fp16'), pytest.param(torch.bfloat16, 8e-3, 2 ** 8, id='bf16')]
# the shapes of test_dynconv_forward / test_dynconv_backward_kernels with h*w a multiple of 8, and config C's per-image conv
SHAPES = [(1, 256, 16, 32, 16), (2, 256, 50, 64, 100), (1, 256, 200, 256, 37), (2, 128, 26, 36, 130), (1, 256, 96, 96, 300),
          (1, 32, 8, 4, 5), (3, 64, 10, 16, 256), (2, 256, 40, 52, 129), (1, 256, 200, 256, 16),
          # channel counts 96..224 (a half-filled second 64-channel K-block), kernel counts at the chunk edges, P = 8 and
          # P % 128 == 8 (136 pixels)
          (2, 96, 2, 4, 33), (1, 160, 8, 17, 65), (2, 192, 12, 20, 127), (1, 224, 16, 24, 257), (1, 96, 24, 40, 1),
          (2, 160, 10, 16, 128), (1, 224, 8, 17, 255)]


def _grads(feat, kern, gout, need=(True, True)):
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    f = feat.detach().requires_grad_(need[0])
    k = kern.detach().requires_grad_(need[1])
    out = dynconv1x1(f, k)
    wrt = [t for t, n in zip((f, k), need) if n]
    gs = iter(torch.autograd.grad(out, wrt, gout))
    return out, (next(gs) if need[0] else None), (next(gs) if need[1] else None)


def _refs(feat, kern, gout):
    f, k, g = feat.double().cpu(), kern.double().cpu(), gout.double().cpu()
    return (torch.einsum('bic,bchw->bihw', k, f), torch.einsum('bic,bihw->bchw', k, g),
            torch.einsum('bihw,bchw->bic', g, f))


@pytest.mark.parametrize('dt,tol,limit', DTYPES)
@pytest.mark.parametrize('B,C,h,w,I', SHAPES)
def test_half_parity_exactness_determinism(B, C, h, w, I, dt, tol, limit):
    gen = torch.Generator().manual_seed(1000 + I + C)
    feat = torch.randn(B, C, h, w, generator=gen).to(dt).to(DEV)
    kern = (torch.randn(B, I, C, generator=gen) * 0.05).to(dt).to(DEV)
    gout = torch.randn(B, I, h, w, generator=gen).to(dt).to(DEV)
    out, gf, gk = _grads(feat, kern, gout)
    assert out.dtype == gf.dtype == gk.dtype == dt
    assert out.shape == (B, I, h, w) and gf.shape == feat.shape and gk.shape == kern.shape
    for got, ref in zip((out, gf, gk), _refs(feat, kern, gout)):
        assert rel_err(got.cpu(), ref) <= tol, rel_err(got.cpu(), ref)
    # determinism: a second call, and each gradient on its own, give the same bits
    out2, gf2, gk2 = _grads(feat, kern, gout)
    _, gf1, _ = _grads(feat, kern, gout, (True, False))
    _, _, gk1 = _grads(feat, kern, gout, (False, True))
    assert torch.equal(out, out2) and torch.equal(gf, gf2) and torch.equal(gk, gk2)
    assert torch.equal(gf, gf1) and torch.equal(gk, gk1)

    # exactness probe: distinct small integers per pixel and per channel; g sparse enough that sums over the pixels stay small
    P = h * w
    fi = torch.randint(-1, 2, (B, C, h, w), generator=gen)
    ki = torch.randint(-1, 2, (B, I, C), generator=gen)
    gi = torch.randint(-1, 2, (B, I, h, w), generator=gen) * (torch.rand(B, I, h, w, generator=gen) < min(1.0, 900 / P))
    refs = _refs(fi, ki, gi)
    assert all(r.abs().max() < limit for r in refs)            # the probe's precondition
    out, gf, gk = _grads(fi.to(dt).to(DEV), ki.to(dt).to(DEV), gi.to(dt).to(DEV))
    for name, got, ref in zip(('forward', 'd/d feat', 'd/d kernel'), (out, gf, gk), refs):
        assert torch.equal(got.cpu().double(), ref), (name, (got.cpu().double() - ref).abs().max().item())


@pytest.mark.parametrize('dt', [torch.float16, torch.bfloat16])
def test_autocast_casts_operands_and_returns_fp32_grads(dt):
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(2, 256, 20, 24, generator=gen).to(DEV).requires_grad_(True)
    k = (torch.randn(2, 48, 256, generator=gen) * 0.05).to(DEV).requires_grad_(True)
    g = torch.randn(2, 48, 20, 24, generator=gen).to(DEV)
    with torch.autocast('cuda', dtype=dt):
        out = dynconv1x1(x, k)
    gx, gk = torch.autograd.grad(out, [x, k], g.to(dt))
    ref, rgx, rgk = _grads(x.detach().to(dt), k.detach().to(dt), g.to(dt))
    assert out.dtype == dt and torch.equal(out, ref)
    assert gx.dtype == gk.dtype == torch.float32
    assert torch.equal(gx, rgx.float()) and torch.equal(gk, rgk.float())


@pytest.mark.parametrize('dt', [torch.float16, torch.bfloat16])
def test_outside_half_envelope_runs_fp32_and_rounds_back(dt):
    """h*w % 8 == 4: the 16-bit kernels cannot take it, the float32 kernels run on promoted copies."""
    gen = torch.Generator().manual_seed(11)
    feat = torch.randn(2, 64, 6, 6, generator=gen).to(dt).to(DEV)
    kern = (torch.randn(2, 10, 64, generator=gen) * 0.05).to(dt).to(DEV)
    gout = torch.randn(2, 10, 6, 6, generator=gen).to(dt).to(DEV)
    out, gf, gk = _grads(feat, kern, gout)
    r_out, r_gf, r_gk = _grads(feat.float(), kern.float(), gout.float())
    assert out.dtype == gf.dtype == gk.dtype == dt
    assert torch.equal(out, r_out.to(dt)) and torch.equal(gf, r_gf.to(dt)) and torch.equal(gk, r_gk.to(dt))


def test_mixed_dtypes_outside_autocast_stay_fp32():
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    gen = torch.Generator().manual_seed(5)
    feat = torch.randn(1, 128, 16, 16, generator=gen).to(DEV)
    kern = (torch.randn(1, 8, 128, generator=gen) * 0.05).to(DEV)
    for a, b in ((feat.half(), kern), (feat, kern.bfloat16()), (feat.half(), kern.bfloat16())):
        out = dynconv1x1(a, b)
        assert out.dtype == torch.float32 and torch.equal(out, dynconv1x1(a.float(), b.float()))


@pytest.mark.parametrize('dt', [torch.float16, torch.bfloat16])
def test_half_cuda_graph_replays_eager_bits(dt):
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    gen = torch.Generator().manual_seed(3)
    feat = torch.randn(1, 256, 64, 80, generator=gen).to(dt).to(DEV)
    kern = (torch.randn(1, 24, 256, generator=gen) * 0.05).to(dt).to(DEV)
    gout = torch.randn(1, 24, 64, 80, generator=gen).to(dt).to(DEV)

    def step():                                                 # fresh leaves: no autograd node outlives its stream
        f, k = feat.clone().requires_grad_(True), kern.clone().requires_grad_(True)
        out = dynconv1x1(f, k)
        return (out,) + tuple(torch.autograd.grad(out, [f, k], gout))

    eager = step()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()                                                  # warm-up outside the capture
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    graph.replay()
    torch.cuda.synchronize()
    assert all(torch.equal(a, b) for a, b in zip(eager, captured))


def test_discobox_step_under_autocast():
    """Config C's DiscoBox mask-loss step with a float16 mask-feature leaf (what the reference's autocast mask-feature head
    hands the loss) under autocast: it runs, loss_ins stays within 1e-3 of the float32 step, the gradients are finite."""
    import bench_configs
    from boxinstseg_b200.models import build_head
    _, info = bench_configs.build_C(torch.device(DEV), 0)
    d = info['data']
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256))

    def step(feat, kern, autocast):
        with torch.autocast('cuda', dtype=torch.float16, enabled=autocast):
            pred = torch.cat([head.dynamic_conv(feat[b], kern[b]) for b in range(2)])
            out = head.mask_loss([pred], [d['labels']], [d['img_inds']], d['color'])
        return out, torch.autograd.grad(out['loss_ins'] + out['loss_ts'], [feat, kern])

    ref, _ = step(d['feat'], d['kern'], False)
    feat16 = d['feat'].detach().half().requires_grad_(True)
    out, (gf, gk) = step(feat16, d['kern'], True)
    assert gf.dtype == torch.float16 and gk.dtype == torch.float32
    assert torch.isfinite(gf).all() and torch.isfinite(gk).all()
    assert torch.isfinite(out['loss_ts'])
    assert abs(out['loss_ins'].item() - ref['loss_ins'].item()) <= 1e-3 * abs(ref['loss_ins'].item())
