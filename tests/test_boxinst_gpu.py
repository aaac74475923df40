"""GPU parity: the CUDA BoxInst path (through the C ABI) against the oracle and the golden
vectors minted from the reference.  Tolerances: index / threshold work bit-exact; floating point
<= 1e-3 relative on loss and gradient (BASELINE.json north_star), in practice ~1e-6."""
import numpy as np
import pytest
import torch

from tests.helpers import boxinst_case, rel_err

pytestmark = pytest.mark.gpu
T = torch.from_numpy


@pytest.fixture(scope='module')
def dev():
    assert torch.cuda.is_available(), 'GPU tests need a CUDA device'
    return torch.device('cuda:0')


# ------------------------------------------------------------------ a7 pairwise op
@pytest.mark.parametrize('tag', ['k3d2', 'k5d1'])
@pytest.mark.parametrize('dtype', [torch.float32, torch.float64])
def test_pairwise_golden(golden, dev, tag, dtype):
    from boxinstseg_b200.ops.pairwise import pairwise_nlog
    g = golden('pairwise_' + tag)
    k, d = int(g['size']), int(g['dilation'])
    x = T(g['logits']).to(dev, dtype).requires_grad_(True)
    out = pairwise_nlog(x, k, d)
    ref = T(g['out64']).to(dev)
    assert torch.allclose(out.double(), ref, rtol=1e-3, atol=2e-6 if dtype == torch.float32 else 1e-12)
    (gx,) = torch.autograd.grad((out * T(g['g_out']).to(dev, dtype)).sum(), x)
    assert torch.allclose(gx.double(), T(g['g_logits64']).to(dev), rtol=1e-3, atol=2e-6 if dtype == torch.float32 else 1e-12)


@pytest.mark.parametrize('shape,k,d', [((3, 1, 37, 53), 3, 2), ((2, 1, 16, 64), 3, 1), ((1, 1, 5, 3), 3, 2),
                                       ((2, 1, 40, 70), 5, 2), ((1, 1, 200, 256), 3, 2), ((1, 1, 30, 30), 7, 3)])
def test_pairwise_vs_oracle(dev, shape, k, d):
    from boxinstseg_b200.ops.pairwise import pairwise_nlog
    from oracle.boxinst import pairwise_nlog as oracle_pw
    gen = torch.Generator().manual_seed(7)
    x = torch.randn(shape, generator=gen) * 4
    x.view(-1)[:4] = torch.tensor([45.0, -45.0, 90.0, -120.0])[: min(4, x.numel())]   # slow-path logits
    gout = torch.rand(shape[0], k * k - 1, *shape[2:], generator=gen)
    x64 = x.double().requires_grad_(True)
    ref = oracle_pw(x64, k, d)
    (gref,) = torch.autograd.grad((ref * gout.double()).sum(), x64)
    xg = x.to(dev).requires_grad_(True)
    out = pairwise_nlog(xg, k, d)
    (gx,) = torch.autograd.grad((out * gout.to(dev)).sum(), xg)
    assert torch.allclose(out.cpu().double(), ref.detach(), rtol=1e-3, atol=2e-6)
    assert torch.allclose(gx.cpu().double(), gref, rtol=1e-3, atol=2e-6)
    # determinism (the reference's atomicAdd backward is not)
    (gx2,) = torch.autograd.grad((pairwise_nlog(xg, k, d) * gout.to(dev)).sum(), xg)
    assert torch.equal(gx, gx2)


def test_pairwise_errors(dev):
    from boxinstseg_b200.ops.pairwise import pairwise_nlog
    with pytest.raises(RuntimeError):
        pairwise_nlog(torch.zeros(1, 1, 4, 4), 3, 2)                     # not CUDA (pairwise.cu:7-13)
    assert pairwise_nlog(torch.zeros(0, 1, 4, 4, device=dev), 3, 2).shape == (0, 8, 4, 4)


# ------------------------------------------------------------------ a5 targets
def _targets(case, dev, **kw):
    from boxinstseg_b200.ops.boxinst import boxinst_targets
    return boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']],
                           want_similarity=True, **kw)


def test_targets_golden(golden, dev):
    g = golden('boxinst_loss')
    from tests.test_oracle_golden import _boxinst_inputs
    img, metas, boxes = _boxinst_inputs(g)
    from boxinstseg_b200.ops.boxinst import boxinst_targets
    t = boxinst_targets(img.to(dev), metas, [b.to(dev) for b in boxes], want_similarity=True)
    bms = t.bitmasks()
    for i in range(2):
        assert torch.equal(bms[i].cpu(), T(g[f'bitmask{i}']))                        # index work: bit-exact
        ref = T(g[f'sim{i}'])
        assert torch.allclose(t.similarity[i].cpu(), ref, rtol=1e-5, atol=1e-7)
        bits = sum(((ref[c] >= 0.3).to(torch.uint8) << c) for c in range(8))
        assert torch.equal(t.edge_bits[i].cpu(), bits)                               # thresholded weights


@pytest.mark.parametrize('ragged', [False, True])
def test_targets_vs_oracle(dev, ragged):
    from oracle.boxinst import boxinst_targets as oracle_targets
    case = boxinst_case(11, B=3, hp=96, wp=160, gts_per_img=4, inst_per_gt=1, ragged=ragged)
    # box edge cases: touching the borders, degenerate, fractional
    case['gt_bboxes'][0] = torch.tensor([[0.0, 0.0, 159.9, 95.9], [10.2, 3.9, 10.9, 4.1], [1.99, 2.01, 5.99, 6.0],
                                         [100.5, 50.5, 160.0, 96.0]])
    t = _targets(case, dev)
    sim, bms = oracle_targets(case['img'], case['metas'], case['gt_bboxes'])
    got = t.bitmasks()
    for i in range(3):
        assert torch.equal(got[i].cpu(), bms[i])
    assert torch.allclose(t.similarity.cpu(), sim, rtol=1e-5, atol=1e-7)
    mism = ((t.similarity.cpu() >= 0.3) != (sim >= 0.3)).sum().item()
    assert mism == 0


def test_targets_forward_empty_images_and_chunks(dev):
    """bxs_boxinst_targets_forward with images without GT boxes, including a batch that ends with one, against the
    oracle; and a batch of more images than one launch carries the metadata of (64) against the same call on its two
    halves, with images without GT boxes on both sides of the chunk boundary."""
    from boxinstseg_b200 import _lib as L
    from oracle.boxinst import boxinst_targets as oracle_targets
    case = boxinst_case(5, B=4, hp=64, wp=96, gts_per_img=3, inst_per_gt=1, ragged=True)
    case['gt_bboxes'][1] = case['gt_bboxes'][1][:0]
    case['gt_bboxes'][3] = case['gt_bboxes'][3][:0]
    t = _targets(case, dev)
    sim, bms = oracle_targets(case['img'], case['metas'], case['gt_bboxes'])
    for got, want in zip(t.bitmasks(), bms):
        assert torch.equal(got.cpu(), want)
    assert torch.allclose(t.similarity.cpu(), sim, rtol=1e-5, atol=1e-7)
    assert torch.equal(t.edge_bits.cpu(), sum(((sim[:, c] >= 0.3).to(torch.uint8) << c) for c in range(8)))
    assert t.gt_img.cpu().tolist() == np.repeat(np.arange(4), [len(b) for b in case['gt_bboxes']]).tolist()

    big = boxinst_case(6, B=70, hp=32, wp=48, gts_per_img=3, inst_per_gt=1, ragged=True)
    num_gts = [0 if b in (3, 62, 63, 64, 66, 69) else b % 4 for b in range(70)]
    big['gt_bboxes'] = [boxes[:n] for boxes, n in zip(big['gt_bboxes'], num_gts)]
    whole = _targets(big, dev)
    halves = [_targets(dict(img=big['img'][s], metas=big['metas'][s], gt_bboxes=big['gt_bboxes'][s]), dev)
              for s in (slice(0, 64), slice(64, 70))]
    for name in ('lab', 'valid', 'similarity', 'edge_bits', 'rects'):
        assert torch.equal(getattr(whole, name), torch.cat([getattr(h, name) for h in halves])), name
    assert whole.gt_img.cpu().tolist() == np.repeat(np.arange(70), num_gts).tolist()

    # argument errors of the C entry point
    img = case['img'].to(dev).contiguous()
    B, _, Hp, Wp = img.shape
    boxes = torch.cat(case['gt_bboxes']).float().to(dev).contiguous()
    ng = np.asarray([len(b) for b in case['gt_bboxes']], np.int32)
    hw = np.asarray([m['img_shape'][:2] for m in case['metas']], np.int32)
    rem = np.asarray([int(10 * float(m['img_shape'][0]) / float(m['ori_shape'][0])) for m in case['metas']], np.int32)
    mean = np.ascontiguousarray(np.asarray(case['metas'][0]['img_norm_cfg']['mean'], np.float32))
    std = np.ascontiguousarray(np.asarray(case['metas'][0]['img_norm_cfg']['std'], np.float32))
    lib = L.lib()

    def call(Bx, ngx=ng, lab_=t.lab):
        return lib.bxs_boxinst_targets_forward(L.ptr(img), L.ptr(boxes), hw.ctypes.data, rem.ctypes.data, ngx.ctypes.data,
                                               mean.ctypes.data, std.ctypes.data, L.ptr(lab_), L.ptr(t.valid),
                                               L.ptr(t.similarity), L.ptr(t.edge_bits), L.ptr(t.rects), L.ptr(t.gt_img), Bx,
                                               Hp, Wp, 4, 3, 2, 0.3, L.stream())
    assert call(B) == 0
    assert call(B, lab_=None) == -1
    assert call(B, ngx=np.asarray([1, -1, 0, 0], np.int32)) == -1


def test_lab_of_all_uint8_colours(dev):
    """The colour conversion of the target build over ALL 2^24 uint8 colours against the oracle's float64 restatement of
    scikit-image rgb2lab (cast to float32 as condinst_head.py:1413-1414 does).  Both sides evaluate in float64; libm and
    CUDA pow / cbrt may differ in the last float64 bit, which can move the float32 cast by one ulp in rare cases."""
    from boxinstseg_b200 import _lib as L
    from oracle.boxinst import rgb2lab_u8
    v = torch.arange(1 << 24, dtype=torch.int32)
    rgb = torch.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], 1).to(torch.uint8)
    d_rgb = rgb.to(dev).contiguous()
    lab = torch.empty(1 << 24, 3, device=dev)
    assert L.lib().bxs_rgb_u8_to_lab(L.ptr(d_rgb), L.ptr(lab), 1 << 24, L.stream()) == 0
    got = lab.cpu()
    worst, differing = 0.0, 0
    for lo in range(0, 1 << 24, 1 << 21):                            # 2M colours at a time (float64 temporaries)
        ref = torch.from_numpy(rgb2lab_u8(rgb[lo:lo + (1 << 21)].numpy()).astype(np.float32))
        d = (got[lo:lo + (1 << 21)] - ref).abs()
        worst = max(worst, float(d.max()))
        differing += int((d > 0).sum())
    assert worst <= 1.6e-5, worst                                    # <= 1 float32 ulp at |value| < 128 (2^-17 .. 2^-16)
    assert differing <= (3 << 24) * 1e-4, differing                 # and rare


# ------------------------------------------------------------------ a6+a7+a8 fused loss
def _oracle_loss(case, warm, dtype=torch.float64):
    from oracle import boxinst as ob
    sim, bms = ob.boxinst_targets(case['img'], case['metas'], case['gt_bboxes'])
    x = case['logits'].to(dtype).requires_grad_(True)
    bm = torch.cat(bms)[case['gt_inds']][:, None].to(dtype)
    prj, pair = ob.boxinst_mask_loss(x, sim[case['img_inds']].to(dtype), bm, warmup_factor=warm)
    return x, prj, pair


def _cuda_loss(case, dev, iters, warmup_iters=10000):
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss
    t = _targets(case, dev)
    x = case['logits'].to(dev).requires_grad_(True)
    it = torch.tensor([float(iters)], device=dev)
    prj, pair = boxinst_mask_loss(x, t, case['gt_inds'].to(dev), it, warmup_iters)
    return x, prj, pair


def test_fused_loss_golden(golden, dev):
    g = golden('boxinst_loss')
    from tests.test_oracle_golden import _boxinst_inputs
    img, metas, boxes = _boxinst_inputs(g)
    case = dict(img=img, metas=metas, gt_bboxes=boxes, gt_inds=T(g['gt_inds']), img_inds=T(g['img_inds']),
                logits=T(g['logits']))
    x, prj, pair = _cuda_loss(case, dev, iters=5000)          # warm-up factor 0.5 as in the golden run
    assert abs(prj.item() - float(g['loss_prj'])) <= 1e-5 * abs(float(g['loss_prj']))
    assert abs(pair.item() - float(g['loss_pairwise'])) <= 1e-5 * abs(float(g['loss_pairwise']))
    (gx,) = torch.autograd.grad(prj * float(g['g_prj']) + pair * float(g['g_pair']), x)
    assert torch.allclose(gx.cpu(), T(g['g_logits']), rtol=1e-3, atol=1e-8)


@pytest.mark.parametrize('cfg', [dict(B=2, hp=96, wp=160, gts_per_img=3, inst_per_gt=2),
                                 dict(B=1, hp=64, wp=52, gts_per_img=2, inst_per_gt=3),       # W%4 != 0 at stride 4 -> scalar path
                                 dict(B=2, hp=200, wp=2200, gts_per_img=2, inst_per_gt=1),    # W > 512: multi-panel
                                 dict(B=3, hp=160, wp=256, gts_per_img=5, inst_per_gt=4, ragged=True)])
def test_fused_loss_vs_oracle(dev, cfg):
    case = boxinst_case(5, logit_std=3.0, **cfg)
    x64, prj64, pair64 = _oracle_loss(case, warm=0.25)
    (g64,) = torch.autograd.grad(prj64 * 1.5 + pair64 * 0.5, x64)
    x, prj, pair = _cuda_loss(case, dev, iters=2500)
    (gx,) = torch.autograd.grad(prj * 1.5 + pair * 0.5, x)
    assert abs(prj.item() - prj64.item()) <= 1e-4 * abs(prj64.item())
    assert abs(pair.item() - pair64.item()) <= 1e-4 * abs(pair64.item())
    assert rel_err(gx.cpu(), g64) <= 1e-4
    # element-wise too, modulo arg-max ties (none expected on random data)
    assert torch.allclose(gx.cpu().double(), g64, rtol=1e-3, atol=1e-9)
    # run-to-run determinism
    x2, prj2, pair2 = _cuda_loss(case, dev, iters=2500)
    (gx2,) = torch.autograd.grad(prj2 * 1.5 + pair2 * 0.5, x2)
    assert torch.equal(gx, gx2) and prj.item() == prj2.item() and pair.item() == pair2.item()


def test_fused_loss_edge_cases(dev):
    # extreme logits (log-space slow path), empty box (covers no sample point), zero total weight
    case = boxinst_case(9, B=2, hp=64, wp=96, gts_per_img=2, inst_per_gt=2, logit_std=1.0)
    case['gt_bboxes'][1] = torch.tensor([[5.0, 5.0, 5.5, 5.5], [0.0, 0.0, 95.0, 63.0]])
    case['logits'][0, 0, :4, :4] = torch.tensor([[50.0, -50.0, 80.0, -80.0]] * 4)
    case['logits'][5] = 100.0
    x64, prj64, pair64 = _oracle_loss(case, warm=1.0)
    (g64,) = torch.autograd.grad(prj64 + pair64, x64)
    x, prj, pair = _cuda_loss(case, dev, iters=20000)
    (gx,) = torch.autograd.grad(prj + pair, x)
    assert abs(prj.item() - prj64.item()) <= 1e-4 * abs(prj64.item())
    assert abs(pair.item() - pair64.item()) <= 1e-4 * abs(pair64.item())
    assert torch.isfinite(gx).all()
    assert rel_err(gx.cpu(), g64) <= 1e-3


def test_fused_loss_full_size_properties(dev):
    """Config A size (N=128, 200x256): properties that do not need the oracle at full size."""
    case = boxinst_case(1234, B=2, hp=800, wp=1024, gts_per_img=8, inst_per_gt=8)
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss, boxinst_targets
    from boxinstseg_b200.ops.pairwise import pairwise_nlog
    t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']], want_similarity=True)
    x = case['logits'].to(dev).requires_grad_(True)
    it = torch.tensor([10000.0], device=dev)
    gi = case['gt_inds'].to(dev)
    prj, pair = boxinst_mask_loss(x, t, gi, it)
    (gx,) = torch.autograd.grad(prj + pair, x)
    # unfused composition from the fine-grained drop-in ops (different kernels, same maths)
    xs = x.detach().clone().requires_grad_(True)
    bm = torch.cat(t.bitmasks())[gi][:, None]
    scores = xs.sigmoid()

    def dice(a, b):
        a, b = a.flatten(1), b.flatten(1)
        return 1 - 2 * (a * b).sum(1) / ((a * a).sum(1) + (b * b).sum(1) + 1e-5)
    prj_ref = (dice(scores.amax(2), bm.amax(2)) + dice(scores.amax(3), bm.amax(3))).mean()
    w = (t.similarity[case['img_inds'].to(dev)] >= 0.3).float() * bm
    pair_ref = (pairwise_nlog(xs, 3, 2) * w).sum() / w.sum().clamp(min=1.0)
    (gref,) = torch.autograd.grad(prj_ref + pair_ref, xs)
    assert abs(prj.item() - prj_ref.item()) <= 1e-4 * abs(prj_ref.item())
    assert abs(pair.item() - pair_ref.item()) <= 1e-4 * abs(pair_ref.item())
    assert rel_err(gx, gref) <= 1e-3
    # gradient is exactly zero where it must be: outside each instance's box grown by the dilation (2), except at the row /
    # column arg-max positions of the logits (torch.max(dim))
    from oracle.boxinst import logit_argmax_mask
    assert torch.isfinite(gx).all()
    N, _, H, W = x.shape
    j0, j1, i0, i1 = (t.rects[gi].long().cpu()[:, k].view(-1, 1, 1) for k in range(4))
    ys, xs = torch.arange(H).view(1, H, 1), torch.arange(W).view(1, 1, W)
    span = (j0 <= j1) & (i0 <= i1) & (ys >= j0 - 2) & (ys <= j1 + 2) & (xs >= i0 - 2) & (xs <= i1 + 2)
    allowed = span[:, None] | logit_argmax_mask(x.detach().cpu())
    assert (gx.cpu()[~allowed] == 0).all()
    assert (gx.cpu()[~span[:, None].expand(N, 1, H, W)] != 0).any()      # the arg-max positions do carry gradient


# ------------------------------------------------------------------ a6+a7+a8 single-pass schedule (boxinst_onepass.cu)
def _two_call(case, t, dev, dil, g_prj, g_pair, iters=10000.0):
    """loss + gradient from the two-call kernels (forward, then backward re-reading the logits), through the C ABI."""
    from boxinstseg_b200 import _lib as L
    lib = L.lib()
    x = case['logits'].to(dev).contiguous()
    N, _, H, W = x.shape
    ws = torch.empty(lib.bxs_boxinst_loss_workspace_bytes(N, H, W), dtype=torch.uint8, device=dev)
    out = torch.empty(4, device=dev)
    it = torch.tensor([iters], device=dev)
    gi = case['gt_inds'].to(dev, torch.int32)
    L.check(lib.bxs_boxinst_loss_forward(L.ptr(x), L.ptr(t.edge_bits), L.ptr(t.rects), L.ptr(gi), L.ptr(t.gt_img), L.ptr(it),
                                         10000.0, L.ptr(ws), L.ptr(out), N, H, W, dil, L.stream()), 'fwd')
    g = torch.tensor([g_prj, g_pair], device=dev)
    gx = torch.empty_like(x)
    L.check(lib.bxs_boxinst_loss_backward(L.ptr(x), L.ptr(t.edge_bits), L.ptr(t.rects), L.ptr(gi), L.ptr(t.gt_img), L.ptr(ws),
                                          L.ptr(g), L.ptr(gx), N, H, W, dil, L.stream()), 'bwd')
    return out, gx


@pytest.mark.parametrize('cfg', [dict(B=2, hp=96, wp=160, gts_per_img=3, inst_per_gt=2, dil=2),       # H=24: one short strip + one full
                                 dict(B=1, hp=200, wp=512, gts_per_img=4, inst_per_gt=3, dil=1),      # W=128, H=50
                                 dict(B=2, hp=264, wp=1024, gts_per_img=3, inst_per_gt=4, dil=3),     # W=256, H=66
                                 dict(B=1, hp=132, wp=2048, gts_per_img=5, inst_per_gt=2, dil=4),     # W=512 (4 chunks), H=33
                                 dict(B=3, hp=128, wp=240, gts_per_img=6, inst_per_gt=40, dil=2)])    # N=720: many items per CTA
def test_single_pass_matches_two_call_and_oracle(dev, cfg):
    from boxinstseg_b200 import _lib as L
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss, boxinst_targets
    cfg = dict(cfg)
    dil = cfg.pop('dil')
    case = boxinst_case(21, logit_std=3.0, **cfg)
    N, _, H, W = case['logits'].shape
    assert L.lib().bxs_boxinst_loss_fused_supported(N, H, W, dil) == 1
    t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']], pairwise_dilation=dil,
                        want_similarity=True)
    it = torch.tensor([10000.0], device=dev)
    for g_prj, g_pair in [(1.0, 1.0), (0.75, 2.5)]:
        x = case['logits'].to(dev).requires_grad_(True)
        prj, pair = boxinst_mask_loss(x, t, case['gt_inds'].to(dev), it, pairwise_dilation=dil)
        (gx,) = torch.autograd.grad(prj * g_prj + pair * g_pair, x)
        out2, gx2 = _two_call(case, t, dev, dil, g_prj, g_pair)
        assert abs(prj.item() - out2[0].item()) <= 1e-5 * abs(out2[0].item())
        assert abs(pair.item() - out2[1].item()) <= 1e-5 * abs(out2[1].item()) + 1e-9
        assert rel_err(gx, gx2) <= 1e-5
        assert torch.allclose(gx, gx2, rtol=1e-4, atol=1e-9)
    if N <= 64:                                                     # and against the float64 oracle where it is quick
        from oracle import boxinst as ob
        sim, bms = ob.boxinst_targets(case['img'], case['metas'], case['gt_bboxes'], dilation=dil)
        x64 = case['logits'].double().requires_grad_(True)
        bm = torch.cat(bms)[case['gt_inds']][:, None].double()
        p64, q64 = ob.boxinst_mask_loss(x64, sim[case['img_inds']].double(), bm, dilation=dil)
        (g64,) = torch.autograd.grad(p64 * 0.75 + q64 * 2.5, x64)
        assert abs(prj.item() - p64.item()) <= 1e-4 * abs(p64.item())
        assert abs(pair.item() - q64.item()) <= 1e-4 * abs(q64.item())
        assert rel_err(gx.cpu(), g64) <= 1e-4


def test_single_pass_retain_graph_and_no_grad(dev):
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss, boxinst_targets
    case = boxinst_case(33, B=2, hp=160, wp=256, gts_per_img=3, inst_per_gt=3, logit_std=2.0)
    t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']])
    it = torch.tensor([4000.0], device=dev)
    gi = case['gt_inds'].to(dev)
    x = case['logits'].to(dev).requires_grad_(True)
    prj, pair = boxinst_mask_loss(x, t, gi, it)
    (ga,) = torch.autograd.grad(prj * 3.0 + pair * 0.5, x, retain_graph=True)      # single-pass buffer, converted in place
    ga = ga.clone()
    (gb,) = torch.autograd.grad(prj * 3.0 + pair * 0.5, x, retain_graph=True)      # second call: two-call kernels
    (gc,) = torch.autograd.grad(prj + pair, x)
    _, g2 = _two_call(case, t, dev, 2, 3.0, 0.5, iters=4000.0)
    _, g1 = _two_call(case, t, dev, 2, 1.0, 1.0, iters=4000.0)
    assert torch.allclose(ga, g2, rtol=1e-4, atol=1e-9) and torch.equal(gb, g2) and torch.equal(gc, g1)
    with torch.no_grad():                                                          # forward only: two-call forward kernel
        p0, q0 = boxinst_mask_loss(case['logits'].to(dev), t, gi, it)
    assert abs(p0.item() - prj.item()) <= 1e-6 * abs(prj.item()) and abs(q0.item() - pair.item()) <= 1e-6 * abs(pair.item())


def test_single_pass_scheduler_state_is_reusable(dev):
    """Back-to-back calls on two streams and a CUDA-graph replay: the work-item counter always returns to zero."""
    from boxinstseg_b200.ops.boxinst import boxinst_mask_loss, boxinst_targets
    case = boxinst_case(4, B=2, hp=320, wp=512, gts_per_img=4, inst_per_gt=8, logit_std=2.0)
    t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']])
    it = torch.tensor([10000.0], device=dev)
    gi = case['gt_inds'].to(dev)
    ones = torch.ones((), device=dev)

    def run(x):
        prj, pair = boxinst_mask_loss(x, t, gi, it)
        torch.autograd.backward([prj, pair], [ones, ones])
        return prj, pair

    x = case['logits'].to(dev).requires_grad_(True)
    run(x)
    ref = x.grad.clone()
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    xs = [case['logits'].to(dev).requires_grad_(True) for _ in streams]
    for _ in range(5):
        for s_, xi in zip(streams, xs):
            s_.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s_):
                xi.grad = None
                run(xi)
    torch.cuda.synchronize()
    assert torch.equal(xs[0].grad, ref) and torch.equal(xs[1].grad, ref)
    xg = case['logits'].to(dev).requires_grad_(True)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run(xg)
        xg.grad = None
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        prj, pair = run(xg)
    for _ in range(3):
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(xg.grad, ref)
