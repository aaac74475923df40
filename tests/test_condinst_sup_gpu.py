"""CondInst's mask-supervised losses on the GPU: the dice mask loss of ``CondInstMaskHead.loss`` with
``boxinst_enabled=False`` (``ops.condinst.dice_mask_loss``, csrc/condinst_sup.cu) and ``CondInstSegmHead``'s semantic
targets and loss.  Against the golden vectors minted from the reference's own code, the float64 oracle and the reference's
float32 lines on the same CUDA tensors: label maps bit for bit (area ties, nested and overlapping masks, bytes above 1,
G = 0 and G = 100, different G per image), losses and gradients element for element, run-to-run bit identity, strided /
offset / misaligned / 16-bit inputs, no host synchronisation, a CUDA-graph capture of a whole mask-supervised step, and a
stand-in ``CondInst.forward_train`` step against the reference's lines."""
import pytest
import torch

from oracle import condinst_sup as ocs
from oracle.make_golden_condinst_sup import CASES, IN_STRIDE, OUT_STRIDE, case

pytestmark = pytest.mark.gpu
DEV = 'cuda'


def _cuda(masks, labels):
    return [m.to(DEV) for m in masks], [l.to(DEV) for l in labels]


def _dice(logits, masks, gt_inds, dtype=torch.float32, relayout=None):
    from boxinstseg_b200.ops.condinst import dice_mask_loss
    x = logits.to(DEV, dtype).requires_grad_(True)
    arg = relayout(x) if relayout else x
    loss = dice_mask_loss(arg, masks, gt_inds.to(DEV), OUT_STRIDE)
    (g,) = torch.autograd.grad(loss, x)
    return loss, g


def _oracle_dice(logits, masks, gt_inds, dtype=torch.float64):
    x = logits.to(DEV, dtype).requires_grad_(True)
    loss = ocs.mask_loss(x, [m.to(DEV) for m in masks], gt_inds.to(DEV), OUT_STRIDE)['loss_mask']
    (g,) = torch.autograd.grad(loss, x)
    return loss, g


def _exact_grad(logits, masks, gt_inds):
    """(d loss / d x, bound) in float64 from the closed form (2/N) (2 I s / U^2 - t / U) s (1 - s) with 1 - s taken as
    sigmoid(-x): autograd's float64 ``(1 - s) * s`` loses up to 1e-3 of its value at |x| = 30.  ``bound`` is the
    magnitude of the two terms before they cancel, (2/N) (|2 I s / U^2| + |t / U|) s (1 - s)."""
    x = logits.to(DEV, torch.float64).reshape(logits.shape[0], -1)
    s, om = x.sigmoid(), (-x).sigmoid()
    start = OUT_STRIDE // 2
    t = torch.cat([m.to(DEV)[:, start::OUT_STRIDE, start::OUT_STRIDE] for m in masks])[gt_inds.to(DEV)].reshape(x.shape).double()
    I, S, T = (s * t).sum(1, keepdim=True), (s * s).sum(1, keepdim=True), (t * t).sum(1, keepdim=True)
    U = S + T + 1e-5
    k = 2. / x.shape[0]
    grad = k * (2 * I * s / U ** 2 - t / U) * s * om
    bound = k * ((2 * I * s / U ** 2).abs() + (t / U).abs()) * s * om
    return grad.reshape(logits.shape), bound.reshape(logits.shape)


def _check_dice(loss, g, logits, masks, gt_inds, tol=1e-5, scale=1.0):
    """The loss within ``tol`` relative of the float64 oracle; every gradient element within ``tol`` of its terms'
    magnitude of the exact float64 gradient (plus 1e-37 where float32 products underflow to subnormals)."""
    want, want_g = _oracle_dice(logits, masks, gt_inds)
    assert abs(float(loss) - float(want)) <= tol * abs(float(want)) + 1e-7, (float(loss), float(want))
    exact, bound = _exact_grad(logits, masks, gt_inds)
    assert float((exact - want_g).abs().max()) <= 1e-9 * float(want_g.abs().max())          # the closed form is right
    err = (g.double() - scale * exact).abs()
    assert bool((err <= tol * scale * bound + 1e-37).all()), float((err / bound.clamp(min=1e-300)).max())


@pytest.mark.parametrize('seed,kw', CASES)
def test_golden(golden, seed, kw):
    g = golden('condinst_sup')
    masks, labels, logits, gt_inds, segm = case(seed, dtype=torch.float32, **kw)
    masks, labels = _cuda(masks, labels)
    C = kw.get('C', 5)
    loss, gx = _dice(logits, masks, gt_inds)
    want = float(g[f's{seed}_loss_mask'])
    assert abs(float(loss.detach()) - want) <= 1e-5 * abs(want) + 1e-7
    gw = torch.as_tensor(g[f's{seed}_g_mask'])
    if gw.numel():
        assert float((gx.cpu().double() - gw).abs().max()) <= 1e-5 * float(gw.abs().max())
    from boxinstseg_b200.ops.condinst import semantic_targets
    t = semantic_targets(masks, labels, IN_STRIDE, C)
    assert t.dtype == torch.int64 and torch.equal(t.cpu(), torch.as_tensor(g[f's{seed}_targets']).long())
    head = _segm_head(C)
    p = segm.to(DEV).requires_grad_(True)
    ls = head.loss(p, masks, labels)['loss_segm']
    (gp,) = torch.autograd.grad(ls, p)
    want = float(g[f's{seed}_loss_segm'])
    assert abs(float(ls.detach()) - want) <= 1e-5 * abs(want)
    gw = torch.as_tensor(g[f's{seed}_g_segm'])
    assert float((gp.cpu().double() - gw).abs().max()) <= 1e-5 * float(gw.abs().max())
    if kw.get('N', 12) == 0:
        assert float(loss) == 0 and loss.requires_grad and not gx.any()


def _segm_head(C, **kw):
    from boxinstseg_b200.models import build_head
    return build_head(dict(type='CondInstSegmHead', num_classes=C, in_channels=256, in_stride=IN_STRIDE, **kw))


def _masks(gen, G, H, W, kind):
    m = torch.zeros(G, H, W, dtype=torch.uint8)
    for k in range(G):
        y0, x0 = int(torch.randint(0, H - 16, (1,), generator=gen)), int(torch.randint(0, W - 16, (1,), generator=gen))
        hh, ww = int(torch.randint(8, H - y0 + 1, (1,), generator=gen)), int(torch.randint(8, W - x0 + 1, (1,), generator=gen))
        if kind == 'ties':                              # equal areas, overlapping
            hh, ww = 40, 48
            y0, x0 = min(y0, H - hh), min(x0, W - ww)
        m[k, y0:y0 + hh, x0:x0 + ww] = 1
        if kind == 'nested' and k:                      # inside the previous mask
            m[k] = 0
            m[k, 8 + 4 * k:40 + 2 * k, 8 + 4 * k:48 + 2 * k] = 1
    if kind == 'bytes':
        m *= torch.randint(1, 256, m.shape, generator=gen, dtype=torch.int64).to(torch.uint8)
    return m


@pytest.mark.parametrize('Gs,kind', [((8, 8), 'random'), ((5, 3), 'ties'), ((6,), 'nested'), ((4, 9), 'bytes'),
                                     ((0, 3), 'random'), ((100,), 'random'), ((1, 0, 50, 2), 'ties')])
def test_semantic_targets_bit_exact(Gs, kind):
    from boxinstseg_b200.ops.condinst import semantic_targets
    gen = torch.Generator().manual_seed(len(Gs) * 7 + sum(Gs))
    H, W, C = 200, 264, 80
    masks = [_masks(gen, G, H, W, kind).to(DEV) for G in Gs]
    labels = [torch.randint(0, C, (G,), generator=gen).to(DEV) for G in Gs]
    t, areas = semantic_targets(masks, labels, IN_STRIDE, C, return_areas=True)
    want = torch.cat([m.long().sum(dim=(1, 2)) for m in masks])
    assert torch.equal(areas, want)
    ref = torch.stack([ocs.semantic_targets([m], [l], IN_STRIDE, C)[0] if m.shape[0] else
                       torch.full_like(t[0], C) for m, l in zip(masks, labels)])
    assert torch.equal(t, ref)
    assert torch.equal(t.cpu(), ocs.first_min_targets([m.cpu() for m in masks], [l.cpu() for l in labels], IN_STRIDE, C))
    # strided masks (a window of a wider buffer, and a transposed copy viewed back) read in place
    wide = [torch.zeros(m.shape[0], H, W + 13, dtype=torch.uint8, device=DEV) for m in masks]
    for w_, m in zip(wide, masks):
        w_[:, :, 5:5 + W] = m
    assert torch.equal(semantic_targets([w_[:, :, 5:5 + W] for w_ in wide], labels, IN_STRIDE, C), t)
    tr = [m.transpose(1, 2).contiguous().transpose(1, 2) for m in masks]
    assert torch.equal(semantic_targets(tr, labels, IN_STRIDE, C), t)


def test_semantic_targets_sentinel_and_more_than_64_images():
    """An area of exactly 1e8 reads as the sentinel (num_classes), as in the reference; 70 images take two launch pairs."""
    from boxinstseg_b200.ops.condinst import semantic_targets
    m = torch.zeros(2, 784, 1000, dtype=torch.uint8, device=DEV)
    m[0] = 255
    m[0].view(-1)[:392157] = 1                          # area = 392157 + 255 * 391843 = 100312122: above 1e8
    m[1, :8, :8] = 1
    lab = torch.tensor([3, 4], device=DEV)
    t = semantic_targets([m], [lab], IN_STRIDE, 9)
    assert torch.equal(t, ocs.semantic_targets([m.cpu()], [lab.cpu()], IN_STRIDE, 9).to(DEV))
    gen = torch.Generator().manual_seed(3)
    masks = [_masks(gen, 2, 64, 64, 'random').to(DEV) for _ in range(70)]
    labels = [torch.randint(0, 5, (2,), generator=gen).to(DEV) for _ in range(70)]
    t = semantic_targets(masks, labels, IN_STRIDE, 5)
    assert torch.equal(t.cpu(), ocs.semantic_targets([m.cpu() for m in masks], [l.cpu() for l in labels], IN_STRIDE, 5))


def _dice_case(seed, N, G=(8, 8), H=800, W=1024):
    gen = torch.Generator().manual_seed(seed)
    masks = [_masks(gen, g, H, W, 'random').to(DEV) for g in G]
    h, w = len(range(OUT_STRIDE // 2, H, OUT_STRIDE)), len(range(OUT_STRIDE // 2, W, OUT_STRIDE))
    logits = 4 * torch.randn(N, 1, h, w, generator=gen)
    logits[: N // 8] = 30 * torch.sign(logits[: N // 8])          # saturated instances
    gt_inds = torch.randint(0, sum(G), (N,), generator=gen)
    return masks, logits, gt_inds


@pytest.mark.parametrize('N', [1, 2, 37, 128, 500])
def test_dice_against_float64_oracle_and_reference_lines(N):
    masks, logits, gt_inds = _dice_case(N, N)
    loss, g = _dice(logits, masks, gt_inds)
    _check_dice(loss, g, logits, masks, gt_inds)
    ref, ref_g = _oracle_dice(logits, masks, gt_inds, torch.float32)          # the reference's float32 lines
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref))
    assert float((g - ref_g).abs().max()) <= 1e-5 * float(ref_g.abs().max())
    loss2, g2 = _dice(logits, masks, gt_inds)
    assert torch.equal(loss, loss2) and torch.equal(g, g2)


def test_dice_upstream_gradient_bytes_and_mixed_images():
    from boxinstseg_b200.ops.condinst import dice_mask_loss
    gen = torch.Generator().manual_seed(11)
    masks = [_masks(gen, g, 96, 128, k).to(DEV) for g, k in ((3, 'bytes'), (0, 'random'), (5, 'nested'), (1, 'ties'))]
    gt_inds = torch.randint(0, 9, (40,), generator=gen)
    logits = 3 * torch.randn(40, 1, 24, 32, generator=gen)
    x = logits.to(DEV).requires_grad_(True)
    loss = dice_mask_loss(x, masks, gt_inds.to(DEV), OUT_STRIDE)
    (0.37 * loss).backward()
    _check_dice(loss, x.grad, logits, masks, gt_inds, scale=0.37)


def _views(x):
    """(name, view) pairs of the same values: strided, offset in a larger buffer, misaligned."""
    N, _, h, w = x.shape
    t = torch.empty(N, 1, w, h, device=DEV, dtype=x.dtype).transpose(2, 3)
    t.copy_(x)
    flat = torch.empty(x.numel() + 1, device=DEV, dtype=x.dtype)
    mis = flat[1:].view(x.shape)
    mis.copy_(x)
    big = torch.zeros(N, 2, h, w + 3, device=DEV, dtype=x.dtype)
    big[:, 1:, :, 2:2 + w] = x
    return [('transposed', t), ('misaligned', mis), ('window', big[:, 1:, :, 2:2 + w])]


@pytest.mark.parametrize('dtype', [torch.float32, torch.float16, torch.bfloat16])
def test_dice_layouts_and_dtypes(dtype):
    masks, logits, gt_inds = _dice_case(5, 64, G=(4, 6), H=200, W=256)
    logits = logits.to(dtype)
    loss, g = _dice(logits.float(), masks, gt_inds)                  # dense float32 of the same values
    from boxinstseg_b200.ops.condinst import dice_mask_loss
    for name, v in _views(logits.to(DEV)):
        src = v.detach().requires_grad_(True)
        l2 = dice_mask_loss(src, masks, gt_inds.to(DEV), OUT_STRIDE)
        (g2,) = torch.autograd.grad(l2, src)
        assert g2.dtype == dtype and g2.shape == src.shape, name
        assert torch.equal(l2, loss), name
        assert torch.equal(g2, g.to(dtype)), name
    wide = [torch.zeros(m.shape[0], m.shape[1], m.shape[2] + 9, dtype=torch.uint8, device=DEV) for m in masks]
    for w_, m in zip(wide, masks):
        w_[:, :, 3:3 + m.shape[2]] = m
    l3, g3 = _dice(logits.float(), [w_[:, :, 3:-6] for w_ in wide], gt_inds)
    assert torch.equal(l3, loss) and torch.equal(g3, g)


def test_no_host_synchronisation():
    from boxinstseg_b200.ops.condinst import dice_mask_loss
    masks, logits, gt_inds = _dice_case(6, 50, G=(4, 6), H=200, W=256)
    labels = [torch.randint(0, 80, (m.shape[0],)).to(DEV) for m in masks]
    head = _segm_head(80)
    x = logits.to(DEV).requires_grad_(True)
    p = torch.randn(2, 80, 25, 32, device=DEV, requires_grad=True)
    gi = gt_inds.to(DEV)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        total = dice_mask_loss(x, masks, gi, OUT_STRIDE) + head.loss(p, masks, labels)['loss_segm']
        total.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(x.grad).all() and torch.isfinite(p.grad).all()


def _mask_head():
    from boxinstseg_b200.models import build_head
    return build_head(dict(type='CondInstMaskHead', in_channels=8, in_stride=8, out_stride=OUT_STRIDE, max_proposals=-1,
                           boxinst_enabled=False)).to(DEV)


def _step_inputs(seed=0, B=2, H=200, W=256, G=(4, 6), N=40, C=80):
    gen = torch.Generator().manual_seed(seed)
    masks = [_masks(gen, g, H, W, 'random').to(DEV) for g in G]
    labels = [torch.randint(0, C, (g,), generator=gen).to(DEV) for g in G]
    feat = torch.randn(B, 8, H // 8, W // 8, generator=gen).to(DEV)
    head = _mask_head()
    params = (0.3 * torch.randn(N, head.num_gen_params, generator=gen)).to(DEV)
    coors = (torch.rand(N, 2, generator=gen) * torch.tensor([float(W), float(H)])).to(DEV)
    levels = torch.randint(0, 5, (N,), generator=gen).to(DEV)
    img_inds = torch.randint(0, B, (N,), generator=gen).to(DEV)
    gt_inds = torch.tensor([int(torch.randint(0, G[b], (1,), generator=gen)) + sum(G[:b]) for b in img_inds.tolist()]).to(DEV)
    segm = torch.randn(B, C, H // 8, W // 8, generator=gen).to(DEV)
    return head, masks, labels, feat, params, coors, levels, img_inds, gt_inds, segm


def test_whole_step_matches_reference_lines():
    """A stand-in CondInst.forward_train tail with boxinst_enabled=False and a segm_head (condinst.py:62-75): same loss
    dict keys and values as the reference's lines on the same tensors."""
    head, masks, labels, feat, params, coors, levels, img_inds, gt_inds, segm = _step_inputs()
    segm_head = _segm_head(80)
    losses = {}
    losses.update(segm_head.loss(segm, masks, labels))
    pred = head(feat, params, coors, levels, img_inds)
    losses.update(head.loss(None, None, pred, gt_inds, None, masks, labels))
    assert list(losses) == ['loss_segm', 'loss_mask']
    want = {}
    want.update(ocs.segm_loss(segm, masks, labels, IN_STRIDE, 80))
    want.update(ocs.mask_loss(pred.detach(), masks, gt_inds, OUT_STRIDE))
    assert list(want) == list(losses)
    for k in want:
        assert abs(float(losses[k]) - float(want[k])) <= 1e-5 * abs(float(want[k])), (k, float(losses[k]), float(want[k]))


def test_cuda_graph_capture():
    head, masks, labels, feat, params, coors, levels, img_inds, gt_inds, segm = _step_inputs(1)
    segm_head = _segm_head(80)
    feat_s = feat.clone().requires_grad_(True)
    par_s = params.clone().requires_grad_(True)
    seg_s = segm.clone().requires_grad_(True)

    def step():
        pred = head(feat_s, par_s, coors, levels, img_inds)
        lm = head.loss(None, None, pred, gt_inds, None, masks, labels)['loss_mask']
        ls = segm_head.loss(seg_s, masks, labels)['loss_segm']
        g = torch.autograd.grad(lm + ls, [feat_s, par_s, seg_s])
        return lm.detach(), ls.detach(), *g

    ref = [t.clone() for t in step()]
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(out, ref):
            assert torch.equal(a, b)
