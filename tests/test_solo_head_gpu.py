"""GPU: BoxSOLOv2Head's training ``forward`` + ``loss`` on the positive grid cells, and the focal kernel under it.

* ``sigmoid_focal_loss_levels`` against a float64 restatement of ``py_sigmoid_focal_loss`` + ``weight_reduce_loss``
  (1e-5 relative for the loss, 1e-5 of the gradient's scale), bit-identical from run to run, sync-free.
* ``head.forward`` + ``head.loss`` against the reference's lines (oracle/solo_head.py: dense conv over every cell,
  interpolate, boolean indexing, per-instance targets, torch focal lines) on the same stand-in towers: the three losses and
  every gradient within 1e-3 (the TF32 bar of the dynamic-convolution tests)."""
import warnings

import pytest
import torch

from oracle import solo_head as osh
from tests.helpers import rel_err, synth_boxes

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
GRIDS = [40, 36, 24, 16, 12]
HEAD = dict(type='BoxSOLOv2Head', num_classes=80, stacked_convs=4, strides=[8, 8, 16, 32, 32],
            scale_ranges=((1, 96), (48, 192), (96, 384), (192, 768), (384, 2048)), sigma=0.2, num_grids=GRIDS,
            cate_down_pos=0, loss_cate=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0))


# ------------------------------------------------------------------------------------------------------------------
# focal kernel
# ------------------------------------------------------------------------------------------------------------------
def _focal64(preds, labels, avg, gamma, alpha, w):
    """float64: py_sigmoid_focal_loss on the permuted / concatenated rows, a label outside [0, C) all-negative."""
    C = preds[0].shape[1]
    x = torch.cat([p.double().permute(0, 2, 3, 1).reshape(-1, C) for p in preds])
    lab = torch.cat([t.reshape(-1) for t in labels])
    t = (lab[:, None] == torch.arange(C, device=lab.device)[None]).double()
    p = x.sigmoid()
    pt = (1 - p) * t + p * (1 - t)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(x, t, reduction='none') * (alpha * t + (1 - alpha) * (1 - t)) * pt.pow(gamma)
    return w * loss.sum() / (avg + torch.finfo(torch.float32).eps)


def _focal_case(seed, kind, B=2, C=80, scale=2.0):
    gen = torch.Generator().manual_seed(seed)
    preds = [(torch.randn(B, C, S, S, generator=gen) * scale).to(DEV) for S in GRIDS]
    labels = [torch.full((B, S * S), C, dtype=torch.int64) for S in GRIDS]
    if kind != 'background':
        for t in labels:
            pos = torch.rand(t.shape, generator=gen) < 0.05
            t[pos] = torch.randint(0, C, (int(pos.sum()),), generator=gen)
    if kind == 'outside':
        labels[1][0, :7] = torch.tensor([-1, -100, C + 1, 1000, C, 0, C - 1])
    return preds, [t.to(DEV) for t in labels]


@pytest.mark.parametrize('kind', ['background', 'planted', 'outside'])
@pytest.mark.parametrize('gamma,alpha', [(0.0, 0.25), (1.0, 0.5), (2.0, 0.25), (2.0, 0.75)])
def test_focal_levels_vs_float64(kind, gamma, alpha):
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    preds, labels = _focal_case(int(gamma * 10 + alpha * 100), kind)
    avg = sum(int(((t >= 0) & (t < 80)).sum()) for t in labels) + 1
    xs = [p.clone().requires_grad_(True) for p in preds]
    loss = sigmoid_focal_loss_levels(xs, labels, torch.tensor(avg, device=DEV), gamma, alpha, 1.5)
    grads = torch.autograd.grad(loss * 3.0, xs)
    x64 = [p.double().requires_grad_(True) for p in preds]
    ref = _focal64(x64, labels, float(avg), gamma, alpha, 1.5)
    g64 = torch.autograd.grad(ref * 3.0, x64)
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()), (loss.item(), ref.item())
    scale = max(g.abs().max().item() for g in g64)
    for g, r in zip(grads, g64):
        assert g.shape == r.shape and (g.double() - r).abs().max().item() <= 1e-5 * scale


@pytest.mark.parametrize('gamma', [0.0, 1.0, 2.0])
def test_focal_levels_saturated_logits(gamma):
    """logits of +-30: the stable softplus keeps every term finite and exact to float32."""
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    preds, labels = _focal_case(3, 'planted', scale=1.0)
    preds = [torch.where(p > 0, 30.0, -30.0) for p in preds]
    xs = [p.clone().requires_grad_(True) for p in preds]
    loss = sigmoid_focal_loss_levels(xs, labels, 17.0, gamma, 0.25, 1.0)
    grads = torch.autograd.grad(loss, xs)
    x64 = [p.double().requires_grad_(True) for p in preds]
    ref = _focal64(x64, labels, 17.0, gamma, 0.25, 1.0)
    g64 = torch.autograd.grad(ref, x64)
    assert torch.isfinite(loss) and abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item())
    scale = max(g.abs().max().item() for g in g64)
    for g, r in zip(grads, g64):
        assert torch.isfinite(g).all() and (g.double() - r).abs().max().item() <= 1e-5 * scale


def test_focal_levels_bit_identical_and_sync_free():
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    preds, labels = _focal_case(11, 'planted')
    avg = torch.tensor(40, device=DEV)
    xs = [p.clone().requires_grad_(True) for p in preds]
    runs = []
    for _ in range(2):
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            loss = sigmoid_focal_loss_levels(xs, labels, avg)
            grads = torch.autograd.grad(loss, xs)
        finally:
            torch.cuda.set_sync_debug_mode(0)
        runs.append((loss, grads))
    assert torch.equal(runs[0][0], runs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))


# ------------------------------------------------------------------------------------------------------------------
# head forward + loss
# ------------------------------------------------------------------------------------------------------------------
def _case(seed, B, H, W, C, gts, boxes=None, mask_sizes=None):
    """FPN inputs (P2..P6), images, box-shaped ground-truth masks, and a head with seeded stand-in towers on the GPU.
    ``mask_sizes[b]``: the (H_b, W_b) of image b's masks, as mmdet pads them to each image's own pad shape."""
    from boxinstseg_b200.models import build_head
    gen = torch.Generator().manual_seed(seed)
    head = osh.attach_towers(build_head(dict(HEAD, in_channels=C, seg_feat_channels=C)), C, C, 80, seed=seed).to(DEV)
    feats = [torch.randn(B, C, -(-H // s), -(-W // s), generator=gen).to(DEV) for s in (4, 8, 16, 32, 64)]
    img = torch.randn(B, 3, H, W, generator=gen).to(DEV)
    bboxes, labels, masks = [], [], []
    for b in range(B):
        hb, wb = mask_sizes[b] if mask_sizes else (H, W)
        bx = boxes[b] if boxes is not None else synth_boxes(gen, gts[b], hb, wb, lo=12, hi=min(400, hb - 2))
        m = torch.zeros(len(bx), hb, wb, dtype=torch.uint8)
        for g, (x1, y1, x2, y2) in enumerate(bx.tolist()):
            m[g, int(y1):int(y2) + 1, int(x1):int(x2) + 1] = 1
        bboxes.append(bx.float().to(DEV))
        labels.append(torch.randint(0, 80, (len(bx),), generator=gen).to(DEV))
        masks.append(m.to(DEV))
    return head, feats, img, bboxes, labels, masks


def _grads(out, params):
    total = out['loss_boxpro'] + out['loss_levelset'] + out['loss_cate']
    return torch.autograd.grad(total, params, allow_unused=True)


def _run_new(head, feats, img, bboxes, labels, masks):
    xs = [f.clone().requires_grad_(True) for f in feats]
    ins, cate, lst = head(xs)
    out = head.loss(ins, cate, lst, bboxes, labels, masks, img, None, None)
    return out, _grads(out, xs + list(head.parameters()))


def _run_ref(head, feats, img, bboxes, labels, masks):
    xs = [f.clone().requires_grad_(True) for f in feats]
    ins, cate, lst = osh.forward(head, xs)
    out = osh.loss(head, ins, cate, lst, bboxes, labels, masks, img)
    return out, _grads(out, xs + list(head.parameters()))


def _run_ref_fp32(*case):
    """The reference lines with TF32 off in cuDNN and cuBLAS: how far the reference's own gradients move under a change of
    convolution precision."""
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    try:
        return _run_ref(*case)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved


def _compare(a, b, b32, tol=1e-3):
    """Losses within ``tol``.  Gradients: each within ``tol``, or within twice the distance between the reference's own
    TF32 and FP32 gradients of that tensor when that is larger -- the projection loss's row / column maxima route a
    gradient to one pixel, so rounding noise that swaps two nearly tied maxima moves the reference's own gradients by
    percents (at config D, 4.6 % between its TF32 and FP32 runs).  A gradient that is zero in exact arithmetic (the
    level-set branch's biases: the losses see only differences of its channels) holds rounding noise alone; it is compared
    against 1e-6 of the largest gradient instead."""
    (oa, ga), (ob, gb), (_, g32) = a, b, b32
    for k in ('loss_boxpro', 'loss_levelset', 'loss_cate'):
        assert abs(oa[k].item() - ob[k].item()) <= tol * abs(ob[k].item()), (k, oa[k].item(), ob[k].item())
    top = max(y.norm().item() for y in gb if y is not None)
    for i, (x, y, z) in enumerate(zip(ga, gb, g32)):
        if y is None or x is None:
            assert (x is None or not x.any()) and (y is None or not y.any()), i
        elif y.norm().item() <= 1e-6 * top:
            assert (x.double() - y.double()).norm().item() <= 1e-6 * top, i
        else:
            bar = max(tol, 2 * rel_err(z, y))
            assert rel_err(x, y) < bar, (i, rel_err(x, y), bar)
            if bar > tol:                       # a widened bar must hold against the other reference run as well
                assert rel_err(x, z) < bar, (i, rel_err(x, z), bar)


def test_head_small_vs_reference_lines():
    """2 images of 128x160, three ground truths each, 64 channels."""
    case = _case(0, 2, 128, 160, 64, [3, 3])
    _compare(_run_new(*case), _run_ref(*case), _run_ref_fp32(*case))


def test_head_config_d_vs_reference_lines_dense_path_never_runs(monkeypatch):
    """config D's shapes (2 x 800x1024, 8 ground truths per image, 256 channels).  The dense convolution is patched to raise
    during the step, and the step's peak allocation stays below the 1.59 GB of the dense output alone."""
    from boxinstseg_b200.models.dense_heads import mask_loss_heads as mlh
    case = _case(1, 2, 800, 1024, 256, [8, 8])
    ref, ref32 = _run_ref(*case), _run_ref_fp32(*case)

    def dense(*a, **k):
        raise AssertionError('the dense dynamic convolution ran during training')
    monkeypatch.setattr(mlh, 'solo_dynamic_conv', dense)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    new = _run_new(*case)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    assert peak < 2 * 3872 * 200 * 256 * 4, peak
    _compare(new, ref, ref32)


def test_loss_has_one_host_read():
    case = _case(2, 2, 128, 160, 64, [3, 3])
    head, feats, img, bboxes, labels, masks = case
    _run_new(*case)                                       # first call: allocator / module warm-up
    ins, cate, lst = head(feats)
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            head.loss(ins, cate, lst, bboxes, labels, masks, img, None, None)
        finally:
            torch.cuda.set_sync_debug_mode(0)
    syncs = [w for w in seen if 'synchroniz' in str(w.message)]
    assert len(syncs) == 1, [str(w.message) for w in syncs]


def test_loss_takes_either_forward():
    """``loss`` fed the reference's dense ins_preds equals ``loss`` fed ``SoloInsPreds``."""
    head, feats, img, bboxes, labels, masks = _case(3, 2, 128, 160, 64, [3, 4])
    ins, cate, lst = head(feats)
    a = head.loss(ins, cate, lst, bboxes, labels, masks, img, None, None)
    b = head.loss([p.dense() for p in ins], cate, lst, bboxes, labels, masks, img, None, None)
    r_ins, _, _ = osh.forward(head, feats)
    c = head.loss(r_ins, cate, lst, bboxes, labels, masks, img, None, None)
    for k in a:
        assert abs(a[k].item() - b[k].item()) <= 1e-3 * abs(b[k].item()), k
        assert abs(a[k].item() - c[k].item()) <= 1e-3 * abs(c[k].item()), k


def test_head_vs_reference_golden():
    """forward + loss on the GPU against tests/golden/solo_head.npz, minted from the reference's own BoxSOLOv2Head methods
    and FocalLoss on the CPU (FP32).  cuDNN / cuBLAS run in FP32 here, so the towers match the golden's arithmetic; the
    positive-cell convolution is TF32.  Losses within 1e-3; gradients (FPN inputs, levelset_bottom.weight) as ``_compare``
    judges them, with the reference lines run on the GPU with TF32 convolutions as the second reference."""
    import os
    import numpy as np
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'solo_head.npz'))
    head, feats, img, bboxes, labels, masks = osh.golden_case()
    case = (head.to(DEV), [f.to(DEV) for f in feats], img.to(DEV), [b.to(DEV) for b in bboxes], [l.to(DEV) for l in labels],
            [torch.from_numpy(m).to(DEV) for m in masks])
    wrt = lambda xs: xs + [head.levelset_bottom.weight]            # noqa: E731

    def run(lines):
        xs = [f.clone().requires_grad_(True) for f in case[1]]
        if lines:
            ins, cate, lst = osh.forward(head, xs)
            out = osh.loss(head, ins, cate, lst, *case[3:], case[2])
        else:
            ins, cate, lst = head(xs)
            out = head.loss(ins, cate, lst, *case[3:6], case[2], None, None)
        return out, torch.autograd.grad(out['loss_boxpro'] + out['loss_levelset'] + out['loss_cate'], wrt(xs))
    saved = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    try:
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        new = run(False)
        torch.backends.cudnn.allow_tf32 = True
        ref_tf32 = run(True)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = saved
    golden = ({k: torch.tensor(float(gold[k])) for k in ('loss_boxpro', 'loss_levelset', 'loss_cate')},
              [torch.from_numpy(gold[f'grad_{i}']).to(DEV) for i in range(len(new[1]))])
    _compare(new, golden, ref_tf32)


def test_head_masks_of_different_sizes_vs_reference_lines():
    """mmdet pads each image's masks to that image's own pad shape: a batch of 128x160 with one image's masks at 96x128."""
    case = _case(9, 2, 128, 160, 64, [3, 3], mask_sizes=[(128, 160), (96, 128)])
    _compare(_run_new(*case), _run_ref(*case), _run_ref_fp32(*case))


@pytest.mark.parametrize('name', ['image_without_gt', 'one_image', 'two_levels'])
def test_head_edge_cases_vs_reference_lines(name):
    """an image without ground truth; B = 1; a ground truth whose scale (sqrt area 64, in (1,96) and (48,192)) spans two
    levels."""
    if name == 'image_without_gt':
        case = _case(4, 2, 128, 160, 64, [3, 0])
    elif name == 'one_image':
        case = _case(5, 1, 128, 160, 64, [4])
    else:
        case = _case(6, 2, 128, 160, 64, None, boxes=[torch.tensor([[30.0, 20.0, 94.0, 84.0]]),
                                                      torch.tensor([[10.0, 10.0, 70.0, 80.0], [90.0, 40.0, 150.0, 120.0]])])
    _compare(_run_new(*case), _run_ref(*case), _run_ref_fp32(*case))


def test_head_17_images_vs_reference_lines():
    """17 images of 64x64, 64 channels: the positive-cell convolution runs in two groups (16 + 1 images)."""
    case = _case(10, 17, 64, 64, 64, [2] * 17)
    _compare(_run_new(*case), _run_ref(*case), _run_ref_fp32(*case))


def test_batch_without_positives():
    """no positive anywhere (no ground truth at all): zero mask losses on the graph, finite gradients, and loss_cate over the
    all-background labels (the reference raises at box_solov2_head.py:366)."""
    head, feats, img, bboxes, labels, masks = _case(7, 2, 128, 160, 64, [0, 0])
    out, grads = _run_new(head, feats, img, bboxes, labels, masks)
    assert out['loss_boxpro'].item() == 0 and out['loss_levelset'].item() == 0
    assert all(g is None or torch.isfinite(g).all() for g in grads)
    cate = osh.forward(head, feats)[1]
    ref = osh.py_sigmoid_focal_loss(torch.cat([c.permute(0, 2, 3, 1).reshape(-1, 80) for c in cate]),
                                    torch.zeros(sum(2 * s * s for s in GRIDS), 80, device=DEV), 2.0, 0.25, 1.0, 1.0)
    assert abs(out['loss_cate'].item() - ref.item()) <= 1e-4 * ref.item()      # float32 torch lines


def test_eval_forward_matches_reference_inference():
    head, feats, *_ = _case(8, 2, 128, 160, 64, [1, 1])
    with torch.no_grad():
        ins, cate, lst = head(feats, eval=True)
        r_ins, r_cate, r_lst = osh.forward(head, feats, eval=True)
    assert (lst - r_lst).abs().max().item() < 1e-5
    for c, rc in zip(cate, r_cate):
        assert c.shape == rc.shape and (c - rc).abs().max().item() < 1e-6
    for p, r in zip(ins, r_ins):
        assert p.shape == r.shape and (p - r).abs().max().item() < 1e-3
