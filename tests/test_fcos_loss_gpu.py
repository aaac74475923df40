"""CondInstBoxHead.loss on the GPU (condinst_head.py:364-476): the golden vectors minted from the reference's own code and
the float64 oracle at config A's shapes (2 images of 800x1024, 8 ground truths each, 80 classes) -- returned index
tensors bit for bit, losses within 1e-4 relative, every gradient within 1e-5 of its largest magnitude -- planted ties, a
batch without positives, float16 / bfloat16 inputs, strided and misaligned inputs, no host synchronisation, a CUDA-graph
capture of loss + backward, and the focal op on rectangular levels."""
import pytest
import torch

from oracle import fcos_loss as ofl
from oracle import fcos_targets as oft
from oracle.make_golden_fcos_loss import CASES, RANGES, STRIDES, case

pytestmark = pytest.mark.gpu
DEV = 'cuda'
KEYS = ('loss_cls', 'loss_bbox', 'loss_centerness')


def _head(C):
    from boxinstseg_b200.models import build_head
    return build_head(dict(type='CondInstBoxHead', num_classes=C, in_channels=256, strides=list(STRIDES),
                           loss_bbox=dict(type='GIoULoss', loss_weight=1.0)))


def _run(head, inputs, dtype=torch.float32, relayout=None):
    cls, bbox, ctr, boxes, labels = inputs
    leaves = [t.to(DEV, dtype).requires_grad_(True) for t in cls + bbox + ctr]
    n = len(cls)
    args = [relayout(t) if relayout else t for t in leaves]
    out = head.loss(args[:n], args[n:2 * n], args[2 * n:], [b.to(DEV) for b in boxes], [l.to(DEV) for l in labels], None)
    grads = torch.autograd.grad(sum(out[0].values()), leaves)
    return out, grads


def _check(out, grads, want, want_grads, n, bbox_tol=1e-5):
    for k in KEYS:
        w = float(want[0][k])
        assert abs(float(out[0][k]) - w) <= 1e-4 * abs(w) + 1e-7, (k, float(out[0][k]), w)
    assert torch.equal(out[1].cpu(), want[1].float())
    for a, b in zip(out[2:], want[2:]):
        assert a.dtype == torch.int64 and torch.equal(a.cpu(), b)
    for j in range(3):
        g = torch.cat([t.reshape(-1) for t in grads[j * n:(j + 1) * n]]).double().cpu()
        w = torch.cat([t.reshape(-1) for t in want_grads[j * n:(j + 1) * n]]).double()
        assert g.shape == w.shape
        scale = max(float(w.abs().max()), 1e-30)
        tol = bbox_tol if j == 1 else 1e-5
        assert float((g - w).abs().max()) <= tol * scale, (j, float((g - w).abs().max()) / scale)


def _oracle(inputs, C, dtype=torch.float64):
    cls, bbox, ctr, boxes, labels = inputs
    leaves = [t.to(dtype).clone().requires_grad_(True) for t in cls + bbox + ctr]
    n = len(cls)
    out = ofl.loss(leaves[:n], leaves[n:2 * n], leaves[2 * n:], boxes, labels, STRIDES, C)
    return out, torch.autograd.grad(sum(out[0].values()), leaves)


@pytest.mark.parametrize('seed,kw', CASES)
def test_golden(golden, seed, kw):
    g = golden('fcos_loss')
    inputs = case(seed, **kw)
    C, n = kw.get('C', 4), len(inputs[0])
    out, grads = _run(_head(C), inputs)
    want = ({k: torch.tensor(g[f's{seed}_{k}']) for k in KEYS}, torch.tensor(g[f's{seed}_points']),
            *[torch.tensor(g[f's{seed}_{k}']).long() for k in ('level_inds', 'img_inds', 'gt_inds')])
    sizes = [t.numel() for t in inputs[0] + inputs[1] + inputs[2]]
    flat = [torch.tensor(g[f's{seed}_g_{k}']) for k in ('cls', 'bbox', 'ctr')]
    want_grads = [*flat[0].split(sizes[:n]), *flat[1].split(sizes[n:2 * n]), *flat[2].split(sizes[2 * n:])]
    _check(out, grads, want, want_grads, n)
    if kw.get('no_pos'):
        assert float(out[0]['loss_bbox']) == 0 and float(out[0]['loss_centerness']) == 0
        assert out[0]['loss_bbox'].requires_grad and out[0]['loss_centerness'].requires_grad
        assert not any(t.any() for t in grads[n:])


def _config_a(seed=0, C=80, G=8):
    return case(seed, B=2, H=800, W=1024, G=(G,), C=C)


def test_config_a_against_the_oracle():
    """Against the reference's lines in float32 -- the precision ``@force_fp32`` runs them in -- and in float64.  The
    reference decodes stride-normalised distances around points in pixels (600 + 0.67 at config A), so each box corner
    carries up to ulp(point) / 2 of rounding: about 3e-5 of a small box's width at 800x1024.  The float32 reference and
    the kernel round those corners identically; against float64 the d/d bbox_pred bar is therefore 1e-4."""
    inputs = _config_a()
    out, grads = _run(_head(80), inputs)
    assert [tuple(t.shape[-2:]) for t in inputs[0]] == [(100, 128), (50, 64), (25, 32), (13, 16), (7, 8)]
    want, want_grads = _oracle(inputs, 80, torch.float32)
    assert int((want[4] >= 0).sum()) > 100
    _check(out, grads, want, want_grads, len(inputs[0]))
    want, want_grads = _oracle(inputs, 80)
    _check(out, grads, want, want_grads, len(inputs[0]), bbox_tol=1e-4)


def test_centerness_targets_bit_exact_with_the_reference_on_cuda():
    from boxinstseg_b200.ops.fcos import fcos_box_stats, fcos_points
    cls, bbox, ctr, boxes, labels = _config_a(3)
    head = _head(80)
    sizes = [tuple(t.shape[-2:]) for t in cls]
    pts = fcos_points(sizes, STRIDES, DEV)
    for p, q in zip(pts, oft.grid_points(sizes, STRIDES)):
        assert torch.equal(p.cpu(), q)
    lab, tgt, _ = head.get_targets(pts, [b.to(DEV) for b in boxes], [l.to(DEV) for l in labels])
    f_lab, f_tgt = torch.cat(lab), torch.cat(tgt)
    pos = ((f_lab >= 0) & (f_lab < 80)).nonzero().reshape(-1)
    ct = ofl.centerness_target(f_tgt[pos])                  # the reference's lines, on CUDA
    stats = fcos_box_stats(lab, tgt, sizes, STRIDES, 2, 80)
    assert float(stats[0]) == len(pos)
    assert abs(float(stats[1]) - float(ct.double().sum())) <= 1e-5 * float(ct.double().sum())
    # the kernel's per-point targets: d loss_centerness / d logit = (sigmoid(x) - ct) / num_pos with a zero logit
    zeros = [torch.zeros(2, 1, h, w, device=DEV, requires_grad=True) for h, w in sizes]
    from boxinstseg_b200.ops.fcos import fcos_box_losses
    den = torch.tensor([1.0, 1.0], device=DEV)
    _, l_ctr = fcos_box_losses([torch.ones(2, 4, h, w, device=DEV) for h, w in sizes], zeros, lab, tgt, den, STRIDES, 80)
    g = torch.autograd.grad(l_ctr, zeros)
    flat = torch.cat([t.permute(0, 2, 3, 1).reshape(-1) for t in g])[pos]
    assert torch.equal(flat, (0.5 - ct) * (1.0 / (1.0 + torch.finfo(torch.float32).eps)))


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_half_inputs_are_promoted(dtype):
    inputs = case(5, B=2, H=160, W=224, C=4)
    rounded = [[t.to(dtype).double() for t in part] for part in inputs[:3]] + list(inputs[3:])
    head = _head(4)
    out, grads = _run(head, inputs, dtype=dtype)
    ref, ref_grads = _run(head, rounded)
    for k in KEYS:
        assert out[0][k].dtype == torch.float32 and torch.equal(out[0][k], ref[0][k])
    for g, r in zip(grads, ref_grads):
        assert g.dtype == dtype and torch.equal(g, r.to(dtype))


_KINDS = {
    'transposed': lambda t: t.transpose(-1, -2).contiguous().transpose(-1, -2),
    'channels_last': lambda t: t.contiguous(memory_format=torch.channels_last),
    'sliced': lambda t: torch.zeros(t.shape[:-1] + (2 * t.shape[-1],), device=t.device, dtype=t.dtype)
    .index_copy(-1, torch.arange(0, 2 * t.shape[-1], 2, device=t.device), t)[..., ::2],
    'offset1': lambda t: torch.cat([t.new_zeros(1), t.reshape(-1)])[1:].view(t.shape),
}


@pytest.mark.parametrize('kind', sorted(_KINDS))
def test_layouts(kind):
    inputs = case(6, B=2, H=160, W=224, C=4)
    head = _head(4)
    ref, ref_grads = _run(head, inputs)
    out, grads = _run(head, inputs, relayout=_KINDS[kind])
    for k in KEYS:
        assert torch.equal(out[0][k], ref[0][k])
    for g, r in zip(grads, ref_grads):
        assert g.shape == r.shape and torch.equal(g, r)


def test_no_host_synchronisation_and_fixed_launches():
    from torch.profiler import ProfilerActivity, profile
    head = _head(80)
    counts = []
    for G in (1, 8, 40):
        inputs = _config_a(7, G=G)
        cls, bbox, ctr, boxes, labels = inputs
        leaves = [t.to(DEV, torch.float32).requires_grad_(True) for t in cls + bbox + ctr]
        bx, lb = [b.to(DEV) for b in boxes], [l.to(DEV) for l in labels]
        n = len(cls)
        head.loss(leaves[:n], leaves[n:2 * n], leaves[2 * n:], bx, lb, None)       # warm-up
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            torch.cuda.set_sync_debug_mode('error')
            try:
                out = head.loss(leaves[:n], leaves[n:2 * n], leaves[2 * n:], bx, lb, None)
                torch.autograd.backward(sum(out[0].values()))
            finally:
                torch.cuda.set_sync_debug_mode(0)
            torch.cuda.synchronize()
        counts.append(sum(1 for e in prof.events() if e.device_type.name == 'CUDA' and 'emcpy' not in e.name))
    assert counts[0] == counts[1] == counts[2], counts


def test_cuda_graph_replay_is_bit_identical():
    inputs = _config_a(8)
    cls, bbox, ctr, boxes, labels = inputs
    head = _head(80)
    n = len(cls)
    leaves = [t.to(DEV, torch.float32).requires_grad_(True) for t in cls + bbox + ctr]
    bx, lb = [b.to(DEV) for b in boxes], [l.to(DEV) for l in labels]

    def step():
        out = head.loss(leaves[:n], leaves[n:2 * n], leaves[2 * n:], bx, lb, None)
        grads = torch.autograd.grad(sum(out[0].values()), leaves)
        # detached: a loss kept alive with its graph would keep the eager AccumulateGrad nodes on the default stream
        return [out[0][k].detach() for k in KEYS] + list(out[1:]) + list(grads)

    eager = step()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        step()
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = step()
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(static, eager):
            assert torch.equal(a, b)


def test_each_loss_differentiates_into_its_own_inputs():
    inputs = case(0)
    cls, bbox, ctr, boxes, labels = inputs
    n = len(cls)
    leaves = [t.to(DEV, torch.float32).requires_grad_(True) for t in cls + bbox + ctr]
    out = _head(4).loss(leaves[:n], leaves[n:2 * n], leaves[2 * n:], [b.to(DEV) for b in boxes],
                        [l.to(DEV) for l in labels], None)
    g = torch.autograd.grad(out[0]['loss_bbox'], leaves, allow_unused=True, retain_graph=True)
    assert all(t is None for t in g[:n] + g[2 * n:]) and all(t is not None for t in g[n:2 * n])
    g2 = torch.autograd.grad(out[0]['loss_bbox'] * 3.0, leaves[n:2 * n])      # a second backward, scaled
    for a, b in zip(g[n:2 * n], g2):
        assert torch.allclose(b, 3.0 * a, rtol=1e-6, atol=0)


def test_focal_on_rectangular_levels_against_the_oracle():
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    gen = torch.Generator().manual_seed(11)
    B, C = 2, 7
    sizes = [(13, 21), (7, 11), (3, 1), (1, 5)]
    preds = [torch.randn(B, C, h, w, generator=gen, dtype=torch.float64) * 3 for h, w in sizes]
    labels = [torch.randint(0, C + 1, (B, h * w), generator=gen) for h, w in sizes]
    x = [p.to(DEV, torch.float32).requires_grad_(True) for p in preds]
    loss = sigmoid_focal_loss_levels(x, [l.to(DEV) for l in labels], torch.tensor(9.0, device=DEV), 2.0, 0.25, 1.5)
    gx = torch.autograd.grad(loss, x)
    leaves = [p.clone().requires_grad_(True) for p in preds]
    flat = torch.cat([p.permute(0, 2, 3, 1).reshape(-1, C) for p in leaves])
    lab = torch.cat([l.reshape(B, h, w).reshape(-1) for l, (h, w) in zip(labels, sizes)])
    onehot = torch.nn.functional.one_hot(lab, C + 1)[:, :C]
    want = 1.5 * (ofl.focal_elementwise(flat, onehot).sum() / (9.0 + ofl.FLT_EPS))
    want_g = torch.autograd.grad(want, leaves)
    assert abs(float(loss) - float(want)) <= 1e-5 * float(want)
    for g, w in zip(gx, want_g):
        assert float((g.double().cpu() - w).abs().max()) <= 1e-5 * float(w.abs().max())
