"""GPU: Box2MaskHead's training loss.

1. ``ops.cross_entropy.softmax_cross_entropy_layers`` (csrc/cross_entropy.cu) against float64 ``F.cross_entropy(weight=w,
   reduction='none')`` + ``weight_reduce_loss``, bit-identical from run to run and without host synchronisation.
2. ``get_targets_layers`` equals L calls of ``get_targets`` bit for bit, with one matching launch per ``loss``.
3. ``loss`` against the golden minted from the reference's own methods, and against the restated reference lines
   (oracle/box2mask_loss.py with the package's GPU parts): small, config E's shapes, an image without ground truth, no
   ground truth at all, G > Q.  Losses and gradients within 1e-3.
4. ``loss`` without host synchronisation and, with the stand-in decoder of oracle/box2mask_head.py, forward + loss +
   backward in a CUDA graph; a NaN image; float16 / bfloat16 inputs."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import box2mask_head as obh
from oracle import box2mask_loss as obl
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


# ------------------------------------------------------------------------------------------------- 1. the kernel
def _ce_reference(scores, labels, cw, loss_weight):
    """float64 F.cross_entropy(weight=w, reduction='none') + weight_reduce_loss(avg_factor=w[labels].sum()), labels outside
    [0, K) dropped."""
    out = []
    for x, y in zip(scores, labels):
        x, y = x.double().flatten(0, 1), y.flatten()
        K = x.shape[1]
        w = torch.ones(K, dtype=torch.float64, device=x.device) if cw is None else cw.double()
        keep = (y >= 0) & (y < K)
        loss = F.cross_entropy(x[keep], y[keep], weight=w, reduction='none')
        out.append(loss_weight * loss.sum() / (w[y[keep]].sum() + torch.finfo(torch.float32).eps))
    return torch.stack(out)


def _ce_case(L, B, K, Q=100, seed=0, scale=3.0, labels='mixed'):
    gen = torch.Generator().manual_seed(seed)
    scores = [(torch.randn(B, Q, K, generator=gen) * scale).to(DEV) for _ in range(L)]
    if labels == 'background':
        y = torch.full((L, B, Q), K - 1, dtype=torch.long)
    elif labels == 'foreground':
        y = torch.randint(0, K - 1, (L, B, Q), generator=gen) if K > 1 else torch.zeros(L, B, Q, dtype=torch.long)
    else:
        y = torch.where(torch.rand(L, B, Q, generator=gen) < 0.2, torch.randint(0, K, (L, B, Q), generator=gen), K - 1)
    cw = torch.cat([torch.rand(K - 1, generator=gen) + 0.5, torch.tensor([0.1])]).to(DEV)
    return scores, y.to(DEV), cw


def _check_ce(scores, labels, cw, loss_weight):
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    xs = [s.clone().requires_grad_(True) for s in scores]
    got = softmax_cross_entropy_layers(xs, labels, cw, loss_weight)
    ref_x = [s.double().requires_grad_(True) for s in scores]
    want = _ce_reference(ref_x, labels, cw, loss_weight)
    assert got.shape == (len(scores),) and got.dtype == torch.float32
    assert torch.allclose(got.double(), want, rtol=1e-5, atol=1e-7), (got, want)
    up = torch.linspace(0.5, 2.0, len(scores), device=DEV)              # distinct upstream gradients per layer
    g_got = torch.autograd.grad((got * up).sum(), xs)
    g_want = torch.autograd.grad((want * up.double()).sum(), ref_x)
    for a, b in zip(g_got, g_want):
        scale = b.abs().max().item()
        assert (a.double() - b).abs().max().item() <= 1e-5 * max(scale, 1e-30)
    return got


@pytest.mark.parametrize('L', [1, 10])
@pytest.mark.parametrize('B', [1, 2, 8])
@pytest.mark.parametrize('K', [2, 81, 134])
def test_cross_entropy_matches_float64(L, B, K):
    scores, labels, cw = _ce_case(L, B, K, seed=L * 100 + B * 10 + K)
    _check_ce(scores, labels, cw, 2.0)


@pytest.mark.parametrize('labels', ['background', 'foreground'])
@pytest.mark.parametrize('loss_weight', [0.5, 1.0, 2.0])
def test_cross_entropy_label_extremes_and_weights(labels, loss_weight):
    scores, y, cw = _ce_case(3, 2, 81, seed=7, labels=labels)
    _check_ce(scores, y, cw, loss_weight)
    _check_ce(scores, y, None, loss_weight)                             # no class weight: all ones


def test_cross_entropy_large_logits_and_out_of_range_labels():
    scores, y, cw = _ce_case(10, 2, 134, seed=3, scale=30.0)
    scores = [s.clamp(-30, 30) for s in scores]
    y[0, 0, :5] = -1
    y[3, 1, 7] = 134
    y[9, 0, 50] = 10 ** 6                                               # adds nothing anywhere
    got = _check_ce(scores, y, cw, 2.0)
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    xs = [s.clone().requires_grad_(True) for s in scores]
    loss = softmax_cross_entropy_layers(xs, y, cw, 2.0)
    g = torch.autograd.grad(loss.sum(), xs)
    assert torch.equal(g[0][0, :5], torch.zeros_like(g[0][0, :5])) and torch.equal(g[3][1, 7], torch.zeros_like(g[3][1, 7]))
    assert torch.equal(loss, got)


def test_cross_entropy_bit_identical_and_sync_free():
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    scores, y, cw = _ce_case(10, 8, 134, seed=5)
    xs = [s.clone().requires_grad_(True) for s in scores]

    def run():
        loss = softmax_cross_entropy_layers(xs, y, cw, 2.0)
        return [loss] + list(torch.autograd.grad((loss * torch.arange(1., 11., device=DEV)).sum(), xs))
    first = run()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        again = [run() for _ in range(3)]
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for r in again:
        for a, b in zip(r, first):
            assert torch.equal(a, b)


def test_cross_entropy_second_backward():
    """retain_graph: a second backward through the same node gives the same gradient (the in-place one is spent)."""
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    scores, y, cw = _ce_case(2, 2, 81, seed=9)
    xs = [s.clone().requires_grad_(True) for s in scores]
    loss = softmax_cross_entropy_layers(xs, y, cw, 2.0)
    g1 = [g.clone() for g in torch.autograd.grad(loss.sum() * 3.0, xs, retain_graph=True)]
    g2 = torch.autograd.grad(loss.sum() * 3.0, xs)
    for a, b in zip(g1, g2):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------- 2. matching
def _head(Q=100, num_classes=80, class_weight=None):
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import Box2MaskHead
    cw = class_weight or [1.0] * num_classes + [0.1]
    return Box2MaskHead(num_queries=Q, num_things_classes=num_classes, num_stuff_classes=0,
                        loss_cls=dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=2.0, reduction='mean',
                                      class_weight=cw),
                        train_cfg=dict(assigner=obl.ASSIGNER, sampler=dict(type='MaskPseudoSampler')))


def _case(seed, Gs, Q=100, layers=3, num_classes=80, pred=64, mask=256, margin=6.0):
    """Device tensors of ``obl.golden_case`` at the given sizes."""
    cls, masks, lsts, labels, gts, img = obl.golden_case(seed=seed, B=len(Gs), gts=Gs, Q=Q, num_classes=num_classes,
                                                         layers=layers, pred=pred, mask=mask, margin=margin)
    to = lambda ts: [t.to(DEV) for t in ts]                                 # noqa: E731
    return to(cls), to(masks), to(lsts), to(labels), to(gts), img.to(DEV)


def test_get_targets_layers_equals_per_layer_get_targets():
    head = _head()
    for seed, Gs in [(0, (7, 0, 50)), (1, (100,)), (2, (150, 1))]:
        cls, masks, _, labels, gts, _ = _case(seed, Gs, layers=4)
        metas = [dict() for _ in Gs]
        got = head.get_targets_layers(cls, masks, labels, gts, metas)
        assert head.lsap_status.shape == (4, len(Gs)) and head.lsap_status.dtype == torch.int32
        assert head.lsap_status.eq(0).all()
        assert len(got) == 4
        for l in range(4):
            want = head.get_targets([c for c in cls[l]], [m for m in masks[l]], labels, gts, metas)
            for g_list, w_list in zip(got[l][:4], want[:4]):
                for g, w in zip(g_list, w_list):
                    assert g.dtype == w.dtype and torch.equal(g, w)
            assert got[l][4:] == want[4:]


def test_loss_matches_every_layer_in_one_launch(monkeypatch):
    from boxinstseg_b200.models.dense_heads import mask_loss_heads as mlh
    calls = []
    real = mlh.solve_batched
    monkeypatch.setattr(mlh, 'solve_batched', lambda costs: calls.append(len(costs)) or real(costs))
    head = _head()
    cls, masks, lsts, labels, gts, img = _case(3, (5, 2), layers=10, pred=32, mask=128)
    head.loss(cls, masks, lsts, labels, gts, [dict(), dict()], img)
    assert calls == [20]


# ------------------------------------------------------------------------------------------------- 3. the head's losses
def _run(fn, cls, masks, lsts):
    leaves = [[t.clone().requires_grad_(True) for t in ts] for ts in (cls, masks, lsts)]
    out = fn(*leaves)
    flat = [t for ts in leaves for t in ts]
    grads = torch.autograd.grad(sum(out.values()), flat, allow_unused=True)
    return out, [torch.zeros_like(t) if g is None else g for g, t in zip(grads, flat)]


def _compare(head, case, tol=1e-3):
    cls, masks, lsts, labels, gts, img = case
    Q, K = cls[0].shape[1:]
    metas = [dict() for _ in labels]
    out, grads = _run(lambda c, m, f: head.loss(c, m, f, labels, gts, metas, img), cls, masks, lsts)
    ref, ref_grads = _run(lambda c, m, f: obl.loss(obl.gpu_parts(head), Q, K - 1, head.cls_class_weight, head.cls_loss_weight,
                                                   c, m, f, labels, gts, img), cls, masks, lsts)
    assert list(out) == list(ref)
    for k in ref:
        a, b = out[k].item(), ref[k].item()
        assert abs(a - b) <= tol * max(abs(b), 1e-6), (k, a, b)
    for i, (a, b) in enumerate(zip(grads, ref_grads)):
        if b.abs().max() == 0:
            assert a.abs().max() == 0, i
        else:
            assert rel_err(a, b) <= tol, (i, rel_err(a, b))
    return out


def test_loss_against_the_golden():
    gold = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'box2mask_loss.npz'))
    head = _head(Q=8, num_classes=obl.GOLDEN_NUM_CLASSES, class_weight=obl.GOLDEN_CLASS_WEIGHT)
    cls, masks, lsts, labels, gts, img = (([t.to(DEV) for t in x] if isinstance(x, list) else x.to(DEV))
                                          for x in obl.golden_case())
    # the golden matched on the up-sampled cost, the head on the low-resolution profiles: the same queries, the same gts
    targets = head.get_targets_layers(cls, masks, labels, gts, [dict(), dict()])
    match = torch.from_numpy(gold['matches']).to(DEV)
    for l, t in enumerate(targets):
        for b in range(2):
            m = match[l * 2 + b]
            assert torch.equal(t[3][b] > 0, m >= 0)
            assert torch.equal(t[2][b].squeeze(1), gts[b][m[m >= 0]])
    out, grads = _run(lambda c, m, f: head.loss(c, m, f, labels, gts, [dict(), dict()], img), cls, masks, lsts)
    lines, line_grads = _run(lambda c, m, f: obl.loss(obl.gpu_parts(head), 8, obl.GOLDEN_NUM_CLASSES,
                                                      obl.GOLDEN_CLASS_WEIGHT, 2.0, c, m, f, labels, gts, img),
                             cls, masks, lsts)
    assert list(out) == list(gold['keys'])
    for k, v in out.items():
        assert abs(v.item() - float(gold[k])) <= 1e-3 * abs(float(gold[k])), (k, v.item(), float(gold[k]))
    # every gradient within 1e-3 of the golden and of the reference lines run on the package's GPU parts
    for i, (g, r) in enumerate(zip(grads, line_grads)):
        ref = torch.from_numpy(gold[f'grad_{i}']).to(DEV)
        assert rel_err(g, ref) <= 1e-3, (i, rel_err(g, ref))
        assert rel_err(g, r) <= 1e-3, (i, rel_err(g, r))


def test_loss_against_reference_lines_small():
    _compare(_head(Q=20, num_classes=10), _case(11, (4, 2), Q=20, layers=3, num_classes=10, pred=48, mask=192))


def test_loss_against_reference_lines_config_e_shapes():
    """B = 1, 10 layers (9 transformer layers + the query-feature head), Q = 100, 256x256 predictions, 1024x1024 box masks,
    8 ground truths."""
    _compare(_head(), _case(12, (8,), layers=10, pred=256, mask=1024))


def test_loss_image_without_ground_truth():
    out = _compare(_head(), _case(13, (5, 0), layers=2, pred=64, mask=256))
    assert all(torch.isfinite(v) for v in out.values())


def test_loss_without_any_ground_truth():
    head = _head()
    cls, masks, lsts, labels, gts, img = _case(14, (0, 0), layers=3, pred=32, mask=128)
    out = _compare(head, (cls, masks, lsts, labels, gts, img))
    for k, v in out.items():
        if 'loss_cls' not in k:
            assert v.item() == 0.0 and v.requires_grad, k


def test_loss_more_ground_truths_than_queries():
    _compare(_head(Q=100), _case(15, (150,), layers=2, pred=64, mask=256, margin=1.0))


def test_loss_single_is_one_layer_of_loss():
    head = _head()
    cls, masks, lsts, labels, gts, img = _case(16, (3, 1), layers=2, pred=32, mask=128)
    metas = [dict(), dict()]
    full = head.loss(cls, masks, lsts, labels, gts, metas, img)
    one = head.loss_single(cls[-1], masks[-1], lsts[-1], labels, gts, metas, img)
    assert len(one) == 3
    for v, k in zip(one, ('loss_cls', 'loss_project', 'loss_levelset')):
        assert torch.allclose(v, full[k], rtol=1e-6, atol=0), k


# ------------------------------------------------------------------------------------------------- 4. capture, NaN, dtypes
def test_loss_sync_free():
    head = _head()
    case = _case(17, (6, 3), layers=4, pred=64, mask=256)
    metas = [dict(), dict()]
    ref, ref_g = _run(lambda c, m, f: head.loss(c, m, f, *case[3:5], metas, case[5]), *case[:3])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        out, grads = _run(lambda c, m, f: head.loss(c, m, f, *case[3:5], metas, case[5]), *case[:3])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for k in ref:
        assert torch.equal(out[k], ref[k]), k
    for a, b in zip(grads, ref_g):
        assert torch.equal(a, b)


def test_forward_loss_backward_cuda_graph():
    """forward (stand-in decoder) + loss + backward: after one eager step, a captured graph replays bit-identically."""
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import Box2MaskHead
    attrs, feats = obh.standins(seed=3, Q=8, num_classes=4)
    head = obh.attach(Box2MaskHead(num_queries=8, num_things_classes=4, num_stuff_classes=0,
                                   train_cfg=dict(assigner=obl.ASSIGNER, sampler=dict(type='MaskPseudoSampler'))),
                      attrs).to(DEV)
    feats = [f.to(DEV) for f in feats]
    gen = torch.Generator().manual_seed(4)
    gts, labels = [], []
    for G in (3, 1):
        m = torch.zeros(G, 64, 64, dtype=torch.long)
        for g in range(G):
            m[g, 4 + 9 * g:30 + 9 * g, 6 + 7 * g:40 + 5 * g] = 1
        gts.append(m.to(DEV))
        labels.append(torch.randint(0, 4, (G,), generator=gen).to(DEV))
    img = torch.randn(2, 3, 64, 64, generator=gen).to(DEV)
    metas = [dict(), dict()]
    params = [p for p in head.parameters() if p.requires_grad]

    def step():
        cls, masks, lsts = head(feats, metas)
        out = head.loss(cls, masks, lsts, labels, gts, metas, img)
        total = sum(out.values())
        return [total] + list(out.values()) + list(torch.autograd.grad(total, params, allow_unused=True))

    eager = [t.detach().clone() if t is not None else None for t in step()]     # nothing of the eager graph kept alive
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(captured, eager):
            assert (a is None and b is None) or torch.equal(a, b)


def test_nan_image_gives_nan_loss_cls_without_raising():
    head = _head()
    cls, masks, lsts, labels, gts, img = _case(18, (4, 3), layers=3, pred=32, mask=128)
    cls[1] = cls[1].clone()
    cls[1][1, 5, 2] = float('nan')                                        # layer 1, image 1: a NaN row of costs
    out = head.loss(cls, masks, lsts, labels, gts, [dict(), dict()], img)
    assert head.lsap_status.tolist() == [[0, 0], [0, 1], [0, 0]]
    assert torch.isnan(out['d1.loss_cls'])
    assert torch.isfinite(out['loss_cls']) and torch.isfinite(out['d0.loss_cls'])


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_half_inputs_give_the_float32_result_of_their_promoted_copies(dtype):
    head = _head()
    cls, masks, lsts, labels, gts, img = _case(19, (4, 2), layers=3, pred=64, mask=256)
    cls_h, masks_h = [c.to(dtype) for c in cls], [m.to(dtype) for m in masks]
    metas = [dict(), dict()]
    out = head.loss(cls_h, masks_h, lsts, labels, gts, metas, img)
    want = head.loss([c.float() for c in cls_h], [m.float() for m in masks_h], lsts, labels, gts, metas, img)
    for k in want:
        assert out[k].dtype == torch.float32 and torch.equal(out[k], want[k]), k
    xs = [c.clone().requires_grad_(True) for c in cls_h]
    g = torch.autograd.grad(sum(head.loss(xs, masks_h, lsts, labels, gts, metas, img).values()), xs)
    assert all(t.dtype == dtype for t in g)


def test_grouped_tree_filter_edge_weight_gradient_is_fixed_order():
    """The level-set tree filter of ``mask_loss_single`` shares one tree per image among its instances (``tree_of``) and sums
    d/d edge_weight over them: in a fixed order (bit-identical from run to run, also with 5 instances on one tree), equal to
    the per-instance filter's gradient up to rounding, and an Inf in one image's instances does not reach another image."""
    head = _head()
    gen = torch.Generator().manual_seed(21)
    embed = torch.randn(2, 1, 96, 96, generator=gen).to(DEV)
    feature = torch.rand(7, 1, 96, 96, generator=gen).to(DEV)
    tree_of = torch.tensor([0, 0, 0, 0, 0, 1, 1], dtype=torch.int32, device=DEV)
    tree = head.mst(embed)
    order = head.tree_filter.order(tree, embed.shape)
    up = torch.randn(7, 1, 96, 96, generator=gen).to(DEV)

    def grouped(f=feature):
        e = embed.clone().requires_grad_(True)
        out = head.tree_filter(f, e, tree, low_tree=False, tree_of=tree_of, order=order)
        return torch.autograd.grad((out * up).sum(), e)[0]

    first = grouped()
    for _ in range(3):
        assert torch.equal(grouped(), first)
    e = embed.clone().requires_grad_(True)
    ii = tree_of.long()
    out = head.tree_filter(feature, e.index_select(0, ii), tree.index_select(0, ii), low_tree=False)
    (per_instance,) = torch.autograd.grad((out * up).sum(), e)
    assert rel_err(first, per_instance) <= 1e-5
    bad = feature.clone()
    bad[6, 0, 5, 5] = float('inf')                                       # an instance of image 1
    g = grouped(bad)
    assert torch.isfinite(g[0]).all() and torch.equal(g[0], first[0])
