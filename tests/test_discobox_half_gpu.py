"""GPU: the DiscoBox mask loss on float16 / bfloat16 logits (ops/discobox.py, csrc/discobox_loss.cu and
bxs_meanfield_forward_logits) against the float64 restatement in tests/discobox_half_oracle.py fed torch.sigmoid of the same
16-bit tensor; first-index arg-max on ties; the pseudo-label against MeanField.forward; the head's routing; determinism,
CUDA-graph replay and the absence of host synchronisation."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.discobox_half_oracle import disco_half_loss
from tests.helpers import tied_logits

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
DTYPES = [torch.float16, torch.bfloat16]
TOL_G = {torch.float16: 1e-3, torch.bfloat16: 8e-3}


def _targets(n, h, w, gen, zero=()):
    """binary uint8 targets: a box with a notch and a hole (not a rectangle) per instance; `zero`: all-zero instances"""
    t = torch.zeros(n, h, w, dtype=torch.uint8)
    for i in range(n):
        y0 = int(torch.randint(0, max(h // 2, 1), (1,), generator=gen))
        x0 = int(torch.randint(0, max(w // 2, 1), (1,), generator=gen))
        y1 = y0 + 1 + int(torch.randint(0, h - y0, (1,), generator=gen))
        x1 = x0 + 1 + int(torch.randint(0, w - x0, (1,), generator=gen))
        t[i, y0:y1, x0:x1] = 1
        if y1 - y0 > 2 and x1 - x0 > 2:
            t[i, y0, x0] = 0
            t[i, (y0 + y1) // 2, (x0 + x1) // 2] = 0
    for i in zero:
        t[i] = 0
    return t


def _mean_field(n_img, h, w, seed):
    from boxinstseg_b200.models.dense_heads.meanfield import MeanField
    gen = torch.Generator().manual_seed(seed)
    color = F.interpolate(torch.randn(n_img, 3, max(h // 8, 1), max(w // 8, 1), generator=gen), size=(h, w), mode='bilinear',
                          align_corners=True)
    return MeanField(color.to(DEV), alpha0=2.0, theta0=0.5, theta1=30.0, theta2=20.0, iter=10, kernel_size=3, base=0.1)


def _case(n, h, w, dt, seed, scale=3.0, zero=(0,), teacher=False):
    gen = torch.Generator().manual_seed(seed)
    x = (torch.randn(n, h, w, generator=gen) * scale).to(dt)
    xt = (torch.randn(n, h, w, generator=gen) * scale).to(dt) if teacher else None
    tg = _targets(n, h, w, gen, zero=[z for z in zero if z < n])
    ii = (torch.arange(n) % 2).to(torch.int32)
    return x, xt, tg, ii


def _run(x, xt, tg, ii, mf, use_ts=True, g_up=(1.0, 1.0)):
    from boxinstseg_b200.ops.discobox import discobox_mask_loss
    xg = x.to(DEV).requires_grad_(True)
    ni, nt, cnt = discobox_mask_loss(xg, tg.to(DEV), ii.to(DEV), mf, None if xt is None else xt.to(DEV), use_ts)
    (g,) = torch.autograd.grad(g_up[0] * ni + g_up[1] * nt, xg) if x.shape[0] else (torch.empty_like(xg),)
    return ni, nt, cnt, g


def _pseudo_ref(x, xt, tg, ii, mf):
    """the float32 mean field (MeanField.forward) on ((t + s) / 2).float(), computed by torch in the 16-bit dtype"""
    s = torch.sigmoid(x.to(DEV))
    t = s if xt is None else torch.sigmoid(xt.to(DEV))
    ret, _ = mf(((t + s) / 2).float().unsqueeze(1), tg.to(DEV).float().unsqueeze(1), obj_img=ii.to(DEV))
    return ret[:, 0].to(torch.uint8)


def _oracle(x, xt, tg, ii, mf, use_ts=True, g_up=(1.0, 1.0)):
    s = torch.sigmoid(x.to(DEV)).cpu()
    pseudo = _pseudo_ref(x, xt, tg, ii, mf).cpu() if use_ts else None
    return disco_half_loss(s, tg, pseudo, *g_up)


def _check(x, xt, tg, ii, mf, dt, use_ts=True, g_up=(1.0, 1.0)):
    ni, nt, cnt, g = _run(x, xt, tg, ii, mf, use_ts, g_up)
    oi, ot, oc, og = _oracle(x, xt, tg, ii, mf, use_ts, g_up)
    assert g.dtype == dt and g.shape == x.shape
    for a, b in ((ni.detach(), oi), (nt.detach(), ot)):
        assert abs(float(a) - float(b)) <= 1e-4 * abs(float(b)) + 1e-12, (float(a), float(b))
    assert float(cnt.detach()) == float(oc)
    gc = g.detach().cpu().double()
    if og.numel() and float(og.norm()) > 0:
        assert float((gc - og).norm() / og.norm()) <= TOL_G[dt]
    keep = tg.flatten(1).sum(1) > 0
    if (~keep).any():
        assert float(gc[~keep].abs().max()) == 0.0                     # weight 0: exactly zero
    return g


SHAPES = [(32, 200, 256), (1, 1, 1), (1, 1, 37), (1, 23, 1), (3, 17, 301), (1, 40, 50), (2, 33, 257)]


@pytest.mark.parametrize('dt', DTYPES)
@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_parity_with_oracle(dt, shape):
    n, h, w = shape
    mf = _mean_field(2, h, w, 1)
    x, xt, tg, ii = _case(n, h, w, dt, seed=n * 7 + h + w, zero=(0,) if n > 1 else ())
    _check(x, xt, tg, ii, mf, dt)


@pytest.mark.parametrize('dt', DTYPES)
def test_independent_teacher_and_no_teacher_term(dt):
    n, h, w = 6, 64, 80
    mf = _mean_field(2, h, w, 2)
    x, xt, tg, ii = _case(n, h, w, dt, seed=5, zero=(2,), teacher=True)
    _check(x, xt, tg, ii, mf, dt, g_up=(0.7, 1.3))
    _check(x, None, tg, ii, mf, dt, use_ts=False, g_up=(2.0, 0.0))
    _check(x, None, tg, ii, None, dt, use_ts=False)


@pytest.mark.parametrize('dt', DTYPES)
def test_empty_level(dt):
    from boxinstseg_b200.ops.discobox import discobox_mask_loss
    mf = _mean_field(1, 8, 8, 3)
    x = torch.zeros(0, 8, 8, dtype=dt, device=DEV, requires_grad=True)
    ni, nt, cnt = discobox_mask_loss(x, torch.zeros(0, 8, 8, dtype=torch.uint8, device=DEV), None, mf)
    (g,) = torch.autograd.grad(ni + nt, x)
    assert float(ni) == float(nt) == float(cnt) == 0.0 and g.shape == x.shape and g.dtype == dt


@pytest.mark.parametrize('dt', DTYPES)
@pytest.mark.parametrize('kind', ['saturated', 'quantised', 'constant', 'boundaries'])
def test_ties_go_to_first_index(dt, kind):
    n, h, w = 4, 70, 530
    gen = torch.Generator().manual_seed(17)
    x = tied_logits(n, h, w, dt, kind, gen)
    tg = _targets(n, h, w, gen, zero=(3,))
    ii = torch.zeros(n, dtype=torch.int32)
    mf = _mean_field(1, h, w, 4)
    # upstream gradients scaled as the reference's fp16 training scales its loss (loss_scale=512): near-saturated scores
    # give s * (1 - s) ~ 1e-4, whose products would otherwise be float16 subnormals
    g = _check(x, None, tg, ii, mf, dt, use_ts=False, g_up=(512.0, 0.0))
    *_, og = _oracle(x, None, tg, ii, mf, use_ts=False, g_up=(512.0, 0.0))
    assert torch.equal(g.detach().cpu() != 0, og.to(dt) != 0)         # support = the first-index arg-max set
    _check(x, None, tg, ii, mf, dt, g_up=(512.0, 512.0))               # and with the teacher term


@pytest.mark.parametrize('dt', DTYPES)
@pytest.mark.parametrize('teacher', [False, True])
@pytest.mark.parametrize('per_object', [False, True])
def test_pseudo_label_equals_meanfield_forward(dt, teacher, per_object):
    from boxinstseg_b200 import _lib as L
    from boxinstseg_b200.ops.discobox import HALF_DTYPES
    n, h, w = 9, 100, 128
    mf = _mean_field(2, h, w, 6)
    x, xt, tg, ii = _case(n, h, w, dt, seed=9, teacher=teacher)
    x = (x.float() * 0.3).to(dt)                                        # many pixels near the 0.5 threshold
    s, t, tgd, iid = x.to(DEV), None if xt is None else xt.to(DEV), tg.to(DEV), ii.to(DEV)
    lib = L.lib()
    ws = None if per_object else torch.empty(lib.bxs_meanfield_workspace_bytes(n, h, w), dtype=torch.uint8, device=DEV)
    out = torch.empty(n, h, w, dtype=torch.uint8, device=DEV)
    L.check(lib.bxs_meanfield_forward_logits(L.ptr(mf.kernel), L.ptr(iid), L.ptr(s), L.ptr(t), L.ptr(tgd), HALF_DTYPES[dt],
                                             mf._neglog.ctypes.data, L.ptr(out), L.ptr(ws), n, h, w, 3, mf.iter, L.stream()),
            'meanfield_forward_logits')
    ref = _pseudo_ref(x, xt, tg, ii, mf)
    assert torch.equal(out, ref)
    assert 0 < int(ref.sum()) < int(tg.sum())


def _head_inputs(dt, seed=0):
    gen = torch.Generator().manual_seed(seed)
    h, w = 100, 128
    color = F.interpolate(torch.randn(2, 3, 13, 16, generator=gen), size=(h, w), mode='bilinear', align_corners=True).to(DEV)
    preds, labels, inds = [], [], []
    for n in (5, 3):
        preds.append((torch.randn(n, h, w, generator=gen) * 3).to(dt).to(DEV))
        labels.append(_targets(n, h, w, gen, zero=(1,)).float().to(DEV))
        inds.append((torch.arange(n) % 2).to(torch.int32).to(DEV))
    return preds, labels, inds, color


@pytest.mark.parametrize('dt', DTYPES)
def test_head_routes_half_levels(dt):
    from boxinstseg_b200.models import build_head
    from boxinstseg_b200.models.dense_heads.meanfield import MeanField
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256))
    preds, labels, inds, color = _head_inputs(dt)
    leaves = [p.clone().requires_grad_(True) for p in preds]
    out = head.mask_loss(leaves, labels, inds, color)
    grads = torch.autograd.grad(out['loss_ins'] + out['loss_ts'], leaves)
    assert all(g.dtype == dt for g in grads)
    # the old composition on the same 16-bit predictions
    mf = MeanField(color, alpha0=head.alpha0, theta0=head.theta0, theta1=head.theta1, theta2=head.theta2,
                   iter=head.crf_max_iter, kernel_size=head.mkernel, base=head.crf_base)
    eager = [head._mask_loss_level_eager(p, None, i, t, mf, True) for p, i, t in zip(preds, inds, labels)]
    cnt = torch.stack([e[2] for e in eager]).sum().clamp(min=1.0)
    l_ins = torch.stack([e[0] for e in eager]).sum() / cnt
    l_ts = torch.stack([e[1] for e in eager]).sum() / cnt
    assert abs(float(out['loss_ins']) - float(l_ins)) <= 1e-3 * abs(float(l_ins))
    assert abs(float(out['loss_ts']) - float(l_ts)) <= 1e-3 * abs(float(l_ts))
    # float32 predictions still take the old composition
    out32 = head.mask_loss([p.float() for p in preds], labels, inds, color)
    assert out32['loss_ins'].dtype == torch.float32


def test_autocast_config_c_step_launches_new_kernels():
    import bench_configs
    from boxinstseg_b200.models import build_head
    _, info = bench_configs.build_C(torch.device(DEV), 0)
    d = info['data']
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256))
    feat = d['feat'].detach().half().requires_grad_(True)

    def step():
        with torch.autocast('cuda', dtype=torch.float16):
            pred = torch.cat([head.dynamic_conv(feat[b], d['kern'][b]) for b in range(2)])
            out = head.mask_loss([pred], [d['labels']], [d['img_inds']], d['color'])
        return torch.autograd.grad(out['loss_ins'] + out['loss_ts'], [feat, d['kern']])
    step()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        g = step()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert any('db_forward_kernel' in k for k in names) and any('db_backward_kernel' in k for k in names)
    assert any('mf_step_global' in k or 'mf_fused_kernel' in k for k in names)
    assert not any('prj_' in k for k in names), [k for k in names if 'prj_' in k]
    assert g[0].dtype == torch.float16


@pytest.mark.parametrize('dt', DTYPES)
def test_deterministic_graph_replay_and_sync_free(dt):
    from boxinstseg_b200.ops.discobox import discobox_mask_loss
    n, h, w = 12, 200, 256
    mf = _mean_field(2, h, w, 8)
    x, xt, tg, ii = _case(n, h, w, dt, seed=21, teacher=True)
    xs, xts, tgs, iis = x.to(DEV), xt.to(DEV), tg.to(DEV), ii.to(DEV)

    def once():
        leaf = xs.detach().requires_grad_(True)         # a fresh leaf per call: no autograd node outlives its call
        ni, nt, cnt = discobox_mask_loss(leaf, tgs, iis, mf, xts)
        (g,) = torch.autograd.grad(ni + 0.5 * nt, leaf)
        return torch.stack((ni, nt, cnt)).detach(), g

    a = once()
    b = once()
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        once()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        once()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        c = once()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(c[0], a[0]) and torch.equal(c[1], a[1])
    assert np.isfinite(a[0].detach().cpu().numpy()).all()
