"""GPU: DiscoBoxSOLOv2Head.loss and the packed dynamic convolution under it.
  * bxs_disco_cells_pack / _unpack_grad against a float64 torch gather / index_add restatement: repeated cells summed in row
    order, zero padding rows, bit-identical backward passes, a bad cell reported through the status word;
  * disco_cells_conv == one dynconv1x1 call per (level, image), bit for bit, in float32, float16 and bfloat16;
  * loss against the golden vectors of the reference (float32) and against the oracle on the same 16-bit convolution outputs
    (autocast float16 / bfloat16), every flag combination, an image without ground truth, an image and a level without
    covered cells, a level whose targets are all zero;
  * the correspondence branch is corr_loss_levels plus the reference's assembly;
  * host reads: only the target builder's."""
import warnings

import numpy as np
import pytest
import torch

from oracle import discobox_loss as odl
from oracle.make_golden_discobox_loss import CASES, CFG, FLAGS, GRIDS, NUM_CLASSES, case

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
BANK_CFG = dict(feat_height=7, feat_width=7, mask_height=28, mask_width=28, min_size=8, len_object_queues=10, fg_iou_thresh=0.7,
                bg_iou_thresh=0.7, ratio_range=[0.9, 1.2], appear_thresh=0.7, max_retrieval_objs=5)
LOSS_CORR = dict(loss_weight=1.0, corr_exp=1.0, corr_eps=0.05, gaussian_filter_size=3, low_score=0.3, corr_num_iter=10,
                 corr_num_smooth_iter=1, dist_kernel=9, obj_bank=BANK_CFG)


# ------------------------------------------------------------------------------------------------------ pack / unpack
def _cells_case(seed, B=3, C=64, grids=(40, 36, 24, 16, 12)):
    gen = torch.Generator().manual_seed(seed)
    orders = []
    for S in grids:
        per = []
        for b in range(B):
            n = int(torch.randint(0, 40, (1,), generator=gen)) if (b + S) % 5 else 0
            c = torch.randint(0, S * S, (n,), generator=gen)
            if n > 4:
                c[n // 2:n // 2 + 3] = c[1]                                 # a cell repeated 4 times, not adjacent
            per.append(c)
        orders.append(per)
    grids_t = [torch.randn(B, C, S, S, generator=gen) for S in grids]
    return grids_t, orders


def _pack_ref(grids, orders, I_pad):
    B, C = grids[0].shape[:2]
    out = torch.zeros(B, I_pad, C, dtype=torch.float64)
    for b in range(B):
        rows = torch.cat([g[b].reshape(C, -1)[:, o[b]].t().double() for g, o in zip(grids, orders)])
        out[b, :rows.shape[0]] = rows
    return out


def _unpack_ref(g_packed, grids, orders, acc_dtype):
    """index_add of every row into its cell, one row at a time in row order, accumulated in ``acc_dtype``."""
    B, C = grids[0].shape[:2]
    outs = [torch.zeros(g.shape, dtype=acc_dtype).reshape(B, C, -1) for g in grids]
    for b in range(B):
        r = 0
        for lv, o in enumerate(orders):
            for k in range(o[b].numel()):
                outs[lv][b][:, o[b][k]] += g_packed[b, r + k].to(acc_dtype)
            r += o[b].numel()
    return [o.view(g.shape) for o, g in zip(outs, grids)]


@pytest.mark.parametrize('dt', DTYPES)
def test_pack_and_unpack_against_torch(dt):
    from boxinstseg_b200.ops.dynconv import _DiscoPack
    grids, orders = _cells_case(1)
    B = grids[0].shape[0]
    counts = [int(orders[l][b].numel()) for l in range(len(grids)) for b in range(B)]
    I_pad = max(sum(counts[l * B + b] for l in range(len(grids))) for b in range(B))
    cells = torch.cat([orders[l][b] for l in range(len(grids)) for b in range(B)]).to(DEV, torch.int32)
    leaves = [g.to(DEV, dt).requires_grad_(True) for g in grids]
    packed = _DiscoPack.apply(counts, I_pad, cells, *leaves)
    assert packed.dtype == dt and packed.shape == (B, I_pad, grids[0].shape[1])
    want = _pack_ref([g.to(dt) for g in grids], orders, I_pad)
    assert torch.equal(packed.cpu().double(), want)                                   # a gather: exact, zero padding
    g_up = torch.randn(packed.shape, generator=torch.Generator().manual_seed(2)).to(DEV, dt)
    g1 = torch.autograd.grad(packed, leaves, g_up, retain_graph=True)
    g2 = torch.autograd.grad(packed, leaves, g_up)
    assert all(torch.equal(a, b) for a, b in zip(g1, g2))
    exact = _unpack_ref(g_up.cpu(), grids, orders, torch.float32)      # FP32 in row order, rounded once: bit for bit
    ref64 = _unpack_ref(g_up.cpu(), grids, orders, torch.float64)
    tol = {torch.float32: 1e-6, torch.float16: 2 ** -10, torch.bfloat16: 2 ** -7}[dt]
    for got, w, w64 in zip(g1, exact, ref64):
        assert got.dtype == dt
        assert torch.equal(got.cpu(), w.to(dt))
        assert torch.allclose(got.cpu().double(), w64, rtol=tol, atol=1e-5)
        untouched = w64 == 0
        assert torch.equal(got.cpu()[untouched], torch.zeros_like(got.cpu()[untouched]))


def test_pack_reports_a_bad_cell():
    from boxinstseg_b200 import _lib as L
    from boxinstseg_b200.ops.dynconv import _i64, _ptrs
    grid = torch.randn(1, 32, 4, 4, device=DEV)
    cells = torch.tensor([3, 16, -1, 5], dtype=torch.int32, device=DEV)
    packed = torch.full((1, 4, 32), 7.0, device=DEV)
    status = torch.zeros(1, dtype=torch.int32, device=DEV)
    L.check(L.lib().bxs_disco_cells_pack(_ptrs([grid]), _i64([4]), _i64([4]), L.ptr(cells), 4, L.ptr(packed), L.ptr(status), 1,
                                         1, 32, 4, 0, L.stream()), 'disco_cells_pack')
    assert int(status) == -1
    assert torch.equal(packed[0, 1:3], torch.zeros(2, 32, device=DEV))
    assert torch.equal(packed[0, 0], grid[0].reshape(32, -1)[:, 3]) and torch.equal(packed[0, 3], grid[0].reshape(32, -1)[:, 5])


# ------------------------------------------------------------------------------------------------ batched convolution
def _head(**kw):
    from boxinstseg_b200.models import build_head
    return build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=NUM_CLASSES, in_channels=256, num_grids=list(GRIDS),
                           scale_ranges=CFG['scale_ranges'], strides=CFG['strides'], sigma=CFG['sigma'], **kw))


def _gpu_case(seed, dt=torch.float32, **kw):
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = case(seed, **kw)
    d = lambda t: t.to(DEV, dt)                                          # noqa: E731
    return ([d(t) for t in cate], [d(t) for t in s_k], [d(t) for t in t_k], d(s_in), d(t_in),
            [b.to(DEV) for b in boxes], [l.to(DEV) for l in labels], [torch.from_numpy(m).to(DEV) for m in masks], d(img))


@pytest.mark.parametrize('dt', DTYPES)
@pytest.mark.parametrize('teacher', [False, True])
def test_batched_conv_equals_per_level_image(dt, teacher):
    head = _head()
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = _gpu_case(0)
    ctx = torch.autocast('cuda', dtype=dt) if dt != torch.float32 else torch.autocast('cuda', enabled=False)
    with ctx:
        new = head.corr_inputs(s_k, t_k, s_in, t_in, boxes, labels, masks, use_ind_teacher=teacher, best=False)
        old = head.corr_inputs(s_k, t_k, s_in, t_in, boxes, labels, masks, use_ind_teacher=teacher, best=False,
                               conv=head.dynamic_conv)
    for a_list, b_list in zip(new, old):
        for a, b in zip(a_list, b_list):
            assert (a is None) == (b is None)
            if a is not None:
                assert a.dtype == b.dtype and torch.equal(a, b)
    assert any(p is not None and p.dtype == dt for p in new[0])


@pytest.mark.parametrize('dt', DTYPES)
def test_batched_conv_equals_per_level_image_beyond_16_images(dt):
    """17 images: the kernels are packed in two groups (16 + 1 images, one bxs_disco_cells_pack call each, the batch's
    I_pad) and convolved in one dynconv1x1 call; every network's rows and image indices equal one convolution per (level,
    image), bit for bit."""
    head = _head()
    G = (3, 4, 3, 5, 3, 3, 4, 3, 3, 4, 3, 5, 3, 3, 4, 3, 3)
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = _gpu_case(2, G=G, empty_image=2)   # image 2: no covered cell
    assert s_in.shape[0] == 17
    ctx = torch.autocast('cuda', dtype=dt) if dt != torch.float32 else torch.autocast('cuda', enabled=False)
    with ctx:
        new = head.corr_inputs(s_k, t_k, s_in, t_in, boxes, labels, masks, use_ind_teacher=True, best=False)
        old = head.corr_inputs(s_k, t_k, s_in, t_in, boxes, labels, masks, use_ind_teacher=True, best=False,
                               conv=head.dynamic_conv)
    assert {int(i) for i in torch.cat([i for i in new[2] if i is not None])} == set(range(17)) - {2}
    for a_list, b_list in zip(new, old):
        for a, b in zip(a_list, b_list):
            assert (a is None) == (b is None)
            if a is not None:
                assert a.dtype == b.dtype and torch.equal(a, b)


# ---------------------------------------------------------------------------------------------------------- the loss
def _run_loss(head, inputs, ts, ind, use_corr=False, s_feat=None, t_feat=None):
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = inputs
    leaves = [t.detach().clone().requires_grad_(True) for t in cate + s_k + [s_in]]
    n = len(cate)
    out = head.loss(leaves[:n], leaves[n:2 * n], t_k, leaves[2 * n], t_in, boxes, labels, masks, None, None, img=img,
                    use_loss_ts=ts, use_ind_teacher=ind, use_corr=use_corr, s_feat=s_feat, t_feat=t_feat)
    grads = torch.autograd.grad(sum(out.values()), leaves, allow_unused=True)
    grads = [torch.zeros_like(x) if g is None else g for x, g in zip(leaves, grads)]
    n = len(GRIDS)
    return out, (torch.cat([g.reshape(-1) for g in grads[:n]]), torch.cat([g.reshape(-1) for g in grads[n:2 * n]]), grads[-1])


def _close(got, want, tol, what):
    got, want = got.detach().double().cpu().reshape(-1), want.detach().double().cpu().reshape(-1)
    scale = max(float(want.abs().max()), 1e-12)
    err = float((got - want).abs().max()) / scale
    assert err <= tol, f'{what}: {err:.3g} > {tol}'


RUNS = [(seed, kw, ts, ind) for seed, kw, flags in CASES for ts, ind in flags]


@pytest.mark.parametrize('seed,kw,ts,ind', RUNS, ids=[f's{r[0]}_ts{int(r[2])}_ind{int(r[3])}' for r in RUNS])
def test_float32_loss_against_reference_golden(golden, seed, kw, ts, ind):
    g = golden('discobox_loss')
    tag = f's{seed}_ts{int(ts)}_ind{int(ind)}'
    out, grads = _run_loss(_head(), _gpu_case(seed, **kw), ts, ind)
    for k in ('loss_ins', 'loss_ts', 'loss_cate', 'loss_corr'):
        assert out[k].dtype == torch.float32 and out[k].dim() == 0
        _close(out[k], torch.from_numpy(np.array(g[f'{tag}_{k}'])), 1e-3, k)
    _close(grads[0], torch.from_numpy(g[f's{seed}_g_cate']), 1e-3, 'g_cate')
    # the convolutions run on TF32 operands (10-bit mantissa): where a MIL row / column maximum is nearly tied it can pick
    # another pixel than the float64 reference and move single gradient entries, so these two are compared by norm
    for name, got in zip(('g_kern', 'g_ins'), grads[1:]):
        want = torch.from_numpy(g[f'{tag}_{name}']).double()
        err = float((got.detach().cpu().double().reshape(-1) - want.reshape(-1)).norm() / want.norm())
        assert err <= REL_NORM_TF32, f'{name}: {err:.3g}'
    # against the oracle fed the same TF32 convolution: everything within 1e-3
    want, w_grads = _oracle_same_conv(_gpu_case(seed, **kw), ts, ind, None)
    for k in ('loss_ins', 'loss_ts', 'loss_cate', 'loss_corr'):
        _close(out[k], want[k], 1e-3, k)
    for name, got, w in zip(('g_cate', 'g_kern', 'g_ins'), grads, w_grads):
        _close(got, w, 1e-3, name)


REL_NORM_TF32 = 1e-3


def _oracle_same_conv(inputs, ts, ind, dt):
    """The oracle on the GPU with the convolutions of the product's per-(level, image) path, under the same autocast (dt
    None: none)."""
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import DiscoBoxSOLOv2Head
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = inputs
    leaves = [t.detach().clone().requires_grad_(True) for t in cate + s_k + [s_in]]
    n = len(cate)
    with torch.autocast('cuda', dtype=dt or torch.float16, enabled=dt is not None):
        out = odl.loss(leaves[:n], leaves[n:2 * n], t_k, leaves[2 * n], t_in, [b.cpu() for b in boxes],
                       [l.cpu() for l in labels], [m.cpu().numpy() for m in masks], img, GRIDS, NUM_CLASSES, ts, ind, CFG,
                       conv=DiscoBoxSOLOv2Head.dynamic_conv)
    grads = torch.autograd.grad(sum(out.values()), leaves, allow_unused=True)
    grads = [torch.zeros_like(x) if g is None else g for x, g in zip(leaves, grads)]
    n = len(GRIDS)
    return out, (torch.cat([g.reshape(-1) for g in grads[:n]]), torch.cat([g.reshape(-1) for g in grads[n:2 * n]]), grads[-1])


TOL16 = {torch.float16: (1e-3, 1e-2), torch.bfloat16: (8e-3, 3e-2)}


@pytest.mark.parametrize('dt', [torch.float16, torch.bfloat16])
@pytest.mark.parametrize('ts,ind', FLAGS)
def test_autocast_loss_against_oracle(dt, ts, ind):
    inputs = _gpu_case(0)
    with torch.autocast('cuda', dtype=dt):
        out, grads = _run_loss(_head(), inputs, ts, ind)
    want, w_grads = _oracle_same_conv(inputs, ts, ind, dt)
    tl, tg = TOL16[dt]
    for k in ('loss_ins', 'loss_ts', 'loss_cate', 'loss_corr'):
        _close(out[k], want[k], tl, k)
    for name, got, w in zip(('g_cate', 'g_kern', 'g_ins'), grads, w_grads):
        _close(got, w, tg, name)


def test_empty_cases_against_oracle():
    """An image without ground truth (the reference cannot take one: its target builder indexes gt_labels_raw[0]) gives the
    losses of the same image with ground truths that cover no cell; a ground truth whose 1/4-scale mask vanishes makes a
    level whose targets are all zero, which the reference skips."""
    head = _head()
    inputs = list(_gpu_case(1, G=(5, 3), empty_image=1))
    out, grads = _run_loss(head, inputs, True, True)
    none = list(inputs)
    none[5] = [inputs[5][0], inputs[5][1][:0]]
    none[6] = [inputs[6][0], inputs[6][1][:0]]
    none[7] = [inputs[7][0], inputs[7][1][:0]]
    out0, grads0 = _run_loss(head, none, True, True)
    for k in out:
        assert torch.equal(out[k], out0[k]), k
    for a, b in zip(grads, grads0):
        assert torch.equal(a, b)
    # a single-pixel mask inside a box of the first level's range: its 1/4 rescale is all zero
    vanish = list(inputs)
    boxes0, masks0 = inputs[5][0].clone(), inputs[7][0].clone()
    boxes0[0] = torch.tensor([10., 10., 22., 22.], device=DEV)
    masks0[0] = 0
    masks0[0, 13, 13] = 1
    vanish[5] = [boxes0, inputs[5][1]]
    vanish[7] = [masks0, inputs[7][1]]
    out, grads = _run_loss(head, vanish, True, False)
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = vanish
    leaves = [t.detach().clone().requires_grad_(True) for t in cate + s_k + [s_in]]
    n = len(cate)
    want = odl.loss(leaves[:n], leaves[n:2 * n], t_k, leaves[2 * n], t_in, [b.cpu() for b in boxes], [l.cpu() for l in labels],
                    [m.cpu().numpy() for m in masks], img, GRIDS, NUM_CLASSES, True, False, CFG,
                    conv=lambda f, k: head.dynamic_conv(f, k))
    for k in out:
        _close(out[k], want[k], 1e-4, k)
    assert all(torch.isfinite(g).all() for g in grads)


def test_corr_branch_is_corr_loss_levels_plus_assembly():
    inputs = _gpu_case(0)
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = inputs
    gen = torch.Generator().manual_seed(5)
    s_feat = torch.randn(2, 32, *s_in.shape[-2:], generator=gen).to(DEV)
    t_feat = torch.randn(2, 32, *s_in.shape[-2:], generator=gen).to(DEV)
    a, b = _head(loss_corr=LOSS_CORR), _head(loss_corr=LOSS_CORR)
    out, _ = _run_loss(a, inputs, True, False, use_corr=True, s_feat=[s_feat], t_feat=[t_feat])
    from boxinstseg_b200.ops.resize import bilinear_resize
    color = bilinear_resize(img, tuple(s_in.shape[-2:]), align_corners=True)
    c = b.corr_inputs(s_k, t_k, s_in, t_in, boxes, labels, masks, best=True)
    loss_corr, corr_ts = b.corr_loss_levels(*c, s_feat, t_feat, color)
    s_list, _, img_list, ins_labels, _ = b.corr_inputs(s_k, t_k, s_in, t_in, boxes, labels, masks, best=False)
    m = b.mask_loss(s_list, ins_labels, img_list, color, None, True)
    assert torch.equal(out['loss_corr'].detach(), loss_corr.detach())
    assert torch.equal(out['loss_ts'].detach(), (m['loss_ts'] + corr_ts * b.ts_loss_weight).detach())
    assert torch.equal(out['loss_ins'].detach(), m['loss_ins'].detach())


def _count_syncs(fn):
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('warn')
    try:
        with warnings.catch_warnings(record=True) as rec:
            warnings.simplefilter('always')
            out = fn()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    return out, [str(w.message) for w in rec if 'synchroniz' in str(w.message)]


@pytest.mark.parametrize('dt', [torch.float32, torch.float16])
def test_host_reads_are_the_target_builders_only(dt):
    from boxinstseg_b200.models.dense_heads.disco_targets import disco_target_single
    head = _head()
    inputs = _gpu_case(0)
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = inputs
    ctx = lambda: torch.autocast('cuda', dtype=dt, enabled=dt != torch.float32)        # noqa: E731
    with ctx():
        _run_loss(head, inputs, True, True)

    def loss():
        with ctx():
            return head.loss(cate, s_k, t_k, s_in, t_in, boxes, labels, masks, None, None, img=img, use_loss_ts=True,
                             use_ind_teacher=True)
    out, syncs = _count_syncs(loss)
    _, builder = _count_syncs(lambda: [disco_target_single(b, l, m, tuple(s_in.shape[-2:]), CFG['scale_ranges'],
                                                           CFG['strides'], GRIDS, CFG['sigma'], NUM_CLASSES)
                                       for b, l, m in zip(boxes, labels, masks)])
    # the per-(level, image) counts are the target builder's output shapes: the convolution and the losses read nothing
    assert len(builder) > 0 and len(syncs) == len(builder), (syncs, builder)
    assert all(torch.isfinite(v).all() for v in out.values())
