"""f4 on the GPU: DiscoBox's semantic-correspondence path through the C ABI (``bxs_corr_solve``, ``bxs_corr_transfer``) and the
device-resident object bank, against the oracle restatement and the golden vectors of the reference's own classes
(oracle/make_golden_corr.py).  Tolerances: the regularised table 5e-6 of its scale (row sums in another order than ATen's
reductions), the transferred maps 2e-5 absolute on values in [0, 1], the InfoNCE term and its gradient 1e-4 relative (north
star: 1e-3); retrieval indices and the bank contents exact."""
import numpy as np
import pytest
import torch

from oracle import corr as oc
from oracle.make_golden_corr import BANK, CH, FEAT, MASK, SOLVER, bank_case, blob, case

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'


def _solver():
    from boxinstseg_b200.models.dense_heads.disco_corr import SemanticCorrSolver
    return SemanticCorrSolver(**SOLVER)


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_solve_and_transfer_match_reference_golden(golden, seed):
    from types import SimpleNamespace
    g = golden('corr')
    f0, f1, m0, m1 = case(seed)
    s = _solver()
    Cu, T, fgm, bgm = s.solve(SimpleNamespace(mask=m0.to(DEV)), dict(feature=f1.to(DEV), mask=m1.to(DEV)), f0.to(DEV))
    assert fgm is None and bgm is None
    assert np.abs(Cu.cpu().numpy() - g[f's{seed}_Cu']).max() <= 2e-6
    ref_T = g[f's{seed}_T']
    # the table computed from the reference's own Cu (isolates the kernel from the GEMM's rounding)
    T_ref_in = s.votes(torch.from_numpy(g[f's{seed}_Cu']).to(DEV), FEAT, FEAT)
    assert np.abs(T_ref_in.cpu().numpy() - ref_T).max() <= 5e-6 * np.abs(ref_T).max()
    assert np.abs(T.cpu().numpy() - ref_T).max() <= 2e-5 * np.abs(ref_T).max()
    fg, bg = s.transfer(torch.from_numpy(ref_T).to(DEV), torch.from_numpy(g[f's{seed}_Cu']).to(DEV), m0.to(DEV), m1.to(DEV), FEAT, FEAT)
    assert np.abs(fg.cpu().numpy() - g[f's{seed}_fg']).max() <= 2e-5 and np.abs(bg.cpu().numpy() - g[f's{seed}_bg']).max() <= 2e-5
    _, fgm, bgm = s.solve(SimpleNamespace(mask=m0.to(DEV)), dict(feature=f1.to(DEV), mask=m1.to(DEV)), f0.to(DEV), return_masks=True)[1:]
    assert fgm.shape == (5, MASK * MASK, MASK * MASK) and bgm.shape == fgm.shape


@pytest.mark.parametrize('seed,shape,dk,iters,smooth,Hm', [(3, (5, 8), 3, 4, 2, 20), (4, (6, 4), 5, 0, 1, 9), (5, (3, 3), 1, 3, 0, 12),
                                                           (6, (12, 12), 9, 2, 1, 24)])
def test_other_shapes_against_oracle(seed, shape, dk, iters, smooth, Hm):
    """Non-square grids, no rounds / no smoothing, window 1, and the largest grid that needs the > 48 KB shared-memory opt-in."""
    from boxinstseg_b200.models.dense_heads.disco_corr import SemanticCorrSolver
    h, w = shape
    f0, f1, m0, m1 = case(seed, K=3, h=h, w=w, Hm=Hm)
    s = SemanticCorrSolver(1.0, 0.05, 3, 0.3, iters, smooth, dk)
    Cu = oc.cosine_table(f0, f1)
    want = oc.solve_votes(Cu, h, w, dk, iters, smooth)
    got = s.votes(Cu.to(DEV), h, w).cpu()
    assert (got - want).abs().max() <= 5e-6 * want.abs().max()
    _, fg, bg = oc.transfer(want, Cu, m0, m1, h, w)
    gfg, gbg = s.transfer(want.to(DEV), Cu.to(DEV), m0.to(DEV), m1.to(DEV), h, w)
    assert (gfg.cpu() - fg).abs().max() <= 2e-5 * max(1.0, float(fg.abs().max()))
    assert (gbg.cpu() - bg).abs().max() <= 2e-5 * max(1.0, float(bg.abs().max()))
    again = s.votes(Cu.to(DEV), h, w).cpu()
    assert torch.equal(again, got)                                        # fixed-order sums: run-to-run identical


def test_corr_objects_loop_against_oracle():
    """The per-object body of corr_loss (:1056-1125): a bank pre-filled with similar objects, six query objects of two
    classes; InfoNCE sum, number of terms, the pasted inter-image maps, the bank after the loop, and d loss / d RoI feature."""
    from boxinstseg_b200.models.dense_heads.disco_corr import ObjectQueues, corr_objects
    feats, masks, boxes = bank_case(0)
    bank_cfg = dict(BANK, len_queue=8)
    mine, orc = ObjectQueues(num_class=3, **bank_cfg), oc.Queues(num_class=3, **bank_cfg)
    for i in range(feats.shape[0]):
        mine.append(1, i, feats.to(DEV), masks.to(DEV), boxes.to(DEV))
        orc.append(1, i, feats, masks, boxes)
    gen = torch.Generator().manual_seed(42)
    n, H, W = 6, 50, 64
    s_feat = oc.relu_and_l2_norm_feat(feats[:1] + 0.15 * torch.randn(n, CH, FEAT, FEAT, generator=gen))
    t_feat = oc.relu_and_l2_norm_feat(feats[:1] + 0.15 * torch.randn(n, CH, FEAT, FEAT, generator=gen))
    s_mask = blob(gen, n, MASK, MASK / 2, MASK / 2, MASK * 0.36, MASK * 0.3)
    t_mask = blob(gen, n, MASK, MASK / 2, MASK / 2, MASK * 0.36, MASK * 0.3)
    qboxes = torch.tensor([[2, 3, 44, 41], [10, 5, 52, 43], [0, 0, 42, 40], [20, 8, 30, 18], [5, 5, 47, 45], [1, 2, 43, 42]],
                          dtype=torch.float32)
    labels = torch.tensor([1, 1, 2, 1, 1, 2])
    want_x = s_feat.clone().requires_grad_(True)
    iiu_o = torch.zeros(2 * n, H, W)
    lo, no = oc.corr_objects(orc, want_x, t_feat, s_mask, t_mask, qboxes, labels, iiu_o, SOLVER, min_size=32)
    assert no >= 3
    (go,) = torch.autograd.grad(lo, want_x)
    got_x = s_feat.clone().to(DEV).requires_grad_(True)
    iiu = torch.zeros(2 * n, H, W, device=DEV)
    lm, nm, qobj = corr_objects(_solver(), mine, None, got_x, t_feat.to(DEV), s_mask.to(DEV), t_mask.to(DEV), qboxes.to(DEV),
                                labels.to(DEV), iiu, objbank_min_size=32)
    (gm,) = torch.autograd.grad(lm, got_x)
    assert nm == no and qobj is not None
    assert abs(float(lm) - float(lo)) <= 1e-4 * abs(float(lo))
    assert (gm.cpu() - go).norm() <= 1e-4 * go.norm()
    assert (iiu.cpu() - iiu_o).abs().max() <= 5e-5 and float(iiu_o.abs().max()) > 0.05
    for c in (1, 2):
        assert torch.equal(mine.queues[c].feature.cpu(), orc.banks[c].feature) and mine.queues[c].ptr == orc.banks[c].ptr
        assert torch.equal(mine.queues[c].mask.cpu(), orc.banks[c].mask) and torch.equal(mine.queues[c].box.cpu(), orc.banks[c].box)


def test_corr_loss_levels_against_oracle():
    """The per-level body of corr_loss (:1013-1139) end to end: empty targets dropped, boxes from the masks, RoIAlign
    (torchvision's, third party on both sides), the per-object loop, the mean field WITH the transferred inter-image maps, dice.
    The bank is warmed up by one oracle iteration and copied to the device; the compared iteration must give the same loss,
    per-object dice terms, gradients (RoI feature path and mask path) and the same bank afterwards."""
    from torchvision.ops import roi_align
    from boxinstseg_b200.models.dense_heads import MeanField
    from boxinstseg_b200.models.dense_heads.disco_corr import DiscoCorr, ObjectElements, create_one
    from oracle.make_golden_corr import levels_case
    bank = dict(feat_height=7, feat_width=7, mask_height=28, mask_width=28, min_size=8, len_object_queues=10, fg_iou_thresh=0.7,
                bg_iou_thresh=0.7, ratio_range=[0.9, 1.2], appear_thresh=0.7, max_retrieval_objs=5)
    mf_cfg = dict(kernel_size=3, theta0=0.5, theta1=30.0, alpha0=2.0, iter=10, base=0.1, gamma=0.5)
    loss_corr = dict(loss_weight=1.0, corr_exp=1.0, corr_eps=0.05, gaussian_filter_size=3, low_score=0.3, corr_num_iter=10,
                     corr_num_smooth_iter=1, dist_kernel=9, obj_bank=bank)
    orc = oc.Queues(num_class=3, **dict(BANK, len_queue=10))
    ra = lambda x, rois, size: roi_align(x, rois, size, 1.0, 0, True)
    state = {'first': True}
    s_feat, t_feat, color, s_list, img_list, tgt_list, lab_list = levels_case(0)
    oc.corr_loss_levels(orc, s_list, img_list, tgt_list, lab_list, s_feat, t_feat, color, SOLVER, bank, mf_cfg, ra, state=state)
    dc = DiscoCorr(3, loss_corr)
    for c, b in enumerate(orc.banks):                                     # the warmed-up bank, copied to the device
        if b is not None:
            q = ObjectElements(size=10, feat_size=7, mask_size=28, n_channel=CH, device=DEV, category=c)
            q.feature.copy_(b.feature); q.mask.copy_(b.mask); q.box.copy_(b.box); q.ptr = b.ptr
            dc.object_queues.queues[c] = q
    dc.qobj = create_one(torch.zeros(1, 28, 28, device=DEV), torch.zeros(1, CH, 7, 7, device=DEV), torch.zeros(1, 4, device=DEV), 0)
    s_feat, t_feat, color, s_list, img_list, tgt_list, lab_list = levels_case(1)
    # oracle side
    of = s_feat.clone().requires_grad_(True)
    ol_ = [s.clone().requires_grad_(True) for s in s_list]
    lo, tso = oc.corr_loss_levels(orc, ol_, img_list, tgt_list, lab_list, of, t_feat, color, SOLVER, bank, mf_cfg, ra, state=state)
    obj_o = lo + torch.cat(tso).mean()
    go = torch.autograd.grad(obj_o, [of] + ol_)
    # product side
    gf = s_feat.clone().to(DEV).requires_grad_(True)
    gl = [s.clone().to(DEV).requires_grad_(True) for s in s_list]
    mf = MeanField(color.to(DEV), kernel_size=3, theta0=0.5, theta1=30.0, theta2=10, alpha0=2.0, iter=10, base=0.1, gamma=0.5)
    lm, tsm = dc.levels(gl, [None] * len(gl), [i.to(DEV) for i in img_list], [t.to(DEV) for t in tgt_list],
                        [l.to(DEV) for l in lab_list], gf, t_feat.to(DEV), mf)
    obj_m = lm + torch.cat(tsm).mean()
    gm = torch.autograd.grad(obj_m, [gf] + gl)
    assert float(lo) > 1.0 and abs(float(lm) - float(lo)) <= 1e-4 * abs(float(lo))
    for a, b in zip(tsm, tso):
        assert a.shape == b.shape and (a.cpu() - b).abs().max() <= 1e-5
    for a, b in zip(gm, go):
        assert (a.cpu() - b).norm() <= 1e-3 * b.norm() + 1e-9, (float((a.cpu() - b).norm()), float(b.norm()))
    for c, b in enumerate(orc.banks):
        if b is not None:
            q = dc.object_queues.queues[c]
            assert q.ptr == b.ptr and (q.feature.cpu() - b.feature).abs().max() <= 1e-5 and (q.mask.cpu() - b.mask).abs().max() <= 1e-5
            assert torch.equal(q.box.cpu(), b.box)
    # the same through the head (DiscoBoxSOLOv2Head.corr_loss_levels builds the mean field from its own CRF settings), next iteration
    from boxinstseg_b200.models import build_head
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=3, in_channels=CH, loss_corr=loss_corr))
    head.corr = dc
    s_feat, t_feat, color, s_list, img_list, tgt_list, lab_list = levels_case(2)
    lo2, tso2 = oc.corr_loss_levels(orc, s_list, img_list, tgt_list, lab_list, s_feat, t_feat, color, SOLVER, bank, mf_cfg, ra, state=state)
    l2, ts2 = head.corr_loss_levels([s.to(DEV) for s in s_list], None, [i.to(DEV) for i in img_list], [t.to(DEV) for t in tgt_list],
                                    [l.to(DEV) for l in lab_list], s_feat.to(DEV), t_feat.to(DEV), color.to(DEV), gamma=0.5)
    assert abs(float(l2) - float(lo2)) <= 1e-4 * abs(float(lo2)) and abs(float(ts2) - float(torch.cat(tso2).mean())) <= 1e-5


def test_head_corr_loss_with_the_reference_signature():
    """DiscoBoxSOLOv2Head.corr_loss (discobox_head.py:900-1139) from the raw head outputs: SOLO targets, kernel gathering, the
    wgmma dynamic convolutions (against F.conv2d on the same tensors, TF32 tolerance), the colour features (align_corners=True
    resize), and two training steps of the level body on top of them (the first fills the bank): finite values, a gradient to the
    mask features, the kernels and the RoI feature map, the bank advancing."""
    import torch.nn.functional as F
    from boxinstseg_b200.models import build_head
    from boxinstseg_b200.models.dense_heads import MeanField
    from oracle.make_golden_disco import CFG as DCFG, case as dcase
    bank = dict(feat_height=7, feat_width=7, mask_height=28, mask_width=28, min_size=2, len_object_queues=16, fg_iou_thresh=0.7,
                bg_iou_thresh=0.7, ratio_range=[0.9, 1.2], appear_thresh=0.7, max_retrieval_objs=5)
    loss_corr = dict(loss_weight=1.0, corr_exp=1.0, corr_eps=0.05, gaussian_filter_size=3, low_score=0.3, corr_num_iter=10,
                     corr_num_smooth_iter=1, dist_kernel=9, obj_bank=bank)
    B, C = 2, 32
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=DCFG['num_classes'], in_channels=C, loss_corr=loss_corr,
                           scale_ranges=DCFG['scale_ranges'], strides=DCFG['strides'], num_grids=DCFG['seg_num_grids'],
                           sigma=DCFG['sigma']))
    gen = torch.Generator().manual_seed(8)
    cases = [dcase(s) for s in (0, 1)]
    fsize = cases[0][3]
    boxes, labels = [c[0].to(DEV) for c in cases], [c[1].to(DEV) for c in cases]
    masks = [torch.from_numpy(c[2]).to(DEV) for c in cases]
    kraw = [(0.2 * torch.randn(B, C, g, g, generator=gen)).to(DEV).requires_grad_(True) for g in DCFG['seg_num_grids']]
    feat = torch.randn(B, C, fsize[0], fsize[1], generator=gen).to(DEV).requires_grad_(True)
    s_feat = torch.randn(B, 16, fsize[0], fsize[1], generator=gen).to(DEV).requires_grad_(True)
    img = torch.randn(B, 3, 160, 192, generator=gen).to(DEV)
    # the front part against F.conv2d on the same tensors
    got = head.corr_inputs(kraw, None, feat, None, boxes, labels, masks)
    ref = head.corr_inputs(kraw, None, feat, None, boxes, labels, masks, conv=lambda f, k: F.conv2d(f[None], k.t()[:, :, None, None])[0])
    n_obj = 0
    for a, b in zip(got[0], ref[0]):
        assert (a is None) == (b is None)
        if a is not None:
            assert (a - b).norm() <= 1e-3 * b.norm()
            n_obj += a.shape[0]
    assert n_obj >= 8
    mfs = [MeanField(F.interpolate(img[b:b + 1], fsize, mode='bilinear', align_corners=True), gamma=0.5) for b in range(B)]
    for step in range(2):
        loss, ts = head.corr_loss(None, kraw, None, feat, None, boxes, labels, masks, mfs, None, None, img=img,
                                  s_feat=s_feat, t_feat=s_feat.detach())
        assert torch.isfinite(loss) and len(ts) >= 1 and all(torch.isfinite(t).all() for t in ts)
        assert sum(t.numel() for t in ts) <= n_obj
        total = loss + torch.cat(ts).mean()
        grads = torch.autograd.grad(total, [feat] + kraw + [s_feat], allow_unused=True)
        assert grads[0] is not None and torch.isfinite(grads[0]).all() and float(grads[0].abs().sum()) > 0
    filled = sum(q.ptr for q in head.corr.object_queues.queues if q is not None)
    assert filled > 0
