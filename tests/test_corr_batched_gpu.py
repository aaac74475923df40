"""f4 on the GPU, batched: the per-object body of corr_loss for all objects of a level at once (``corr_level``:
``bxs_corr_retrieve``, the batched solve / transfer, ``bxs_corr_paste``, ``bxs_corr_bank_append``) against the oracle's
sequential loop (oracle/corr.py ``corr_objects``) over multi-level, multi-class sequences (tests/corr_sequences.py).
Exact: the retrieved slots, the number of InfoNCE terms, the append slots, the bank after every level (feature, mask, box,
ptr -- copies).  Within the bars of tests/test_corr_gpu.py: the loss 1e-4 relative, iiu 5e-5, the gradient 1e-3 relative.
Then the training entry point: no host synchronisation, CUDA-graph replay bit-identical to eager calls, and a number of
launches per level that does not grow with the number of objects."""
import pytest
import torch

from oracle import corr as oc
from oracle.make_golden_corr import CH, FEAT, MASK, SOLVER, levels_case
from tests import corr_sequences as cs

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
BANK_CFG = dict(feat_height=7, feat_width=7, mask_height=28, mask_width=28, min_size=8, len_object_queues=10, fg_iou_thresh=0.7,
                bg_iou_thresh=0.7, ratio_range=[0.9, 1.2], appear_thresh=0.7, max_retrieval_objs=5)
LOSS_CORR = dict(loss_weight=1.0, corr_exp=1.0, corr_eps=0.05, gaussian_filter_size=3, low_score=0.3, corr_num_iter=10,
                 corr_num_smooth_iter=1, dist_kernel=9, obj_bank=BANK_CFG)


def _product_bank(orc):
    from boxinstseg_b200.models.dense_heads.disco_corr import ObjectElements, ObjectQueues
    mine = ObjectQueues(num_class=cs.NUM_CLASS, **cs.BANK)
    for c, b in enumerate(orc.banks):
        if b is not None:
            q = ObjectElements(size=cs.BANK['len_queue'], feat_size=FEAT, mask_size=MASK, n_channel=CH, device=DEV, category=c)
            q.feature.copy_(b.feature); q.mask.copy_(b.mask); q.box.copy_(b.box); q.ptr = b.ptr
            mine.queues[c] = q
    return mine


@pytest.mark.parametrize('ind_teacher', [True, False])
@pytest.mark.parametrize('seed', [0, 1])
def test_level_body_against_sequential_oracle(seed, ind_teacher):
    from boxinstseg_b200.models.dense_heads.disco_corr import SemanticCorrSolver, corr_level
    solver = SemanticCorrSolver(**SOLVER)
    orc, levels = cs.sequence(seed, ind_teacher=ind_teacher)
    mine = _product_bank(orc)
    first = torch.ones(1, dtype=torch.int32, device=DEV)
    state = {'first': True}
    terms, H, W = 0, 56, 64
    for lv in levels:
        s_feat, t_feat, s_mask, t_mask, boxes, labels, valid = lv
        keep = valid.nonzero().flatten()
        n, nk = s_feat.shape[0], keep.numel()
        want, appends, margin, _, _, _ = cs.replay(cs.clone(orc), state['first'], *lv)
        assert margin >= 1e-5
        # oracle: the reference's loop over the objects with a non-empty target
        xo = s_feat[keep].clone().requires_grad_(True)
        iiu_o = torch.zeros(2 * nk, H, W)
        lo, no = oc.corr_objects(orc, xo, t_feat[keep], s_mask[keep], t_mask[keep], boxes[keep], labels[keep], iiu_o, SOLVER,
                                 min_size=cs.MIN_SIZE, state=state)
        # product: all n objects in one pass
        xm = s_feat.clone().to(DEV).requires_grad_(True)
        iiu = torch.zeros(2 * n, H, W, device=DEV)
        lm, nm, rec = corr_level(solver, mine, first, xm, t_feat.to(DEV), s_mask.to(DEV), t_mask.to(DEV), boxes.to(DEV),
                                 labels.to(DEV), valid.to(DEV), iiu, cs.MIN_SIZE)
        src, count, slot = rec['src'].cpu(), rec['count'].cpu(), rec['slot'].cpu()
        assert slot.tolist() == appends
        for i, w in enumerate(want):
            if w is None:
                assert int(count[i]) == 0
            else:
                assert cs.decode(src[i], count[i], slot) == w, (i, w)
        assert int(nm) == no and int(first) == 0
        terms += no
        if no:
            go = torch.autograd.grad(lo, xo)[0]
            gm = torch.autograd.grad(lm, xm)[0].cpu()
            assert abs(float(lm) - float(lo)) <= 1e-4 * abs(float(lo))
            assert (gm[keep] - go).norm() <= 1e-3 * go.norm() and float(gm[~valid].abs().sum()) == 0
        else:
            assert float(lm) == 0
        want_iiu = torch.zeros(n, 2, H, W)
        want_iiu[keep] = iiu_o.view(nk, 2, H, W)
        assert (iiu.cpu().view(n, 2, H, W) - want_iiu).abs().max() <= 5e-5
        for c, b in enumerate(orc.banks):
            q = mine.queues[c]
            assert (q is None) == (b is None)
            if b is not None:
                assert torch.equal(q.feature.cpu(), b.feature) and torch.equal(q.mask.cpu(), b.mask)
                assert torch.equal(q.box.cpu(), b.box) and q.ptr == b.ptr
    assert terms >= 5


def _head():
    from boxinstseg_b200.models import build_head
    return build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=3, in_channels=CH, loss_corr=LOSS_CORR))


def _head_inputs(seed, per_level=(5, 4)):
    s_feat, t_feat, color, s_list, img_list, tgt_list, lab_list = levels_case(seed, per_level=per_level)
    return ([s.to(DEV) for s in s_list], None, [i.to(DEV) for i in img_list], [t.to(DEV) for t in tgt_list],
            [l.to(DEV) for l in lab_list], s_feat.to(DEV), t_feat.to(DEV), color.to(DEV))


def _bank_state(head):
    q = head.corr.object_queues
    return [t.clone() for t in (q.feature, q.mask, q.box, q.ptr, q.exists, head.corr.first)]


def _restore(head, snap):
    q = head.corr.object_queues
    for t, s in zip((q.feature, q.mask, q.box, q.ptr, q.exists, head.corr.first), snap):
        t.copy_(s)


def test_head_corr_loss_levels_is_sync_free():
    head = _head()
    args = _head_inputs(0)
    head.corr_loss_levels(*args, gamma=0.5)                        # allocates the bank and the first-query flag
    args = _head_inputs(1)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        loss, ts = head.corr_loss_levels(*args, gamma=0.5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(loss) and torch.isfinite(ts)


def test_cuda_graph_replay_equals_eager_calls():
    head = _head()
    for seed in (0, 1):                                            # a bank that retrieves
        head.corr_loss_levels(*_head_inputs(seed), gamma=0.5)
    args = _head_inputs(2)
    snap = _bank_state(head)
    with torch.no_grad():
        eager = [torch.stack(head.corr_loss_levels(*args, gamma=0.5)) for _ in range(3)]
    eager_bank = _bank_state(head)
    assert float(eager[0][0]) > 0
    _restore(head, snap)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.no_grad():                 # warm-up on the capture stream, then back to the start
        head.corr_loss_levels(*args, gamma=0.5)
    torch.cuda.current_stream().wait_stream(side)
    _restore(head, snap)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph), torch.no_grad():
        out = torch.stack(head.corr_loss_levels(*args, gamma=0.5))
    _restore(head, snap)                                           # capturing runs nothing, but start from the same bank
    replayed = []
    for _ in range(3):
        graph.replay()
        replayed.append(out.clone())
    torch.cuda.synchronize()
    for a, b in zip(replayed, eager):
        assert torch.equal(a, b), (a, b)
    for a, b in zip(_bank_state(head), eager_bank):
        assert torch.equal(a, b)


def test_launches_per_level_do_not_grow_with_objects():
    from torch.profiler import ProfilerActivity, profile

    def launches(n):
        head = _head()
        args = _head_inputs(3, per_level=(n, 4))
        head.corr_loss_levels(*args, gamma=0.5)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            head.corr_loss_levels(*args, gamma=0.5)
            torch.cuda.synchronize()
        return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)

    few, many = launches(4), launches(32)
    assert few == many and few > 0, (few, many)
