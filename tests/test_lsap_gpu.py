"""GPU: the batched linear-sum-assignment kernel (csrc/lsap.cu, ops.lsap) against scipy.optimize.linear_sum_assignment --
bit-exact row_ind / col_ind, scipy's errors -- and the two callers built on it: MaskHungarianAssigner.assign and
Box2MaskHead.get_targets (box2mask_head.py:135-189), the latter against a restatement of the reference's
_get_target_single with scipy and MaskPseudoSampler, without host synchronisation and inside a CUDA graph."""
import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment as scipy_lsa

from tests.test_lsap_cpu import INFEASIBLE, INVALID, OK, scipy_result, seeded_matrix

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
ASSIGNER = dict(type='MaskHungarianAssigner', cls_cost=dict(type='ClassificationCost', weight=2.0),
                dice_cost=dict(type='BoxMatchingCost', weight=5.0, pred_act=True, eps=1.0))


def check_batch(cs):
    """Solve the numpy matrices `cs` in one batched call and compare each problem with scipy."""
    from boxinstseg_b200.ops.lsap import solve_batched
    matches, status = solve_batched([torch.from_numpy(c).to(DEV) for c in cs])
    status = status.cpu().numpy()
    for c, m, st in zip(cs, matches, status):
        want, r, k = scipy_result(c)
        m = m.cpu().numpy()
        assert st == want, (c.shape, st, want)
        if want != OK:
            assert (m == -1).all()
            continue
        rows = np.nonzero(m >= 0)[0]
        assert np.array_equal(rows, r) and np.array_equal(m[rows], k), c.shape
    return matches, status


@pytest.mark.parametrize('kind', ['normal', 'int3', 'zeros', 'inf'])
def test_lsap_kernel_matches_scipy(kind):
    rng = np.random.default_rng(100 + ['normal', 'int3', 'zeros', 'inf'].index(kind))
    cs = [seeded_matrix(rng, kind, *(int(v) for v in rng.integers(1, 40, 2))) for _ in range(800)]
    check_batch(cs)
    check_batch([c.astype(np.float64) for c in cs[:100]])


def test_lsap_kernel_invalid_infeasible_empty():
    cs = []
    for bad in (np.nan, -np.inf):
        for shape in [(4, 6), (6, 4), (1, 1)]:
            c = np.ones(shape, np.float32)
            c[shape[0] - 1, 0] = bad
            cs.append(c)
    c = np.ones((3, 3), np.float32)
    c[1, :] = np.inf
    cs += [c, np.ascontiguousarray(c.T)]
    c = np.full((2, 5), np.inf, np.float32)
    c[0, 0] = c[1, 0] = 1.0
    cs.append(c)
    cs += [np.zeros(s, np.float32) for s in [(0, 5), (5, 0), (0, 0)]]
    _, status = check_batch(cs)
    assert list(status[:6]) == [INVALID] * 6 and list(status[6:9]) == [INFEASIBLE] * 3 and list(status[9:]) == [OK] * 3


def test_lsap_scipy_signature():
    from boxinstseg_b200.ops.lsap import linear_sum_assignment
    rng = np.random.default_rng(5)
    for shape in [(100, 50), (50, 100), (7, 7), (1, 9), (0, 4), (4, 0)]:
        c = rng.integers(0, 3, shape).astype(np.float32)
        r, k = linear_sum_assignment(torch.from_numpy(c).to(DEV))
        rr, kk = scipy_lsa(c)
        assert r.dtype == torch.int64 and k.dtype == torch.int64 and r.is_cuda
        assert np.array_equal(r.cpu().numpy(), rr) and np.array_equal(k.cpu().numpy(), kk)
    c = torch.ones(3, 4, device=DEV)
    c[1, 2] = float('nan')
    with pytest.raises(ValueError, match='matrix contains invalid numeric entries'):
        linear_sum_assignment(c)
    c = torch.full((2, 3), float('inf'), device=DEV)
    c[:, 0] = 0
    with pytest.raises(ValueError, match='cost matrix is infeasible'):
        linear_sum_assignment(c)


def _box2mask_cost(gen, Q, G):
    from boxinstseg_b200.core import BoxMatchingCost, ClassificationCost
    pr, pc = torch.sigmoid(torch.randn(Q, 64, generator=gen) * 3), torch.sigmoid(torch.randn(Q, 80, generator=gen) * 3)
    gr, gc = (torch.rand(G, 64, generator=gen) > 0.6).float(), (torch.rand(G, 80, generator=gen) > 0.6).float()
    return (ClassificationCost(2.0)(torch.randn(Q, 81, generator=gen), torch.randint(0, 80, (G,), generator=gen)) +
            BoxMatchingCost(5.0, pred_act=True, eps=1.0)._cost(pr, pc, gr, gc)).numpy()


def test_lsap_kernel_box2mask_costs():
    gen = torch.Generator().manual_seed(11)
    check_batch([_box2mask_cost(gen, 100, G) for G in (0, 1, 7, 50, 100, 150) for _ in range(5)])


def test_lsap_kernel_large_problems():
    """Problems whose state does not fit in shared memory run on the caller's workspace; a chunk mixing them with small
    ones, in both orientations."""
    rng = np.random.default_rng(13)
    big = rng.standard_normal((600, 1500)).astype(np.float32)
    check_batch([big, rng.integers(0, 3, (9, 4)).astype(np.float32), np.ascontiguousarray(big.T[:, :500]),
                 rng.integers(0, 5, (300, 800)).astype(np.float64)])


def test_lsap_ragged_chunks_and_repeats():
    """200 ragged problems (4 launches of the 64-problem chunk) equal the same problems solved one at a time, and repeated
    runs give identical bits."""
    from boxinstseg_b200.ops.lsap import solve_batched
    rng = np.random.default_rng(9)
    cs = []
    for i in range(200):
        nr, nc = (int(v) for v in rng.integers(0, 60, 2))
        cs.append(seeded_matrix(rng, ['normal', 'int3', 'inf'][i % 3], nr, nc))
    ts = [torch.from_numpy(c).to(DEV) for c in cs]
    batched, status = check_batch(cs)
    for t, m, st in zip(ts, batched, status):
        (m1,), s1 = solve_batched([t])
        assert torch.equal(m1, m) and int(s1[0]) == st
    for _ in range(3):
        again, st2 = solve_batched(ts)
        assert torch.equal(torch.cat(again), torch.cat(batched)) and np.array_equal(st2.cpu().numpy(), status)


def _assign_case(seed, Q=100, G=6, h=64, w=64, H=256, W=256):
    gen = torch.Generator().manual_seed(seed)
    cls_pred = torch.randn(Q, 81, generator=gen)
    mask_pred = torch.randn(Q, h, w, generator=gen) * 3
    gt_labels = torch.randint(0, 80, (G,), generator=gen)
    gt = torch.zeros(G, H, W)
    for i in range(G):
        y0, x0 = (int(v) for v in torch.randint(0, H // 2, (2,), generator=gen))
        gt[i, y0:y0 + 20 + 7 * i, x0:x0 + 30 + 5 * i] = 1
    return cls_pred.to(DEV), mask_pred.to(DEV), gt_labels.to(DEV), gt.to(DEV)


def _scipy_assign(asg, cls_pred, mask_pred, gt_labels, gt):
    """Step 3-4 of the reference (mask_hungarian_assigner.py:113-132) on the same cost matrix."""
    Q = mask_pred.shape[0]
    cost = asg.cost_matrix(cls_pred, mask_pred, gt_labels, gt, lowres=True).cpu()
    r, c = scipy_lsa(cost)
    gt_inds, labels = torch.zeros(Q, dtype=torch.long), torch.full((Q,), -1, dtype=torch.long)
    gt_inds[torch.from_numpy(r)] = torch.from_numpy(c) + 1
    labels[torch.from_numpy(r)] = gt_labels.cpu()[torch.from_numpy(c)]
    return gt_inds, labels


@pytest.mark.parametrize('seed,Q,G', [(0, 100, 6), (1, 100, 50), (2, 30, 60), (3, 100, 1)])
def test_assign_equals_scipy(seed, Q, G):
    from boxinstseg_b200.core import MaskHungarianAssigner
    asg = MaskHungarianAssigner(**{k: v for k, v in ASSIGNER.items() if k != 'type'})
    case = _assign_case(seed, Q=Q, G=G)
    res = asg.assign(*case, None, lowres=True)
    gt_inds, labels = _scipy_assign(asg, *case)
    assert res.num_gts == G and res.max_overlaps is None
    assert res.gt_inds.dtype == torch.long and res.labels.dtype == torch.long
    assert torch.equal(res.gt_inds.cpu(), gt_inds) and torch.equal(res.labels.cpu(), labels)


def test_assign_errors_equal_scipy():
    from boxinstseg_b200.core import MaskHungarianAssigner
    asg = MaskHungarianAssigner(**{k: v for k, v in ASSIGNER.items() if k != 'type'})
    cls_pred, mask_pred, gt_labels, gt = _assign_case(4)
    cls_pred[3, 0] = float('nan')
    with pytest.raises(ValueError) as ref:
        scipy_lsa(asg.cost_matrix(cls_pred, mask_pred, gt_labels, gt, lowres=True).cpu())
    with pytest.raises(ValueError) as ours:
        asg.assign(cls_pred, mask_pred, gt_labels, gt, None, lowres=True)
    assert str(ours.value) == str(ref.value) == 'matrix contains invalid numeric entries'


def _head():
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import Box2MaskHead
    return Box2MaskHead(num_queries=100, train_cfg=dict(assigner=ASSIGNER, sampler=dict(type='MaskPseudoSampler')))


def _targets_case(seed, Gs=(7, 0, 50), Q=100):
    gen = torch.Generator().manual_seed(seed)
    cls, masks, labels, gts = [], [], [], []
    for G in Gs:
        c, m, l, g = _assign_case(int(torch.randint(0, 1 << 30, (1,), generator=gen)), Q=Q, G=G, H=128, W=160)
        cls.append(c), masks.append(m), labels.append(l), gts.append(g)
    return cls, masks, labels, gts, [dict() for _ in Gs]


def _reference_targets(head, cls_list, mask_list, labels_list, gts_list):
    """box2mask_head.py:135-189 with scipy (mask_hungarian_assigner.py:113-132) and MaskPseudoSampler.sample, on the same
    low-resolution cost matrix."""
    out = [[], [], [], []]
    num_pos = num_neg = 0
    for cls, mp, gl, gm in zip(cls_list, mask_list, labels_list, gts_list):
        Q, G = mp.shape[0], gl.shape[0]
        gt_inds = torch.zeros(Q, dtype=torch.long)
        if G:
            gt_inds, _ = _scipy_assign(head.hungarian, cls, mp, gl, gm)
        pos_inds = torch.nonzero(gt_inds > 0, as_tuple=False).squeeze(-1).unique()
        neg_inds = torch.nonzero(gt_inds == 0, as_tuple=False).squeeze(-1).unique()
        pos_assigned = gt_inds[pos_inds] - 1
        labels = torch.full((head.num_queries,), head.num_classes, dtype=torch.long)
        labels[pos_inds] = gl.cpu()[pos_assigned]
        mask_weights = torch.zeros(head.num_queries)
        mask_weights[pos_inds] = 1.0
        for lst, v in zip(out, (labels, torch.ones(head.num_queries, dtype=torch.long), gm.cpu().unsqueeze(1)[pos_assigned],
                                mask_weights)):
            lst.append(v)
        num_pos += pos_inds.numel()
        num_neg += neg_inds.numel()
    return (*out, num_pos, num_neg)


def _assert_targets_equal(got, want):
    for g_list, w_list in zip(got[:4], want[:4]):
        assert len(g_list) == len(w_list)
        for g, w in zip(g_list, w_list):
            assert g.is_cuda and g.dtype == w.dtype and g.shape == w.shape
            assert torch.equal(g.cpu(), w)
    assert got[4:] == want[4:]


def test_get_targets_equals_reference():
    head = _head()
    for seed, Gs in [(0, (7, 0, 50)), (1, (100,)), (2, (150, 1))]:
        case = _targets_case(seed, Gs)
        got = head.get_targets(*case)
        assert len(got) == 6
        _assert_targets_equal(got, _reference_targets(head, *case[:4]))
        assert head.lsap_status.tolist() == [0] * len(Gs)


def test_get_targets_no_sync():
    head = _head()
    case = _targets_case(3)
    head.get_targets(*case)                        # warm-up: library load, allocator
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        got = head.get_targets(*case)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    _assert_targets_equal(got, _reference_targets(head, *case[:4]))


def test_get_targets_cuda_graph():
    head = _head()
    static = _targets_case(4)
    fresh = _targets_case(5)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        head.get_targets(*static)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = head.get_targets(*static)
    for lst_s, lst_f in zip(static[:4], fresh[:4]):
        for a, b in zip(lst_s, lst_f):
            a.copy_(b)
    graph.replay()
    torch.cuda.synchronize()
    eager = head.get_targets(*fresh)
    _assert_targets_equal(out, tuple([t.cpu() for t in lst] for lst in eager[:4]) + eager[4:])
    _assert_targets_equal(out, _reference_targets(head, *fresh[:4]))


def test_get_targets_nan_image_is_background():
    """A NaN prediction cannot raise without a synchronisation: that image's queries come back as background, the other
    images are unaffected, and the per-image status stays on the head."""
    head = _head()
    cls, masks, labels, gts, metas = _targets_case(6, Gs=(7, 12))
    cls[0][5, 3] = float('nan')
    got = head.get_targets(cls, masks, labels, gts, metas)
    assert head.lsap_status.is_cuda and head.lsap_status.tolist() == [INVALID, OK]
    assert torch.equal(got[0][0].cpu(), torch.full((100,), head.num_classes, dtype=torch.long))
    assert torch.equal(got[3][0].cpu(), torch.zeros(100))
    assert got[2][0].shape == (7, 1, 128, 160)
    assert got[4] == 7 + 12 and got[5] == 2 * 100 - 19
    want = _reference_targets(head, cls[1:], masks[1:], labels[1:], gts[1:])
    for i in range(4):
        assert torch.equal(got[i][1].cpu(), want[i][0])
