"""GPU parity of the tree-filter ops (a12-a15): MST edge set bit-exact against the reference's Boruvka
(golden fixtures + the Kruskal oracle), BFS validity, refine forward/backward against the C oracle and the
float64 closed form."""
import numpy as np
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
T = torch.from_numpy
DEV = 'cuda:0'


def _edge_ids(tree, h, w):
    from oracle.tree import edges_to_ids
    return edges_to_ids(tree.cpu().numpy(), h, w)


def test_mst_golden(golden):
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    g = golden('tree')
    gm = T(g['guide']).to(DEV)
    mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
    assert torch.equal(mst._build_feature_weight(gm).cpu(), T(g['edge_weight']))          # weights bit-identical
    tree = mst(gm)
    assert tree.dtype == torch.int32 and tree.shape == (3, 9 * 13 - 1, 2)
    for b in range(3):
        assert np.array_equal(_edge_ids(tree[b], 9, 13), g['mst_edge_ids'][b])            # reference Boruvka edge set


@pytest.mark.parametrize('B,C,h,w,quant', [(2, 3, 40, 56, False), (3, 5, 25, 31, True), (1, 3, 200, 256, False),
                                           (2, 1, 96, 96, True), (1, 2, 2, 2, False), (1, 2, 1, 7, False)])
def test_mst_vs_oracle(B, C, h, w, quant):
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    from oracle import tree as ot
    gen = torch.Generator().manual_seed(h * w)
    gm = torch.randn(B, C, h, w, generator=gen)
    if quant:
        gm = torch.round(gm * 2) / 2                          # massive weight ties -> the (weight, id) order decides
    tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(gm.to(DEV))
    ei = ot.grid_edges(h, w)
    ew = ot.grid_edge_weights(gm).numpy()
    for b in range(B):
        assert np.array_equal(_edge_ids(tree[b], h, w), ot.mst_edge_ids(ei, ew[b], h * w))


def _check_bfs(idx, par, chd, tree, V):
    i, p, c = idx.cpu().numpy(), par.cpu().numpy(), chd.cpu().numpy()
    assert sorted(i.tolist()) == list(range(V)) and i[0] == 0 and p[0] == 0
    assert np.all(p[1:] < np.arange(1, V)) and np.all(np.diff(p) >= 0)
    edges = {tuple(sorted(e)) for e in tree.cpu().numpy().tolist()}
    assert {tuple(sorted((int(i[k]), int(i[p[k]])))) for k in range(1, V)} == edges       # same tree
    for pos in range(V):
        kids = [k for k in c[pos] if k > 0]
        assert all(p[k] == pos for k in kids) and len(kids) == int(np.sum(p[1:] == pos))
        # the deterministic order both BFS paths promise: children adjacent in position, ascending in vertex id
        assert kids == list(range(kids[0], kids[0] + len(kids))) if kids else True
        assert [int(i[k]) for k in kids] == sorted(int(i[k]) for k in kids)


def test_bfs_generic_path_on_a_non_grid_tree():
    """A random (non-grid) tree takes the generic adjacency-list BFS; a grid tree takes the shared-memory bit-adjacency
    fast path.  Both must satisfy the same contract."""
    from boxinstseg_b200.ops.tree_filter import bfs
    gen = torch.Generator().manual_seed(3)
    V = 700
    par = (torch.rand(V - 1, generator=gen) * torch.arange(1, V)).long().clamp(max=V - 2)      # parent of vertex k+1 in [0, k]
    deg = torch.zeros(V, dtype=torch.long)
    edges = []
    for k in range(1, V):                       # keep every degree <= 4 (bfs_forward's max_adj)
        cand = int(par[k - 1])
        while deg[cand] >= 3:
            cand = (cand + 1) % k
        deg[cand] += 1; deg[k] += 1
        edges.append((cand, k))
    tree = torch.tensor(edges, dtype=torch.int32).unsqueeze(0).to(DEV)
    idx, p, c = bfs(tree, 4)
    _check_bfs(idx[0], p[0], c[0], tree[0], V)


def test_bfs_valid_and_deterministic():
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D, bfs
    gen = torch.Generator().manual_seed(1)
    gm = torch.randn(3, 3, 30, 41, generator=gen).to(DEV)
    tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(gm)
    idx, par, chd = bfs(tree, 4)
    for b in range(3):
        _check_bfs(idx[b], par[b], chd[b], tree[b], 30 * 41)
    idx2, par2, chd2 = bfs(tree, 4)
    assert torch.equal(idx, idx2) and torch.equal(par, par2) and torch.equal(chd, chd2)   # the reference's order is racy
    # level boundaries recomputed from sorted_parent agree with the ones bfs produced
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as _C
    lvl, nlv = _C.levels_of(idx, par)
    lvl2, nlv2 = _C.levels_of(idx.clone(), par)
    assert torch.equal(nlv, nlv2)
    order = _C.bfs_order(tree, 4)                          # the same order as one value, level table included
    assert all(torch.equal(a, b) for a, b in zip(order[:3], (idx, par, chd)))
    assert torch.equal(order.num_levels, nlv)
    for b in range(3):
        L = int(nlv[b])
        assert torch.equal(lvl[b, :L + 1], lvl2[b, :L + 1])
        assert torch.equal(order.level_start[b, :L + 1], lvl[b, :L + 1])


def test_refine_golden_closed_form(golden):
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    g = golden('tree')
    gm = T(g['guide']).to(DEV)
    tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(gm)
    out = TreeFilter2D(sigma=0.02)(T(g['feature']).to(DEV), gm, tree, low_tree=False)
    assert torch.allclose(out.cpu().double(), T(g['filtered_high']), rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize('B,C,h,w,low', [(2, 1, 24, 30, True), (2, 1, 24, 30, False), (3, 4, 17, 9, False),
                                         (1, 1, 200, 256, False), (2, 2, 96, 96, True), (1, 1, 250, 260, False)])
def test_tree_filter_vs_oracle(B, C, h, w, low):
    """Module-level parity (MinimumSpanningTree + TreeFilter2D, autograd) against the C restatement of the reference's
    refine kernels.  The reference's BFS order is racy and every valid order gives a slightly different fp32 recursion,
    so the restatement is driven with OUR order (all three gradients <= 1e-4), and a float64 run of the same recursion
    arbitrates the absolute accuracy (<= 1e-3 as BASELINE.json asks, or no worse than the fp32 restatement itself)."""
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D, bfs
    from oracle import tree as ot
    gen = torch.Generator().manual_seed(7 + h)
    guide = torch.randn(B, 3, h, w, generator=gen)
    embed = torch.randn(B, 5, h, w, generator=gen) * (0.05 if low else 0.4)
    feat = torch.rand(B, C, h, w, generator=gen)
    gout = torch.randn(B, C, h, w, generator=gen)

    tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(guide.to(DEV))
    f = feat.to(DEV).requires_grad_(True)
    e = embed.to(DEV).requires_grad_(True)
    out = TreeFilter2D(sigma=0.02)(f, e, tree, low_tree=low)
    gf, ge = torch.autograd.grad((out * gout.to(DEV)).sum(), [f, e], allow_unused=True)

    idx, par, chd = (t.cpu() for t in bfs(tree, 4))                    # our order, handed to the restatement
    f_ref = feat.clone().requires_grad_(True)
    e_ref = embed.clone().requires_grad_(True)
    w_ref = ot.build_edge_weight(e_ref, idx, par, low)
    ref = ot.refine(f_ref.reshape(B, C, -1), w_ref, idx, par, chd, low).reshape(feat.shape)
    gf_ref, ge_ref = torch.autograd.grad((ref * gout).sum(), [f_ref, e_ref], allow_unused=True)
    assert rel_err(out.cpu(), ref.detach()) < 1e-4
    assert rel_err(gf.cpu(), gf_ref) < 1e-4
    if low:
        assert ge is None and ge_ref is None              # low_tree: no gradient to the embedding (refine.py:36-37)
        return
    assert rel_err(ge.cpu(), ge_ref) < 1e-4               # same order: same arithmetic up to summation order
    # float64 arbiter
    f64 = feat.double().requires_grad_(True)
    e64 = embed.double().requires_grad_(True)
    out64 = ot.tree_filter_f64(f64, e64, idx, par, low_tree=low)
    gf64, ge64 = torch.autograd.grad((out64 * gout.double()).sum(), [f64, e64])
    assert rel_err(out.cpu(), out64.detach()) < 1e-4 and rel_err(gf.cpu(), gf64) < 1e-4
    err_ours, err_fp32_ref = rel_err(ge.cpu(), ge64), rel_err(ge_ref, ge64)
    assert err_ours <= max(1e-3, 1.5 * err_fp32_ref), (err_ours, err_fp32_ref)


def test_channel_groups_equal_one_filter_per_group():
    """groups=2 (tree_filter.py:110-120, split_group): each half of the channels is filtered with the edge weights of its
    half of the embedding on the image's tree -- bit for bit what groups=1 gives for each half on its own."""
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    gen = torch.Generator().manual_seed(5)
    guide = torch.randn(2, 3, 20, 12, generator=gen).to(DEV)
    feat = torch.rand(2, 4, 20, 12, generator=gen).to(DEV)
    embed = (torch.randn(2, 4, 20, 12, generator=gen) * 0.4).to(DEV)
    gout = torch.randn(2, 4, 20, 12, generator=gen).to(DEV)
    tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(guide)

    def run(tf, f, e, g):
        f, e = f.clone().requires_grad_(True), e.clone().requires_grad_(True)
        out = tf(f, e, tree, low_tree=False)
        return (out.detach(),) + torch.autograd.grad((out * g).sum(), [f, e])

    both = run(TreeFilter2D(groups=2), feat, embed, gout)
    halves = [run(TreeFilter2D(groups=1), feat[:, s], embed[:, s], gout[:, s]) for s in (slice(0, 2), slice(2, 4))]
    for got, lo, hi in zip(both, *halves):
        assert torch.equal(got, torch.cat((lo, hi), dim=1))


def test_box2mask_call_pattern():
    """Box2Mask (box2mask_head.py:269-325): trees built once per image at 96x96 and repeated per query."""
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    gen = torch.Generator().manual_seed(11)
    img = torch.randn(2, 3, 96, 96, generator=gen).to(DEV)
    lst = torch.randn(2, 1, 96, 96, generator=gen).to(DEV).requires_grad_(True)
    mst, tf = MinimumSpanningTree(TreeFilter2D.norm2_distance), TreeFilter2D()
    t_img, t_lst = mst(img), mst(lst)
    rep = torch.tensor([3, 2], device=DEV)
    preds = torch.rand(5, 1, 96, 96, generator=gen).to(DEV).requires_grad_(True)
    img_r, lst_r = img.repeat_interleave(rep, 0), lst.repeat_interleave(rep, 0)
    s1 = tf(preds, img_r, t_img.repeat_interleave(rep, 0))
    s2 = tf(s1, lst_r, t_lst.repeat_interleave(rep, 0), low_tree=False)
    (s1.sum() + s2.sum()).backward()
    assert torch.isfinite(preds.grad).all() and torch.isfinite(lst.grad).all()
    assert 0.0 <= float(s2.min()) and float(s2.max()) <= 1.0 + 1e-5       # a normalised filter of values in [0,1]


@pytest.mark.parametrize('G,per,C,h,w,low', [(2, [3, 2], 1, 24, 30, True), (2, [1, 4], 1, 24, 30, False), (3, [2, 2, 1], 2, 96, 96, False)])
def test_grouped_tree_filter_equals_repeated_trees(G, per, C, h, w, low):
    """tree_of: n instances sharing G trees == the reference's repeat-per-instance call pattern (box2mask_head.py:271-276)."""
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    gen = torch.Generator().manual_seed(G * h)
    guide = torch.randn(G, 3, h, w, generator=gen).to(DEV)
    embed = (torch.randn(G, 5, h, w, generator=gen) * (0.05 if low else 0.4)).to(DEV)
    rep = torch.tensor(per, device=DEV)
    n = int(rep.sum())
    tree_of = torch.repeat_interleave(torch.arange(G, device=DEV), rep).to(torch.int32)
    feat = torch.rand(n, C, h, w, generator=gen).to(DEV)
    gout = torch.randn(n, C, h, w, generator=gen).to(DEV)
    tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(guide)
    tf = TreeFilter2D()
    f1, e1 = feat.clone().requires_grad_(True), embed.clone().requires_grad_(True)
    o1 = tf(f1, e1, tree, low_tree=low, tree_of=tree_of)
    f2, e2 = feat.clone().requires_grad_(True), embed.clone().requires_grad_(True)
    o2 = tf(f2, e2.repeat_interleave(rep, 0), tree.repeat_interleave(rep, 0), low_tree=low)
    assert rel_err(o1, o2) <= 1e-6
    g1 = torch.autograd.grad((o1 * gout).sum(), [f1, e1], allow_unused=True)
    g2 = torch.autograd.grad((o2 * gout).sum(), [f2, e2], allow_unused=True)
    assert rel_err(g1[0], g2[0]) <= 1e-6
    if low:
        assert g1[1] is None and g2[1] is None
    else:
        assert rel_err(g1[1], g2[1]) <= 1e-5
