"""The tree filter on trees built to reach its limits (tests/tree_shapes.py): paths, serpentines up to the grid-BFS
limit and past it, combs whose anti-diagonal levels hold every width up to 257 at level counts on both sides of the
256-level window refills, H-trees whose widest level is 1 024, 1 025 or over 4 096, brooms (generic trees) with a wide
fan-out after a path, and random MSTs.

- BFS: ``bfs(tree, 4, root)`` equals the canonical order bit for bit, from vertex 0 and from the centre, and the path
  that ordered the tree (grid fast path, or the generic path from the start or after the fast path declined) is the
  one the launch rule predicts.
- Refine and ``TreeFilter2D``: output, d/d feature and d/d edge weight against the C restatement driven with the
  GPU's order (1e-4), and output, d/d feature and d/d embed against a float64 recursion over positions; closed forms
  (unit weights, weights that underflow to zero) and run-to-run bit identity on every shape.
- Grouped launches mixing the shapes, a foreign (DFS) order, MSTs of guides that force these shapes, the zero-size
  shared-tree filter, and the kernels the profiler sees on both sides of each limit."""
import re

import numpy as np
import pytest
import torch

from tests import tree_shapes as ts
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
NAMES = list(ts.SHAPES)
KINDS = ('root0', 'centre')


def _tree(name):
    edges, (h, w) = ts.build(name)
    return torch.from_numpy(edges)[None].to(DEV), h, w


# ------------------------------------------------------------------------------------------------------------- BFS
def _align(n):
    return (n + 255) // 256 * 256


def _bfs_with_path(tree, V, root):
    """bxs_bfs_forward_rooted with a workspace of our own, so that its per-tree flag (1: ordered by bfs_grid_kernel, 0:
    by the generic bfs_block_kernel) can be read afterwards.  The offsets restate carve_bfs (deg, adj, counts, flags,
    each 256-byte aligned; 256 bytes behind them for the error word)."""
    from boxinstseg_b200 import _lib as L
    lib = L.lib()
    B = 1
    off_flags = _align(4 * B * V) + _align(16 * B * V) + _align(4 * B * V)
    nbytes = lib.bxs_bfs_workspace_bytes(B, V)
    assert nbytes == off_flags + _align(4 * B) + 256, 'the BFS workspace layout changed'
    ws = torch.full((nbytes,), 0xA5, dtype=torch.uint8, device=DEV)
    idx = torch.empty((B, V), dtype=torch.int32, device=DEV)
    par, lvl, nlv = torch.empty_like(idx), torch.empty((B, V + 1), dtype=torch.int32, device=DEV), \
        torch.empty(B, dtype=torch.int32, device=DEV)
    chd = torch.empty((B, V, 4), dtype=torch.int32, device=DEV)
    L.check(lib.bxs_bfs_forward_rooted(L.ptr(tree), L.ptr(idx), L.ptr(par), L.ptr(chd), L.ptr(lvl), L.ptr(nlv), L.ptr(ws),
                                       B, V, 4, int(root), L.stream()), 'bfs')
    flag = int(ws[off_flags:off_flags + 4].view(torch.int32)[0])
    return idx[0], par[0], chd[0], lvl[0], int(nlv[0]), flag


@pytest.mark.parametrize('name,kind', [(n, k) for n in NAMES for k in KINDS],
                         ids=[ts.case_id(n, k) for n in NAMES for k in KINDS])
def test_bfs_equals_canonical_order(name, kind):
    from boxinstseg_b200.ops.tree_filter import bfs
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as _C
    edges, (h, w) = ts.build(name)
    V = h * w
    root = ts.root_vertex(name, kind)
    tree = torch.from_numpy(edges)[None].to(DEV)
    r_idx, r_par, r_chd, r_lvl, r_L = ts.canonical_bfs(edges, V, root)
    assert (r_L, int(np.diff(r_lvl).max())) == ts.PROFILE[name][KINDS.index(kind)]
    idx, par, chd = bfs(tree, 4, root)
    lvl, nlv = _C.levels_of(idx, par)
    assert np.array_equal(idx[0].cpu().numpy(), r_idx)
    assert np.array_equal(par[0].cpu().numpy(), r_par)
    assert np.array_equal(chd[0].cpu().numpy(), r_chd)
    assert int(nlv[0]) == r_L and np.array_equal(lvl[0, :r_L + 1].cpu().numpy(), r_lvl)
    order = _C.bfs_order(tree, 4, root)                    # the same order as one value, and a copy of it, which is adopted
    lvl_c, nlv_c = _C.levels_of(idx.clone(), par)
    assert all(torch.equal(a, b) for a, b in zip(order[:3], (idx, par, chd)))
    assert torch.equal(order.num_levels, nlv) and torch.equal(nlv_c, nlv)
    assert torch.equal(order.level_start[0, :r_L + 1], lvl[0, :r_L + 1])
    assert torch.equal(lvl_c[0, :r_L + 1], lvl[0, :r_L + 1])
    # the path: the grid fast path is tried iff its shared memory fits, and keeps the tree iff the tree is 4-connected
    # on the pitch it infers and no level is wider than its frontier
    i2, p2, c2, l2, n2, flag = _bfs_with_path(tree, V, root)
    grid = ts.grid_bfs_tried(V) and ts.grid_pitch(edges, V) is not None and int(np.diff(r_lvl).max()) <= ts.BFS_FRONT
    assert flag == int(grid)
    assert torch.equal(i2, idx[0]) and torch.equal(p2, par[0]) and torch.equal(c2, chd[0]) and n2 == r_L
    assert torch.equal(l2[:r_L + 1], lvl[0, :r_L + 1])


# ---------------------------------------------------------------------------------------------------------- refine
# every shape runs all four (low_tree, C) combinations, two from each root
VARIANTS = {'root0': [(False, 3), (True, 1)], 'centre': [(False, 1), (True, 3)]}
REFINE_CASES = [(n, k, low, C) for n in NAMES for k in KINDS for low, C in VARIANTS[k]]


def _inputs(name, C, low, seed):
    _, (h, w) = ts.build(name)
    gen = torch.Generator().manual_seed(seed)
    feat = torch.rand(1, C, h, w, generator=gen)
    gout = torch.randn(1, C, h, w, generator=gen)
    embed = torch.randn(1, 5, h, w, generator=gen) * (0.05 if low else 0.4)
    return feat, gout, embed


def _f64_objective(x, g, embed, idx, par, sigma):
    V = x.shape[-1]
    w = ts.edge_weight_f64(embed.reshape(embed.shape[0], V), idx, par, sigma)
    return float((ts.refine_f64(x, w, idx, par) * g).sum())


@pytest.mark.parametrize('name,kind,low,C', REFINE_CASES,
                         ids=[f'{ts.case_id(n, k)}-{"low" if low else "high"}-C{C}' for n, k, low, C in REFINE_CASES])
def test_refine_and_tree_filter(name, kind, low, C):
    from boxinstseg_b200.ops.tree_filter import TreeFilter2D, bfs
    from boxinstseg_b200.ops.tree_filter.functions.refine import refine
    from oracle import tree as ot
    tree, h, w = _tree(name)
    V = h * w
    root = ts.root_vertex(name, kind)
    feat, gout, embed = _inputs(name, C, low, V + C)
    order = bfs(tree, 4, root)
    idx, par, chd = order
    tf = TreeFilter2D()
    outs = []
    for _ in range(2):
        f = feat.to(DEV).requires_grad_(True)
        e = embed.to(DEV).requires_grad_(True)
        out = tf(f, e, tree, low_tree=low, order=order)
        gf, ge = torch.autograd.grad((out * gout.to(DEV)).sum(), [f, e], allow_unused=True)
        outs.append((out.detach(), gf, ge))
    (out, gf, ge), (out2, gf2, ge2) = outs
    assert torch.equal(out, out2) and torch.equal(gf, gf2)                     # run to run
    assert (ge is None) == low and (ge2 is None) == low and (low or torch.equal(ge, ge2))

    # refine itself against the C restatement, driven with the GPU's order and edge weights
    wgt = tf.build_edge_weight(embed.to(DEV), idx, par, low, chd).detach()
    fr = feat.reshape(1, C, V).to(DEV).requires_grad_(True)
    wr = wgt.clone().requires_grad_(True)
    o = refine(fr, wr, idx, par, chd, False)
    gfr, gwr = torch.autograd.grad((o * gout.reshape(1, C, V).to(DEV)).sum(), [fr, wr])
    assert torch.equal(o.reshape(out.shape), out)
    i_c, p_c, c_c = idx.cpu(), par.cpu(), chd.cpu()
    f_ref = feat.reshape(1, C, V).clone().requires_grad_(True)
    w_ref = wgt.cpu().clone().requires_grad_(True)
    ref = ot.refine(f_ref, w_ref, i_c, p_c, c_c, False)
    gf_ref, gw_ref = torch.autograd.grad((ref * gout.reshape(1, C, V)).sum(), [f_ref, w_ref])
    assert rel_err(o.detach().cpu(), ref.detach()) < 1e-4
    assert rel_err(gfr.cpu(), gf_ref) < 1e-4
    assert rel_err(gwr.cpu(), gw_ref) < 1e-4

    # the whole filter against float64
    sigma = 0.02 if low else 1.0
    i_n, p_n = i_c[0].numpy(), p_c[0].numpy()
    x64, g64, e64 = (t.reshape(t.shape[1], V).double().numpy() for t in (feat, gout, embed))
    w64 = ts.edge_weight_f64(e64, i_n, p_n, sigma)
    assert rel_err(out.cpu().reshape(C, V), torch.from_numpy(ts.refine_f64(x64, w64, i_n, p_n))) < 1e-4
    assert rel_err(gf.cpu().reshape(C, V), torch.from_numpy(ts.refine_f64_grad_feature(g64, w64, i_n, p_n))) < 1e-4
    if low:
        return
    # d/d embed: the fp32 restatement through autograd, and float64 central differences along it
    e_ref = embed.clone().requires_grad_(True)
    w_e = ot.build_edge_weight(e_ref, i_c, p_c, False)
    r2 = ot.refine(feat.reshape(1, C, V), w_e, i_c, p_c, c_c, False)
    (ge_ref,) = torch.autograd.grad((r2 * gout.reshape(1, C, V)).sum(), [e_ref])
    assert rel_err(ge.cpu(), ge_ref) < 1e-4
    v = (ge_ref / ge_ref.norm()).reshape(5, V).double().numpy()
    eps = 1e-5
    fd = (_f64_objective(x64, g64, e64 + eps * v, i_n, p_n, sigma) -
          _f64_objective(x64, g64, e64 - eps * v, i_n, p_n, sigma)) / (2 * eps)
    ours = float((ge.cpu().double().reshape(5, V).numpy() * v).sum())
    theirs = float((ge_ref.double().reshape(5, V).numpy() * v).sum())
    err_ours, err_ref = abs(ours - fd) / abs(fd), abs(theirs - fd) / abs(fd)
    assert err_ours <= max(1e-3, 1.5 * err_ref), (err_ours, err_ref)


@pytest.mark.parametrize('name,kind', [(n, k) for n in NAMES for k in KINDS],
                         ids=[ts.case_id(n, k) for n in NAMES for k in KINDS])
def test_closed_forms(name, kind):
    """Unit weights (a constant embedding): every output is the channel mean and d/d feature is sum(g) / V, the same
    value at every vertex.  Weights that underflow to 0 (low_tree, embedding steps of 3): the filter is the identity, bit
    for bit, and so is its d/d feature."""
    from boxinstseg_b200.ops.tree_filter import TreeFilter2D, bfs
    tree, h, w = _tree(name)
    V = h * w
    C = 3
    order = bfs(tree, 4, ts.root_vertex(name, kind))
    gen = torch.Generator().manual_seed(V)
    feat = torch.rand(1, C, h, w, generator=gen).to(DEV)
    gout = (torch.randn(1, C, h, w, generator=gen) + 0.5).to(DEV)
    tf = TreeFilter2D()

    f = feat.clone().requires_grad_(True)
    e = torch.full((1, 2, h, w), 0.7, device=DEV, requires_grad=True)
    out = tf(f, e, tree, low_tree=False, order=order)
    gf, ge = torch.autograd.grad((out * gout).sum(), [f, e])
    o, g = out.detach().reshape(C, V), gf.reshape(C, V)
    assert torch.equal(o, o[:, :1].expand(C, V)) and torch.equal(g, g[:, :1].expand(C, V))
    assert rel_err(o[:, 0], feat.double().reshape(C, V).mean(1)) < 1e-4
    assert rel_err(g[:, 0], gout.double().reshape(C, V).sum(1) / V) < 1e-4
    assert torch.isfinite(ge).all()

    f = feat.clone().requires_grad_(True)
    e = (3.0 * torch.arange(V, dtype=torch.float32, device=DEV)).reshape(1, 1, h, w)
    out = tf(f, e, tree, low_tree=True, order=order)
    (gf,) = torch.autograd.grad((out * gout).sum(), [f])
    assert torch.equal(out.detach(), feat) and torch.equal(gf, gout)


# --------------------------------------------------------------------------------------------------------- grouped
GROUPED = {63: ('serpentine', 'comb', (5,), 'random'), 255: ('serpentine', 'comb', (7,), 'random')}


def _group_trees(n):
    out = []
    for kind in GROUPED[n]:
        if kind == 'serpentine':
            out.append(ts.serpentine(n, n)[0])
        elif kind == 'comb':
            out.append(ts.comb(n, n)[0])
        elif kind == 'random':
            out.append(ts.random_mst(n, n, seed=n)[0])
        else:
            out.append(ts.htree(*kind)[0])
    return out


@pytest.mark.parametrize('n', [63, 255], ids=['63x63-smem', '255x255-global'])
@pytest.mark.parametrize('low', [False, True], ids=['high', 'low'])
def test_grouped_mixed_shapes(n, low):
    """One launch over a serpentine, a comb, an H-tree and a random MST of the same map, with a non-monotone tree_of
    and more instances than trees: equal to the repeated trees, and to float64 per instance."""
    from boxinstseg_b200.ops.tree_filter import TreeFilter2D, bfs
    trees = torch.from_numpy(np.stack(_group_trees(n))).to(DEV)
    G, V, C = trees.shape[0], n * n, 2
    tree_of = torch.tensor([2, 0, 3, 1, 2, 0, 3, 3, 1], dtype=torch.int32, device=DEV)
    N = tree_of.numel()
    gen = torch.Generator().manual_seed(n + low)
    embed = (torch.randn(G, 5, n, n, generator=gen) * (0.05 if low else 0.4)).to(DEV)
    feat = torch.rand(N, C, n, n, generator=gen).to(DEV)
    gout = torch.randn(N, C, n, n, generator=gen).to(DEV)
    tf = TreeFilter2D()
    f1, e1 = feat.clone().requires_grad_(True), embed.clone().requires_grad_(True)
    o1 = tf(f1, e1, trees, low_tree=low, tree_of=tree_of)
    g1 = torch.autograd.grad((o1 * gout).sum(), [f1, e1], allow_unused=True)
    rep = tree_of.long()
    f2, e2 = feat.clone().requires_grad_(True), embed.clone().requires_grad_(True)
    o2 = tf(f2, e2[rep], trees[rep], low_tree=low)
    g2 = torch.autograd.grad((o2 * gout).sum(), [f2, e2], allow_unused=True)
    assert rel_err(o1, o2) <= 1e-6 and rel_err(g1[0], g2[0]) <= 1e-6
    if low:
        assert g1[1] is None and g2[1] is None
    else:
        assert rel_err(g1[1], g2[1]) <= 1e-5
    idx, par, _ = bfs(trees, 4, ts.centre((n, n)))
    sigma = 0.02 if low else 1.0
    for i, t in enumerate(tree_of.tolist()):
        i_n, p_n = idx[t].cpu().numpy(), par[t].cpu().numpy()
        w64 = ts.edge_weight_f64(embed[t].reshape(5, V).double().cpu().numpy(), i_n, p_n, sigma)
        x = feat[i].reshape(C, V).double().cpu().numpy()
        g = gout[i].reshape(C, V).double().cpu().numpy()
        assert rel_err(o1[i].detach().cpu().reshape(C, V), torch.from_numpy(ts.refine_f64(x, w64, i_n, p_n))) < 1e-4
        assert rel_err(g1[0][i].cpu().reshape(C, V), torch.from_numpy(ts.refine_f64_grad_feature(g, w64, i_n, p_n))) < 1e-4


# --------------------------------------------------------------------------------------------------- foreign order
FOREIGN = [(n, k) for n in ('htree-m5-w1024', 'broom-L257-W1025', 'comb129x640', 'random64x80') for k in KINDS]


@pytest.mark.parametrize('name,kind', FOREIGN, ids=[ts.case_id(n, k) for n, k in FOREIGN])
def test_foreign_order_is_adopted_bit_for_bit(name, kind):
    """A depth-first order of the same tree, rooted at the same vertex, through refine_forward / refine_backward_*:
    every result equals the canonical order's, bit for bit, moved to the foreign positions."""
    from boxinstseg_b200.ops.tree_filter import bfs
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as _C
    edges, (h, w) = ts.build(name)
    V, C = h * w, 3
    root = ts.root_vertex(name, kind)
    tree = torch.from_numpy(edges)[None].to(DEV)
    idx, par, chd = bfs(tree, 4, root)
    d_idx, d_par, d_chd = (torch.from_numpy(a)[None].to(DEV) for a in ts.dfs_order(edges, V, root))
    gen = torch.Generator().manual_seed(V)
    feat = torch.rand(1, C, V, generator=gen).to(DEV)
    gout = torch.randn(1, C, V, generator=gen).to(DEV)
    w_vertex = (torch.rand(1, V, generator=gen) * 0.9).to(DEV)            # edge weight of each vertex to its parent
    w_can = torch.gather(w_vertex, 1, idx.long())
    w_dfs = torch.gather(w_vertex, 1, d_idx.long())
    pos = torch.empty(V, dtype=torch.long, device=DEV)
    pos[idx[0].long()] = torch.arange(V, device=DEV)
    perm = pos[d_idx[0].long()]                                            # foreign position -> canonical position
    can = _C.refine_forward(feat, w_can, idx, par, chd)
    dfs = _C.refine_forward(feat, w_dfs, d_idx, d_par, d_chd)
    for k in (0, 1, 3):                                                    # out, aggr, wsum: vertex order
        assert torch.equal(dfs[k], can[k])
    for k in (2, 4):                                                       # aggr_up, wsum_up: position order
        assert torch.equal(dfs[k], can[k][..., perm])
    args_c = (feat, w_can, idx, par, chd, can[0], can[1], can[2], can[3], can[4], gout)
    args_d = (feat, w_dfs, d_idx, d_par, d_chd, dfs[0], dfs[1], dfs[2], dfs[3], dfs[4], gout)
    assert torch.equal(_C.refine_backward_feature(*args_d), _C.refine_backward_feature(*args_c))
    assert torch.equal(_C.refine_backward_weight(*args_d), _C.refine_backward_weight(*args_c)[..., perm])


# ------------------------------------------------------------------------------------------------------------- MST
def _ramp_guide(order_of_vertex, h, w):
    return torch.from_numpy(order_of_vertex.astype(np.float32)).reshape(1, 1, h, w)


MST_CASES = {'serpentine63x63': lambda: ts.serpentine(63, 63), 'serpentine256x748': lambda: ts.serpentine(256, 748),
             'serpentine438x438': lambda: ts.serpentine(438, 438), 'comb129x640': lambda: ts.comb(129, 640),
             'comb256x748': lambda: ts.comb(256, 748)}


@pytest.mark.parametrize('name', list(MST_CASES))
def test_mst_of_guides_that_force_the_shape(name):
    """A serpentine's guide is each pixel's index along the path: path edges weigh 2, every other edge at least 10.  A
    comb's guide is the pixel's id r * w + c: horizontal edges weigh 2, all vertical edges tie at w^2 + 1 and the
    (weight, id) order takes the one in column 0 for each pair of rows.  The GPU's edge set equals Kruskal's and the
    builder's tree."""
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    from oracle import tree as ot
    edges, (h, w) = MST_CASES[name]()
    V = h * w
    if name.startswith('serpentine'):
        idx, _, _, _, _ = ts.canonical_bfs(edges, V, 0)
        t = np.empty(V, np.int64)
        t[idx] = np.arange(V)
        guide = _ramp_guide(t, h, w)
    else:
        guide = _ramp_guide(np.arange(V), h, w)
    mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
    g = guide.to(DEV)
    tree = mst(g)
    torch.cuda.synchronize()
    ids = ot.edges_to_ids(tree[0].cpu().numpy(), h, w)
    ei = ot.grid_edges(h, w)
    ew = ot.grid_edge_weights(guide).numpy()[0]
    assert np.array_equal(ids, ot.mst_edge_ids(ei, ew, V))
    assert np.array_equal(ids, ot.edges_to_ids(edges, h, w))
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    times = []
    for _ in range(5):
        start.record()
        mst(g)
        end.record()
        torch.cuda.synchronize()
        times.append(start.elapsed_time(end))
    print(f'[mst] {name} V={V}: {sorted(times)[2]:.3f} ms (median of 5, {torch.cuda.get_device_name()})')


# ------------------------------------------------------------------------------------------------------- zero size
@pytest.mark.parametrize('low', [False, True], ids=['high', 'low'])
def test_zero_size_shared_tree_filter(low):
    """No instance shares the trees: an empty output, an empty d/d feature, and a zero d/d embed (None for low_tree)."""
    from boxinstseg_b200.ops.tree_filter import TreeFilter2D
    trees = torch.from_numpy(np.stack([ts.comb(9, 11)[0], ts.serpentine(9, 11)[0]])).to(DEV)
    feat = torch.rand(0, 3, 9, 11, device=DEV, requires_grad=True)
    embed = torch.randn(2, 4, 9, 11, device=DEV, requires_grad=True)
    out = TreeFilter2D()(feat, embed, trees, low_tree=low, tree_of=torch.zeros(0, dtype=torch.int32, device=DEV))
    assert out.shape == (0, 3, 9, 11)
    gf, ge = torch.autograd.grad(out.sum(), [feat, embed], allow_unused=True)
    assert gf.shape == feat.shape
    if low:
        assert ge is None
    else:
        assert ge.shape == embed.shape and not ge.any()


# -------------------------------------------------------------------------------------------------------- profiler
KERNEL = re.compile(r'\b(bfs_\w+_kernel|refine_\w+_kernel)\b')
PATH_SHAPES = ['comb215x244', 'comb201x261', 'serpentine215x244', 'serpentine201x261', 'comb256x748',
               'serpentine256x748', 'path1x191489', 'serpentine438x438', 'htree-m5-w1025']


def _traced(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    for _ in range(5):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]):
            torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = {e.name for e in prof.events() if KERNEL.search(e.name)}
        if any('refine_bwd_weight_kernel' in n for n in names):
            return names
    return names


def check_paths():
    """Per shape: bfs_grid_kernel is launched iff grid_bfs_tried(V), and the refine kernels are the shared-memory (true)
    or global-memory (false) instantiations iff refine_in_smem(V)."""
    from boxinstseg_b200.ops.tree_filter import TreeFilter2D
    for name in PATH_SHAPES:
        tree, h, w = _tree(name)
        V = h * w
        f = torch.rand(1, 1, h, w, device=DEV, requires_grad=True)
        e = (torch.randn(1, 2, h, w, device=DEV) * 0.4).requires_grad_(True)

        def run():
            TreeFilter2D()(f, e, tree, low_tree=False).sum().backward()
        names = _traced(run)
        print(f'[kernels] {name} V={V}: {sorted({re.search(r"\w+_kernel(<[^>]*>)?", n).group(0) for n in names})}',
              flush=True)
        grid = any('bfs_grid_kernel' in n for n in names)
        assert grid == ts.grid_bfs_tried(V), (name, names)
        s, o = ('true', 'false') if ts.refine_in_smem(V) else ('false', 'true')
        for want in (rf'refine_updown_kernel<(\(int\))?0, {s}>', rf'refine_updown_kernel<(\(int\))?1, {s}>',
                     rf'refine_bwd_weight_kernel<{s}>'):
            assert any(re.search(want, n) for n in names), (name, want, names)
        assert not any(re.search(rf'<((\(int\))?\d, )?{o}>', n) for n in names if 'refine_' in n), (name, names)


def test_profiler_sees_the_predicted_paths():
    """check_paths in a process of its own (as test_dispatch_paths_gpu does: the profiler's kernel records are complete
    in a fresh process)."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, '-c', 'from tests.test_tree_shapes_gpu import check_paths; check_paths()'],
                       cwd=root, capture_output=True, text=True, timeout=900)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert r.stdout.count('[kernels] ') == len(PATH_SHAPES)
