"""GPU parity against the REFERENCE'S OWN CUDA kernels: oracle/make_golden_ref_ext.py runs the reference's
mmdet/ops/pairwise and mmdet/ops/tree_filter extensions (compiled unmodified by oracle/Makefile into oracle/_ref/) on the
inputs built here and stores their outputs in tests/golden/ref_ext.npz.  These tests pin rows a7, a12, a13, a15 on the
reference itself rather than on restatements.  Outputs larger than a few thousand entries are stored as a fixed, seeded
sample of their entries (sample_index)."""
import numpy as np
import pytest
import torch

from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'

PAIRWISE_CASES = [((3, 1, 37, 53), 3, 2), ((2, 1, 16, 64), 3, 1), ((2, 1, 40, 70), 5, 2), ((4, 1, 200, 256), 3, 2)]
MST_CASES = [(2, 3, 24, 40), (1, 5, 50, 64)]
REFINE_CASES = [(2, 4, 24, 40), (1, 1, 50, 64)]
SAMPLE = 4096


def sample_index(n, k=SAMPLE, seed=0):
    """The entries of a flattened output of n elements that the golden file keeps (all of them when n <= k)."""
    if n <= k:
        return torch.arange(n)
    return torch.randperm(n, generator=torch.Generator().manual_seed(seed))[:k].sort().values


def case_key(*args):
    return '_'.join(str(a) for a in args)


# ------------------------------------------------------------------ inputs (shared with oracle/make_golden_ref_ext.py)
def pairwise_inputs(shape, k):
    gen = torch.Generator().manual_seed(3)
    x = (torch.randn(shape, generator=gen) * 3).to(DEV)
    x.view(-1)[:4] = torch.tensor([45.0, -45.0, 30.0, -60.0], device=DEV)[: min(4, x.numel())]
    g = torch.rand(shape[0], k * k - 1, *shape[2:], generator=gen).to(DEV)
    return x, g


def grid_problem(B, C, h, w, seed):
    from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
    gen = torch.Generator().manual_seed(seed)
    guide = torch.randn(B, C, h, w, generator=gen).to(DEV)
    mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
    index = mst._build_matrix_index(guide).contiguous()
    weight = mst._build_feature_weight(guide)
    return guide, index, weight


def refine_inputs(B, C, h, w):
    """Our MST and our deterministic BFS order (fed to both implementations), features, edge weights, upstream grads."""
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as ours
    _, index, weight = grid_problem(B, 3, h, w, seed=7 * h)
    V = h * w
    tree = ours.mst_forward(index, weight, V)
    idx, par, chd = ours.bfs_forward(tree, 4)
    gen = torch.Generator().manual_seed(1)
    feat = torch.rand(B, C, V, generator=gen).to(DEV)
    ew = torch.rand(B, V, generator=gen).to(DEV) * 0.9 + 0.05     # edge weights in (0, 1), entry 0 ignored
    gout = torch.randn(B, C, V, generator=gen).to(DEV)
    return feat, ew, idx, par, chd, gout


BFS_CASE = (2, 2, 20, 28)


def bfs_inputs():
    """The tree of the foreign-order case, features, upstream grads and edge weights (per position of the order)."""
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as ours
    B, C, h, w = BFS_CASE
    _, index, weight = grid_problem(B, 3, h, w, seed=11)
    tree = ours.mst_forward(index, weight, h * w)
    gen = torch.Generator().manual_seed(2)
    feat = torch.rand(B, C, h * w, generator=gen).to(DEV)
    gout = torch.randn(B, C, h * w, generator=gen).to(DEV)
    ew = torch.rand(B, h * w, generator=gen).to(DEV) * 0.9 + 0.05
    return tree, feat, gout, ew


def _edge_set(tree):
    e = np.sort(np.asarray(tree.cpu() if torch.is_tensor(tree) else tree).astype(np.int64), axis=-1)
    return [set(map(tuple, e[b].tolist())) for b in range(e.shape[0])]


@pytest.fixture(scope='module')
def ref(golden):
    return golden('ref_ext')


def _stored(ref, key):
    return torch.from_numpy(ref[key]).to(DEV)


# ------------------------------------------------------------------ a7: pairwise_nlog (pairwise.cu:68-149)
@pytest.mark.parametrize('shape,k,d', PAIRWISE_CASES)
def test_pairwise_matches_reference_cuda(ref, shape, k, d):
    from boxinstseg_b200.ops.pairwise import pairwise_ext as ours
    key = case_key('pw', *shape, k, d)
    x, g = pairwise_inputs(shape, k)
    pw = ours.pairwise_nlog_forward(k, d, x)
    assert list(pw.shape) == list(ref[key + '_shape'])
    sel = sample_index(pw.numel()).to(DEV)
    pw_ref = _stored(ref, key + '_fwd')
    assert torch.allclose(pw.flatten()[sel], pw_ref, rtol=1e-4, atol=1e-5)
    gx = ours.pairwise_nlog_backward(k, d, x, pw, g).flatten()[sample_index(x.numel()).to(DEV)]
    gx_ref = _stored(ref, key + '_bwd')
    assert torch.allclose(gx, gx_ref, rtol=1e-3, atol=1e-5) and rel_err(gx, gx_ref) <= 1e-4   # theirs: float atomics


# ------------------------------------------------------------------ a12 / a13 / a15: tree filter (src/mst, src/bfs, src/refine)
@pytest.mark.parametrize('B,C,h,w', MST_CASES)
def test_mst_edge_set_matches_reference(ref, B, C, h, w):
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as ours
    _, index, weight = grid_problem(B, C, h, w, seed=h)
    t = ours.mst_forward(index, weight, h * w)
    assert _edge_set(t) == _edge_set(ref[case_key('mst', B, C, h, w)])


@pytest.mark.parametrize('B,C,h,w', REFINE_CASES)
def test_refine_matches_reference_cuda(ref, B, C, h, w):
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as ours
    key = case_key('refine', B, C, h, w)
    feat, ew, idx, par, chd, gout = refine_inputs(B, C, h, w)
    o = ours.refine_forward(feat, ew, idx, par, chd)
    r0 = _stored(ref, key + '_out')
    assert rel_err(o[0], r0) <= 1e-5 and torch.allclose(o[0], r0, rtol=1e-3, atol=1e-5)
    gf = ours.refine_backward_feature(feat, ew, idx, par, chd, o[0], o[1], o[2], o[3], o[4], gout)
    assert rel_err(gf, _stored(ref, key + '_gfeat')) <= 1e-5
    gw = ours.refine_backward_weight(feat, ew, idx, par, chd, o[0], o[1], o[2], o[3], o[4], gout)
    assert rel_err(gw[:, 1:], _stored(ref, key + '_gweight')[:, 1:]) <= 1e-4               # entry 0 is the root (no edge)


def test_reference_bfs_order_is_accepted(ref):
    """The reference's own (racy, any parent-before-child) BFS order, fed to OUR refine entry points, gives the
    reference's results: the shim adopts foreign orders (tree_filter_cuda._adopt) instead of assuming its own.  The
    order is the one the reference produced when the golden file was made."""
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as ours
    tree, feat, gout, ew = bfs_inputs()
    assert _edge_set(tree) == _edge_set(ref['bfs_tree'])
    ridx, rpar, rchd = (_stored(ref, 'bfs_' + n) for n in ('idx', 'par', 'chd'))
    o = ours.refine_forward(feat, ew, ridx, rpar, rchd)
    for i, a in enumerate(o):
        assert rel_err(a, _stored(ref, f'bfs_out{i}')) <= 1e-5
    gf = ours.refine_backward_feature(feat, ew, ridx, rpar, rchd, o[0], o[1], o[2], o[3], o[4], gout)
    assert rel_err(gf, _stored(ref, 'bfs_gfeat')) <= 1e-5
    gw = ours.refine_backward_weight(feat, ew, ridx, rpar, rchd, o[0], o[1], o[2], o[3], o[4], gout)
    assert rel_err(gw[:, 1:], _stored(ref, 'bfs_gweight')[:, 1:]) <= 1e-4
    # the same order through the grouped path (autograd, one tree per instance: tree_of = arange(B)) is adopted as well,
    # never run with the level table of another order
    from boxinstseg_b200.ops.tree_filter import refine
    B, V = ew.shape
    f, w = feat.clone().requires_grad_(True), ew.clone().requires_grad_(True)
    og = refine(f, w, ridx, rpar, rchd, False, torch.arange(B, dtype=torch.int32, device=DEV))
    assert rel_err(og, _stored(ref, 'bfs_out0')) <= 1e-5
    gfg, gwg = torch.autograd.grad((og * gout).sum(), [f, w])
    assert rel_err(gfg, _stored(ref, 'bfs_gfeat')) <= 1e-5
    assert rel_err(gwg[:, 1:], _stored(ref, 'bfs_gweight')[:, 1:]) <= 1e-4
    # and the same tree through our own deterministic order gives the same filter output
    idx, par, chd = ours.bfs_forward(tree, 4)
    wv = torch.zeros(B, V, device=DEV).scatter_(1, ridx.long(), ew)   # weight of the edge (vertex -> parent), by vertex id
    o2 = ours.refine_forward(feat, torch.gather(wv, 1, idx.long()), idx, par, chd)[0]
    assert rel_err(o2, o[0]) <= 1e-5
