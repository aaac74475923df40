"""The tree builders of tests/tree_shapes.py deliver what they advertise (spanning trees of degree <= 4, 4-adjacent on
the grid where they claim a grid tree, the level profile of the table), the canonical BFS matches the C oracle at
root 0, and the float64 recursion over positions matches the level-by-level and dense float64 references."""
import numpy as np
import pytest
import torch

from tests import tree_shapes as ts

GRID = {ts.path, ts.serpentine, ts.comb, ts.htree, ts.random_mst}


@pytest.mark.parametrize('name', list(ts.SHAPES))
def test_builder_delivers_its_profile(name):
    edges, (h, w) = ts.build(name)
    V = h * w
    assert edges.dtype == np.int32 and edges.shape == (V - 1, 2)
    assert len({(min(a, b), max(a, b)) for a, b in edges.tolist()}) == V - 1
    assert np.bincount(edges.ravel(), minlength=V).max() <= 4
    idx, par, chd, lvl, L = ts.canonical_bfs(edges, V, 0)                  # raises unless every vertex is reached
    assert sorted(idx.tolist()) == list(range(V))
    if ts.SHAPES[name][0] in GRID:
        a, b = edges.min(1).astype(np.int64), edges.max(1).astype(np.int64)
        assert np.all(((b - a == 1) & (a // w == b // w)) | (b - a == w)), 'not 4-adjacent'
        assert ts.grid_pitch(edges, V) in (w, V)
    else:
        assert ts.grid_pitch(edges, V) is None                             # the grid fast path must reject it
    for kind in ('root0', 'centre'):
        assert ts.profile(edges, V, ts.root_vertex(name, kind)) == ts.PROFILE[name][kind != 'root0'], kind


def test_limits_restated_from_the_constants():
    assert ts.GRID_BFS_MAX_V == 191488 and ts.grid_bfs_tried(191488) and not ts.grid_bfs_tried(191489)
    assert ts.REFINE_SMEM_MAX_V == 52460 and ts.refine_in_smem(52460) and not ts.refine_in_smem(52461)
    assert ts._RING_BYTES == 22528


def test_shapes_cover_the_limits():
    prof = {n: p for n, p in ts.PROFILE.items()}
    Ls = {p[0][0] for p in prof.values()}
    for M in range(256, 1281, 256):
        assert {M - 1, M, M + 1} <= Ls, M
    assert set(range(2, 9)) <= Ls
    widths = {p[k][1] for p in prof.values() for k in (0, 1)}                # widest levels
    for name in ('comb33x224', 'comb129x384', 'comb257x200'):                  # every width up to min(h, w) inside a comb
        _, _, _, lvl, _ = ts.canonical_bfs(ts.build(name)[0], int(np.prod(ts.build(name)[1])), 0)
        widths |= set(np.diff(lvl).tolist())
    assert {32, 33, 127, 128, 129, 255, 256, 257, 511, 512, 513, 1024, 1025} <= widths and max(widths) > 4096
    V = {n: np.prod(ts.build(n)[1]) for n in ('serpentine256x748', 'path1x191489', 'serpentine215x244',
                                               'serpentine201x261')}
    assert V['serpentine256x748'] == ts.GRID_BFS_MAX_V and V['path1x191489'] == ts.GRID_BFS_MAX_V + 1
    assert V['serpentine215x244'] == ts.REFINE_SMEM_MAX_V and V['serpentine201x261'] == ts.REFINE_SMEM_MAX_V + 1


@pytest.mark.parametrize('name', ['htree-m5-w1024', 'broom-L257-W1025', 'comb33x224', 'random64x80', 'path1x7'])
def test_canonical_bfs_equals_oracle_at_root0(name):
    from oracle import tree as ot
    edges, (h, w) = ts.build(name)
    idx, par, chd = (t[0].numpy() for t in ot.bfs(torch.from_numpy(edges)[None]))
    r_idx, r_par, r_chd, _, _ = ts.canonical_bfs(edges, h * w, 0)
    assert np.array_equal(idx, r_idx) and np.array_equal(par, r_par) and np.array_equal(chd, r_chd)


def test_dfs_order_is_a_parent_first_order_of_the_same_tree():
    edges, (h, w) = ts.build('htree-m5-w1024')
    V = h * w
    idx, par, chd = ts.dfs_order(edges, V, ts.centre((h, w)))
    assert idx[0] == ts.centre((h, w)) and sorted(idx.tolist()) == list(range(V))
    assert np.all(par[1:] < np.arange(1, V))
    assert {(min(a, b), max(a, b)) for a, b in zip(idx[1:].tolist(), idx[par[1:]].tolist())} == \
        {(min(a, b), max(a, b)) for a, b in edges.tolist()}
    c_idx = ts.canonical_bfs(edges, V, ts.centre((h, w)))[0]
    assert not np.array_equal(idx, c_idx)


@pytest.mark.parametrize('name,kind', [('broom-L6-W257', 'root0'), ('comb33x224', 'centre'), ('htree-m5-w1025', 'root0'),
                                       ('random64x80', 'centre')])
def test_f64_recursion_over_positions(name, kind):
    """refine_f64 equals oracle.tree.tree_filter_f64 (levels in torch) on the same order, and its d/d feature equals
    torch autograd through tree_filter_f64."""
    from oracle import tree as ot
    edges, (h, w) = ts.build(name)
    V, C = h * w, 2
    idx, par, _, _, _ = ts.canonical_bfs(edges, V, ts.root_vertex(name, kind))
    gen = torch.Generator().manual_seed(V)
    x = torch.rand(1, C, h, w, generator=gen, dtype=torch.float64).requires_grad_(True)
    g = torch.randn(1, C, h, w, generator=gen, dtype=torch.float64)
    e = torch.randn(1, 3, h, w, generator=gen, dtype=torch.float64) * 0.4
    ti, tp = torch.from_numpy(idx)[None], torch.from_numpy(par)[None]
    ref = ot.tree_filter_f64(x, e, ti, tp, low_tree=False)
    (gref,) = torch.autograd.grad((ref * g).sum(), [x])
    w64 = ts.edge_weight_f64(e.reshape(3, V).numpy(), idx, par, 1.0)
    out = ts.refine_f64(x.detach().reshape(C, V).numpy(), w64, idx, par)
    gx = ts.refine_f64_grad_feature(g.reshape(C, V).numpy(), w64, idx, par)
    np.testing.assert_allclose(out, ref.detach().reshape(C, V).numpy(), rtol=1e-12, atol=1e-14)
    np.testing.assert_allclose(gx, gref.reshape(C, V).numpy(), rtol=1e-10, atol=1e-13)


def test_f64_recursion_equals_dense_closed_form():
    """On a tiny tree of each kind: the closed form sum_j prod(w on the path) x_j / sum_j prod(w on the path)."""
    from oracle import tree as ot
    for edges, (h, w) in (ts.comb(4, 5), ts.serpentine(3, 4), ts.broom(2, [3, 5]), ts.htree(1)):
        V = h * w
        gen = torch.Generator().manual_seed(V)
        x = torch.rand(1, 2, h, w, generator=gen, dtype=torch.float64)
        e = torch.randn(1, 3, h, w, generator=gen, dtype=torch.float64) * 0.3
        dense = ot.tree_filter_dense(x, e, torch.from_numpy(edges)[None], low_tree=False).reshape(2, V).numpy()
        for root in (0, V // 2):
            idx, par, _, _, _ = ts.canonical_bfs(edges, V, root)
            w64 = ts.edge_weight_f64(e.reshape(3, V).numpy(), idx, par, 1.0)
            np.testing.assert_allclose(ts.refine_f64(x.reshape(2, V).numpy(), w64, idx, par), dense, rtol=1e-12)
