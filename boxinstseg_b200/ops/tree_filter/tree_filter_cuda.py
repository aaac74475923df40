"""Stand-in for the reference's pybind module ``tree_filter_cuda``
(mmdet/ops/tree_filter/src/tree_filter.cpp:7-13): the same five functions with the same argument
order and return values, implemented on the C ABI of libboxseg_b200."""
from typing import NamedTuple

import torch

from ... import _lib as L

_LEVELS = '_bxs_levels'        # the attribute _remember / _recall keep on a sorted_index tensor object


class TreeOrder(NamedTuple):
    """A batch of trees in BFS order, with the level table the level-by-level refine kernels walk (all int32)."""
    sorted_index: torch.Tensor      # [B,V]    vertex at each position
    sorted_parent: torch.Tensor     # [B,V]    position of each position's parent
    sorted_child: torch.Tensor      # [B,V,4]  positions of each position's children, 0-padded
    level_start: torch.Tensor       # [B,V+1]  first position of each level
    num_levels: torch.Tensor        # [B]


def _i32(t):
    return t if t.dtype == torch.int32 and t.is_contiguous() else t.to(torch.int32).contiguous()


def _f32(t):
    return t if t.dtype == torch.float32 and t.is_contiguous() else t.float().contiguous()


def _edges(t):
    """An edge list [B,E,2] as the kernels read it: int32, dense, and 8-byte aligned (one ``int2`` load per edge)."""
    return L.dense_aligned(_i32(t), 8)


def mst_forward(edge_index, edge_weight, vertex_count):
    ei, ew = _edges(edge_index), _f32(edge_weight)
    L.require_cuda(ei, ew)
    B, E = ei.shape[0], ei.shape[1]
    V = int(vertex_count)
    out = torch.empty((B, V - 1, 2), dtype=torch.int32, device=ei.device)
    lib = L.lib()
    ws = torch.empty(lib.bxs_mst_workspace_bytes(B, E, V), dtype=torch.uint8, device=ei.device)
    with torch.cuda.device(ei.device):
        L.check(lib.bxs_mst_forward(L.ptr(ei), L.ptr(ew), L.ptr(out), L.ptr(ws), B, E, V, L.stream()), 'mst_forward')
    return out


def bfs_order(edge_index, max_adj_per_node, root=0):
    """The deterministic level order of each tree, rooted at vertex ``root``, as a TreeOrder."""
    te = _edges(edge_index)
    L.require_cuda(te)
    B, V = te.shape[0], te.shape[1] + 1
    dev = te.device
    idx = torch.empty((B, V), dtype=torch.int32, device=dev)
    par = torch.empty((B, V), dtype=torch.int32, device=dev)
    chd = torch.empty((B, V, max_adj_per_node), dtype=torch.int32, device=dev)
    lvl = torch.empty((B, V + 1), dtype=torch.int32, device=dev)
    nlv = torch.empty(B, dtype=torch.int32, device=dev)
    lib = L.lib()
    ws = torch.empty(lib.bxs_bfs_workspace_bytes(B, V), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.bxs_bfs_forward_rooted(L.ptr(te), L.ptr(idx), L.ptr(par), L.ptr(chd), L.ptr(lvl), L.ptr(nlv), L.ptr(ws), B, V,
                                           int(max_adj_per_node), int(root), L.stream()), 'bfs_forward')
    return TreeOrder(idx, par, chd, lvl, nlv)


# The reference's five functions pass an order as three bare tensors, with no place for its level table.  So that code
# written against them stays free of host synchronisation, bfs_forward remembers the table on the sorted_index it
# returns and the refine_* functions recall it; everything else in the package carries a TreeOrder instead.
def _remember(sorted_index, level_start, num_levels):
    setattr(sorted_index, _LEVELS, (level_start, num_levels, sorted_index._version))


def _recall(sorted_index):
    """(level_start, num_levels) remembered for exactly this tensor object in its current state, else None: a tensor
    written since (another `_version`), e.g. a buffer modified in place or reused as an output, counts as foreign."""
    memo = getattr(sorted_index, _LEVELS, None)
    if memo is None or memo[2] != sorted_index._version:
        return None
    return memo[0], memo[1]


def bfs_forward(edge_index, max_adj_per_node, root=0):
    order = bfs_order(edge_index, max_adj_per_node, root)
    _remember(order.sorted_index, order.level_start, order.num_levels)
    return order.sorted_index, order.sorted_parent, order.sorted_child


def levels_of(sorted_index, sorted_parent):
    """level boundaries of an order produced by bfs_forward (remembered), else of the equivalent canonical order."""
    levels = _recall(sorted_index)
    if levels is not None:
        return levels
    order = _adopt(sorted_index, sorted_parent)[0]
    return order.level_start, order.num_levels


def _adopt(sorted_index, sorted_parent):
    """Any parent-before-child order (e.g. the reference's own racy bfs_forward output, bfs.cu:46-98) -> the
    deterministic level order of the SAME tree that the refine kernels need (levels contiguous, children of a node
    adjacent): (order, perm) with perm[b, foreign position] = position here.
    The adopted order keeps each tree's root (the foreign order's first vertex): a position's edge weight belongs to the
    edge to ITS parent, and re-rooting would hand the weights of the edges between the two roots to the wrong edges."""
    idx, par = _i32(sorted_index), _i32(sorted_parent)
    B, V = idx.shape
    up = torch.gather(idx, 1, par[:, 1:].long())                       # vertex id of each non-root node's parent
    edges = torch.stack((idx[:, 1:], up), dim=2).contiguous()          # the tree as an edge list [B,V-1,2]
    roots = idx[:, 0].tolist()
    if all(r == roots[0] for r in roots):
        order = bfs_order(edges, 4, roots[0])
    else:                                                              # one BFS per tree
        parts = [bfs_order(edges[b:b + 1], 4, r) for b, r in enumerate(roots)]
        order = TreeOrder(*(torch.cat(ts) for ts in zip(*parts)))
    pos_of_vertex = torch.empty((B, V), dtype=torch.int64, device=idx.device)
    pos_of_vertex.scatter_(1, order.sorted_index.long(), torch.arange(V, device=idx.device).expand(B, V))
    perm = torch.gather(pos_of_vertex, 1, idx.long())
    return order, perm


def _own(sorted_index, sorted_parent, sorted_child):
    """-> (order, perm): the caller's tensors with their remembered level table when bfs_forward produced them (perm
    None), else the adopted order."""
    levels = _recall(sorted_index)
    if levels is not None:
        return TreeOrder(_i32(sorted_index), _i32(sorted_parent), _i32(sorted_child), *levels), None
    return _adopt(sorted_index, sorted_parent)


def _resolve(edge_weight, sorted_index, sorted_parent, sorted_child):
    """-> (w, order, perm): ``_own`` with the per-position edge weights carried over by vertex to an adopted order."""
    order, perm = _own(sorted_index, sorted_parent, sorted_child)
    w = _f32(edge_weight)
    return (w if perm is None else torch.zeros_like(w).scatter_(1, perm, w)), order, perm


def _to_ours(t, perm):      # position-ordered [B,V] or [B,C,V] tensor: foreign order -> adopted order
    if perm is None or t is None:
        return t
    out = torch.empty_like(t)
    out.scatter_(t.dim() - 1, perm if t.dim() == 2 else perm.unsqueeze(1).expand_as(t), t)
    return out


def _to_theirs(t, perm):
    if perm is None:
        return t
    return torch.gather(t, t.dim() - 1, perm if t.dim() == 2 else perm.unsqueeze(1).expand_as(t))


def _scratch(B, C, V, dev):
    return torch.empty(max(L.lib().bxs_refine_scratch_bytes(B, C, V), 4), dtype=torch.uint8, device=dev)


def refine_forward(feature_in, edge_weight, sorted_index, sorted_parent, sorted_child):
    w, order, perm = _resolve(edge_weight, sorted_index, sorted_parent, sorted_child)
    out, aggr, aggr_up, wsum, wsum_up = refine_forward_grouped(feature_in, w, order, None)
    # out / aggr / wsum are vertex-ordered; the two *_up tensors are position-ordered (refine.cu:201-260)
    return out, aggr, _to_theirs(aggr_up, perm), wsum, _to_theirs(wsum_up, perm)


def refine_backward_feature(feature_in, edge_weight, sorted_index, sorted_parent, sorted_child, feature_out,
                            feature_aggr, feature_aggr_up, weight_sum, weight_sum_up, grad_out):
    w, order, _ = _resolve(edge_weight, sorted_index, sorted_parent, sorted_child)
    return refine_backward_feature_grouped(w, order, None, _f32(weight_sum), grad_out)


def refine_backward_weight(feature_in, edge_weight, sorted_index, sorted_parent, sorted_child, feature_out,
                           feature_aggr, feature_aggr_up, weight_sum, weight_sum_up, grad_out):
    w, order, perm = _resolve(edge_weight, sorted_index, sorted_parent, sorted_child)
    gw = refine_backward_weight_grouped(w, order, None, _f32(feature_out), _f32(feature_aggr),
                                        _to_ours(_f32(feature_aggr_up), perm), _f32(weight_sum),
                                        _to_ours(_f32(weight_sum_up), perm), grad_out)
    return _to_theirs(gw, perm)


# ----------------------------------------------------------------------------------------------------------------
# grouped forms (not part of the reference's pybind surface): n instances share G trees, tree_of [n] -> tree (None:
# instance i uses tree i, n == G).  ``order`` is a TreeOrder: from bfs_order, or an adopted one (see _resolve).
# ----------------------------------------------------------------------------------------------------------------
def refine_forward_grouped(feature_in, edge_weight, order, tree_of):
    f, w = _f32(feature_in), _f32(edge_weight)
    idx, par, chd, lvl, nlv = (_i32(t) for t in order)
    L.require_cuda(f, w, idx, par, chd, lvl, nlv, tree_of)
    n, C, V = f.shape
    G = w.shape[0]
    out, aggr, aggr_up = torch.empty_like(f), torch.empty_like(f), torch.empty_like(f)
    wsum = torch.empty((G, V), dtype=torch.float32, device=f.device)
    wsum_up = torch.empty_like(wsum)
    if n == 0:                  # no instance: nothing to filter, and no backward reads the normaliser
        return out, aggr, aggr_up, wsum.zero_(), wsum_up.zero_()
    with torch.cuda.device(f.device):
        L.check(L.lib().bxs_refine_forward_grouped(L.ptr(f), L.ptr(w), L.ptr(idx), L.ptr(par), L.ptr(chd), L.ptr(lvl), L.ptr(nlv),
                                                   L.ptr(tree_of), L.ptr(out), L.ptr(aggr), L.ptr(aggr_up), L.ptr(wsum),
                                                   L.ptr(wsum_up), L.ptr(_scratch(max(n, G), C, V, f.device)), n, G, C, V,
                                                   L.stream()), 'refine_forward_grouped')
    return out, aggr, aggr_up, wsum, wsum_up


def refine_backward_feature_grouped(edge_weight, order, tree_of, weight_sum, grad_out):
    w, g, wsum = _f32(edge_weight), _f32(grad_out), _f32(weight_sum)
    idx, par, chd, lvl, nlv = (_i32(t) for t in order)
    L.require_cuda(w, g, wsum, idx, par, chd, lvl, nlv, tree_of)
    n, C, V = g.shape
    G = w.shape[0]
    gf = torch.empty_like(g)
    if n == 0:
        return gf
    with torch.cuda.device(g.device):
        L.check(L.lib().bxs_refine_backward_feature_grouped(L.ptr(w), L.ptr(idx), L.ptr(par),
                                                            L.ptr(chd), L.ptr(lvl), L.ptr(nlv), L.ptr(tree_of),
                                                            L.ptr(wsum), L.ptr(g), L.ptr(gf),
                                                            L.ptr(_scratch(max(n, G), C, V, g.device)), n, G, C, V, L.stream()),
                'refine_backward_feature_grouped')
    return gf


def refine_backward_weight_grouped(edge_weight, order, tree_of, feature_out, feature_aggr, feature_aggr_up, weight_sum,
                                   weight_sum_up, grad_out):
    w, g = _f32(edge_weight), _f32(grad_out)
    idx, par, chd, lvl, nlv = (_i32(t) for t in order)
    out, aggr, aggr_up = _f32(feature_out), _f32(feature_aggr), _f32(feature_aggr_up)
    wsum, wsum_up = _f32(weight_sum), _f32(weight_sum_up)
    L.require_cuda(w, g, idx, par, chd, lvl, nlv, out, aggr, aggr_up, wsum, wsum_up, tree_of)
    n, C, V = g.shape
    G = w.shape[0]
    gw = torch.empty((n, V), dtype=torch.float32, device=g.device)
    if n == 0:                  # the callers sum the rows of a tree: a tree without instances gets a zero d/d w
        return gw
    with torch.cuda.device(g.device):
        L.check(L.lib().bxs_refine_backward_weight_grouped(L.ptr(w), L.ptr(idx), L.ptr(par),
                                                           L.ptr(chd), L.ptr(lvl), L.ptr(nlv), L.ptr(tree_of),
                                                           L.ptr(out), L.ptr(aggr), L.ptr(aggr_up),
                                                           L.ptr(wsum), L.ptr(wsum_up), L.ptr(g), L.ptr(gw),
                                                           L.ptr(_scratch(max(n, G), C, V, g.device)), n, G, C, V, L.stream()),
                'refine_backward_weight_grouped')
    return gw
