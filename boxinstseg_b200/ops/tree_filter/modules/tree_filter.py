"""``MinimumSpanningTree`` and ``TreeFilter2D`` -- drop-ins for
mmdet/ops/tree_filter/modules/tree_filter.py:9-150 (same constructor arguments and forward signatures).

The grid-graph construction and the MST edge weights stay in torch, written so that the float32 results are
bit-identical to the reference's (near-ties decide the tree, SURVEY appendix A13); the tree selection, ordering,
the FILTER's edge weights (build_edge_weight, forward and autograd) and the aggregation run in libboxseg_b200.
"""
import torch
from torch import nn

from .... import _lib as L

from .. import tree_filter_cuda as _C
from ..functions.mst import mst
from ..functions.refine import refine_ordered


def _squared_distance(a, b):
    d = a - b
    return (d * d).sum(dim=1)


class _EdgeWeight(torch.autograd.Function):
    """w[p] = exp(-|E(v_p) - E(v_par(p))|^2 / sigma) for the default norm2 distance (tree_filter.py:72-108): one gather
    kernel forward, one gather kernel backward (the reference: two [n,C,V] torch.gather + elementwise ops + their
    autograd scatters)."""

    @staticmethod
    def forward(ctx, embed, sorted_index, sorted_parent, sorted_child, groups, sigma):
        e = embed.contiguous().float()
        L.require_cuda(e, sorted_index, sorted_parent, sorted_child)
        B, Ctot = e.shape[0], e.shape[1]
        V = e.shape[2] * e.shape[3]
        C = Ctot // groups
        w = torch.empty((B * groups, V), dtype=torch.float32, device=e.device)
        with torch.cuda.device(e.device):
            L.check(L.lib().bxs_tree_edge_weight_forward(L.ptr(e), L.ptr(sorted_index), L.ptr(sorted_parent), L.ptr(w), B,
                                                         groups, C, V, float(sigma), L.stream()), 'tree_edge_weight_forward')
        ctx.save_for_backward(e, sorted_index, sorted_parent, sorted_child, w)
        ctx.cfg = (groups, float(sigma))
        ctx.set_materialize_grads(False)        # refine returns no d/d weight when low_tree (refine.py:36-37): embed gets None
        return w

    @staticmethod
    def backward(ctx, g_w):
        if g_w is None:
            return None, None, None, None, None, None
        e, idx, par, chd, w = ctx.saved_tensors
        groups, sigma = ctx.cfg
        B, Ctot = e.shape[0], e.shape[1]
        V = e.shape[2] * e.shape[3]
        g = torch.empty_like(e)
        with torch.cuda.device(e.device):
            L.check(L.lib().bxs_tree_edge_weight_backward(L.ptr(e), L.ptr(idx), L.ptr(par), L.ptr(chd), L.ptr(w),
                                                          L.ptr(g_w.contiguous().float()), L.ptr(g), B, groups,
                                                          Ctot // groups, V, sigma, L.stream()), 'tree_edge_weight_backward')
        return g, None, None, None, None, None


class MinimumSpanningTree(nn.Module):
    def __init__(self, distance_func):
        super().__init__()
        self.distance_func = distance_func

    @staticmethod
    def _build_matrix_index(fm):
        """int32 [B,E,2]: vertical edges (v, v+W) first, then horizontal (v, v+1); tree_filter.py:15-25."""
        b, h, w = fm.shape[0], fm.shape[2], fm.shape[3]
        ids = torch.arange(h * w, dtype=torch.int32, device=fm.device).view(h, w)
        vert = torch.stack((ids[:-1], ids[1:]), dim=2).reshape(-1, 2)
        hori = torch.stack((ids[:, :-1], ids[:, 1:]), dim=2).reshape(-1, 2)
        return torch.cat((vert, hori), dim=0).unsqueeze(0).expand(b, -1, -1)

    def _build_feature_weight(self, fm):
        """distance along both grid directions + 1; tree_filter.py:27-34."""
        b = fm.shape[0]
        vert = self.distance_func(fm[:, :, :-1, :], fm[:, :, 1:, :]).reshape(b, -1)
        hori = self.distance_func(fm[:, :, :, :-1], fm[:, :, :, 1:]).reshape(b, -1)
        return torch.cat((vert, hori), dim=1) + 1

    def _build_label_weight(self, fm):
        """tree_filter.py:36-51 (never used by the heads; kept for API parity)."""
        b = fm.shape[0]
        diff = torch.cat((self.distance_func(fm[:, :, :-1, :], fm[:, :, 1:, :]).reshape(b, -1),
                          self.distance_func(fm[:, :, :, :-1], fm[:, :, :, 1:]).reshape(b, -1)), dim=1)
        both = torch.cat(((fm[:, :, :-1, :] + fm[:, :, 1:, :]).sum(1).reshape(b, -1),
                          (fm[:, :, :, :-1] + fm[:, :, :, 1:]).sum(1).reshape(b, -1)), dim=1)
        return diff * both

    def forward(self, guide_in, label=None):
        with torch.no_grad():
            index = self._build_matrix_index(guide_in).contiguous()
            weight = self._build_feature_weight(guide_in)
            if label is not None:
                sel = self._build_label_weight(label) > 0
                weight[sel] = torch.sigmoid(weight[sel])
            return mst(index, weight.contiguous(), guide_in.shape[2] * guide_in.shape[3])


class TreeFilter2D(nn.Module):
    def __init__(self, groups=1, sigma=0.02, distance_func=None, enable_log=False):
        super().__init__()
        self.groups = groups
        self.enable_log = enable_log
        self.distance_func = distance_func if distance_func is not None else self.norm2_distance
        self.sigma = sigma

    @staticmethod
    def norm2_distance(fm_ref, fm_tar):
        return _squared_distance(fm_ref, fm_tar)

    @staticmethod
    def batch_index_opr(data, index):
        with torch.no_grad():
            index = index.long().unsqueeze(1).expand(-1, data.shape[1], -1)
        return torch.gather(data, 2, index)

    @staticmethod
    def _root(shape):
        """The filter A x / A 1 does not depend on where the tree is rooted, the DEPTH of the recursion does: every pass
        is one dependent step per BFS level.  The reference roots at vertex 0, a corner (bfs.cu:100-135); the centre
        pixel roughly halves the number of levels (1898 -> ~1000 at 200x256)."""
        h, w = shape[-2], shape[-1]
        return (h // 2) * w + w // 2

    def build_edge_weight(self, fm, sorted_index, sorted_parent, low_tree, sorted_child=None):
        """w[pos] = exp(-dist(E(v_pos), E(v_par)) / (sigma if low_tree else 1)); tree_filter.py:91-108.
        With the default distance and the BFS child table at hand this is one kernel (and one for its autograd);
        a custom ``distance_func`` keeps the reference's torch formulation."""
        if self.distance_func is TreeFilter2D.norm2_distance and sorted_child is not None and fm.is_cuda and \
                sorted_index.dtype == torch.int32 and sorted_index.is_contiguous() and sorted_parent.is_contiguous() and \
                sorted_child.is_contiguous():
            return _EdgeWeight.apply(fm, sorted_index, sorted_parent, sorted_child, self.groups,
                                     self.sigma if low_tree else 1.0)
        b, c = fm.shape[0], fm.shape[1]
        v = fm.shape[2] * fm.shape[3]
        flat = fm.reshape(b, c, -1)
        src = self.batch_index_opr(flat, sorted_index)
        dst = self.batch_index_opr(src, sorted_parent)
        src = src.reshape(-1, c // self.groups, v)
        dst = dst.reshape(-1, c // self.groups, v)
        dist = self.distance_func(src, dst)
        return torch.exp(-dist / self.sigma) if low_tree else torch.exp(-dist)

    def order(self, tree, shape):
        """The order ``forward`` would compute for ``tree`` (a TreeOrder rooted at the centre pixel of ``shape``): lets a
        caller build it ahead of time, e.g. on a side stream while another filter runs, and pass it back as ``order=``."""
        return _C.bfs_order(tree, 4, self._root(shape))

    def forward(self, feature_in, embed_in, tree, low_tree=True, tree_of=None, order=None):
        """``tree_of`` (optional, int32 [n]): feature_in holds n instances that share the G trees / embeddings given
        (embed_in [G,C,h,w], tree [G,V-1,2]); instance i uses tree ``tree_of[i]``.  Same result as repeating the trees
        and embeddings per instance (what the reference's heads do), computed once per tree.
        ``order`` (optional): ``self.order(tree, feature_in.shape)`` computed by the caller, or the three tensors of
        ``bfs(tree, 4, root)`` for any root."""
        assert tree_of is None or self.groups == 1
        shape = feature_in.shape
        if order is None:
            order = self.order(tree, shape)
        elif not isinstance(order, _C.TreeOrder):
            order = _C._own(*order)[0]
        edge_weight = self.build_edge_weight(embed_in, order.sorted_index, order.sorted_parent, low_tree, order.sorted_child)
        # n may be 0, so the last extent is spelled out
        feat = feature_in.reshape(shape[0] * self.groups, shape[1] // self.groups, shape[2] * shape[3]).contiguous()
        if self.groups > 1:                                  # tree_filter.py:110-120 (split_group)
            order = _C.TreeOrder(*(t.repeat_interleave(self.groups, dim=0).contiguous() for t in order))
        if tree_of is not None:
            tree_of = tree_of.to(torch.int32).contiguous()
        return refine_ordered(feat, edge_weight, order, low_tree, tree_of).reshape(shape)
