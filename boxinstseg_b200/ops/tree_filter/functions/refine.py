"""``refine(feature_in, edge_weight, sorted_index, sorted_parent, sorted_child, low_tree)`` --
mmdet/ops/tree_filter/functions/refine.py:9-41: differentiable wrt feature_in always and wrt
edge_weight when ``low_tree`` is False."""
import torch
from torch.autograd import Function
from torch.autograd.function import once_differentiable

from .. import tree_filter_cuda as _C

from ..._streams import Forked


def _both(device, feature_fn, weight_fn):
    """-> (feature_fn(), weight_fn()).  d/d feature and d/d edge_weight are independent level walks (two and three dependent
    passes over ~1000-1900 tree levels) on a handful of SMs each: the second one runs on the side stream."""
    forked = Forked(weight_fn, device)
    gf = feature_fn()
    return gf, forked.join()


class _Refine(Function):
    """``tree_of`` (optional, [n] int32 -> tree): n instances share the G trees given.  The instances of one image share the
    image's tree in both heads that use the filter (box_solov2_head.py:300-305,353; box2mask_head.py:271-276), so the
    BFS order, the edge weights and the normaliser are computed once per image, and d/d edge_weight is summed over the
    instances of a tree.  Without it instance i uses tree i, as in the reference.  An order that bfs_forward did not
    produce is replaced by the equivalent canonical order of the same tree (tree_filter_cuda._resolve)."""

    @staticmethod
    def forward(ctx, feature_in, edge_weight, sorted_index, sorted_parent, sorted_child, low_tree, tree_of=None):
        w, idx, par, chd, levels, perm = _C._resolve(edge_weight, sorted_index, sorted_parent, sorted_child)
        out, aggr, aggr_up, wsum, wsum_up = _C.refine_forward_grouped(feature_in, w, idx, par, chd, levels, tree_of)
        ctx.save_for_backward(w, idx, par, chd, *levels, tree_of, perm, out, aggr, aggr_up, wsum, wsum_up)
        ctx.low_tree = low_tree
        return out

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        (w, idx, par, chd, lvl, nlv, tree_of, perm, out, aggr, aggr_up, wsum, wsum_up) = ctx.saved_tensors
        g = grad_output.contiguous()

        def d_feature():
            return _C.refine_backward_feature_grouped(w, idx, par, chd, (lvl, nlv), tree_of, wsum, g)

        def d_weight():
            gw = _C.refine_backward_weight_grouped(w, idx, par, chd, (lvl, nlv), tree_of, out, aggr, aggr_up, wsum, wsum_up, g)
            if tree_of is not None:
                gw = torch.zeros_like(w).index_add_(0, tree_of.long(), gw)
            return _C._to_theirs(gw, perm)

        if ctx.low_tree:
            return d_feature(), None, None, None, None, None, None
        grad_feature, grad_weight = _both(g.device, d_feature, d_weight)
        return grad_feature, grad_weight, None, None, None, None, None


def refine(feature_in, edge_weight, sorted_index, sorted_parent, sorted_child, low_tree, tree_of=None):
    return _Refine.apply(feature_in, edge_weight, sorted_index, sorted_parent, sorted_child, low_tree, tree_of)
