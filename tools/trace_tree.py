"""Per-level clock-stamp trace of the refine up pass (needs a -DBXS_TREE_TRACE build:
   python tools/build_variant.py treetrace --src=tree_filter -DBXS_TREE_TRACE ;  BXS_LIB_PATH=.../libboxseg_b200_treetrace.so)."""
import ctypes
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.nn.functional as F

from boxinstseg_b200 import _lib as L
from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
from boxinstseg_b200.ops.tree_filter.functions.refine import refine_ordered
from boxinstseg_b200.ops.tree_filter.tree_filter_cuda import bfs_order

dev = torch.device('cuda:0')
g = torch.Generator(device=dev).manual_seed(0)
n, h, w = 2, 200, 256
guide = F.interpolate(torch.randn(n, 3, h // 8, w // 8, device=dev, generator=g), size=(h, w), mode='bilinear') + 0.05 * torch.randn(n, 3, h, w, device=dev, generator=g)
tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(guide)
tf = TreeFilter2D()
order = bfs_order(tree, 4)
feat = torch.rand(n, 1, h * w, device=dev, generator=g)
ew = tf.build_edge_weight(guide, order.sorted_index, order.sorted_parent, False, order.sorted_child).detach()
for _ in range(3):
    refine_ordered(feat, ew, order, False)
torch.cuda.synchronize()
handle = ctypes.CDLL(L.LIB_PATH)
buf = np.zeros((6, 4096), dtype=np.int64)
assert handle.bxs_debug_tree_trace(ctypes.c_void_p(buf.ctypes.data)) == 0
levels = int(order.num_levels[0])
m = min(levels, 4096) - 1
c0, c1, c2, p0, p1, p2 = (buf[k][:m] for k in range(6))
c0n, p0n = buf[0][1:m + 1], buf[3][1:m + 1]
lvl = order.level_start[0].cpu().numpy()
width = (lvl[1:levels + 1] - lvl[:levels])[::-1][:m]        # the up pass starts at the deepest level


def stat(name, x):
    x = x[8:]
    print(f'{name:38s} mean {x.mean():7.1f}  p50 {np.median(x):7.1f}  p90 {np.percentile(x, 90):7.1f}  max {x.max():7.0f} cycles')


print(f'levels {levels}, level width mean {width.mean():.1f} p90 {np.percentile(width, 90):.0f} max {width.max()}')
stat('level period (consumer top -> top)', c0n - c0)
stat('consumer: top -> store issued', c1 - c0)
stat('consumer: store -> at barrier', c2 - c1)
stat('consumer: barrier wait', c0n - c2)
stat('producer: top -> copies issued', p1 - p0)
stat('producer: cp.async group wait', p2 - p1)
stat('producer: barrier wait', p0n - p2)
narrow = width[8:] <= 32
print('period, levels <= 32 wide:', (c0n - c0)[8:][narrow].mean(), ' wider:', (c0n - c0)[8:][~narrow].mean() if (~narrow).any() else '-')
