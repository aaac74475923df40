"""Per-level clock-stamp trace of bfs_grid_kernel's warp 0 (needs a -DBXS_TREE_TRACE build, see tools/trace_tree.py)."""
import ctypes, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np, torch
import torch.nn.functional as F
from boxinstseg_b200 import _lib as L
from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D
from boxinstseg_b200.ops.tree_filter.tree_filter_cuda import bfs_order
dev = torch.device('cuda:0')
g = torch.Generator(device=dev).manual_seed(0)
n, h, w = 2, 200, 256
guide = F.interpolate(torch.randn(n, 3, h // 8, w // 8, device=dev, generator=g), size=(h, w), mode='bilinear') + 0.05 * torch.randn(n, 3, h, w, device=dev, generator=g)
tree = MinimumSpanningTree(TreeFilter2D.norm2_distance)(guide)
for _ in range(3):
    order = bfs_order(tree, 4)
torch.cuda.synchronize()
handle = ctypes.CDLL(L.LIB_PATH)
buf = np.zeros((6, 4096), dtype=np.int64)
assert handle.bxs_debug_tree_trace(ctypes.c_void_p(buf.ctypes.data)) == 0
levels = int(order.num_levels[0])
m = min(levels, 4096) - 1
t = [buf[k][:m] for k in range(5)]
nxt = buf[0][1:m + 1]
def stat(name, x):
    x = x[8:]
    print(f'{name:40s} mean {x.mean():7.1f}  p50 {np.median(x):7.1f}  p90 {np.percentile(x, 90):7.1f} cycles')
print('levels', levels)
stat('level period', nxt - t[0])
stat('top -> adjacency bits + popc', t[1] - t[0])
stat('bits -> ballots / prefix', t[2] - t[1])
stat('prefix -> next frontier stored', t[3] - t[2])
stat('store -> past pair barrier', t[4] - t[3])
stat('barrier -> next level top', nxt - t[4])
