"""debug: is the grid BFS fast path engaged, and how long do the BFS / MST / refine calls take (CUDA events)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.nn.functional as F
from benchkit import time_call
from boxinstseg_b200 import _lib as L
from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D, bfs
from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as C
dev = torch.device('cuda:0')
lib = L.lib()
g = torch.Generator(device=dev).manual_seed(0)
us = lambda fn: time_call(fn, reps=5, warmup=1)[0] * 1e3  # noqa: E731
for (n, h, w) in [(2, 200, 256), (16, 200, 256), (2, 96, 96), (2, 50, 64)]:
    guide = F.interpolate(torch.randn(n, 3, h // 8, w // 8, device=dev, generator=g), size=(h, w), mode='bilinear') + 0.05 * torch.randn(n, 3, h, w, device=dev, generator=g)
    mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
    tree = mst(guide)
    B, V = n, h * w
    idx = torch.empty((B, V), dtype=torch.int32, device=dev); par = torch.empty_like(idx)
    chd = torch.empty((B, V, 4), dtype=torch.int32, device=dev)
    lvl = torch.empty((B, V + 1), dtype=torch.int32, device=dev); nlv = torch.empty(B, dtype=torch.int32, device=dev)
    nbytes = lib.bxs_bfs_workspace_bytes(B, V)
    ws = torch.zeros(nbytes, dtype=torch.uint8, device=dev)
    rc = lib.bxs_bfs_forward_rooted(L.ptr(tree), L.ptr(idx), L.ptr(par), L.ptr(chd), L.ptr(lvl), L.ptr(nlv), L.ptr(ws), B, V, 4, 0,
                                    L.stream())
    torch.cuda.synchronize()
    al = lambda v: (v + 255) // 256 * 256
    off = al(4 * B * V); off = al(off + 16 * B * V); off = al(off + 4 * B * V)
    flags = ws[off:off + 4 * B].view(torch.int32)
    print(f'{n}x{h}x{w}: rc={rc} flags={flags.tolist()} levels={nlv.tolist()[:4]}', flush=True)
    print('  ',
          f'bfs {us(lambda: bfs(tree, 4)):.0f} us  mst {us(lambda: mst(guide)):.0f} us')
    tf = TreeFilter2D()
    feat = torch.rand(n, 1, h, w, device=dev, generator=g).requires_grad_(True)
    emb = guide.clone().requires_grad_(True)
    idx, par, chd = bfs(tree, 4)
    from boxinstseg_b200.ops.tree_filter.functions.refine import refine
    f3 = feat.reshape(n, 1, -1)
    ew0 = tf.build_edge_weight(emb, idx, par, False, chd).detach()
    def fb():
        ew = tf.build_edge_weight(emb, idx, par, False, chd)
        return torch.autograd.grad(refine(f3, ew, idx, par, chd, False).sum(), [feat, emb])
    print('   refine fwd', f'{us(lambda: refine(f3.detach(), ew0, idx, par, chd, False)):.0f} us', 'fwd+bwd', f'{us(fb):.0f} us', flush=True)
