"""Raw C-ABI loop of the single-pass BoxInst loss (config A) for ncu / timing (diagnostic, GPU box).
   python tools/raw_loop1.py [steps] [graph]"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bench import synthetic_case, N_INST, H, W
from boxinstseg_b200 import _lib as L
from boxinstseg_b200.ops.boxinst import boxinst_loss_plan, boxinst_targets
dev = torch.device('cuda:0')
case = synthetic_case(1234)
t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']])
it = torch.tensor([10000.0], device=dev)
lib = L.lib()
R = 8
xs = [torch.randn(N_INST, 1, H, W, device=dev) * 2 for _ in range(R)]
gls = [torch.empty_like(xs[0]) for _ in range(R)]
inst_gt = case['gt_inds'].to(dev).to(torch.int32)
ws = torch.empty(lib.bxs_boxinst_loss_fused_workspace_bytes(N_INST, H, W), dtype=torch.uint8, device=dev)
sched = torch.zeros(int(lib.bxs_boxinst_loss_fused_sched_bytes()), dtype=torch.uint8, device=dev)
out = torch.empty(4, device=dev); g = torch.ones(2, device=dev)
plan = boxinst_loss_plan(t, inst_gt, H, W, 2)
def raw(i, st):
    x, gl = xs[i % R], gls[i % R]
    rc = lib.bxs_boxinst_loss_fused_forward_planned(L.ptr(x), L.ptr(t.edge_bits), L.ptr(plan), L.ptr(it), 10000.0, L.ptr(ws), L.ptr(sched), L.ptr(out), L.ptr(gl), N_INST, H, W, 2, st)
    assert rc == 0, rc
    rc = lib.bxs_boxinst_loss_fused_backward(L.ptr(ws), L.ptr(g[0:1]), L.ptr(g[1:2]), L.ptr(gl), N_INST, H, W, st)
    assert rc == 0, rc
n = int(sys.argv[1]) if len(sys.argv) > 1 else 40
use_graph = len(sys.argv) > 2 and sys.argv[2] == 'graph'
for i in range(R): raw(i, L.stream())
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
if use_graph:
    gr = torch.cuda.CUDAGraph()
    with torch.cuda.graph(gr):
        for i in range(R): raw(i, L.stream())
    gr.replay(); torch.cuda.synchronize()
    e0.record()
    for i in range(n // R): gr.replay()
    e1.record(); torch.cuda.synchronize()
    print(f'single-pass C ABI, graph of {R} rotating sets: {e0.elapsed_time(e1)/(n // R * R)*1e3:.2f} us/step', out.tolist())
else:
    e0.record()
    for i in range(n): raw(i, L.stream())
    e1.record(); torch.cuda.synchronize()
    print(f'single-pass C ABI, eager rotating {R} sets: {e0.elapsed_time(e1)/n*1e3:.1f} us/step', out.tolist())
