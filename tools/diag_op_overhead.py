"""Where does the op-level step lose time against the raw C-ABI step?  Each variant: 8 rotating steps in ONE CUDA graph."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from bench import synthetic_case, N_INST, H, W
from benchkit import capture, replay_ms
from boxinstseg_b200 import _lib as L
from boxinstseg_b200.ops import boxinst as OB
from boxinstseg_b200.ops.boxinst import boxinst_mask_loss, boxinst_targets
dev = torch.device('cuda:0')
lib = L.lib()
case = synthetic_case(1234)
t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']])
it = torch.tensor([10000.0], device=dev)
gi = case['gt_inds'].to(dev).to(torch.int32)
ones = torch.ones((), device=dev)
R = 8
xs = [(torch.randn(N_INST, 1, H, W, device=dev) * 2).requires_grad_(True) for _ in range(R)]
keep = []

def v_full(x):
    prj, pair = boxinst_mask_loss(x, t, gi, it)
    torch.autograd.backward([prj, pair], [ones, ones])
    keep.append(x.grad); x.grad = None

def v_fwd_only(x):
    prj, pair = boxinst_mask_loss(x, t, gi, it)
    keep.append((prj, pair))

def v_grad(x):
    prj, pair = boxinst_mask_loss(x, t, gi, it)
    keep.append(torch.autograd.grad([prj, pair], [x], [ones, ones]))

def v_sum_backward(x):
    prj, pair = boxinst_mask_loss(x, t, gi, it)
    (prj + pair).backward()
    keep.append(x.grad); x.grad = None

ws1 = [torch.empty(lib.bxs_boxinst_loss_fused_workspace_bytes(N_INST, H, W), dtype=torch.uint8, device=dev) for _ in range(R)]
gl = [torch.empty(N_INST, 1, H, W, device=dev) for _ in range(R)]
outs = [torch.empty(4, device=dev) for _ in range(R)]
sched = torch.zeros(int(lib.bxs_boxinst_loss_fused_sched_bytes()), dtype=torch.uint8, device=dev)
g2 = torch.ones(2, device=dev)
idx = {id(x): i for i, x in enumerate(xs)}

def v_raw(x):
    i = idx[id(x)]
    st = L.stream()
    lib.bxs_boxinst_loss_fused_forward(L.ptr(x.detach()), L.ptr(t.edge_bits), L.ptr(t.rects), L.ptr(gi), L.ptr(t.gt_img), L.ptr(it),
                                       10000.0, L.ptr(ws1[i]), L.ptr(sched), L.ptr(outs[i]), L.ptr(gl[i]), N_INST, H, W, 2, st)
    lib.bxs_boxinst_loss_fused_backward(L.ptr(ws1[i]), L.ptr(g2[0:1]), L.ptr(g2[1:2]), L.ptr(gl[i]), N_INST, H, W, st)

def v_raw_fresh(x):           # raw calls but with per-step torch.empty buffers like the op
    st = L.stream()
    ws = torch.empty(lib.bxs_boxinst_loss_fused_workspace_bytes(N_INST, H, W), dtype=torch.uint8, device=dev)
    g = torch.empty_like(x)
    o = torch.empty(4, device=dev)
    lib.bxs_boxinst_loss_fused_forward(L.ptr(x.detach()), L.ptr(t.edge_bits), L.ptr(t.rects), L.ptr(gi), L.ptr(t.gt_img), L.ptr(it),
                                       10000.0, L.ptr(ws), L.ptr(OB._sched_state(dev)), L.ptr(o), L.ptr(g), N_INST, H, W, 2, st)
    lib.bxs_boxinst_loss_fused_backward(L.ptr(ws), L.ptr(g2[0:1]), L.ptr(g2[1:2]), L.ptr(g), N_INST, H, W, st)
    keep.append((ws, g, o))

def measure(fn, name):
    keep.clear()
    g = capture(lambda: [fn(x) for x in xs])
    print(f'{name:28s} {replay_ms(g, 50) / R * 1e3:7.2f} us/step', flush=True)

for fn, name in [(v_raw, 'raw C ABI'), (v_raw_fresh, 'raw, fresh buffers per step'), (v_fwd_only, 'op forward only'),
                 (v_full, 'op + autograd.backward'), (v_grad, 'op + autograd.grad'), (v_sum_backward, 'op + (prj+pair).backward()')]:
    measure(fn, name)
