"""Per-CTA timeline of onepass_main_kernel (diagnostic build with -DBXS_OP_TRACE).
   build:  python tools/trace_onepass.py build      (here, writes boxinstseg_b200/lib/libboxseg_b200_trace.so)
   run:    python tools/trace_onepass.py            (GPU box)"""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from boxinstseg_b200 import build as B
TRACE_LIB = os.path.join(B.LIBDIR, 'libboxseg_b200_trace.so')
if len(sys.argv) > 1 and sys.argv[1] == 'build':
    objs = []
    os.makedirs(os.path.join(B.LIBDIR, 'obj_trace'), exist_ok=True)
    for src in B.sources():
        obj = os.path.join(B.LIBDIR, 'obj_trace', os.path.basename(src)[:-3] + '.o')
        if 'onepass' in src or not os.path.exists(obj):
            subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ['-DBXS_OP_TRACE', '-c', src, '-o', obj], check=True)
        objs.append(obj)
    subprocess.run([B._nvcc(), '-shared', '-o', TRACE_LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'], check=True)
    print(TRACE_LIB); sys.exit(0)
import ctypes
import numpy as np, torch
from boxinstseg_b200 import _lib as L
L.LIB_PATH = TRACE_LIB
from bench import synthetic_case, N_INST, H, W
from boxinstseg_b200.ops.boxinst import boxinst_targets
dev = torch.device('cuda:0')
lib = L.lib()
case = synthetic_case(1234)
t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']])
it = torch.tensor([10000.0], device=dev)
xs = [torch.randn(N_INST, 1, H, W, device=dev) * 2 for _ in range(4)]
gl = torch.empty_like(xs[0])
inst_gt = case['gt_inds'].to(dev).to(torch.int32)
ws = torch.empty(lib.bxs_boxinst_loss_fused_workspace_bytes(N_INST, H, W), dtype=torch.uint8, device=dev)
sched = torch.zeros(int(lib.bxs_boxinst_loss_fused_sched_bytes()), dtype=torch.uint8, device=dev)
out = torch.empty(4, device=dev)
trace = torch.zeros(1024 * 64 * 2, dtype=torch.int64, device=dev)
h = ctypes.CDLL(TRACE_LIB)
h.bxs_debug_set_trace.argtypes = [ctypes.c_void_p]
def run(i):
    rc = lib.bxs_boxinst_loss_fused_forward(L.ptr(xs[i % 4]), L.ptr(t.edge_bits), L.ptr(t.rects), L.ptr(inst_gt), L.ptr(t.gt_img), L.ptr(it), 10000.0, L.ptr(ws), L.ptr(sched), L.ptr(out), L.ptr(gl), N_INST, H, W, 2, L.stream())
    assert rc == 0
for i in range(4): run(i)
torch.cuda.synchronize()
assert h.bxs_debug_set_trace(ctypes.c_void_p(trace.data_ptr())) == 0
run(5)
torch.cuda.synchronize()
tr = trace.cpu().numpy().reshape(1024, 64, 2)
ctas = [c for c in range(1024) if tr[c, 0, 0] != 0]
t0 = min(tr[c, 0, 0] for c in ctas)
ends, items = [], {0: [], 1: []}
pro = []
per_sm = {}
for c in ctas:
    ev = [(int(tr[c, j, 0] - t0), int(tr[c, j, 1])) for j in range(64) if tr[c, j, 0] != 0]
    start = ev[0][0]
    role = None
    for (ta, tag), (tb, _) in zip(ev, ev[1:] + [(None, None)]):
        code = tag & 0xff
        if code == 2:
            pro.append(ta - start); role = (tag >> 32) & 1; smid = (tag >> 8) & 0xffffff
            per_sm.setdefault(smid, []).append(role)
        if code in (16, 17) and tb is not None:
            items[code - 16].append(tb - ta)
        if code == 3:
            ends.append(ta)
print(f'CTAs {len(ctas)}; start spread {max(tr[c,0,0] for c in ctas) - t0} ns; prologue mean {np.mean(pro):.0f} max {np.max(pro)} ns')
for k, name in ((0, 'stream'), (1, 'pair')):
    a = np.array(items[k])
    print(f'{name}: n={len(a)} mean {a.mean():.0f} p50 {np.percentile(a,50):.0f} p90 {np.percentile(a,90):.0f} max {a.max()} ns; sum {a.sum()/1e3:.0f} us')
e = np.array(ends)
print(f'CTA end times: min {e.min()} p10 {np.percentile(e,10):.0f} p50 {np.percentile(e,50):.0f} p90 {np.percentile(e,90):.0f} max {e.max()} ns')
roles = [sum(v) for v in per_sm.values()]
print('pair-first CTAs per SM histogram:', np.bincount(roles), ' CTAs per SM:', np.bincount([len(v) for v in per_sm.values()]))
# busy pattern: how many CTAs are in a pair item / stream item over time
edges = np.arange(0, e.max() + 1000, 1000)
occ = np.zeros((2, len(edges)))
for c in ctas:
    ev = [(int(tr[c, j, 0] - t0), int(tr[c, j, 1])) for j in range(64) if tr[c, j, 0] != 0]
    for (ta, tag), (tb, _) in zip(ev, ev[1:]):
        code = tag & 0xff
        if code in (16, 17):
            occ[code - 16, ta // 1000:(tb // 1000) + 1] += 1
print('t(us)  stream-CTAs  pair-CTAs')
for i in range(len(edges)):
    print(f'{i:4d} {int(occ[0, i]):6d} {int(occ[1, i]):6d}')
