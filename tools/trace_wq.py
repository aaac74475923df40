"""Per-WARP timeline of wq_main_kernel (diagnostic build with -DBXS_OP_TRACE).
   build:  python tools/trace_wq.py build      (here, writes boxinstseg_b200/lib/libboxseg_b200_trace.so)
   run:    python tools/trace_wq.py            (GPU box)"""
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
        if 'onepass' in src or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), B._headers_mtime()):
            subprocess.run([B._nvcc()] + B.NVCC_FLAGS + ['-DBXS_OP_TRACE', '-c', src, '-o', obj], check=True)
        objs.append(obj)
    subprocess.run([B._nvcc(), '-shared', '-o', TRACE_LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'], check=True)
    print(TRACE_LIB); sys.exit(0)
import ctypes
import numpy as np, torch
from boxinstseg_b200 import _lib as L
L.LIB_PATH = TRACE_LIB
from bench import synthetic_case, N_INST, H, W
from boxinstseg_b200.ops.boxinst import boxinst_loss_plan, boxinst_targets
dev = torch.device('cuda:0')
lib = L.lib()
case = synthetic_case(1234)
t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']])
it = torch.tensor([10000.0], device=dev)
xs = [torch.randn(N_INST, 1, H, W, device=dev) * 2 for _ in range(6)]
gl = torch.empty_like(xs[0])
inst_gt = case['gt_inds'].to(dev).to(torch.int32)
plan = boxinst_loss_plan(t, inst_gt, H, W, 2)
ws = torch.empty(lib.bxs_boxinst_loss_fused_workspace_bytes(N_INST, H, W), dtype=torch.uint8, device=dev)
sched = torch.zeros(int(lib.bxs_boxinst_loss_fused_sched_bytes()), dtype=torch.uint8, device=dev)
out = torch.empty(4, device=dev)
NWMAX = 148 * 4 * 8
trace = torch.zeros((NWMAX * 16 + 2048 * 8) * 2, dtype=torch.int64, device=dev)
h = ctypes.CDLL(TRACE_LIB)
h.bxs_debug_set_trace.argtypes = [ctypes.c_void_p]
def run(i):
    rc = lib.bxs_boxinst_loss_fused_forward_planned(L.ptr(xs[i % 6]), L.ptr(t.edge_bits), L.ptr(plan), L.ptr(it), 10000.0, L.ptr(ws), L.ptr(sched), L.ptr(out), L.ptr(gl), N_INST, H, W, 2, L.stream())
    assert rc == 0
for i in range(5): run(i)
torch.cuda.synchronize()
assert h.bxs_debug_set_trace(ctypes.c_void_p(trace.data_ptr())) == 0
run(5)
torch.cuda.synchronize()
fin = trace.cpu().numpy()[NWMAX * 16 * 2:].reshape(2048, 8, 2)[:N_INST, :, 0]
tr = trace.cpu().numpy()[:NWMAX * 16 * 2].reshape(NWMAX, 16, 2)
os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
np.save(os.path.join(ROOT, 'gpurun_out', 'wq_trace.npy'), tr)
warps = [w for w in range(NWMAX) if tr[w, 0, 0] != 0]
t0 = min(tr[w, 0, 0] for w in warps)
dur = {2: [], 3: [], 'fence': [], 'fin': []}
starts, ends, exits = [], [], []
busy = {2: np.zeros(400), 3: np.zeros(400), 'fin': np.zeros(400)}
for w in warps:
    ev = [(int(tr[w, j, 0] - t0), int(tr[w, j, 1])) for j in range(16) if tr[w, j, 0] != 0]
    starts.append(ev[0][0])
    cur = None
    for (ta, tag) in ev:
        code = tag & 0xff
        if code in (2, 3): cur = (code, ta)
        elif code == 4 and cur: dur[cur[0]].append(ta - cur[1]); busy[cur[0]][cur[1] // 1000: ta // 1000 + 1] += 1; cur = None
        elif code == 7: exits.append(ta)
def st(a):
    a = np.array(a) / 1e3
    return f'n={len(a)} mean={a.mean():.2f} p50={np.median(a):.2f} p90={np.percentile(a, 90):.2f} max={a.max():.2f} us' if len(a) else 'n=0'
print('warps', len(warps), 'first start spread', st(starts))
print('stream items', st(dur[2])); print('pair items  ', st(dur[3]))
print('warp exits  ', st(exits))
print('busy warps per us [stream/pair/fin]:')
T = int(max(exits) // 1000) + 1
for u in range(0, T, max(T // 40, 1)):
    print(f'  t={u:3d}us  {int(busy[2][u]):5d} {int(busy[3][u]):5d} {int(busy["fin"][u]):4d}')
f = (fin - t0) / 1e3
print('finalize CTAs: launch   ', st((fin[:, 0] - t0).tolist()))
print('finalize CTAs: released ', st((fin[:, 1] - t0).tolist()))
print('finalize CTAs: done     ', st((fin[:, 2] - t0).tolist()))
print('finalize CTAs: duration ', st((fin[:, 2] - fin[:, 1]).tolist()))
print('finalize CTAs: released -> first barrier ', st((fin[:, 3] - fin[:, 1]).tolist()))
print('finalize CTAs: released -> partial keys   ', st((fin[:, 4] - fin[:, 1]).tolist()))
print('finalize CTAs: released -> arg-max row    ', st((fin[:, 5] - fin[:, 1]).tolist()))
print('losses', out.tolist())
