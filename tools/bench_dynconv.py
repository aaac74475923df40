"""Time the wgmma dynamic 1x1 convolution (forward, d/d feat, d/d kernel) against cuBLAS (FP32 and TF32) at the
head shapes of configs D / E.  Prints one JSON object."""
import json
import sys

import torch

sys.path.insert(0, '.')
from boxinstseg_b200 import _lib as L  # noqa: E402

DEV = 'cuda:0'
PEAK = json.load(open('MEASURED_PEAKS.json')).get('hbm_gbs', 3350.0)


def timeit(fn, iters=50):
    for _ in range(5):
        fn()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def case(name, B, C, h, w, I):
    P = h * w
    f = torch.randn(B, C, h, w, device=DEV)
    k = torch.randn(B, I, C, device=DEV) * 0.05
    g = torch.randn(B, I, h, w, device=DEV)
    out = torch.empty(B, I, h, w, device=DEV)
    gf, gk = torch.empty_like(f), torch.empty_like(k)
    lib = L.lib()
    ws = torch.empty(lib.bxs_dynconv1x1_backward_workspace_bytes(B, C, P, I), dtype=torch.uint8, device=DEV)
    st = L.stream()
    res = {'shape': [B, C, h, w, I]}
    res['fwd_us'] = timeit(lambda: lib.bxs_dynconv1x1_forward(L.ptr(f), L.ptr(k), L.ptr(out), B, C, P, I, st))
    if I <= 256:
        res['bwd_feat_us'] = timeit(lambda: lib.bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), L.ptr(gf), None, L.ptr(ws), B, C, P, I, st))
    res['bwd_kernel_us'] = timeit(lambda: lib.bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), None, L.ptr(gk), L.ptr(ws), B, C, P, I, st))
    f2, g2 = f.flatten(2), g.flatten(2)
    for tf32 in (False, True):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        tag = 'cublas_tf32' if tf32 else 'cublas_fp32'
        res[tag + '_fwd_us'] = timeit(lambda: torch.bmm(k, f2))
        res[tag + '_bwd_feat_us'] = timeit(lambda: torch.bmm(k.transpose(1, 2), g2))
        res[tag + '_bwd_kernel_us'] = timeit(lambda: torch.bmm(g2, f2.transpose(1, 2)))
    torch.backends.cuda.matmul.allow_tf32 = False
    byts = 4 * (B * C * P + B * I * P + B * I * C)
    for key in ('fwd_us', 'bwd_feat_us', 'bwd_kernel_us'):
        if key in res:
            res[key.replace('_us', '_frac_hbm')] = byts / res[key] / 1e3 / PEAK
    res['algo_mb'] = byts / 1e6
    print(name, json.dumps(res), flush=True)
    return res


if __name__ == '__main__':
    out = {}
    out['boxsolo_D_pos100'] = case('boxsolo_D_pos100', 2, 256, 200, 256, 100)
    out['boxsolo_D_pos16'] = case('boxsolo_D_pos16', 2, 256, 200, 256, 16)
    out['box2mask_E_q100'] = case('box2mask_E_q100', 2, 256, 96, 96, 100)
    out['discobox_pos256'] = case('discobox_pos256', 2, 256, 200, 256, 256)
    json.dump(out, open('gpurun_out/bench_dynconv.json', 'w'), indent=1)
