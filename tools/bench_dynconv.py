"""Time the wgmma dynamic 1x1 convolution (forward, d/d feat, d/d kernel) against cuBLAS at the head shapes of configs
C / D / E: float32 operands (our TF32 kernels vs cuBLAS FP32 and TF32) and float16 / bfloat16 operands (our 16-bit
kernels vs cuBLAS in the same dtype), plus config C's DiscoBox mask-loss step in float32 and under float16 autocast.
Prints one line per case, with the card's name and power limit; `--out PATH` also writes everything to one JSON file.

    python tools/bench_dynconv.py [--out PATH]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, '.')
from benchkit import capture, card, host_ms, replay_ms, time_queued  # noqa: E402
from boxinstseg_b200 import _lib as L  # noqa: E402

DEV = 'cuda:0'
PEAK = json.load(open('MEASURED_PEAKS.json')).get('hbm_gbs', 3350.0) if os.path.exists('MEASURED_PEAKS.json') else 3350.0
HALF = {torch.float16: 0, torch.bfloat16: 1}


def l2_cold_us(fn, iters=50):
    """Median GPU time (µs) of one call queued behind an L2 flush, which also hides the call's launch."""
    for _ in range(5):
        fn()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=DEV)
    ts = []
    for _ in range(iters):
        flush.zero_()
        ts.append(time_queued(fn)[0] * 1e3)
    return sorted(ts)[len(ts) // 2]


def case(name, B, C, h, w, I, dt=torch.float32):
    P = h * w
    f = torch.randn(B, C, h, w, device=DEV).to(dt)
    k = (torch.randn(B, I, C, device=DEV) * 0.05).to(dt)
    g = torch.randn(B, I, h, w, device=DEV).to(dt)
    out = torch.empty(B, I, h, w, device=DEV, dtype=dt)
    gf, gk = torch.empty_like(f), torch.empty_like(k)
    lib = L.lib()
    st = L.stream()
    res = {'shape': [B, C, h, w, I], 'dtype': str(dt).replace('torch.', '')}
    if dt == torch.float32:
        ws = torch.empty(lib.bxs_dynconv1x1_backward_workspace_bytes(B, C, P, I), dtype=torch.uint8, device=DEV)
        fwd = lambda: lib.bxs_dynconv1x1_forward(L.ptr(f), L.ptr(k), L.ptr(out), B, C, P, I, st)   # noqa: E731
        bwd = lambda a, b: lib.bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), a, b, L.ptr(ws), B, C, P, I, st)  # noqa: E731
    else:
        d = HALF[dt]
        ws = torch.empty(lib.bxs_dynconv1x1_half_backward_workspace_bytes(B, C, P, I, d), dtype=torch.uint8, device=DEV)
        fwd = lambda: lib.bxs_dynconv1x1_half_forward(L.ptr(f), L.ptr(k), L.ptr(out), B, C, P, I, d, st)   # noqa: E731
        bwd = lambda a, b: lib.bxs_dynconv1x1_half_backward(L.ptr(f), L.ptr(k), L.ptr(g), a, b, L.ptr(ws), B, C, P, I, d, st)  # noqa: E731
    assert fwd() == 0 and bwd(L.ptr(gf) if I <= 256 else None, L.ptr(gk)) == 0
    res['fwd_us'] = l2_cold_us(fwd)
    if I <= 256:
        res['bwd_feat_us'] = l2_cold_us(lambda: bwd(L.ptr(gf), None))
    res['bwd_kernel_us'] = l2_cold_us(lambda: bwd(None, L.ptr(gk)))
    f2, g2 = f.flatten(2), g.flatten(2)
    for tf32 in ((False, True) if dt == torch.float32 else (False,)):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        tag = 'cublas_' + ('tf32' if tf32 else res['dtype'])
        res[tag + '_fwd_us'] = l2_cold_us(lambda: torch.bmm(k, f2))
        res[tag + '_bwd_feat_us'] = l2_cold_us(lambda: torch.bmm(k.transpose(1, 2), g2))
        res[tag + '_bwd_kernel_us'] = l2_cold_us(lambda: torch.bmm(g2, f2.transpose(1, 2)))
    torch.backends.cuda.matmul.allow_tf32 = False
    byts = f.element_size() * (B * C * P + B * I * P + B * I * C)
    for key in ('fwd_us', 'bwd_feat_us', 'bwd_kernel_us'):
        if key in res:
            res[key.replace('_us', '_frac_hbm')] = byts / res[key] / 1e3 / PEAK
    res['algo_mb'] = byts / 1e6
    print(name, json.dumps(res), flush=True)
    return res


def config_c_step(iters=20):
    """Config C's DiscoBox mask-loss step (forward + backward): float32, and under float16 autocast with a float16
    mask-feature leaf (median ms of `iters` synchronised steps); plus the step's two dynamic convolutions, forward and
    backward, alone with the float16 leaf, through the 16-bit kernels and as a float32 cast + TF32 kernels (GPU µs)."""
    import bench_configs
    from boxinstseg_b200.models import build_head
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    _, info = bench_configs.build_C(torch.device(DEV), 0)
    d = info['data']
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256))
    feat16 = d['feat'].detach().half().requires_grad_(True)
    g = torch.randn(16, 200, 256, device=DEV).half()

    def step(feat, autocast):
        with torch.autocast('cuda', dtype=torch.float16, enabled=autocast):
            pred = torch.cat([head.dynamic_conv(feat[b], d['kern'][b]) for b in range(2)])
            out = head.mask_loss([pred], [d['labels']], [d['img_inds']], d['color'])
        torch.autograd.grad(out['loss_ins'] + out['loss_ts'], [feat, d['kern']])

    def conv_legs(cast_fp32):
        f, k = feat16.detach().requires_grad_(True), d['kern'].detach().requires_grad_(True)
        for b in range(2):
            x = f[b][None]
            with torch.autocast('cuda', dtype=torch.float16, enabled=not cast_fp32):
                out = dynconv1x1(x.float() if cast_fp32 else x, k[b].t()[None].contiguous())
            torch.autograd.grad(out, [f, k], g[None].to(out.dtype))

    def median_step_ms(fn):
        for _ in range(3):
            fn()
        return sorted(host_ms(fn)[0] for _ in range(iters))[iters // 2]

    res = {}
    for _ in range(2):                                           # alternate, to see the spread
        res.setdefault('step_fp32_ms', []).append(median_step_ms(lambda: step(d['feat'], False)))
        res.setdefault('step_autocast_fp16_ms', []).append(median_step_ms(lambda: step(feat16, True)))
        # the eager legs are bound by the host's launch rate: their GPU time comes from a graph replay
        for tag, cast in (('native', False), ('cast_tf32', True)):
            graph = capture(lambda: conv_legs(cast))
            res.setdefault(f'conv_legs_fp16_{tag}_graph_us', []).append(replay_ms(graph, 50) * 1e3)
    print('config_C_step', json.dumps(res), flush=True)
    return res


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', metavar='PATH', default=None, help='write all results to this JSON file')
    args = ap.parse_args()
    out = {'card': card()}
    print('card', json.dumps(out['card']), flush=True)
    shapes = dict(boxsolo_D_pos100=(2, 256, 200, 256, 100), boxsolo_D_pos16=(2, 256, 200, 256, 16),
                  box2mask_E_q100=(2, 256, 96, 96, 100), discobox_pos256=(2, 256, 200, 256, 256),
                  discobox_C_img=(1, 256, 200, 256, 16))
    for name, shape in shapes.items():
        for dt in (torch.float32, torch.float16, torch.bfloat16):
            out[f'{name}_{str(dt)[6:]}'] = case(name, *shape, dt=dt)
    out['config_C_step'] = config_c_step()
    out['card_after'] = card()
    print('card_after', json.dumps(out['card_after']), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            json.dump(out, fh, indent=1)
