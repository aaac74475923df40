"""One Box2Mask decoder layer's head at config E's shapes (B = 1, Q = 100 queries, C = 256, mask features 256x256, 8 heads),
the attention-mask target cycling 32x32, 64x64, 128x128 as the decoder levels do, two arms alternating over the rounds:

  ref  the reference's lines (box2mask_head.py:345-355 and the reset of :397): einsum, F.interpolate, flatten, repeat on
       float32, sigmoid, < 0.5, and attn_mask[torch.where(attn_mask.sum(-1) == attn_mask.shape[-1])] = False;
  new  box2mask_mask_pred (the wgmma kernel) + ops.box2mask.attention_mask(..., reset_full_rows=True).

Per layer: GPU time on CUDA events around the eager call, host time of the eager call (to its return; the reference arm
returns only after its nonzero has synchronised), kernel launches from a torch.profiler run, host synchronisations counted
under torch.cuda.set_sync_debug_mode('warn').  Medians and min / max over the rounds.  `--lib NAME=PATH` (repeatable) also
times the attention-mask kernel alone from other builds of the library (e.g. tools/build_variant.py with
-DBXS_ATTN_CLUSTER=1 to fix the cluster size).  Prints the card's name and power limit, read in the same call.

    python tools/bench_box2mask_head.py [--rounds R] [--iters N] [--lib NAME=PATH ...] [--out PATH]
"""
import argparse
import ctypes
import json
import os
import sys
import time

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from benchkit import card, kernel_launches, summary, syncs, time_call  # noqa: E402

B, Q, C, HF, HEADS = 1, 100, 256, 256, 8
SIZES = ((32, 32), (64, 64), (128, 128))


def ref_arm(embed, feat, size):
    mask_pred = torch.einsum('bqc,bchw->bqhw', embed, feat)
    attn = F.interpolate(mask_pred, size, mode='bilinear', align_corners=False)
    attn = attn.flatten(2).unsqueeze(1).repeat((1, HEADS, 1, 1)).flatten(0, 1)
    attn = (attn.sigmoid() < 0.5).detach()
    attn[torch.where(attn.sum(-1) == attn.shape[-1])] = False
    return mask_pred, attn


def new_arm(embed, feat, size):
    from boxinstseg_b200.ops.box2mask import attention_mask
    from boxinstseg_b200.ops.dynconv import box2mask_mask_pred
    mask_pred = box2mask_mask_pred(embed, feat)
    return mask_pred, attention_mask(mask_pred, size, HEADS, reset_full_rows=True)


def layer_times(fn, embed, feat, iters):
    """(GPU ms, host ms) per layer: the mean over `iters` passes of the three target sizes."""
    def host_clock(size):
        t0 = time.perf_counter()
        fn(embed, feat, size)
        return time.perf_counter() - t0
    host, gpu = 0.0, 0.0
    for _ in range(iters):
        for size in SIZES:
            g, h = time_call(lambda: host_clock(size))
            gpu += g
            host += h
    n = iters * len(SIZES)
    return gpu / n, host * 1e3 / n


def all_sizes(fn, embed, feat):
    return lambda: [fn(embed, feat, size) for size in SIZES]


def kernel_only(path, mask_pred, iters):
    """ms per launch of bxs_box2mask_attn_mask (reset on) from the library at `path`, per target size."""
    from boxinstseg_b200 import _lib as L
    f = getattr(ctypes.CDLL(path), 'bxs_box2mask_attn_mask')
    f.argtypes = L.SIGNATURES['bxs_box2mask_attn_mask']
    out = {}
    for h, w in SIZES:
        attn = torch.empty((B * HEADS, Q, h * w), dtype=torch.bool, device=mask_pred.device)
        args = (L.ptr(mask_pred), L.ptr(attn), B, Q, HF, HF, h, w, HEADS, 0, 1, L.stream())
        for _ in range(3):
            L.check(f(*args), 'warm-up')
        out[f'{h}x{w}'] = time_call(lambda: f(*args), reps=iters)[0]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=7)
    ap.add_argument('--iters', type=int, default=30)
    ap.add_argument('--lib', action='append', default=[], metavar='NAME=PATH')
    ap.add_argument('--out', metavar='PATH', default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'this benchmark measures the GPU'
    res = {'card': card()}
    print('card', json.dumps(res['card']), flush=True)
    gen = torch.Generator(device='cuda').manual_seed(0)
    embed = torch.randn(B, Q, C, generator=gen, device='cuda') * C ** -0.5
    feat = torch.randn(B, C, HF, HF, generator=gen, device='cuda')
    arms = {'ref': ref_arm, 'new': new_arm}
    with torch.no_grad():
        for size in SIZES:                                  # same masks: the new arm is bit-exact on its own mask_pred
            mp, attn = new_arm(embed, feat, size)
            _, attn_ref = ref_arm(embed, feat, size)
            res[f'mask_bits_differing_from_ref_{size[0]}'] = int((attn != attn_ref).sum())
        for fn in arms.values():
            layer_times(fn, embed, feat, 3)
        gpu = {a: [] for a in arms}
        host = {a: [] for a in arms}
        for _ in range(args.rounds):                        # alternate the arms within the call
            for a, fn in arms.items():
                g, h = layer_times(fn, embed, feat, args.iters)
                gpu[a].append(g)
                host[a].append(h)
        for a, fn in arms.items():
            res[a] = {'gpu_ms_per_layer': summary(gpu[a]), 'host_ms_per_layer': summary(host[a]),
                      'launches_per_layer': kernel_launches(all_sizes(fn, embed, feat)) / len(SIZES),
                      'syncs_per_layer': syncs(all_sizes(fn, embed, feat)) / len(SIZES)}
            r = res[a]
            print(f'{a:3s} GPU {r["gpu_ms_per_layer"]["median"]:.4f} ms [{r["gpu_ms_per_layer"]["min"]:.4f}, '
                  f'{r["gpu_ms_per_layer"]["max"]:.4f}]  host {r["host_ms_per_layer"]["median"]:.4f} ms '
                  f'[{r["host_ms_per_layer"]["min"]:.4f}, {r["host_ms_per_layer"]["max"]:.4f}]  launches '
                  f'{r["launches_per_layer"]:.2f}  syncs {r["syncs_per_layer"]:.2f}', flush=True)
        mp = new_arm(embed, feat, SIZES[0])[0].contiguous()
        libs = [('main', os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'boxinstseg_b200', 'lib',
                                      'libboxseg_b200.so'))] + [tuple(s.split('=', 1)) for s in args.lib]
        kt = {name: [] for name, _ in libs}
        for _ in range(args.rounds):
            for name, path in libs:
                kt[name].append(kernel_only(path, mp, args.iters * 10))
        res['kernel_ms'] = {}
        for name, _ in libs:
            res['kernel_ms'][name] = {s: summary([r[s] for r in kt[name]]) for s in kt[name][0]}
            print(f'kernel {name:6s} ' + '  '.join(f'{s} {v["median"] * 1e3:.1f} us [{v["min"] * 1e3:.1f}, '
                                                      f'{v["max"] * 1e3:.1f}]' for s, v in res['kernel_ms'][name].items()),
                  flush=True)
    # algorithmic bytes of the new kernel: mask_pred read once, the bools written once per head
    res['kernel_bytes'] = {f'{h}x{w}': B * Q * HF * HF * 4 + B * HEADS * Q * h * w for h, w in SIZES}
    res['card_after'] = card()
    print('bytes', json.dumps(res['kernel_bytes']), 'card_after', json.dumps(res['card_after']), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
