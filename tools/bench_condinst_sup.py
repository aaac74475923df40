"""Time CondInst's mask-supervised losses -- the dice mask loss of CondInstMaskHead.loss with boxinst_enabled=False and
CondInstSegmHead.loss -- forward and backward, in two arms alternated over rounds on the same CUDA tensors:

  ref  the reference's lines as restated in oracle/condinst_sup.py (dice: the [N, h, w] uint8 gather and its float copy,
       sigmoid, three products and reductions, autograd; segm: the [G, H, W] int64 areas / labels at full resolution, then
       the focal loss in its torch form);
  new  ops.condinst.dice_mask_loss and CondInstSegmHead.loss (csrc/condinst_sup.cu, the masks read in place, and the
       focal-loss kernel).

Shapes: dice at N in {128, 500} instances of 200x256 logits (out_stride 4 over 2 images of 800x1024) with G in {8, 50}
ground truths per image; the segm head at B = 2, C = 80, 800x1024, G in {8, 50}.  Reports per arm the median / min / max
host-clock time of a step ending in a device synchronise, launches (torch.profiler, kernels + memcpys + memsets),
synchronising calls (set_sync_debug_mode('warn')) and the peak allocation a step adds; for the dice loss also the device
time of the new arm's kernels and its achieved bytes over that time against 3.35 TB/s (the H100 SXM's HBM3 data-sheet
figure), with the card's name, power limit and clock read in the same run.  Prints one JSON document; `--out PATH` also
writes it there.

    python tools/bench_condinst_sup.py [--rounds 20] [--out tools/results/bench_condinst_sup_h100.json]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from benchkit import card, host_ms, launches, ms_summary, peak_alloc, profile, syncs  # noqa: E402
from oracle import condinst_sup as ocs  # noqa: E402

DEV = 'cuda:0'
H, W, OUT_STRIDE, IN_STRIDE, C, B = 800, 1024, 4, 8, 80, 2
HBM_BYTES_PER_S = 3.35e12


def masks_of(G, seed):
    """B images of G rectangles each, uint8 [G, H, W] on the device, and int64 labels."""
    gen = torch.Generator().manual_seed(seed)
    masks, labels = [], []
    for _ in range(B):
        m = torch.zeros(G, H, W, dtype=torch.uint8)
        for k in range(G):
            y0, x0 = int(torch.randint(0, H - 64, (1,), generator=gen)), int(torch.randint(0, W - 64, (1,), generator=gen))
            m[k, y0:y0 + int(torch.randint(32, H - y0 + 1, (1,), generator=gen)),
              x0:x0 + int(torch.randint(32, W - x0 + 1, (1,), generator=gen))] = 1
        masks.append(m.to(DEV))
        labels.append(torch.randint(0, C, (G,), generator=gen).to(DEV))
    return masks, labels


def dice_arms(N, G, seed=0):
    from boxinstseg_b200.ops.condinst import dice_mask_loss
    masks, _ = masks_of(G, seed)
    gen = torch.Generator().manual_seed(seed + 1)
    h, w = H // OUT_STRIDE, W // OUT_STRIDE
    x = (4 * torch.randn(N, 1, h, w, generator=gen)).to(DEV).requires_grad_(True)
    gt_inds = torch.randint(0, B * G, (N,), generator=gen).to(DEV)

    def new():
        return torch.autograd.grad(dice_mask_loss(x, masks, gt_inds, OUT_STRIDE), x)

    def ref():
        return torch.autograd.grad(ocs.mask_loss(x, masks, gt_inds, OUT_STRIDE)['loss_mask'], x)
    distinct = int(torch.unique(gt_inds).numel())
    logits = N * h * w * 4
    targets = distinct * h * ((W + 31) // 32) * 32          # each sampled row's 32-byte sectors, once per distinct GT
    bytes_ = dict(formula='2 * N*h*w*4 (logits read by forward and backward) + N*h*w*4 (gradient written) + '
                          'distinct_gts * h * ceil(W/32)*32 (the sampled rows of each referenced mask)',
                  logits_read=2 * logits, gradient_written=logits, target_sectors=targets,
                  total=3 * logits + targets)
    return {'ref': ref, 'new': new}, bytes_


def segm_arms(G, seed=0):
    from boxinstseg_b200.models import build_head
    head = build_head(dict(type='CondInstSegmHead', num_classes=C, in_channels=256, in_stride=IN_STRIDE))
    masks, labels = masks_of(G, seed)
    gen = torch.Generator().manual_seed(seed + 2)
    p = torch.randn(B, C, H // IN_STRIDE, W // IN_STRIDE, generator=gen).to(DEV).requires_grad_(True)

    def new():
        return torch.autograd.grad(head.loss(p, masks, labels)['loss_segm'], p)

    def ref():
        return torch.autograd.grad(ocs.segm_loss(p, masks, labels, IN_STRIDE, C)['loss_segm'], p)
    return {'ref': ref, 'new': new}


def measure(fns, rounds, warmup):
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    times = {k: [] for k in fns}
    for r in range(rounds):                                        # alternate the arms, starting side swapped each round
        for name in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
            times[name].append(host_ms(fns[name])[0])
    out = {}
    for name, fn in fns.items():
        out[name] = dict(**ms_summary(times[name]), launches=launches(fn), host_syncs=syncs(fn),
                         peak_alloc_bytes=peak_alloc(fn)[0])
    out['speedup_median'] = out['ref']['median_ms'] / out['new']['median_ms']
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_condinst_sup needs a CUDA device')
    res = dict(card=card(), rounds=args.rounds, dice={}, segm={})
    for N in (128, 500):
        for G in (8, 50):
            fns, bytes_ = dice_arms(N, G)
            r = measure(fns, args.rounds, args.warmup)
            fns['new']()
            kernels = {k: v for k, v in profile(fns['new']).items() if 'dice' in k}
            dev_ms = sum(ms for _, ms in kernels.values())
            r['new']['dice_kernels_device_ms'] = {k: ms for k, (_, ms) in kernels.items()}
            r['bytes'] = bytes_
            r['achieved_bytes_per_s'] = bytes_['total'] / (dev_ms * 1e-3)
            r['share_of_hbm_peak'] = r['achieved_bytes_per_s'] / HBM_BYTES_PER_S
            res['dice'][f'N{N}_G{G}'] = r
            del fns
            torch.cuda.empty_cache()
    for G in (8, 50):
        res['segm'][f'G{G}'] = measure(segm_arms(G), args.rounds, args.warmup)
        torch.cuda.empty_cache()
    res['card_after'] = card()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
