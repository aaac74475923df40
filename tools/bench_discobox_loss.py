"""Time DiscoBoxSOLOv2Head's training loss -- category logits, student and teacher kernel grids and mask features to
loss_ins, loss_ts and loss_cate, forward and backward -- at config C's shapes (2 images of 800x1024, mask features
[2,256,200,256], the COCO grids 40/36/24/16/12, 8 ground truths per image) under float16 autocast with an independent
teacher, in two arms alternated over rounds on the same CUDA tensors:

  ref  the reference's ``loss`` lines as restated in oracle/discobox_loss.py (host SOLO targets, one F.conv2d per (level,
       image) and network, the host loops, one mean field per image, the torch focal loss on the concatenated logits);
  new  DiscoBoxSOLOv2Head.loss (device targets, one packed dynamic convolution per network, the 16-bit mask-loss kernels,
       the focal kernel on the levels as they lie).

Reports per arm the median / min / max time of an eager step (CUDA events around work ending in a synchronise), kernel
launches per step (torch.profiler, a separate run), synchronising calls per step (torch.cuda.set_sync_debug_mode('warn'))
and the peak allocation of a step; the GPU time of the student convolution alone (forward + backward), one packed call
against one call per (level, image); and the card's name and power limit read in the same run.  Prints one JSON document;
`--out PATH` also writes it there.

    python tools/bench_discobox_loss.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from bench_condinst_box_loss import card, launches, syncs, timed  # noqa: E402
from oracle import discobox_loss as odl  # noqa: E402

DEV = 'cuda:0'
GRIDS = (40, 36, 24, 16, 12)
NUM_CLASSES = 80


def workload(seed=0, B=2, H=800, W=1024, G=8, C=256):
    gen = torch.Generator().manual_seed(seed)
    boxes, labels, masks = [], [], []
    for _ in range(B):
        wh = 16 + torch.rand(G, 2, generator=gen) ** 2 * 400
        xy = torch.rand(G, 2, generator=gen) * (torch.tensor([W, H]) - wh)
        bx = torch.cat([xy, xy + wh], 1).floor()
        m = np.zeros((G, H, W), np.uint8)
        for i, r in enumerate(bx):
            m[i, int(r[1]):int(r[3]), int(r[0]):int(r[2])] = 1
        boxes.append(bx.to(DEV))
        labels.append(torch.randint(0, NUM_CLASSES, (G,), generator=gen).to(DEV))
        masks.append(m)
    cate = [torch.randn(B, NUM_CLASSES, S, S, generator=gen).to(DEV) for S in GRIDS]
    s_k = [(torch.randn(B, C, S, S, generator=gen) * 0.05).to(DEV) for S in GRIDS]
    t_k = [(torch.randn(B, C, S, S, generator=gen) * 0.05).to(DEV) for S in GRIDS]
    s_in = torch.randn(B, C, H // 4, W // 4, generator=gen).to(DEV)
    t_in = torch.randn(B, C, H // 4, W // 4, generator=gen).to(DEV)
    img = torch.randn(B, 3, H, W, generator=gen).to(DEV)
    return cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img


def arms(head, w):
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = w
    leaves = [t.requires_grad_(True) for t in cate + s_k + [s_in]]
    dev_masks = [torch.from_numpy(m).to(DEV) for m in masks]

    def new():
        with torch.autocast('cuda', dtype=torch.float16):
            out = head.loss(cate, s_k, t_k, s_in, t_in, boxes, labels, dev_masks, None, None, img=img, use_loss_ts=True,
                            use_ind_teacher=True)
        return torch.autograd.grad(sum(out.values()), leaves, allow_unused=True)

    def ref():
        with torch.autocast('cuda', dtype=torch.float16):
            out = odl.loss(cate, s_k, t_k, s_in, t_in, [b.cpu() for b in boxes], [l.cpu() for l in labels], masks, img, GRIDS,
                           NUM_CLASSES, use_loss_ts=True, use_ind_teacher=True)
        return torch.autograd.grad(sum(out.values()), leaves, allow_unused=True)
    return {'ref': ref, 'new': new}


def peak_bytes(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def conv_alone(head, w, reps=20):
    """GPU time (ms) of the student convolution of every level and image, forward + backward under float16 autocast."""
    from boxinstseg_b200.ops.dynconv import disco_cells_conv
    cate, s_k, t_k, s_in, t_in, boxes, labels, masks, img = w
    dev_masks = [torch.from_numpy(m).to(DEV) for m in masks]
    (s_list, _, _, _, _), per_img = head._corr_inputs(s_k, None, s_in, None, boxes, labels, dev_masks, False, False, None)
    B = len(per_img)
    orders = [[per_img[b][3][lv] for b in range(B)] for lv in range(len(GRIDS))]
    leaves = [s_in] + s_k

    def packed():
        with torch.autocast('cuda', dtype=torch.float16):
            rows = [r for r in disco_cells_conv(s_in, s_k, orders)[0] if r is not None]
        return torch.autograd.grad(sum(r.float().sum() for r in rows), leaves)

    def per_level_image():
        with torch.autocast('cuda', dtype=torch.float16):
            rows = [head.dynamic_conv(s_in[b], s_k[lv][b].reshape(s_k[lv].shape[1], -1)[:, o])
                    for lv in range(len(GRIDS)) for b, o in enumerate(orders[lv]) if o.numel()]
        return torch.autograd.grad(sum(r.float().sum() for r in rows), leaves)
    fns = {'packed': packed, 'per_level_image': per_level_image}
    for fn in fns.values():
        fn()
    times = {k: [] for k in fns}
    for r in range(reps):
        for name in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
            times[name].append(timed(fns[name]))
    rows = sum(int(o.numel()) for lvl in orders for o in lvl)
    return dict(rows=rows, I_pad=max(sum(int(orders[lv][b].numel()) for lv in range(len(GRIDS))) for b in range(B)),
                **{k: dict(median_ms=statistics.median(v), min_ms=min(v), max_ms=max(v), launches=launches(fns[k]))
                   for k, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_discobox_loss needs a CUDA device')
    from boxinstseg_b200.models import build_head
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=NUM_CLASSES, in_channels=256, num_grids=list(GRIDS),
                           strides=odl.CFG['strides'], scale_ranges=odl.CFG['scale_ranges']))
    w = workload()
    fns = arms(head, w)
    for _ in range(args.warmup):
        for fn in fns.values():
            fn()
    times = {k: [] for k in fns}
    for r in range(args.rounds):                                   # alternate the arms, starting side swapped each round
        for name in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
            times[name].append(timed(fns[name]))
    res = dict(card=card(), workload='DiscoBoxSOLOv2Head.loss at config C: 2 x 800x1024, mask features [2,256,200,256], '
                                     'grids 40/36/24/16/12, 8 GT per image, 80 classes, float16 autocast, independent '
                                     'teacher, use_loss_ts; forward + backward to cate_preds, s_kernel_preds_raw, s_ins_pred',
               rounds=args.rounds)
    for name, fn in fns.items():
        res[name] = dict(median_ms=statistics.median(times[name]), min_ms=min(times[name]), max_ms=max(times[name]),
                         launches=launches(fn), host_syncs=syncs(fn), peak_alloc_bytes=peak_bytes(fn))
    res['speedup_median_eager'] = res['ref']['median_ms'] / res['new']['median_ms']
    res['student_conv_alone'] = conv_alone(head, w)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
