"""Time one BoxLevelset head step -- FPN features to loss_boxpro + loss_levelset + loss_cate, forward and backward -- at
config D's shapes (2 images of 800x1024, 8 ground truths per image drawn as bench_configs draws them, stand-in towers
with 256 channels), in two arms alternated over rounds:

  ref  the reference's training lines (oracle/solo_head.py): dense F.conv2d(groups=B) over all 3872 cells of every level,
       F.interpolate, boolean indexing, per-instance image / level-set targets into this package's mask_loss, focal loss
       as torch lines;
  new  BoxSOLOv2Head.forward + BoxSOLOv2Head.loss (positive cells only, one host read, the focal kernel).

Reports per arm the median / min / max GPU time of a step (CUDA events), kernel launches per step (torch.profiler, a
separate run), synchronising calls per step (torch.cuda.set_sync_debug_mode('warn')), the peak allocation of a step, and
the category loss alone (fwd + bwd: sigmoid_focal_loss_levels against the torch lines), with the card's name and power
limit read in the same run.  Prints one JSON document; `--out PATH` also writes it there.

    python tools/bench_solo_head.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench_configs import HP, WP, _image_and_boxes  # noqa: E402
from oracle import solo_head as osh  # noqa: E402

DEV = 'cuda:0'
HEAD = dict(type='BoxSOLOv2Head', num_classes=80, in_channels=256, seg_feat_channels=256, stacked_convs=4,
            strides=[8, 8, 16, 32, 32], scale_ranges=((1, 96), (48, 192), (96, 384), (192, 768), (384, 2048)), sigma=0.2,
            num_grids=[40, 36, 24, 16, 12], cate_down_pos=0,
            loss_cate=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0))


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def workload(seed=0):
    from boxinstseg_b200.models import build_head
    _, imgs, boxes = _image_and_boxes(seed, 2)
    gen = torch.Generator().manual_seed(seed + 1)
    head = osh.attach_towers(build_head(HEAD), 256, 256, 80, seed=seed).to(DEV)
    feats = [torch.randn(2, 256, -(-HP // s), -(-WP // s), generator=gen).to(DEV) for s in (4, 8, 16, 32, 64)]
    masks, labels = [], []
    for bx in boxes:
        m = torch.zeros(len(bx), HP, WP, dtype=torch.uint8)
        for g, (x1, y1, x2, y2) in enumerate(bx.tolist()):
            m[g, int(y1):int(y2) + 1, int(x1):int(x2) + 1] = 1        # box-shaped masks (GenerateBoxMask)
        masks.append(m.to(DEV))
        labels.append(torch.randint(0, 80, (len(bx),), generator=gen).to(DEV))
    return head, feats, imgs.to(DEV), [b.to(DEV) for b in boxes], labels, masks


def arms(head, feats, img, boxes, labels, masks):
    params = list(head.parameters())

    def new():
        xs = [f.clone().requires_grad_(True) for f in feats]
        ins, cate, lst = head(xs)
        out = head.loss(ins, cate, lst, boxes, labels, masks, img, None, None)
        return out, torch.autograd.grad(sum(out.values()), xs + params, allow_unused=True)

    def ref():
        xs = [f.clone().requires_grad_(True) for f in feats]
        ins, cate, lst = osh.forward(head, xs)
        out = osh.loss(head, ins, cate, lst, boxes, labels, masks, img)
        return out, torch.autograd.grad(sum(out.values()), xs + params, allow_unused=True)
    return {'ref': ref, 'new': new}


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), torch.cuda.max_memory_allocated() - base


def syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as seen:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(0)
    return sum('synchroniz' in str(w.message) for w in seen)


def launches(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def focal_alone(head, feats, reps=50):
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    with torch.no_grad():
        _, cate, _ = osh.forward(head, feats)
    gen = torch.Generator(device=DEV).manual_seed(0)
    labels = [torch.where(torch.rand(2, c.shape[-1] ** 2, device=DEV, generator=gen) < 0.01,
                          torch.randint(0, 80, (2, c.shape[-1] ** 2), device=DEV, generator=gen), 80) for c in cate]
    xs = [c.detach().clone().requires_grad_(True) for c in cate]
    avg = sum((t < 80).sum() for t in labels) + 1

    def kernel():
        torch.autograd.grad(sigmoid_focal_loss_levels(xs, labels, avg, 2.0, 0.25, 1.0), xs)

    def torch_lines():
        pred = torch.cat([c.permute(0, 2, 3, 1).reshape(-1, 80) for c in xs])
        t = torch.nn.functional.one_hot(torch.cat([l.reshape(-1) for l in labels]), 81)[:, :80]
        torch.autograd.grad(osh.py_sigmoid_focal_loss(pred, t, 2.0, 0.25, avg, 1.0), xs)
    out = {}
    for name, fn in (('kernel', kernel), ('torch_lines', torch_lines)):
        for _ in range(5):
            fn()
        ts = [timed(fn)[0] for _ in range(reps)]
        out[name] = dict(median_ms=statistics.median(ts), min_ms=min(ts), max_ms=max(ts), launches=launches(fn))
    out['bytes'] = dict(logits=sum(c.numel() * 4 for c in cate), grad=sum(c.numel() * 4 for c in cate))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_solo_head needs a CUDA device')
    case = workload()
    fns = arms(*case)
    for _ in range(args.warmup):
        for fn in fns.values():
            fn()
    times, peaks = {k: [] for k in fns}, {k: 0 for k in fns}
    for r in range(args.rounds):                                   # alternate the arms, starting side swapped each round
        for name in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
            t, p = timed(fns[name])
            times[name].append(t)
            peaks[name] = max(peaks[name], p)
    res = dict(card=card(), workload='BoxSOLOv2 head step at config D: 2 x 800x1024, 8 GT / image, 256-channel stand-in towers, '
                                     'forward + backward to every parameter and the FPN inputs', rounds=args.rounds)
    for name, fn in fns.items():
        res[name] = dict(median_ms=statistics.median(times[name]), min_ms=min(times[name]), max_ms=max(times[name]),
                         peak_alloc_bytes=peaks[name], launches=launches(fn), host_syncs=syncs(fn))
    res['speedup_median'] = res['ref']['median_ms'] / res['new']['median_ms']
    res['focal'] = focal_alone(case[0], case[1])
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
