"""Time CondInstBoxHead's box-branch loss -- the three prediction lists to loss_cls, loss_bbox and loss_centerness, forward
and backward -- at config A's shapes (2 images of 800x1024, five FCOS levels 100x128 ... 7x8, 80 classes, 8 ground truths
per image), in two arms alternated over rounds on the same CUDA tensors:

  ref  the reference's ``loss`` lines as restated in oracle/fcos_loss.py (permute + cat of every level, the dense
       [points, gts] FCOS assignment per image, nonzero(), Python max() of the reduced counts, gathers, the focal loss in
       its torch form, GIoU and BCE over the positive rows);
  new  CondInstBoxHead.loss (one targets launch, the stats kernel, one focal launch over the rectangular levels, the
       GIoU + centerness kernel, no host read).

Reports per arm the median / min / max time of an eager step (CUDA events around work ending in a synchronise), kernel
launches per step (torch.profiler, a separate run) and synchronising calls per step (torch.cuda.set_sync_debug_mode('warn')),
the device time of the new arm's step replayed from a CUDA graph, the algorithmic bytes of a step computed from the shapes,
and the card's name and power limit read in the same run.  Prints one JSON document; `--out PATH` also writes it there.

    python tools/bench_condinst_box_loss.py [--rounds 20] [--out PATH]
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
from oracle import fcos_loss as ofl  # noqa: E402
from oracle.make_golden_fcos_loss import STRIDES, case  # noqa: E402

DEV = 'cuda:0'


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def workload(seed=0):
    from boxinstseg_b200.models import build_head
    head = build_head(dict(type='CondInstBoxHead', num_classes=80, in_channels=256, strides=list(STRIDES),
                           loss_bbox=dict(type='GIoULoss', loss_weight=1.0)))
    cls, bbox, ctr, boxes, labels = case(seed, B=2, H=800, W=1024, G=(8,), C=80, ties=False, dtype=torch.float32)
    leaves = [t.to(DEV).requires_grad_(True) for t in cls + bbox + ctr]
    return head, leaves, [b.to(DEV) for b in boxes], [l.to(DEV) for l in labels]


def arms(head, leaves, boxes, labels):
    n = len(leaves) // 3
    parts = leaves[:n], leaves[n:2 * n], leaves[2 * n:]

    def new():
        out = head.loss(*parts, boxes, labels, None)
        return torch.autograd.grad(sum(out[0].values()), leaves)

    def ref():
        out = ofl.loss(*parts, boxes, labels, STRIDES, 80)
        return torch.autograd.grad(sum(out[0].values()), leaves)
    return {'ref': ref, 'new': new}


def timed(fn):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


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


def graph_replay_ms(fn, reps=200):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    for _ in range(10):
        g.replay()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        g.replay()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def algorithmic_bytes(leaves):
    """Each prediction read once and its gradient written once (float32), plus the labels (int64) and targets read."""
    n = len(leaves) // 3
    preds = sum(t.numel() for t in leaves) * 4
    points = sum(t.shape[0] * t.shape[2] * t.shape[3] for t in leaves[:n])
    return dict(predictions_read=preds, gradients_written=preds, labels_and_targets=points * (8 + 16),
                total=2 * preds + points * 24)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_condinst_box_loss needs a CUDA device')
    head, leaves, boxes, labels = workload()
    fns = arms(head, leaves, boxes, labels)
    for _ in range(args.warmup):
        for fn in fns.values():
            fn()
    times = {k: [] for k in fns}
    for r in range(args.rounds):                                   # alternate the arms, starting side swapped each round
        for name in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
            times[name].append(timed(fns[name]))
    res = dict(card=card(), workload='CondInstBoxHead.loss at config A: 2 x 800x1024, 8 GT per image, 80 classes, five '
                                     'FCOS levels, forward + backward to cls_scores, bbox_preds and centernesses',
               rounds=args.rounds, bytes=algorithmic_bytes(leaves))
    for name, fn in fns.items():
        res[name] = dict(median_ms=statistics.median(times[name]), min_ms=min(times[name]), max_ms=max(times[name]),
                         launches=launches(fn), host_syncs=syncs(fn))
    res['new']['graph_replay_ms'] = graph_replay_ms(fns['new'])
    res['speedup_median_eager'] = res['ref']['median_ms'] / res['new']['median_ms']
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
