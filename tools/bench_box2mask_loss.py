"""Time Box2MaskHead's training loss -- decoder outputs to the 30 losses of every layer, forward and backward -- at config E's
shapes (B = 1, 10 decoder layers, Q = 100 queries, 80 classes, 256x256 mask logits, 1024x1024 box masks, 8 ground truths),
in two arms alternated over rounds:

  ref  the reference's ``loss`` / ``loss_single`` lines (oracle/box2mask_loss.py with the package's GPU parts): one scipy
       matching per (layer, image) on the host, F.cross_entropy + weight_reduce_loss per layer, boolean indexing,
       ``.cpu()`` of the match counts, the image MST rebuilt per layer, targets repeated per matched query;
  new  Box2MaskHead.loss (one matching launch for every layer, one cross-entropy kernel, the image trees built once, the
       layers' mask losses on lane streams, no host read).

Reports per arm the median / min / max GPU time of a step (CUDA events), kernel launches per step (torch.profiler, a
separate run), synchronising calls per step (torch.cuda.set_sync_debug_mode('warn')), the peak allocation of a step, and
the classification loss alone (fwd + bwd of the 10 layers: softmax_cross_entropy_layers against the torch lines), with the
card's name and power limit read in the same run.  Prints one JSON document; `--out PATH` also writes it there.

    python tools/bench_box2mask_loss.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchkit import card, launches, ms_summary, peak_alloc, syncs, time_call  # noqa: E402
from oracle import box2mask_loss as obl  # noqa: E402

DEV = 'cuda:0'


def workload(seed=0, layers=10):
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import Box2MaskHead
    head = Box2MaskHead(num_queries=100, num_things_classes=80, num_stuff_classes=0,
                        train_cfg=dict(assigner=obl.ASSIGNER, sampler=dict(type='MaskPseudoSampler')))
    case = obl.golden_case(seed=seed, B=1, gts=(8,), Q=100, num_classes=80, layers=layers, pred=256, mask=1024)
    to = lambda x: [t.to(DEV) for t in x] if isinstance(x, list) else x.to(DEV)     # noqa: E731
    return head, [to(x) for x in case]


def arms(head, case):
    cls, masks, lsts, labels, gts, img = case
    metas = [dict()]

    def leaves():
        return [[t.clone().requires_grad_(True) for t in ts] for ts in (cls, masks, lsts)]

    def new():
        lv = leaves()
        out = head.loss(*lv, labels, gts, metas, img)
        return out, torch.autograd.grad(sum(out.values()), [t for ts in lv for t in ts])

    def ref():
        lv = leaves()
        out = obl.loss(obl.gpu_parts(head), 100, 80, head.cls_class_weight, head.cls_loss_weight, *lv, labels, gts, img)
        return out, torch.autograd.grad(sum(out.values()), [t for ts in lv for t in ts], allow_unused=True)
    return {'ref': ref, 'new': new}


def ce_alone(head, case, reps=100):
    """The 10 layers' classification losses, forward + backward: one kernel pair against the reference's torch lines."""
    from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
    cls = case[0]
    gen = torch.Generator(device=DEV).manual_seed(0)
    labels = torch.where(torch.rand(len(cls), 1, 100, device=DEV, generator=gen) < 0.08,
                         torch.randint(0, 80, (len(cls), 1, 100), device=DEV, generator=gen), 80)
    cw = head._class_weight(torch.device(DEV))
    xs = [c.detach().clone().requires_grad_(True) for c in cls]

    def kernel():
        torch.autograd.grad(softmax_cross_entropy_layers(xs, labels, cw, 2.0).sum(), xs)

    def torch_lines():
        total = sum(obl.cross_entropy_loss(x.flatten(0, 1), y.flatten(), torch.ones_like(y.flatten()), cw, 2.0,
                                           cw[y.flatten()].sum()) for x, y in zip(xs, labels))
        torch.autograd.grad(total, xs)
    out = {}
    for name, fn in (('kernel', kernel), ('torch_lines', torch_lines)):
        for _ in range(5):
            fn()
        ts = [time_call(fn)[0] for _ in range(reps)]
        out[name] = dict(**ms_summary(ts), launches=launches(fn))
    out['bytes'] = dict(scores=sum(c.numel() * 4 for c in cls), grad=sum(c.numel() * 4 for c in cls))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_box2mask_loss needs a CUDA device')
    head, case = workload()
    fns = arms(head, case)
    for _ in range(args.warmup):
        for fn in fns.values():
            fn()
    times, peaks = {k: [] for k in fns}, {k: 0 for k in fns}
    for r in range(args.rounds):                                   # alternate the arms, starting side swapped each round
        for name in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
            p, t = peak_alloc(lambda: time_call(fns[name])[0])
            times[name].append(t)
            peaks[name] = max(peaks[name], p)
    res = dict(card=card(), workload='Box2MaskHead.loss at config E: 1 x 1024x1024, 8 GT, 10 decoder layers x 100 queries, '
                                     '256x256 mask logits, forward + backward to every layer\'s scores, logits and level-set '
                                     'feature', rounds=args.rounds)
    for name, fn in fns.items():
        res[name] = dict(**ms_summary(times[name]), peak_alloc_bytes=peaks[name], launches=launches(fn),
                         host_syncs=syncs(fn))
    res['speedup_median'] = res['ref']['median_ms'] / res['new']['median_ms']
    res['cross_entropy'] = ce_alone(head, case)
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
