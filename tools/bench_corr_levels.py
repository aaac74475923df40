"""DiscoBox's correspondence loss per call of ``DiscoBoxSOLOv2Head.corr_loss_levels`` (forward: RoIAlign, retrieval, solve,
InfoNCE, transfer, paste, bank append, mean field, dice) with the COCO bank and solver settings
(configs/discobox/discobox_solov2_coco_r50_fpn_3x.py: 80 classes, 100 slots, 7 x 7 features of 128 channels, 28 x 28 masks,
min_size 32, at most 5 retrieved), B = 2 images of 200 x 336 mask features, one level of n objects of four classes.  The
bank is pre-filled by warm-up calls on similar objects, so that most queries retrieve 5 objects and take the loss.

Per n: the eager time per call (host clock around a synchronised call: the loss is bound by the host issuing launches),
the CUDA-graph replay time (CUDA events; "null" when the tree's code cannot be captured), the kernel launches per call
(torch.profiler).  Medians and min / max over the rounds.

    python tools/bench_corr_levels.py [--trees DIR [DIR ...]] [--rounds R] [--iters N] [--out PATH]

Each tree (a checkout with its library built) runs in its own process, the trees alternating round by round; the card's
name and power limit are read in the same call.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

from benchkit import capture, card, host_ms, launches, replay_ms

DEV = 'cuda:0'
NS = (4, 16, 32)
BANK = dict(feat_height=7, feat_width=7, mask_height=28, mask_width=28, min_size=32, len_object_queues=100, fg_iou_thresh=0.7,
            bg_iou_thresh=0.7, ratio_range=[0.9, 1.2], appear_thresh=0.7, max_retrieval_objs=5)
LOSS_CORR = dict(loss_weight=1.0, corr_exp=1.0, corr_eps=0.05, gaussian_filter_size=3, low_score=0.3, corr_num_iter=10,
                 corr_num_smooth_iter=1, dist_kernel=9, obj_bank=BANK)


def inputs(torch, n, seed, B=2, C=128, H=200, W=336):
    gen = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.arange(H, dtype=torch.float32), torch.arange(W, dtype=torch.float32), indexing='ij')
    pattern = torch.stack([torch.sin(yy / 5 + c) + torch.cos(xx / 7 + 2 * c) for c in range(C)])
    s_feat = pattern[None] + 0.03 * torch.randn(B, C, H, W, generator=gen)
    t_feat = pattern[None] + 0.03 * torch.randn(B, C, H, W, generator=gen)
    color = torch.randn(B, 3, H, W, generator=gen)
    tg = torch.zeros(n, H, W, dtype=torch.uint8)
    inside = []
    for i in range(n):
        y0, x0 = 20 + 30 * (i % 5) + int(torch.randint(0, 3, (1,), generator=gen)), 20 + 50 * (i % 5)
        bh, bw = 44 + int(torch.randint(0, 2, (1,), generator=gen)), 48 + int(torch.randint(0, 2, (1,), generator=gen))
        tg[i, y0:y0 + bh, x0:x0 + bw] = 1
        inside.append(((yy - (y0 + bh / 2)) / (0.4 * bh)) ** 2 + ((xx - (x0 + bw / 2)) / (0.4 * bw)) ** 2 < 1)
    logits = (torch.stack(inside).float() * 2 - 1) * 4 + 0.5 * torch.randn(n, H, W, generator=gen)
    labels = torch.arange(n) % 4
    imgs = torch.arange(n) % B
    return ([logits.to(DEV)], None, [imgs.to(DEV)], [tg.to(DEV)], [labels.to(DEV)], s_feat.to(DEV), t_feat.to(DEV),
            color.to(DEV))


def worker(tree, iters):
    sys.path.insert(0, os.path.abspath(tree))
    import torch
    from boxinstseg_b200.models import build_head
    out = {}
    for n in NS:
        head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=128, loss_corr=LOSS_CORR))
        args = inputs(torch, n, n)
        call = lambda: head.corr_loss_levels(*args, gamma=0.5)
        with torch.no_grad():
            for _ in range(8):                                       # fills the bank: >= 5 similar objects per class
                call()
            times = [host_ms(call)[0] for _ in range(iters)]
            n_launches = launches(call)
            graph_ms = None
            if not hasattr(head.corr, 'levels_masked'):               # a tree whose loss synchronises: no capture
                out[n] = dict(eager_ms=statistics.median(times), graph_ms=None, launches=n_launches)
                continue
            try:
                graph_ms = replay_ms(capture(call), iters)
            except Exception as exc:                                  # a host synchronisation inside the call
                out.setdefault('graph_error', str(exc).splitlines()[0][:200])
        out[n] = dict(eager_ms=statistics.median(times), graph_ms=graph_ms, launches=n_launches)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--trees', nargs='+', default=['.'])
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out')
    ap.add_argument('--worker')
    a = ap.parse_args()
    if a.worker:
        return worker(a.worker, a.iters)
    runs = {t: [] for t in a.trees}
    for _ in range(a.rounds):
        for t in a.trees:
            r = subprocess.run([sys.executable, os.path.abspath(__file__), '--worker', t, '--iters', str(a.iters)],
                               capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit(f'{t}: {r.stderr[-2000:]}')
            runs[t].append(json.loads(r.stdout.strip().splitlines()[-1]))
    res = {'card': card(), 'rounds': a.rounds, 'iters': a.iters, 'trees': {}}
    for t, rs in runs.items():
        res['trees'][t] = {}
        for n in NS:
            per = [r[str(n)] for r in rs]
            row = {}
            for k in ('eager_ms', 'graph_ms'):
                v = [p[k] for p in per if p[k] is not None]
                row[k] = dict(median=statistics.median(v), min=min(v), max=max(v)) if v else None
            row['launches'] = per[0]['launches']
            res['trees'][t][n] = row
        if 'graph_error' in rs[0]:
            res['trees'][t]['graph_error'] = rs[0]['graph_error']
    print(json.dumps(res, indent=1))
    if a.out:
        with open(a.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
