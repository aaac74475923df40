"""Time BoxLevelset's head test path -- FPN features to per-image masks, labels and scores -- both ways, at COCO test shape
(800 x 1333 images padded to 800 x 1344: feature_pred 200 x 336, grids 40/36/24/16/12 = 3872 cells, 80 classes), B = 1 and
2, the 256-channel stand-in towers of tools/bench_solo_head.py, test_cfg score_thr 0.05, mask_thr 0.55, nms_pre 500,
max_per_img 100, in two arms alternated over rounds:

  dense  get_seg(*forward(feats, eval=True)): the dynamic convolution and sigmoid of all 3872 cells at 200 x 336, each
         distinct candidate row read in place;
  cells  BoxSOLOv2Head.simple_test: the same towers, then only the distinct candidate cells packed and convolved.

The category logits are seeded: K (cell, class) pairs per image, K = 100, 500 and 2000, get +4 on the stand-in's logits
(whose sigmoid stays below 0.05 elsewhere), so that about K cells pass score_thr.  Both arms run the same towers on the same
offsets.  Reports per arm the median / min / max GPU time of a call over alternated rounds (CUDA events), kernel launches
per call and the sum of their device times (torch.profiler, a separate run), synchronising calls per call, the peak
allocation of a call, and the time of the towers alone;
checks that both arms return the same masks, labels and scores bit for bit; reads the card's name and power limit in the same
run.  Prints one JSON document; `--out PATH` also writes it.

    python tools/bench_solo_infer.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench_solo_head import HEAD  # noqa: E402
from benchkit import card, ms_summary, peak_alloc, profile, syncs, time_call  # noqa: E402
from oracle import solo_head as osh  # noqa: E402

DEV = 'cuda:0'
HP, WP = 800, 1344
GRIDS, C = HEAD['num_grids'], HEAD['num_classes']
META = dict(img_shape=(800, 1333, 3), ori_shape=(800, 1333, 3), pad_shape=(HP, WP, 3))
CFG = dict(score_thr=0.05, mask_thr=0.55, nms_pre=500, max_per_img=100, kernel='gaussian', sigma=2.0, filter_thr=0.05)
BOOST = 4.0


class SeededCate(nn.Module):
    """The stand-in's ``solo_cate`` plus a fixed logit offset per grid size: the category logits of a head whose K cells
    per image are confident."""

    def __init__(self, conv, offsets):
        super().__init__()
        self.conv, self.offsets = conv, offsets

    def forward(self, x):
        out = self.conv(x)
        return out + self.offsets[out.shape[-1]].to(out.dtype)


def offsets(B, K, gen):
    P = sum(s * s for s in GRIDS)
    flat = torch.zeros(B, P, C)
    for b in range(B):
        cells = torch.randperm(P, generator=gen)[:K]
        flat[b, cells, torch.randint(0, C, (K,), generator=gen)] = BOOST
    out, o = {}, 0
    for s in GRIDS:
        out[s] = flat[:, o:o + s * s].reshape(B, s, s, C).permute(0, 3, 1, 2).contiguous().to(DEV)
        o += s * s
    return out


def workload(B, K, seed=0):
    from boxinstseg_b200.models import build_head
    gen = torch.Generator().manual_seed(seed)
    head = osh.attach_towers(build_head(HEAD), 256, 256, C, seed=seed).to(DEV).eval()
    head.solo_cate = SeededCate(head.solo_cate, offsets(B, K, gen))
    feats = [torch.randn(B, 256, -(-HP // s), -(-WP // s), generator=gen).to(DEV) for s in (4, 8, 16, 32, 64)]
    return head, feats


def arms(head, feats, B):
    metas = [META] * B

    def dense():
        with torch.no_grad():
            return head.get_seg(*head.forward(feats, eval=True), metas, CFG)

    def cells():
        return head.simple_test(feats, metas, cfg=CFG)
    return {'dense': dense, 'cells': cells}


def same(a, b):
    return all(torch.equal(getattr(x, k), getattr(y, k)) and getattr(x, k).dtype == getattr(y, k).dtype
               for x, y in zip(a, b) for k in ('masks', 'labels', 'scores'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_solo_infer needs a CUDA device')
    res = dict(card=card(), rounds=args.rounds, cfg=CFG,
               workload='BoxSOLOv2 head test path at COCO test shape: 800x1344 padded input, feature_pred 200x336, '
                        '256-channel stand-in towers, grids 40/36/24/16/12, K confident (cell, class) pairs per image',
               dense_prediction_bytes_per_image=sum(s * s for s in GRIDS) * (HP // 4) * (WP // 4) * 4, cases={})
    for B in (1, 2):
        for K in (100, 500, 2000):
            head, feats = workload(B, K)
            fns = arms(head, feats, B)
            with torch.no_grad():
                cate = head._towers(feats, True, 'bench')[1]
            rows = [int(sum((c[b] > CFG['score_thr']).any(-1).sum() for c in cate)) for b in range(B)]
            towers = lambda: head._towers(feats, True, 'bench')                 # noqa: E731
            for _ in range(args.warmup):
                for fn in fns.values():
                    fn()
            times = {k: [] for k in fns}
            for r in range(args.rounds):                               # alternate the arms, starting side swapped each round
                for name in (list(fns) if r % 2 == 0 else list(fns)[::-1]):
                    times[name].append(time_call(fns[name])[0])
            with torch.no_grad():
                t_towers = [time_call(towers)[0] for _ in range(args.rounds)]
            rec = dict(candidate_cells_per_image=rows)
            outs = {}
            for name, fn in fns.items():
                peak, outs[name] = peak_alloc(fn)
                kern = {n: v for n, v in profile(fn).items() if 'Memcpy' not in n and 'Memset' not in n}
                rec[name] = dict(**ms_summary(times[name]), peak_alloc_bytes=peak,
                                 kernel_launches=sum(c for c, _ in kern.values()),
                                 kernel_device_ms=sum(ms for _, ms in kern.values()), host_syncs=syncs(fn),
                                 instances=[len(o.scores) for o in outs[name]])
            rec['towers'] = ms_summary(t_towers)
            rec['bit_identical'] = same(outs['cells'], outs['dense'])
            rec['speedup_median'] = rec['dense']['median_ms'] / rec['cells']['median_ms']
            rec['peak_ratio'] = rec['dense']['peak_alloc_bytes'] / rec['cells']['peak_alloc_bytes']
            res['cases'][f'B{B}_K{K}'] = rec
            print(f'B{B}_K{K}', json.dumps(rec), flush=True)
            del head, feats, fns, outs
            torch.cuda.empty_cache()
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as f:
            f.write(text)


if __name__ == '__main__':
    main()
