"""Time SOLOv2 inference -- the head outputs to per-image masks, labels and scores -- at COCO test shapes (800x1344 padded
input, mask features h x w = 200 x 336, grids 40/36/24/16/12, 80 classes, original image 480 x 640), on seeded synthetic
blob masks that pass the stride filter and overlap, about 1000 candidates per image, in two arms alternated over rounds:

  ref  the reference's lines (oracle/solo_seg.py): per image, boolean indexing, one [h,w] row per candidate, the float32
       torch.mm intersection matrix, two full float32 F.interpolate passes;
  new  BoxSOLOv2Head.get_seg / DiscoBoxSOLOv2Head.get_seg (distinct rows once, packed masks, bxs_matrix_nms, fused paste).

BoxLevelset: score_thr 0.05, mask_thr 0.55, nms_pre 500, max_per_img 100, B = 1 and 2, float32 probabilities.  DiscoBox: the
same shapes, score_thr 0.1, mask_thr 0.4, float16 autocast, 256 mask-feature channels.  Reports per arm the median / min /
max GPU time of a call (CUDA events), kernel launches and synchronising calls per call, the peak allocation, and the
per-kernel time of the new arm (torch.profiler, a separate run) with its share of the HBM bound from the bytes computed
below; the card's name and power limit are read in the same run.  Prints one JSON document; `--out PATH` also writes it.

    python tools/bench_solo_seg.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import sys
import types

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchkit import card, ms_summary, peak_alloc, profile, syncs, time_call  # noqa: E402
from oracle import solo_seg as oss  # noqa: E402

DEV = 'cuda:0'
GRIDS, STRIDES = [40, 36, 24, 16, 12], [8, 8, 16, 32, 32]
H, W, C, E = 200, 336, 80, 256
META = dict(img_shape=(800, 1067, 3), ori_shape=(480, 640, 3), pad_shape=(800, 1344, 3))
HBM = 3.35e12


def _cate(gen, B, K):
    """[B,S,S,C] category maps with K (cell, class) scores in (0.12, 1) per image, the rest 0."""
    P = sum(s * s for s in GRIDS)
    flat = torch.zeros(B, P * C)
    for b in range(B):
        idx = torch.randperm(P * C, generator=gen)[:K]
        flat[b, idx] = 0.12 + 0.88 * torch.rand(K, generator=gen)
    flat = flat.view(B, P, C)
    out, o = [], 0
    for s in GRIDS:
        out.append(flat[:, o:o + s * s].reshape(B, s, s, C).to(DEV))
        o += s * s
    return out


def box_workload(B, K=1000, seed=0):
    gen = torch.Generator().manual_seed(seed)
    ys = torch.arange(H, device=DEV, dtype=torch.float32).view(1, H, 1)
    xs = torch.arange(W, device=DEV, dtype=torch.float32).view(1, 1, W)
    seg = []
    for s in GRIDS:
        n = B * s * s
        cy = (torch.rand(n, 1, 1, generator=gen) * H).to(DEV)
        cx = (torch.rand(n, 1, 1, generator=gen) * W).to(DEV)
        r = (12 + torch.rand(n, 1, 1, generator=gen) * 40).to(DEV)
        lvl = torch.empty(n, H, W, device=DEV)
        for c0 in range(0, n, 512):                    # blobs: p = sigmoid(r - distance to the centre)
            d = ((ys - cy[c0:c0 + 512]) ** 2 + (xs - cx[c0:c0 + 512]) ** 2).sqrt()
            lvl[c0:c0 + 512] = torch.sigmoid((r[c0:c0 + 512] - d) * 0.5)
        seg.append(lvl.view(B, s * s, H, W))
    return seg, _cate(gen, B, K)


def disco_workload(B, K=1000, seed=0):
    gen = torch.Generator().manual_seed(seed)
    feat = torch.randn(B, E, H, W, generator=gen) * 0.1
    ys = torch.linspace(-1, 1, H).view(H, 1)
    xs = torch.linspace(-1, 1, W).view(1, W)
    for k in range(0, 16):                              # radial channels: the logits of a cell are blob-shaped
        cy, cx = torch.rand(2, generator=gen) * 2 - 1
        feat[:, k] = 1 - ((ys - cy) ** 2 + (xs - cx) ** 2).sqrt() * 3
    kern = [torch.zeros(B, E, s, s) for s in GRIDS]
    for kk in kern:
        kk[:, :16] = torch.rand(B, 16, *kk.shape[-2:], generator=gen) ** 8 * 8
        kk[:, 16] = -2.0
    return feat.to(DEV), [k.to(DEV) for k in kern], _cate(gen, B, K)


def cfg(disco):
    return dict(score_thr=0.1 if disco else 0.05, mask_thr=0.4 if disco else 0.55, nms_pre=500, max_per_img=100,
                kernel='gaussian', sigma=2.0, filter_thr=0.05)


def arms(disco, B):
    from boxinstseg_b200.models import build_head
    c = cfg(disco)
    metas = [META] * B
    head = types.SimpleNamespace(cate_out_channels=C, kernel_out_channels=E, seg_num_grids=GRIDS, strides=STRIDES)
    if disco:
        feat, kern, cate = disco_workload(B)
        new_head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=C, num_grids=GRIDS, strides=STRIDES))
        ref = lambda: oss.disco_get_seg(head, cate, kern, feat, metas, oss_cfg(c))                  # noqa: E731
        new = lambda: new_head.get_seg(cate, kern, feat, metas, c)                                 # noqa: E731
    else:
        seg, cate = box_workload(B)
        new_head = build_head(dict(type='BoxSOLOv2Head', num_classes=C, num_grids=GRIDS, strides=STRIDES))
        ref = lambda: oss.box_get_seg(head, seg, cate, None, metas, oss_cfg(c))                     # noqa: E731
        new = lambda: new_head.get_seg(seg, cate, None, metas, c)                                  # noqa: E731
    return {'ref': ref, 'new': new}, cate


def oss_cfg(c):
    return types.SimpleNamespace(**c)


def hbm_bytes(cate, thr, out, disco):
    """Algorithmic HBM bytes of the new arm's kernels: the stats kernel reads every distinct candidate row once (float32
    probabilities, or float16 logits for DiscoBox) and writes its packed bits; the paste writes n x H_ori x W_ori bytes (its
    reads are the L1 / L2-resident rows, 134 or 268 KB each).  The NMS reads packed rows that stay in L2: no HBM bound."""
    rows = int(sum((c > thr).any(-1).sum() for c in cate))
    elt = 2 if disco else 4
    words = -(-H * W // 32)
    return {'solo_stats': rows * (H * W * elt + words * 4),
            'solo_paste': sum(len(r.scores) for r in out) * META['ori_shape'][0] * META['ori_shape'][1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--out')
    a = ap.parse_args()
    result = {'card': card(), 'rounds': a.rounds, 'workloads': {}}
    for disco in (False, True):
        for B in (1, 2):
            name = f"{'discobox' if disco else 'boxlevelset'}_B{B}"
            fns, cate = arms(disco, B)
            for f in fns.values():                     # warm up every shape
                f(), f()
            t = {k: [] for k in fns}
            for _ in range(a.rounds):                  # alternated rounds
                for k, f in fns.items():
                    t[k].append(time_call(f)[0])
            rec = {}
            for k, f in fns.items():
                peak, out = peak_alloc(f)
                kern = profile(f)
                rec[k] = {**ms_summary(t[k]), 'launches': sum(c for c, _ in kern.values()), 'syncs': syncs(f),
                          'peak_bytes': peak,
                          'instances': [len(r.scores) for r in out]}
                if k == 'new':
                    hbm = hbm_bytes(cate, cfg(disco)['score_thr'], out, disco)
                    per = {}
                    for n, (c, ms) in kern.items():
                        tag = next((t for t in ('solo_stats', 'nms_inter', 'nms_decay', 'solo_paste') if t in n), None)
                        if tag:
                            per[tag] = {'count': c, 'ms': ms, 'hbm_bytes': hbm.get(tag),
                                        'hbm_bound_share': hbm[tag] / HBM / (ms / 1e3) if tag in hbm and ms else None}
                    rec[k]['kernels'] = per
            rec['speedup_median'] = rec['ref']['median_ms'] / rec['new']['median_ms']
            result['workloads'][name] = rec
            print(name, json.dumps(rec), flush=True)
    doc = json.dumps(result, indent=1)
    print(doc)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(doc + '\n')


if __name__ == '__main__':
    main()
