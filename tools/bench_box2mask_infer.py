"""Time Box2Mask inference -- the last decoder layer's outputs to per-image instance results (Box2MaskHead.simple_test's
upsample, then MaskFormerFusionHead.simple_test with rescale=True) -- at COCO test shapes (configs/box2mask/*_coco.py):
batch_input_shape 800x1088, img_shape 800x1067, original 480x640 (and 427x640 for the second image), mask features
200x272, 100 queries, 80 classes, max_per_image 100; B = 1 and 2; two arms alternated over rounds:

  ref  the reference's lines on CUDA: F.interpolate of all queries to batch_input_shape, then per image the crop,
       F.interpolate to ori_shape, softmax, topk(sorted=False), the gathered masks' sigmoid / threshold products and
       mask2bbox's per-detection loop (oracle/box2mask_infer.py's restatement of mmdet/core/mask/utils.py:68-89);
  new  this library's Box2MaskHead.simple_test output (the low-resolution predictions) and MaskFormerFusionHead.simple_test.

Reports per arm the median / min / max GPU time of a call (CUDA events), kernel launches and synchronising calls per call
and the peak allocation; for the new arm the per-kernel time (torch.profiler, a separate run) with the bytes each kernel
must move (computed below) and the share of the HBM bound that gives; the card's name and power limit are read in the same
run.  Prints one JSON document; `--out PATH` also writes it.

    python tools/bench_box2mask_infer.py [--rounds 20] [--out PATH]
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchkit import card, ms_summary, peak_alloc, profile, syncs, time_call  # noqa: E402
from oracle import box2mask_infer as obi  # noqa: E402

HBM = 3.35e12
Q, K, HW, PAD, IMG, ORI = 100, 80, (200, 272), (800, 1088), (800, 1067), ((480, 640), (427, 640))
KERNELS = ('maskformer_paste_kernel', 'maskformer_stats_kernel')


def workload(B, seed=0):
    g = torch.Generator().manual_seed(seed)
    mask_cls = (torch.randn(B, Q, K + 1, generator=g) * 3).cuda()
    low = torch.randn(B, Q, 25, 34, generator=g) * 4
    mask_pred = F.interpolate(low, HW, mode='bilinear', align_corners=False).cuda()
    metas = [dict(img_shape=IMG + (3,), ori_shape=ORI[b] + (3,), batch_input_shape=PAD) for b in range(B)]
    return mask_cls, mask_pred, metas


def ref_arm(mask_cls, mask_pred, metas):
    pred = F.interpolate(mask_pred, metas[0]['batch_input_shape'], mode='bilinear', align_corners=False)
    out = []
    for cls, mp, meta in zip(mask_cls, pred, metas):
        mp = mp[:, :meta['img_shape'][0], :meta['img_shape'][1]]
        mp = F.interpolate(mp[:, None], meta['ori_shape'][:2], mode='bilinear', align_corners=False)[:, 0]
        scores = F.softmax(cls, dim=-1)[:, :-1]
        labels = torch.arange(K, device=cls.device).unsqueeze(0).repeat(Q, 1).flatten(0, 1)
        s, top = scores.flatten(0, 1).topk(100, sorted=False)
        labels = labels[top]
        mp = mp[top // K]
        is_thing = labels < K
        s, labels, mp = s[is_thing], labels[is_thing], mp[is_thing]
        binary = (mp > 0).float()
        det = s * ((mp.sigmoid() * binary).flatten(1).sum(1) / (binary.flatten(1).sum(1) + 1e-6))
        binary = binary.bool()
        out.append((labels, torch.cat([obi.mask2bbox(binary), det[:, None]], -1), binary))
    return out


def kernel_bytes(B):
    """Bytes each new kernel must move at least once: the paste reads each chosen query's 200x272 float32 logits and
    writes its 480x640 (427x640) bool mask and 64 partial statistics of 32 bytes; the statistics kernel reads the partials
    and writes 24 bytes per mask."""
    n, out_px = 100 * B, 100 * sum(ORI[b][0] * ORI[b][1] for b in range(B))
    return {'maskformer_paste_kernel': n * HW[0] * HW[1] * 4 + out_px + n * 64 * 32,
            'maskformer_stats_kernel': n * 64 * 32 + n * 24}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=20)
    ap.add_argument('--out')
    a = ap.parse_args()
    from boxinstseg_b200.models.dense_heads.box2mask_infer import MaskFormerFusionHead
    head = MaskFormerFusionHead(K, 0, test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True,
                                                     max_per_image=100))
    result = {'card': card(), 'rounds': a.rounds, 'workloads': {}}
    for B in (1, 2):
        mask_cls, mask_pred, metas = workload(B, seed=B)
        fns = {'ref': lambda: ref_arm(mask_cls, mask_pred, metas),
               'new': lambda: [r['ins_results'] for r in head.simple_test(mask_cls, mask_pred, metas, rescale=True)]}
        for f in fns.values():                         # warm up every shape
            f(), f()
        t = {k: [] for k in fns}
        for _ in range(a.rounds):                      # alternated rounds
            for k, f in fns.items():
                t[k].append(time_call(f)[0])
        rec = {}
        for k, f in fns.items():
            peak, out = peak_alloc(f)
            kern = profile(f)
            rec[k] = {**ms_summary(t[k]), 'launches': sum(c for c, _ in kern.values()), 'syncs': syncs(f),
                      'peak_bytes': peak,
                      'detections': [len(o[0]) for o in out]}
            if k == 'new':
                need = kernel_bytes(B)
                per = {}
                for n, (c, ms) in kern.items():
                    tag = next((t for t in KERNELS if t in n), None)
                    if tag:
                        per[tag] = {'count': c, 'ms': ms, 'bytes': need[tag],
                                    'hbm_bound_share': need[tag] / HBM / (ms / 1e3) if ms else None}
                rec[k]['kernels'] = per
        rec['ratio_ref_over_new_median'] = rec['ref']['median_ms'] / rec['new']['median_ms']
        name = f'coco_B{B}'
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
