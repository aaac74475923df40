"""Time ``format_results`` of the SOLOv2-family detectors -- each image's get_seg output to the per-class CPU masks, scores
and float64 boxes that BoxLevelSet and DiscoBoxSOLOv2 return -- on the get_seg outputs of tools/bench_solo_seg.py's
workloads (COCO test shapes, original image 480 x 640, about 100 kept masks per image, B = 1 and 2) and one with about 20
kept masks per image (max_per_img = 20), in two arms alternated over rounds, on the same get_seg outputs:

  ref  the reference's lines (oracle/solo_format.py): per detection seg_mask.sum() > 0, .cpu() copies and a torch.where
       over the whole mask, up to 9 synchronising calls;
  new  models/detectors/solo.py format_results: one bxs_mask_extents call, two non-blocking copies to pinned memory, one
       event wait.

Reports per arm the host-clock time per image (median, min-max over rounds; every call ends in a device synchronise),
synchronising calls and event waits per image, CUDA activities (kernels, memcpys, memsets) per image, and for the new arm
the extents kernels' time from a torch.profiler run with their share of the HBM bound (n*H*W bytes read at 3.35 TB/s).
The device-to-host copy of the masks alone, into pinned and into pageable memory, is timed separately: it is the floor
neither arm goes under.  get_seg's own time is given for scale.  The card's name and power limit are read in the same run.

    python tools/bench_solo_format.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchkit import card, host_ms, profile, summary, syncs  # noqa: E402
from bench_solo_seg import C, GRIDS, META, STRIDES, box_workload, cfg, disco_workload  # noqa: E402
from oracle import solo_format as osf  # noqa: E402
from oracle.make_golden_solo_format import assert_same  # noqa: E402

HBM = 3.35e12


def get_seg_call(disco, B, max_per_img):
    from boxinstseg_b200.models import build_head
    c = dict(cfg(disco), max_per_img=max_per_img)
    metas = [META] * B
    if disco:
        feat, kern, cate = disco_workload(B)
        head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=C, num_grids=GRIDS, strides=STRIDES))
        return lambda: head.get_seg(cate, kern, feat, metas, c)
    seg, cate = box_workload(B)
    head = build_head(dict(type='BoxSOLOv2Head', num_classes=C, num_grids=GRIDS, strides=STRIDES))
    return lambda: head.get_seg(seg, cate, None, metas, c)


def event_waits(fn):
    """Event.synchronize calls in one call of fn (sync-debug mode does not flag them)."""
    n = [0]
    orig = torch.cuda.Event.synchronize

    def counted(self):
        n[0] += 1
        return orig(self)
    torch.cuda.Event.synchronize = counted
    try:
        fn()
    finally:
        torch.cuda.Event.synchronize = orig
    return n[0]


def copy_floor(outs, pinned):
    """Host-clock ms of the device-to-host copy of every image's masks, one copy per image, ending in a synchronise."""
    def run():
        for r in outs:
            if pinned:
                torch.empty(r.masks.shape, dtype=r.masks.dtype, pin_memory=True).copy_(r.masks, non_blocking=True)
            else:
                r.masks.cpu()
    return host_ms(run)[0]


def main():
    from boxinstseg_b200.models.detectors.solo import format_results
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--out')
    a = ap.parse_args()
    result = {'card': card(), 'rounds': a.rounds, 'workloads': {}}
    for disco, B, max_per_img in ((False, 1, 100), (False, 2, 100), (True, 1, 100), (True, 2, 100), (False, 1, 20)):
        name = f"{'discobox' if disco else 'boxlevelset'}_B{B}" + ('' if max_per_img == 100 else f'_max{max_per_img}')
        seg = get_seg_call(disco, B, max_per_img)
        outs = seg()
        seg_ms = statistics.median([host_ms(seg)[0] for _ in range(3)])
        fns = {'ref': lambda: [osf.format_results(r, C) for r in outs],
               'new': lambda: [format_results(r, C) for r in outs]}
        for f in fns.values():                         # warm up, and the two arms agree
            f()
        for x, y in zip(fns['ref'](), fns['new']()):
            assert_same(x, y, name)
        t = {k: [] for k in fns}
        for _ in range(a.rounds):                      # alternated rounds
            for k, f in fns.items():
                t[k].append(host_ms(f)[0] / B)
        rec = {'instances': [len(r.scores) for r in outs], 'get_seg_ms': seg_ms}
        for k, f in fns.items():
            prof = profile(f)
            rec[k] = {'per_image_ms': summary(t[k]), 'syncs_per_image': syncs(f) / B,
                      'event_waits_per_image': event_waits(f) / B,
                      'activities_per_image': sum(c for c, _ in prof.values()) / B}
            if k == 'new':
                nbytes = sum(r.masks.numel() for r in outs)
                ext = {n: v for n, v in prof.items() if 'mask_extents' in n or 'mask_stats_reduce' in n}
                ms = sum(v[1] for v in ext.values())
                rec[k]['extents_kernels'] = {n: {'count': c, 'ms': m} for n, (c, m) in ext.items()}
                rec[k]['extents_bytes'] = nbytes
                rec[k]['extents_ms'] = ms
                rec[k]['extents_hbm_bound_share'] = nbytes / HBM / (ms / 1e3) if ms else None
        rec['d2h_masks_pinned_ms_per_image'] = statistics.median([copy_floor(outs, True) for _ in range(5)]) / B
        rec['d2h_masks_pageable_ms_per_image'] = statistics.median([copy_floor(outs, False) for _ in range(5)]) / B
        rec['speedup_median'] = rec['ref']['per_image_ms']['median'] / rec['new']['per_image_ms']['median']
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
