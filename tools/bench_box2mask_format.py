"""Time Box2Mask's test-result formatting -- each image's ``ins_results`` from MaskFormerFusionHead.simple_test to the
per-class float32 boxes and numpy masks that ``MaskFormer.simple_test`` (``Box2Mask.simple_test``) returns -- on the fusion
head's outputs for tools/bench_box2mask_infer.py's COCO workloads (original 480 x 640, and 427 x 640 for the second image,
100 detections per image, B = 1 and 2) and one with max_per_image = 20, in two arms alternated over rounds, on the same
CUDA results:

  ref  the reference's lines (oracle/box2mask_format.py): bbox2result's two .cpu() copies, then per detection a host read
       of its label and a blocking, pageable .cpu() of its mask;
  new  models/detectors/box2mask.py format_instance_results: per image two non-blocking copies to pinned memory (the
       masks and a packed table of boxes and labels), one event wait for the whole call.

Reports per arm the host-clock time per image (median, min-max over rounds; every call ends in a device synchronise),
synchronising calls and event waits per image, and CUDA activities (kernels, memcpys, memsets) per image from a
torch.profiler run.  The device-to-host copy of the masks alone, into pinned and into pageable memory, is timed separately:
it is the floor neither arm goes under.  The fusion head's own time is given for scale.  The card's name and power limit
are read in the same run.

    python tools/bench_box2mask_format.py [--rounds 10] [--out PATH]
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
from bench_box2mask_infer import K, workload  # noqa: E402
from bench_solo_format import event_waits  # noqa: E402
from oracle import box2mask_format as obf  # noqa: E402


def copy_floor(ins, pinned):
    """Host-clock ms of the device-to-host copy of every image's masks, one copy per image, ending in a synchronise."""
    def run():
        for _, _, masks in ins:
            if pinned:
                torch.empty(masks.shape, dtype=masks.dtype, pin_memory=True).copy_(masks, non_blocking=True)
            else:
                masks.cpu()
    return host_ms(run)[0]


def main():
    from boxinstseg_b200.models.dense_heads.box2mask_infer import MaskFormerFusionHead
    from boxinstseg_b200.models.detectors.box2mask import format_instance_results
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--out')
    a = ap.parse_args()
    result = {'card': card(), 'rounds': a.rounds, 'workloads': {}}
    for B, max_per_image in ((1, 100), (2, 100), (1, 20)):
        name = f'coco_B{B}' + ('' if max_per_image == 100 else f'_max{max_per_image}')
        head = MaskFormerFusionHead(K, 0, test_cfg=dict(panoptic_on=False, semantic_on=False, instance_on=True,
                                                         max_per_image=max_per_image))
        mask_cls, mask_pred, metas = workload(B, seed=B)
        fusion = lambda: [r['ins_results'] for r in head.simple_test(mask_cls, mask_pred, metas, rescale=True)]  # noqa
        ins = fusion()
        fusion_ms = statistics.median([host_ms(fusion)[0] for _ in range(3)])
        fns = {'ref': lambda: obf.maskformer_simple_test_tail(ins, K),
               'new': lambda: format_instance_results(ins, K)}
        for f in fns.values():                         # warm up
            f()
        obf.assert_same(fns['new'](), fns['ref'](), name)
        t = {k: [] for k in fns}
        for _ in range(a.rounds):                      # alternated rounds
            for k, f in fns.items():
                t[k].append(host_ms(f)[0] / B)
        rec = {'detections': [len(i[0]) for i in ins], 'mask_bytes': sum(i[2].numel() for i in ins),
               'fusion_head_ms': fusion_ms}
        for k, f in fns.items():
            prof = profile(f)
            rec[k] = {'per_image_ms': summary(t[k]), 'syncs_per_image': syncs(f) / B,
                      'event_waits_per_image': event_waits(f) / B,
                      'activities_per_image': sum(c for c, _ in prof.values()) / B,
                      'activities': {n: {'count': c, 'ms': ms} for n, (c, ms) in prof.items()}}
        rec['d2h_masks_pinned_ms_per_image'] = statistics.median([copy_floor(ins, True) for _ in range(5)]) / B
        rec['d2h_masks_pageable_ms_per_image'] = statistics.median([copy_floor(ins, False) for _ in range(5)]) / B
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
