"""Time CondInst inference -- the box head's outputs to per-image detections and per-class masks
(CondInstBoxHead.get_bboxes, then CondInstMaskHead.simple_test with rescale=True) -- at COCO test shapes: 800x1344 padded
input, img_shape 800x1067, original 480x640, levels 100x168 ... 7x11 (strides 8 .. 128), 80 classes, 233 dynamic parameters,
mask_feat [B,16,100,168] and the BoxInst configs' test_cfg (nms_pre 2000, score_thr 0.05, iou 0.5, max_per_img 2000).
Two seeded workloads (oracle/condinst_infer.py ``WORKLOADS``): about 3k candidates and 100 detections per image, and about
20k candidates and 300 detections per image; B = 1 and 2; two arms alternated over rounds:

  ref  the reference's lines (oracle/condinst_infer.py): per-level permute / sigmoid / topk / distance2bbox, per image
       nms_with_others and mmcv's batched_nms (per-class loop above 10000 candidates), then the cuDNN dynamic
       convolutions, aligned_bilinear, F.interpolate and the host split.  mmcv's CUDA ``nms`` is not installed here, so
       this arm calls torchvision.ops.nms in its place (same greedy order; it divides the IoU instead of multiplying).
  new  this library's get_bboxes and simple_test.
The ``*_get_bboxes`` arms time the box part alone.

Reports per arm the median / min / max GPU time of a call (CUDA events), kernel launches and synchronising calls per call,
the peak allocation, and for the new arm the per-kernel time (torch.profiler, a separate run) with the bytes each kernel
must move (computed below) and the share of the HBM bound that gives; the card's name and power limit are read in the
same run.  Prints one JSON document; `--out PATH` also writes it.

    python tools/bench_condinst_infer.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import warnings

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import condinst_infer as oci  # noqa: E402

HBM = 3.35e12
SOI = [64, 128, 256, 512, 1024]
KERNELS = ('ci_key_kernel', 'ci_decode_kernel', 'nms_mask_kernel', 'nms_resolve_kernel', 'ci_gather_kernel', 'ci_paste_kernel')


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q.stdout.strip().splitlines()[:1]}


def _tv_nms(boxes, scores, iou_threshold, stable=True):
    import torchvision
    keep = torchvision.ops.nms(boxes, scores, iou_threshold)
    return torch.cat((boxes[keep], scores[keep].reshape(-1, 1)), dim=1), keep


def ref_boxes(cls, bbox, ctr, prm, feat, metas):
    return oci.get_bboxes(cls, bbox, ctr, prm, metas, oci.COCO_TEST_CFG, oci.COCO_STRIDES, True, True, stable=False)


def ref_arm(cls, bbox, ctr, prm, feat, metas):
    dets = ref_boxes(cls, bbox, ctr, prm, feat, metas)
    soi = torch.tensor(SOI, device=feat.device)
    out = []
    for b, (d, labels, p, coors, lvl) in enumerate(dets):
        if len(p) == 0:
            out.append([[] for _ in range(80)])
            continue
        logits = oci.mask_head_forward(feat, p, coors, lvl, torch.full((len(p),), b, dtype=torch.long, device=feat.device), soi)
        m = oci.aligned_bilinear(logits.sigmoid(), 4)[:, :, :800, :1067]
        m = F.interpolate(m, (480, 640), mode='bilinear', align_corners=False).squeeze(1) > 0.5
        m = m.cpu().numpy().astype(np.uint8)
        lab = labels.cpu().numpy()
        out.append([m[lab == i] for i in range(80)])
    return dets, out


def new_arm(box_head, mask_head, cls, bbox, ctr, prm, feat, metas):
    dets = box_head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True)
    segm = mask_head.simple_test(feat, *[[d[i] for d in dets] for i in (1, 2, 3, 4)], metas, 80, rescale=True)
    return dets, segm


def time_call(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def count_syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as rec:
        warnings.simplefilter('always')
        torch.cuda.set_sync_debug_mode('warn')
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode('default')
    return sum('called a synchronizing' in str(r.message) for r in rec)


def profile(fn):
    from torch.profiler import ProfilerActivity, profile as prof
    with prof(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    return {e.key: (e.count, e.device_time_total / 1e3) for e in p.key_averages() if e.device_type.name == 'CUDA' and e.count}


def kernel_bytes(box_head, cls, bbox, ctr, prm, metas, dets, B):
    """Bytes each new kernel must move at least once: key reads cls and centerness and writes the padded keys; decode reads
    C + 5 floats per kept point and writes its box, centerness, point, and per class the flag and the score; the NMS mask
    reads the sorted offset boxes and writes sum_s n_s * ceil(n_s / 64) words; resolve reads them back and writes a byte
    per candidate; gather reads and writes the parameters of the detections; paste reads the logits once and writes the
    480 x 640 bool masks."""
    C, P = 80, prm[0].shape[1]
    hw = [int(c.shape[-2] * c.shape[-1]) for c in cls]
    k = [min(2000, n) for n in hw]
    S = sum(k)
    raw = box_head.get_bboxes(cls, bbox, ctr, prm, metas, rescale=True, with_nms=False)
    counts = torch.stack([(r[1][:, :-1] > 0.05).sum(0) for r in raw]).flatten().tolist()
    N = sum(counts)
    words = sum(n * -(-n // 64) for n in counts) * 8
    n_det = sum(len(d[0]) for d in dets)
    return {'ci_key_kernel': B * sum(hw) * (C + 1) * 4 + B * len(hw) * max(hw) * 4,
            'ci_decode_kernel': B * S * ((C + 5) * 4 + 16 + 4 + 8 + C * 5),
            'nms_mask_kernel': N * 16 + words, 'nms_resolve_kernel': words + N,
            'ci_gather_kernel': n_det * (2 * P * 4 + 16),
            'ci_paste_kernel': n_det * (200 * 336 * 4 + 480 * 640)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--out')
    a = ap.parse_args()
    oci.nms = _tv_nms                                  # the reference arm's NMS: torchvision's in place of mmcv's
    from boxinstseg_b200.models.dense_heads.condinst_box_head import CondInstBoxHead
    from boxinstseg_b200.models.dense_heads.condinst_mask_head import CondInstMaskHead
    box_head = CondInstBoxHead(num_classes=80, strides=oci.COCO_STRIDES, test_cfg=oci.COCO_TEST_CFG)
    mask_head = CondInstMaskHead(in_channels=16, sizes_of_interest=SOI).cuda()
    result = {'card': card(), 'rounds': a.rounds, 'workloads': {}}
    for wname, args in oci.WORKLOADS:
        for B in (1, 2):
            inputs = oci.workload(7, B, *args, device='cuda')
            fns = {'ref': lambda: ref_arm(*inputs), 'new': lambda: new_arm(box_head, mask_head, *inputs),
                   'ref_get_bboxes': lambda: (ref_boxes(*inputs), None),
                   'new_get_bboxes': lambda: (box_head.get_bboxes(*inputs[:4], inputs[5], rescale=True), None)}
            for f in fns.values():                     # warm up every shape
                f(), f()
            t = {k: [] for k in fns}
            for _ in range(a.rounds):                  # alternated rounds
                for k, f in fns.items():
                    t[k].append(time_call(f)[0])
            rec = {}
            for k, f in fns.items():
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                _, out = time_call(f)
                peak = torch.cuda.max_memory_allocated() - base
                kern = profile(f)
                rec[k] = {'median_ms': statistics.median(t[k]), 'min_ms': min(t[k]), 'max_ms': max(t[k]),
                          'launches': sum(c for c, _ in kern.values()), 'syncs': count_syncs(f), 'peak_bytes': peak,
                          'detections': [len(d[0]) for d in out[0]]}
                if k == 'new':
                    need = kernel_bytes(box_head, *inputs[:4], inputs[5], out[0], B)
                    per = {}
                    for n, (c, ms) in kern.items():
                        tag = next((t for t in KERNELS if t in n), None)
                        if tag:
                            per[tag] = {'count': c, 'ms': ms, 'bytes': need[tag],
                                        'hbm_bound_share': need[tag] / HBM / (ms / 1e3) if ms else None}
                    rec[k]['kernels'] = per
            raw = box_head.get_bboxes(*inputs[:4], inputs[5], rescale=True, with_nms=False)
            rec['new']['candidates'] = [int((r[1][:, :-1] > 0.05).sum()) for r in raw]
            rec['ratio_ref_over_new_median'] = rec['ref']['median_ms'] / rec['new']['median_ms']
            name = f'{wname}_B{B}'
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
