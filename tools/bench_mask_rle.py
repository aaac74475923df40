"""Time the COCO RLE encoding of mask results (``encode_mask_results``, mmdet/core/mask/utils.py:38-65) on the get_seg
outputs of tools/bench_solo_seg.py's BoxSOLOv2 workload (COCO test shapes, original image 480 x 640, about 100 kept masks
per image, B = 1 and 2), one with about 20 kept masks per image (max_per_img = 20), and one adversarial workload of 100
noise masks of 480 x 640 (a run every other pixel), in up to four arms alternated over rounds on the same masks:

  ref         the reference's lines on pycocotools' mask.encode, one call per mask on the host; run only where
              pycocotools can be imported (its version, or "absent", is recorded);
  oracle      the same lines on oracle/mask_rle.py, the numpy restatement: a parity check, not the reference;
  new_host    core.mask.encode_mask_results on format_results' host masks (views of one pinned buffer per image): pack into
              one pinned staging buffer, one upload, the RLE kernels, two host waits;
  new_device  ops.mask_rle.encode on the device masks get_seg returns.

Reports per arm the host-clock time per image (median, min-max over rounds; every call ends in a device synchronise), the
synchronising calls and event waits per image, and the CUDA activities per image; for new_host the split into pack (host
clock), upload, kernels and download (torch.profiler); and the RLE kernels' time from a torch.profiler run with their share
of the HBM bound (n*H*W bytes per pass over the masks, two passes, at 3.35 TB/s).  The arms' outputs are asserted equal at every timed
size.  The card's name and power limit are read in the same run.

    python tools/bench_mask_rle.py [--rounds 10] [--out PATH]
"""
import argparse
import json
import os
import statistics
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchkit import card, host_ms, profile, summary, syncs  # noqa: E402
from bench_solo_format import event_waits, get_seg_call  # noqa: E402
from oracle import mask_rle as omr  # noqa: E402

HBM = 3.35e12
MASK_PASSES = 2                  # the boundary kernel reads every mask twice: to count the runs, then to write them
RLE_KERNELS = ('rle_boundary', 'rle_segment_scan', 'rle_offsets_scan', 'rle_tile_chars', 'rle_emit')


def pycocotools_mask():
    try:
        import pycocotools
        import pycocotools.mask as mask_util
    except ImportError:
        return None, 'absent'
    return mask_util, getattr(pycocotools, '__version__', 'unknown')


def reference_lines(mask_util):
    """encode_mask_results's loop (utils.py:54-60) with ``mask_util`` bound: per mask a Fortran copy and one encode."""
    def encode(cls_segms):
        out = [[] for _ in range(len(cls_segms))]
        for i in range(len(cls_segms)):
            for cls_segm in cls_segms[i]:
                out[i].append(mask_util.encode(np.array(cls_segm[:, :, np.newaxis], order='F', dtype='uint8'))[0])
        return out
    return encode


def host_images(outs, num_classes):
    """Per image the per-class host masks of format_results (views of one pinned buffer)."""
    from boxinstseg_b200.models.detectors.solo import format_results
    return [format_results(r, num_classes)[1][0] for r in outs]


def noise_image(n=100, H=480, W=640, seed=0):
    """A get_seg-like result of n noise masks with a run every other pixel on average, its labels spread over 80 classes."""
    g = torch.Generator(device='cuda').manual_seed(seed)
    masks = torch.rand(n, H, W, generator=g, device='cuda') < 0.5
    labels = torch.arange(n, device='cuda') % 80
    scores = torch.linspace(1, 0.1, n, device='cuda')
    return types.SimpleNamespace(labels=labels, scores=scores, masks=masks)


def rle_split(prof):
    """(kernels {name: (count, ms)}, upload ms, download ms) of a torch.profiler table."""
    kern = {n: v for n, v in prof.items() if any(k in n for k in RLE_KERNELS)}
    up = sum(v[1] for n, v in prof.items() if 'HtoD' in n)
    down = sum(v[1] for n, v in prof.items() if 'DtoH' in n)
    return kern, up, down


def main():
    from boxinstseg_b200.core import encode_mask_results
    from boxinstseg_b200.core.mask import stage
    from boxinstseg_b200.ops import mask_rle
    from bench_solo_seg import C
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--out')
    a = ap.parse_args()
    mask_util, version = pycocotools_mask()
    result = {'card': card(), 'rounds': a.rounds, 'pycocotools': version, 'workloads': {}}
    workloads = [('boxsolov2_B1', 1, 100), ('boxsolov2_B2', 2, 100), ('boxsolov2_B1_max20', 1, 20), ('noise_B1', 1, 0)]
    for name, B, max_per_img in workloads:
        outs = [noise_image()] if max_per_img == 0 else get_seg_call(False, B, max_per_img)()
        images = host_images(outs, C)
        fns = {'oracle': lambda: [reference_lines(omr)(im) for im in images],
               'new_host': lambda: [encode_mask_results(im) for im in images],
               'new_device': lambda: [mask_rle.encode(r.masks) for r in outs]}
        if mask_util is not None:
            fns = {'ref': lambda: [reference_lines(mask_util)(im) for im in images], **fns}
        for f in fns.values():                                  # warm up
            f()
        want = fns['oracle']()                                  # the arms agree
        want_device = [omr.encode(np.asfortranarray(r.masks.cpu().numpy().astype(np.uint8).transpose(1, 2, 0)))
                       for r in outs]
        for k, f in fns.items():
            assert f() == (want_device if k == 'new_device' else want), (name, k)
        t = {k: [] for k in fns}
        for _ in range(a.rounds if max_per_img else min(a.rounds, 3)):   # alternated rounds; the noise arms are slow
            for k, f in fns.items():
                t[k].append(host_ms(f)[0] / B)
        nbytes = sum(r.masks.numel() for r in outs)
        counts = [mask_rle.rle_counts(r.masks)[0].numel() for r in outs]
        rec = {'instances': [len(r.scores) for r in outs], 'runs': counts, 'mask_bytes': nbytes,
               'string_bytes': sum(len(x['counts']) for im in want for per in im for x in per)}
        for k, f in fns.items():
            prof = profile(f)
            rec[k] = {'per_image_ms': summary(t[k]), 'syncs_per_image': syncs(f) / B,
                      'event_waits_per_image': event_waits(f) / B,
                      'activities_per_image': sum(c for c, _ in prof.values()) / B}
            if k.startswith('new'):
                kern, up, down = rle_split(prof)
                ms = sum(v[1] for v in kern.values())
                rec[k]['rle_kernels'] = {n: {'count': c, 'ms': m} for n, (c, m) in kern.items()}
                rec[k]['rle_kernels_ms_per_image'] = ms / B
                rec[k]['rle_kernels_hbm_bound_share'] = MASK_PASSES * nbytes / HBM / (ms / 1e3) if ms else None
                rec[k]['upload_ms_per_image'] = up / B
                rec[k]['download_ms_per_image'] = down / B
            if k == 'new_host':
                ms_list = [[m for per in im for m in per] for im in images]
                rec[k]['pack_ms_per_image'] = statistics.median(
                    [host_ms(lambda: [stage(m) for m in ms_list])[0] for _ in range(5)]) / B
        if 'ref' in fns:
            rec['speedup_median_new_host'] = rec['ref']['per_image_ms']['median'] / rec['new_host']['per_image_ms']['median']
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
