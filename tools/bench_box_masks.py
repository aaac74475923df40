"""Time the box-mask data pipeline of the box-supervised configs, two arms alternated over rounds on the same boxes:

  bitmap   the reference's GenerateBoxMask (restated in oracle/box_masks.py) then BitmapMasks' resize, flip, crop and pad
           on the dense uint8 [G, H, W] array (cv2.resize where cv2 imports, else the numpy restatement: "resize" in the
           output says which ran), then to_tensor = torch.tensor(ndarray, device='cuda');
  boxes    the same pipeline on BoxMasks, to_tensor written by the rasterize kernel.

Workloads: DiscoBox / BoxLevelSet multiscale (a 640 x 427 image rescaled into (1333, 800), flip, pad to 32) at G = 7, 20,
100; Box2Mask's large-scale jitter (1024 x 1024, ratio 0.1-2.0, RandomCrop 1024 with the kept masks, pad) at G = 20, 100.
Reports per arm the host pipeline ms and the to_tensor ms (host clock, ending in a device synchronise; median and range
over rounds), the synchronising calls of to_tensor (benchkit.syncs), and the rasterize kernel's time from a CUDA-graph
replay against G*H*W bytes at the data sheet's 3.35 TB/s.  The arms' tensors are asserted equal.  The card is read in the
same run.

    python tools/bench_box_masks.py [--rounds 15] [--out PATH]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from benchkit import card, graph_us, host_ms, summary, syncs  # noqa: E402
from boxinstseg_b200.core import BoxMasks  # noqa: E402
from boxinstseg_b200.datasets import GenerateBoxMask  # noqa: E402
from oracle import box_masks as ob  # noqa: E402

HBM = 3.35e12
DEV = 'cuda:0'


def workloads():
    rng = np.random.default_rng(0)
    out = []
    for G in (7, 20, 100):
        h, w = 427, 640
        ops = [('rescale', (1333, 800)), ('flip', 'horizontal')]
        nw, nh = ob.rescale_size((w, h), (1333, 800))
        ops.append(('pad', (-(-nh // 32) * 32, -(-nw // 32) * 32)))
        out.append((f'discobox_G{G}', ob._boxes(rng, G, h, w, special=False), h, w, ops))
    for G in (20, 100):
        h = w = 1024
        r = float(rng.uniform(1.0, 2.0))                          # an upscale: the crop keeps a full 1024 x 1024 window
        nw, nh = ob.rescale_size((w, h), (int(1024 * r), int(1024 * r)))
        oy, ox = int(rng.integers(0, nh - 1024 + 1)), int(rng.integers(0, nw - 1024 + 1))
        ops = [('flip', 'horizontal'), ('rescale', (int(1024 * r), int(1024 * r))),
               ('index', np.arange(G)), ('crop', [ox, oy, ox + 1024, oy + 1024]), ('pad', (1024, 1024))]
        out.append((f'box2mask_lsj_G{G}_r{r:.2f}', ob._boxes(rng, G, h, w, special=False), h, w, ops))
    return out


def pipeline(make, boxes, h, w, ops):
    m = make(boxes, h, w)
    for op in ops:
        m = ob.apply(m, op)
    return m


def make_boxes(boxes, h, w):
    return GenerateBoxMask()({'gt_bboxes': boxes, 'img': np.zeros((h, w, 3), np.uint8), 'mask_fields': []})['gt_masks']


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=15)
    ap.add_argument('--out', default=os.path.join(ROOT, 'tools', 'results', 'bench_box_masks_h100.json'))
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_box_masks needs a CUDA device'
    res = {'card': card(), 'resize': 'cv2.resize' if ob.cv2 is not None else 'numpy restatement', 'rounds': args.rounds,
           'hbm_bytes_per_s': HBM, 'workloads': {}}
    arms = {'bitmap': ob.generate_box_mask, 'boxes': make_boxes}
    for name, boxes, h, w, ops in workloads():
        t = {a: {'pipeline_ms': [], 'to_tensor_ms': []} for a in arms}
        outs = {}
        for rnd in range(args.rounds + 1):                       # round 0 warms up
            for a in (arms if rnd % 2 == 0 else reversed(list(arms))):
                t0 = time.perf_counter()
                m = pipeline(arms[a], boxes, h, w, ops)
                p_ms = (time.perf_counter() - t0) * 1e3
                tt_ms, out = host_ms(lambda: torch.tensor(m.to_ndarray(), device=DEV) if a == 'bitmap'
                                     else m.to_tensor(torch.uint8, DEV))
                if rnd:
                    t[a]['pipeline_ms'].append(p_ms)
                    t[a]['to_tensor_ms'].append(tt_ms)
                outs[a] = (m, out)
        (mb, ob_), (mx, ox_) = outs['bitmap'], outs['boxes']
        assert ob_.shape == ox_.shape and torch.equal(ob_, ox_), name
        G, H, W = ox_.shape
        entry = {'G': G, 'H': H, 'W': W, 'bytes': G * H * W}
        for a in arms:
            entry[a] = {k: summary(v) for k, v in t[a].items()}
        entry['bitmap']['to_tensor_syncs'] = syncs(lambda: torch.tensor(mb.to_ndarray(), device=DEV))
        entry['boxes']['to_tensor_syncs'] = syncs(lambda: mx.to_tensor(torch.uint8, DEV))
        from boxinstseg_b200.ops.box_masks import rasterize
        rects, size = [mx.rects], [(mx.height, mx.width)]
        us = graph_us(lambda: rasterize(rects, size, torch.uint8, DEV), reps=50, per_graph=10)
        entry['kernel_us_graph_replay'] = us
        if isinstance(us, float):
            entry['hbm_bound_us'] = G * H * W / HBM * 1e6
            entry['share_of_hbm_bound'] = entry['hbm_bound_us'] / us
        res['workloads'][name] = entry
        print(name, json.dumps({k: (v if not isinstance(v, dict) else {kk: vv.get('median') if isinstance(vv, dict)
                                                                        else vv for kk, vv in v.items()})
                                for k, v in entry.items()}))
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, 'w') as f:
        json.dump(res, f, indent=1)
    print('wrote', args.out)


if __name__ == '__main__':
    main()
