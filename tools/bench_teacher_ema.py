"""Time DiscoBox's independent-teacher update -- ``SingleStageWSInsTeacherDetector.momentum_update``
(mmdet/models/detectors/single_stage_ts.py:118-131), once per training step after the teacher turns on -- on R-50 and
R-101 DiscoBox-shaped teacher / student states (torchvision ResNet without fc, FPN, SOLOv2 head and mask-feature head of
configs/discobox), in two arms alternated over rounds on the same CUDA tensors:

  ref  the reference's lines: two state_dict() walks, `cur * (1. - m) + self * m` per entry, load_state_dict;
  new  models/detectors/discobox.py momentum_update: the cached pairing and one bxs_momentum_update launch.

Per arm: host-clock ms per call (ends in a device synchronise), device µs of one call replayed from a CUDA graph, kernel
launches, synchronising calls, the peak allocation a call adds; for the new arm the kernel's share of its HBM bound
(teacher read + student read + teacher write, computed from the shapes, at 3.35 TB/s).

Then forward_train's glue alone, on a stand-in detector whose backbone, heads and loss are stubs (the loss is a fixed
tensor), with the R-50 state as the teacher and student: the reference's lines (reference momentum_update, `float(loss)`
every step) against discobox.forward_train, per step host ms, synchronising calls and event waits.  The card's name, power
limit and maximum SM clock are read in the same run.

    python tools/bench_teacher_ema.py [--rounds 10] [--out PATH]
"""
import argparse
import copy
import json
import os
import sys
import time
import types

import torch
from torch import nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from benchkit import card, graph_us, host_ms, kernel_launches, peak_alloc, summary, syncs  # noqa: E402

HBM = 3.35e12


def discobox_model(depth):
    """A DiscoBox-shaped detector state: torchvision ResNet-``depth`` without fc, FPN (256 channels), the SOLOv2 head
    (4 stacked 3x3 convs of 512 channels with GroupNorm for the kernel branch -- its first conv sees 2 coordinate channels
    -- and for the category branch, a 256-channel kernel output, 80 classes) and the mask-feature head (128 channels, 256
    out), as configs/discobox/*.py build them."""
    import torchvision
    from torchvision.ops import FeaturePyramidNetwork
    m = nn.Module()
    r = getattr(torchvision.models, f'resnet{depth}')()
    del r.fc
    m.backbone = r
    m.neck = FeaturePyramidNetwork([256, 512, 1024, 2048], 256)

    def stack(cin):
        return nn.Sequential(*[nn.Sequential(nn.Conv2d(cin if i == 0 else 512, 512, 3, padding=1, bias=False),
                                             nn.GroupNorm(32, 512)) for i in range(4)])
    m.bbox_head = nn.Module()
    m.bbox_head.kernel_convs = stack(258)
    m.bbox_head.cate_convs = stack(256)
    m.bbox_head.solo_kernel = nn.Conv2d(512, 256, 3, padding=1)
    m.bbox_head.solo_cate = nn.Conv2d(512, 80, 3, padding=1)
    m.mask_feat_head = nn.Module()
    m.mask_feat_head.convs = nn.ModuleList([nn.Sequential(nn.Conv2d(256 + (2 if i == 3 else 0), 128, 3, padding=1,
                                                                    bias=False), nn.GroupNorm(32, 128)) for i in range(4)])
    m.mask_feat_head.conv_pred = nn.Sequential(nn.Conv2d(128, 256, 1, bias=False), nn.GroupNorm(32, 256))
    return m


def ref_momentum_update(teacher, cur_model, m):
    """single_stage_ts.py:118-131, the reference's lines."""
    from collections import OrderedDict
    cur, mine = cur_model.state_dict(), teacher.state_dict()
    fed = OrderedDict()
    for key in cur:
        fed[key] = cur[key] * (1. - m) + mine[key] * m
    teacher.load_state_dict(fed)


def event_waits(fn):
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


def update_arms(depth, rounds):
    from boxinstseg_b200.models.detectors import momentum_update
    torch.manual_seed(depth)
    student = discobox_model(depth).cuda()
    teacher = copy.deepcopy(student)
    sd = teacher.state_dict()
    entries, elems = len(sd), sum(v.numel() for v in sd.values())
    nbytes = 3 * sum(v.numel() * v.element_size() for v in sd.values())
    arms = {'ref': lambda: ref_momentum_update(teacher, student, 0.999),
            'new': lambda: momentum_update(teacher, student, 0.999)}
    for fn in arms.values():
        fn()
        fn()
    host = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            host[k].append(host_ms(fn)[0])
    out = {'state_dict_entries': entries, 'elements': elems, 'hbm_bytes': nbytes, 'hbm_bound_us': nbytes / HBM * 1e6}
    for k, fn in arms.items():
        dev = [graph_us(fn, reps=20) for _ in range(3)]
        out[k] = {'host_ms': summary(host[k]),
                  'device_us_graph': summary(dev) if all(isinstance(d, float) for d in dev) else dev[0],
                  'kernel_launches': kernel_launches(fn), 'syncs': syncs(fn), 'peak_alloc_bytes': peak_alloc(fn)[0]}
    d = out['new']['device_us_graph']
    if isinstance(d, dict):
        out['new']['share_of_hbm_bound'] = out['hbm_bound_us'] / d['median']
    return out


class _Stub:
    start_level, end_level = 0, 3

    def __init__(self, x, loss):
        self.x, self._loss = x, loss

    def __call__(self, feats):
        return feats, feats

    def loss(self, *a, **kw):
        return {'loss_ins': self._loss * 1.0}


def _ref_forward_train(self, img, img_metas, gt_bboxes, gt_labels, gt_bboxes_ignore=None, gt_masks=None):
    """single_stage_ts.py:179-237's glue on the stubs: reference momentum_update and the float() of loss_ins."""
    if self.turn_on_teacher and self.use_ind_teacher:
        ref_momentum_update(self.tsw.teacher, self, self.tsw.teacher.teacher_momentum)
    x = self.extract_feat(img)
    outs = self.bbox_head(x)
    losses = self.bbox_head.loss(*outs, use_loss_ts=self.ref_avg < 0.3, use_corr=self.ref_avg < 0.2 and self.use_corr)
    self.ref_avg = self.ref_avg * 0.9 + 0.1 * float(losses['loss_ins'])
    self.cnt += 1
    return losses


def glue_arms(rounds, steps=20):
    from boxinstseg_b200.models.detectors import DiscoBoxSOLOv2
    torch.manual_seed(0)
    x = [torch.zeros(2, 256, 8, 8, device='cuda')] * 5
    loss = torch.tensor(0.25, device='cuda')

    def make(cls):
        det = cls()
        det.add_module('state', discobox_model(50).cuda())
        teacher = nn.Module()
        teacher.add_module('state', copy.deepcopy(det.state))
        teacher.teacher_momentum = 0.999
        det.tsw = types.SimpleNamespace(teacher=teacher)
        det.bbox_head = det.mask_feat_head = _Stub(x, loss)
        det.extract_feat = teacher.extract_feat = lambda img: x
        teacher.bbox_head = teacher.mask_feat_head = det.bbox_head
        det.use_ind_teacher, det.use_corr, det.train_cfg = True, True, None
        det.cnt, det.turn_on_teacher, det.avg_loss_ins = 20000, True, 0.25
        det.ref_avg = 0.25
        return det

    class New(DiscoBoxSOLOv2, nn.Module):
        pass
    new = make(New)
    ref = make(nn.Module)
    img = torch.zeros(2, 3, 64, 64, device='cuda')
    args = (img, [{}] * 2, [], [])
    arms = {'ref': lambda: [_ref_forward_train(ref, *args) for _ in range(steps)],
            'new': lambda: [new.forward_train(*args) for _ in range(steps)]}
    for fn in arms.values():
        fn()
    host = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            host[k].append((time.perf_counter() - t0) * 1e3 / steps)
    out = {'steps_per_sample': steps}
    for k, fn in arms.items():
        out[k] = {'host_ms_per_step': summary(host[k]), 'syncs_per_step': syncs(fn) / steps,
                  'event_waits_per_step': event_waits(fn) / steps}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=10)
    ap.add_argument('--out', default=os.path.join(ROOT, 'tools', 'results', 'bench_teacher_ema_h100.json'))
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'needs a GPU'
    res = {'card': card(), 'rounds': a.rounds,
           'momentum_update': {f'R-{d}': update_arms(d, a.rounds) for d in (50, 101)},
           'forward_train_glue_R-50': glue_arms(a.rounds)}
    text = json.dumps(res, indent=1)
    print(text)
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, 'w') as f:
        f.write(text)


if __name__ == '__main__':
    main()
