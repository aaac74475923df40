"""Config C's DiscoBox step (the two per-image dynamic convolutions + mask_loss, forward and backward) with a float16 and
then a bfloat16 mask-feature leaf under autocast, three ways:

  new    mask_loss on the 16-bit predictions: the DiscoBox loss kernels (ops/discobox.py);
  eager  the old per-level composition (DiscoBoxSOLOv2Head._mask_loss_level_eager) on the same 16-bit predictions;
  fp32   float32 leaf, no autocast (the float32 kernels and composition).

The arms alternate within one call.  Eager steps are timed on the host clock around a synchronise (the step is bound by
the host issuing launches), CUDA-graph replays of the same step on CUDA events; medians and min / max over the rounds.
Kernel launches per step come from a separate torch.profiler run.  Prints the card's name and power limit, read in the
same call; `--out PATH` also writes everything to one JSON file.

    python tools/bench_discobox_half.py [--rounds R] [--iters N] [--out PATH]
"""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, '.')
from benchkit import capture, card, host_ms, kernel_launches, replay_ms, summary  # noqa: E402

DEV = 'cuda:0'


def make_step(arm, dt):
    import bench_configs
    from boxinstseg_b200.models import build_head
    _, info = bench_configs.build_C(torch.device(DEV), 0)
    d = info['data']
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256))
    feat = d['feat'].detach().to(torch.float32 if arm == 'fp32' else dt).requires_grad_(True)
    kern = d['kern']
    if arm == 'eager':
        def mask_loss(preds, labels, inds, color):
            from boxinstseg_b200.models.dense_heads.meanfield import MeanField
            mf = MeanField(color, alpha0=head.alpha0, theta0=head.theta0, theta1=head.theta1, theta2=head.theta2,
                           iter=head.crf_max_iter, kernel_size=head.mkernel, base=head.crf_base)
            ni, nt, cnt = head._mask_loss_level_eager(preds[0], None, inds[0], labels[0], mf, True)
            cnt = cnt.clamp(min=1.0)
            return dict(loss_ins=ni / cnt * head.ins_loss_weight, loss_ts=nt / cnt * head.ts_loss_weight)
    else:
        mask_loss = head.mask_loss

    def step():
        with torch.autocast('cuda', dtype=dt, enabled=arm != 'fp32'):
            pred = torch.cat([head.dynamic_conv(feat[b], kern[b]) for b in range(2)])
            out = mask_loss([pred], [d['labels']], [d['img_inds']], d['color'])
        return torch.autograd.grad(out['loss_ins'] + out['loss_ts'], [feat, kern])
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', metavar='PATH', default=None)
    args = ap.parse_args()
    res = {'card': card()}
    print('card', json.dumps(res['card']), flush=True)
    for dt in (torch.float16, torch.bfloat16):
        name = str(dt).replace('torch.', '')
        arms = {arm: make_step(arm, dt) for arm in ('new', 'eager', 'fp32')}
        graphs = {arm: capture(s) for arm, s in arms.items()}
        for s in arms.values():
            for _ in range(3):
                s()
        host = {a: [] for a in arms}
        gpu = {a: [] for a in arms}
        for _ in range(args.rounds):                      # alternate the arms within the call
            for arm, s in arms.items():
                host[arm].append(statistics.median(host_ms(s)[0] for _ in range(args.iters)))
                gpu[arm].append(replay_ms(graphs[arm], args.iters))
        r = {arm: {'eager_step_ms': summary(host[arm]), 'graph_step_ms': summary(gpu[arm]),
                   'launches': kernel_launches(s)}
             for arm, s in arms.items()}
        res[name] = r
        for arm in arms:
            print(f'{name:9s} {arm:5s} eager step {r[arm]["eager_step_ms"]["median"]:.3f} ms '
                  f'[{r[arm]["eager_step_ms"]["min"]:.3f}, {r[arm]["eager_step_ms"]["max"]:.3f}]  graph replay '
                  f'{r[arm]["graph_step_ms"]["median"]:.3f} ms [{r[arm]["graph_step_ms"]["min"]:.3f}, '
                  f'{r[arm]["graph_step_ms"]["max"]:.3f}]  launches {r[arm]["launches"]}', flush=True)
        del arms, graphs
    res['card_after'] = card()
    print('card_after', json.dumps(res['card_after']), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
