"""Time Box2Mask's Hungarian matching (MaskHungarianAssigner.assign step 3) for one training step: 10 decoder layers x
B = 2 images, Q = 100 queries, G ground truths per image, two ways:

  scipy   the parent's path, per problem: cost.cpu() + scipy.optimize.linear_sum_assignment + the indices back to the device;
  kernel  ops.lsap.solve_batched: one launch per layer for both images, nothing read back.

Reports the host-clock time of the whole step's matchings ending in a device synchronise (both paths), and the CUDA-event
time of the kernel path alone (back-to-back launches, no host round trip).  Both paths' matchings are checked to be equal.
Prints one line per G, with the card's name and power limit; `--out PATH` also writes everything to one JSON file.

    python tools/bench_lsap.py [--reps N] [--out PATH]
"""
import argparse
import json
import os
import sys

import torch
from scipy.optimize import linear_sum_assignment as scipy_lsa

sys.path.insert(0, '.')
from benchkit import card, host_ms, time_call  # noqa: E402
from boxinstseg_b200.core import MaskHungarianAssigner  # noqa: E402
from boxinstseg_b200.ops.lsap import solve_batched  # noqa: E402

DEV = 'cuda:0'
LAYERS, B, Q = 10, 2, 100


def costs_for(G, seed):
    """[LAYERS][B] cost matrices [Q, G] of the Box2Mask assigner config on seeded predictions (what the layers hand to step 3)."""
    gen = torch.Generator().manual_seed(seed)
    asg = MaskHungarianAssigner(cls_cost=dict(type='ClassificationCost', weight=2.0),
                                dice_cost=dict(type='BoxMatchingCost', weight=5.0, pred_act=True, eps=1.0))
    H, W = 256, 256
    out = []
    for _ in range(LAYERS):
        layer = []
        for _ in range(B):
            cls = torch.randn(Q, 81, generator=gen).to(DEV)
            masks = (torch.randn(Q, 64, 64, generator=gen) * 3).to(DEV)
            labels = torch.randint(0, 80, (G,), generator=gen).to(DEV)
            gt = torch.zeros(G, H, W)
            for g in range(G):
                y, x = (int(v) for v in torch.randint(0, H // 2, (2,), generator=gen))
                gt[g, y:y + 16 + int(torch.randint(0, 100, (1,), generator=gen)), x:x + 16 + int(torch.randint(0, 100, (1,), generator=gen))] = 1
            layer.append(asg.cost_matrix(cls, masks, labels, gt.to(DEV), lowres=True))
        out.append(layer)
    return out


def scipy_step(costs):
    res = []
    for layer in costs:
        for c in layer:
            r, k = scipy_lsa(c.detach().cpu())
            res.append((torch.from_numpy(r).to(DEV), torch.from_numpy(k).to(DEV)))
    torch.cuda.synchronize()
    return res


def kernel_step(costs):
    return [solve_batched(layer) for layer in costs]


def spread(timer, fn, reps):
    """(median, min, max) ms of `reps` calls of fn on `timer` (host_ms or time_call), after three untimed calls."""
    for _ in range(3):
        fn()
    ts = sorted(timer(fn)[0] for _ in range(reps))
    return ts[len(ts) // 2], ts[0], ts[-1]


def case(G, reps):
    costs = costs_for(G, seed=G)
    want = scipy_step(costs)
    got = [m for layer in kernel_step(costs) for m in layer[0]]
    for (r, k), m in zip(want, got):
        rows = torch.nonzero(m >= 0).squeeze(1)
        assert torch.equal(rows, r) and torch.equal(m[rows].long(), k), 'kernel and scipy disagree'
    s = spread(host_ms, lambda: scipy_step(costs), reps)
    k = spread(host_ms, lambda: kernel_step(costs), reps)
    e = spread(time_call, lambda: kernel_step(costs), reps)
    row = {'G': G, 'problems': LAYERS * B, 'scipy_host_ms': s, 'kernel_host_ms': k, 'kernel_event_ms': e}
    print(f'G={G:3d}  {LAYERS}x{B} matchings of {Q}x{G}: scipy path {s[0]:.3f} ms (min {s[1]:.3f}, max {s[2]:.3f}) | '
          f'kernel host clock {k[0]:.3f} ms (min {k[1]:.3f}, max {k[2]:.3f}) | kernel events {e[0]:.3f} ms '
          f'(min {e[1]:.3f}, max {e[2]:.3f})  [median, min, max over {reps}]', flush=True)
    return row


if __name__ == '__main__':
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', metavar='PATH', default=None, help='write all results to this JSON file')
    args = ap.parse_args()
    out = {'card': card()}
    print('card', json.dumps(out['card']), flush=True)
    out['cases'] = [case(G, args.reps) for G in (8, 50)]
    out['card_after'] = card()
    print('card_after', json.dumps(out['card_after']), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, 'w') as fh:
            json.dump(out, fh, indent=1)
