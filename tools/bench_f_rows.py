"""Timings of the f2 / f4 rows on the GPU box next to the reference's own composition (its eager torch code restated in oracle/,
run on the same CUDA tensors -- the reference has no other GPU path for these rows): FCOS point assignment (config A: 2 x 800 x
1024, 8 ground truths per image), DiscoBox SOLO targets (host loops in the reference), SemanticCorrSolver.solve (K = 5, 7 x 7,
10 rounds) and the corr_loss transfer (28 x 28 masks).  `_us` = CUDA events around the eager call (launch overhead included);
`_graph_us` = device time of a CUDA-graph replay.  Prints one JSON object.      python tools/bench_f_rows.py"""
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from benchkit import graph_us, host_ms, time_call  # noqa: E402

dev = torch.device('cuda:0')


def row(ours, ref, ref_graph=True, **extra):
    """Eager and graph-replay µs of this package's call and of the reference's composition, then `extra`."""
    r = dict(us=time_call(ours, reps=20, warmup=3)[0] * 1e3, graph_us=graph_us(ours, 20, per_graph=4),
             reference_eager_us=time_call(ref, reps=5, warmup=3)[0] * 1e3)
    if ref_graph:
        r['reference_graph_us'] = graph_us(ref, 5)
    return dict(r, **extra)


res = {}

# ---- f2: FCOS point assignment, config A ---------------------------------------------------------------------------------
from boxinstseg_b200.models import build_head  # noqa: E402
from oracle import fcos_targets as oft  # noqa: E402
from oracle.make_golden_fcos import CFG, case  # noqa: E402

points, boxes, labels, flags = case(21, B=2, H=800, W=1024, G=(8, 8))
pts, bx, lb = [p.to(dev) for p in points], [b.to(dev) for b in boxes], [l.to(dev) for l in labels]
head = build_head(dict(type='CondInstBoxHead', num_classes=80, in_channels=256, regress_ranges=CFG['regress_ranges'],
                       strides=CFG['strides']))
ours = lambda: head.get_targets(pts, bx, lb)
ref = lambda: oft.get_targets(pts, [b.clone() for b in bx], [l.clone() for l in lb], CFG['regress_ranges'], CFG['strides'], 80)
res['fcos_targets_A'] = row(ours, ref, ref_graph=False, locations=2 * 17064, out_mb=2 * 17064 * 32 / 1e6)

# ---- f2: DiscoBox SOLO targets (the reference: host loops + cv2 per ground truth) ---------------------------------------
from boxinstseg_b200.models.dense_heads.disco_targets import disco_target_single  # noqa: E402
from oracle import solo_targets as ost  # noqa: E402
from oracle.make_golden_disco import CFG as DCFG, case as dcase  # noqa: E402

dbox, dlab, dmask, fsize = dcase(3, H=800, W=1024, G=12)
big = dict(DCFG, scale_ranges=((1, 96), (48, 192), (96, 384), (192, 768), (384, 2048)))
dm = torch.from_numpy(dmask).to(dev)
db, dl = dbox.to(dev), dlab.to(dev)
for best in (False, True):
    ours = lambda: disco_target_single(db, dl, dm, fsize, best=best, **big)
    t0 = time.perf_counter()
    for _ in range(2):
        ost.disco_target_single(dbox, dlab, dmask, fsize, best=best, **big)
    host = (time.perf_counter() - t0) / 2 * 1e6
    ours()
    wall_us = host_ms(lambda: [ours() for _ in range(5)])[0] * 1e3 / 5
    res['disco_targets_best' if best else 'disco_targets'] = dict(wall_us=wall_us, reference_host_loop_us=host, gts=12,
                                                                  mask='800x1024')

# ---- f4: SemanticCorrSolver.solve + transfer -------------------------------------------------------------------------------
from boxinstseg_b200.models.dense_heads.disco_corr import SemanticCorrSolver  # noqa: E402
from oracle import corr as oc  # noqa: E402
from oracle.make_golden_corr import FEAT, SOLVER, case as ccase  # noqa: E402

f0, f1, m0, m1 = [t.to(dev) for t in ccase(0, C=128)]
s = SemanticCorrSolver(**SOLVER)
Cu = s.cosine_table(f0, f1).contiguous()
win = oc.window_mask(FEAT, FEAT, SOLVER['dist_kernel']).to(dev)
oc_window = oc.window_mask
oc.window_mask = lambda h, w, dk: win                      # the reference builds it on the device once per call; keep it resident
ours = lambda: s.votes(Cu, FEAT, FEAT)
ref = lambda: oc.solve_votes(Cu, FEAT, FEAT, SOLVER['dist_kernel'], SOLVER['num_iter'], SOLVER['num_smooth_iter'])
T = ours()
res['corr_solve_K5_7x7_10it'] = row(ours, ref, max_abs_diff=float((T - ref()).abs().max()))
ours = lambda: s.transfer(T, Cu, m0, m1, FEAT, FEAT)
ref = lambda: oc.transfer(T, Cu, m0, m1, FEAT, FEAT)
fg, bg = ours()
_, rfg, rbg = ref()
res['corr_transfer_K5_28x28'] = row(ours, ref, reference_intermediates_mb=6 * 5 * 784 * 784 * 4 / 1e6,
                                     max_abs_diff=float(max((fg - rfg).abs().max(), (bg - rbg).abs().max())))
oc.window_mask = oc_window
print(json.dumps({k: {kk: (round(vv, 2) if isinstance(vv, float) else vv) for kk, vv in v.items()} for k, v in res.items()}, indent=1))
