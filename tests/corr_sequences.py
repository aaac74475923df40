"""TEST INFRASTRUCTURE: seeded object sequences for the batched correspondence path (``corr_level`` / ``bxs_corr_retrieve``)
and a sequential replay of the oracle's retrieval (oracle/corr.py ``Queues.similar`` / ``append``) that records, per query,
the retrieved slots and how far every retrieval test value lies from its threshold (float64).

The sequences cover: a bank with never-written (all-zero) slots and a slot with a zero box, a class created mid-level, more
appends of one class in a level than slots before the ring wraps (and than slots at all: the last writer wins), objects with
an all-zero target mixed in, degenerate boxes, objects that fail the IoU tests or the ratio test, and the head's first query
(re-normalised feature)."""
import copy

import torch
import torch.nn.functional as F

from oracle import corr as oc
from oracle.make_golden_corr import CH, FEAT, MASK, blob

BANK = dict(len_queue=6, fg_iou_thresh=0.7, bg_iou_thresh=0.7, ratio_range=[0.9, 1.2], appear_thresh=0.7, max_retrieval_objs=5)
NUM_CLASS = 4
MIN_SIZE = 8

# per level: (class, variant) of each object; variant 'ok' similar to its class, 'shape' another mask (fails the IoU tests),
# 'ratio' another aspect ratio, 'tiny' a degenerate 3 x 3 box (never appended), 'flat' a zero-height box, 'empty' an
# all-zero target (takes no part)
LEVELS = (
    [(1, 'ok'), (1, 'ok'), (0, 'ok'), (1, 'shape'), (0, 'empty'), (1, 'ok'), (1, 'tiny'), (2, 'ok'), (3, 'ok'), (1, 'ok'),
     (0, 'ok'), (1, 'ratio'), (1, 'ok')],
    [(1, 'ok'), (1, 'ok'), (1, 'empty'), (1, 'ok'), (1, 'ok'), (1, 'ok'), (1, 'ok'), (2, 'ok'), (1, 'ok'), (1, 'flat'),
     (1, 'ok'), (0, 'ok'), (0, 'ok'), (0, 'ok'), (0, 'ok')],
    [(0, 'ok'), (1, 'ok'), (2, 'ok'), (1, 'ok'), (0, 'empty'), (1, 'shape'), (0, 'ok'), (1, 'ok')],
)


def _proto(gen, C):
    return [torch.randn(1, C, FEAT, FEAT, generator=gen) for _ in range(NUM_CLASS)]


def _objects(gen, protos, spec, C):
    """RoI tensors of one level: s_feat, t_feat [n,C,7,7], s_mask, t_mask [n,28,28], boxes [n,4] (integer valued), labels [n],
    valid [n] bool."""
    n = len(spec)
    labels = torch.tensor([c for c, _ in spec])
    valid = torch.tensor([v != 'empty' for _, v in spec])
    base = torch.cat([protos[c] for c, _ in spec])
    s_feat = oc.relu_and_l2_norm_feat(base + 0.25 * torch.randn(n, C, FEAT, FEAT, generator=gen))
    t_feat = oc.relu_and_l2_norm_feat(base + 0.25 * torch.randn(n, C, FEAT, FEAT, generator=gen))
    s_mask = blob(gen, n, MASK, MASK / 2, MASK / 2, MASK * 0.36, MASK * 0.3)
    t_mask = blob(gen, n, MASK, MASK / 2, MASK / 2, MASK * 0.36, MASK * 0.3)
    xy = torch.randint(0, 12, (n, 2), generator=gen).float()
    wh = torch.stack([40 + torch.randint(0, 2, (n,), generator=gen), 40 + torch.randint(0, 2, (n,), generator=gen)], 1).float()
    for i, (_, v) in enumerate(spec):
        if v == 'shape':
            s_mask[i] = t_mask[i] = blob(gen, 1, MASK, 6.0, 6.0, 4.0, 4.0)[0]
        elif v == 'ratio':
            wh[i, 1] = 2 * wh[i, 0]
        elif v == 'tiny':
            wh[i] = 3.0
        elif v == 'flat':
            wh[i, 1] = 0.0
    boxes = torch.cat([xy, xy + wh], 1)
    return s_feat, t_feat, s_mask, t_mask, boxes, labels, valid


def initial_bank(gen, protos, C):
    """The oracle's bank before the sequence: class 1 with 4 of 6 slots written (two all-zero slots, one written slot with a
    zero box), class 2 full and wrapped (ptr 2); classes 0 and 3 without a bank."""
    orc = oc.Queues(num_class=NUM_CLASS, **BANK)
    for c, count in ((1, 4), (2, 8)):
        spec = [(c, 'ok')] * count
        _, t_feat, _, t_mask, boxes, _, _ = _objects(gen, protos, spec, C)
        if c == 1:
            boxes[2] = 0.0
        for i in range(count):
            orc.append(c, i, t_feat, t_mask, boxes)
    return orc


def sequence(seed, C=CH, ind_teacher=True):
    """(initial oracle bank, [per-level RoI tensors]) of seed; without ind_teacher the teacher mask is the student's (what
    DiscoCorr.levels passes when use_ind_teacher is False)."""
    gen = torch.Generator().manual_seed(500 + seed)
    protos = _proto(gen, C)
    orc = initial_bank(gen, protos, C)
    levels = []
    for spec in LEVELS:
        s_feat, t_feat, s_mask, t_mask, boxes, labels, valid = _objects(gen, protos, spec, C)
        if not ind_teacher:
            t_mask = s_mask.clone()
        levels.append((s_feat, t_feat, s_mask, t_mask, boxes, labels, valid))
    return orc, levels


def _values64(bank, q_mask, q_feat, q_box):
    """The four retrieval test values of get_similar_obj (:174-221) in float64, for every slot of a bank."""
    A, B = q_mask.double(), bank.mask.double()
    fg = (A * B).sum([1, 2]) / ((A + B) >= 1).double().sum([1, 2])
    bg = ((1 - A) * (1 - B)).sum([1, 2]) / ((2 - A - B) >= 1).double().sum([1, 2])
    fs = q_feat.shape[2:]
    a = F.interpolate(A[:, None], fs, mode='bilinear', align_corners=False)[:, 0]
    b = F.interpolate(B[:, None], fs, mode='bilinear', align_corners=False)[:, 0]
    app = (q_feat.double() * bank.feature.double() * a[:, None] * b[:, None]).sum([1, 2, 3]) / ((a * b).sum([1, 2]) + 1e-6)
    ratio = lambda x: (x[:, 2] - x[:, 0]) / (x[:, 3] - x[:, 1] + 1e-5)
    rr = ratio(q_box.double())[:, None] / ratio(bank.box.double())[None, :]
    return fg, bg, app, rr[0]


def replay(orc, first, s_feat, t_feat, s_mask, t_mask, boxes, labels, valid, min_size=MIN_SIZE):
    """The retrieval and append steps of the per-object loop (oracle.corr.corr_objects :1056-1125) on ``orc`` (mutated).
    Returns (per query: None (not valid / no bank) or the retrieved slots as a list, per query the append slot or -1,
    the smallest distance of any finite test value to its threshold, number of passing and of failing slot tests, first)."""
    slots, appends, margin, passing, failing = [], [], float('inf'), 0, 0
    for i in range(s_feat.shape[0]):
        if not bool(valid[i]):
            slots.append(None)
            appends.append(-1)
            continue
        c = int(labels[i])
        qf = s_feat[i:i + 1]
        if first:
            qf, first = oc.relu_and_l2_norm_feat(qf), False
        idx = orc.similar(c, s_mask[i:i + 1], qf, boxes[i:i + 1])
        slots.append(None if idx is None else [int(v) for v in idx])
        if idx is not None:
            fg, bg, app, rr = _values64(orc.banks[c], s_mask[i:i + 1], qf, boxes[i:i + 1])
            for v, t in ((fg, BANK['fg_iou_thresh']), (bg, BANK['bg_iou_thresh']), (app, BANK['appear_thresh']),
                         (rr, BANK['ratio_range'][0]), (rr, BANK['ratio_range'][1])):
                fin = torch.isfinite(v)
                if fin.any():
                    margin = min(margin, float((v[fin] - t).abs().min()))
            ok = ((fg > BANK['fg_iou_thresh']) & (bg > BANK['bg_iou_thresh']) & (app > BANK['appear_thresh']) &
                  (rr >= BANK['ratio_range'][0]) & (rr <= BANK['ratio_range'][1]))
            passing += int(ok.sum())
            failing += int((~ok).sum())
        x1, y1, x2, y2 = [int(v) for v in boxes[i]]
        if (x2 - x1) > min_size and (y2 - y1) > min_size:
            appends.append(0 if orc.banks[c] is None else orc.banks[c].ptr)
            orc.append(c, i, t_feat, t_mask, boxes)
        else:
            appends.append(-1)
    return slots, appends, margin, passing, failing, first


def packed(orc, C=CH):
    """The oracle bank as the product's packed store: feature [num_class*L, C,7,7], mask, box, ptr, exists (CPU)."""
    L = BANK['len_queue']
    feat = torch.zeros(NUM_CLASS * L, C, FEAT, FEAT)
    mask = torch.zeros(NUM_CLASS * L, MASK, MASK)
    box = torch.zeros(NUM_CLASS * L, 4)
    ptr = torch.zeros(NUM_CLASS, dtype=torch.int32)
    exists = torch.zeros(NUM_CLASS, dtype=torch.int32)
    for c, b in enumerate(orc.banks):
        if b is not None:
            feat[c * L:(c + 1) * L], mask[c * L:(c + 1) * L], box[c * L:(c + 1) * L] = b.feature, b.mask, b.box
            ptr[c], exists[c] = b.ptr, 1
    return feat, mask, box, ptr, exists


def decode(src, count, slot_out, L=BANK['len_queue']):
    """The product's retrieval record of one query as bank slots: a store row -> row % L, the level's object j -> the slot
    object j's append wrote."""
    return [int(s) % L if s >= 0 else int(slot_out[-int(s) - 1]) for s in src[:int(count)]]


def clone(orc):
    return copy.deepcopy(orc)
