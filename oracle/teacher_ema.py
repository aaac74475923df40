"""Oracle of DiscoBox's independent teacher (mmdet/models/detectors/single_stage_ts.py:118-131, 179-237), in numpy:

* ``ema_state``: ``SingleStageWSInsTeacherDetector.momentum_update``'s arithmetic on state dicts of numpy arrays:
  ``cur * (1. - m) + self * m`` as torch evaluates it, then ``load_state_dict``'s cast back to the teacher's dtype.
* ``gates``: the host-side control flow of ``SingleStageWSInsTSDetector.forward_train`` for a given ``loss_ins`` sequence:
  per step the gates handed to the head's loss, ``turn_on_teacher``, ``cnt`` and ``avg_loss_ins``.

Also the small model and the seeded states the golden vectors (oracle/make_golden_teacher_ema.py) are minted on.
"""
import numpy as np
import torch
from torch import nn

MOMENTA = (0.999, 0.0, 0.5)


def ema_state(teacher, student, m):
    """{key: new teacher array} for state dicts of numpy arrays (float32, float16, float64 or integer/bool)."""
    a, b = 1. - m, m
    out = {}
    with np.errstate(invalid='ignore', over='ignore'):          # inf * 0 and inf - inf are NaN, as in torch
        for k, s in student.items():
            out[k] = _ema(teacher[k], s, a, b)
    return out


def _ema(t, s, a, b):
    if t.dtype == np.float64:
        return s * a + t * b
    if t.dtype in (np.float32, np.float16):
        # float32 opmath with the Python scalars cast to float; float16 rounds each product and the sum
        p = (s.astype(np.float32) * np.float32(a)).astype(t.dtype).astype(np.float32)
        q = (t.astype(np.float32) * np.float32(b)).astype(t.dtype).astype(np.float32)
        return (p + q).astype(t.dtype)
    # int * float promotes to float32; load_state_dict's copy_ converts back toward zero
    r = s.astype(np.float32) * np.float32(a) + t.astype(np.float32) * np.float32(b)
    return (r != 0) if t.dtype == np.bool_ else np.trunc(r).astype(np.int64).astype(t.dtype)


def gates(use_ind_teacher, use_corr, avg0, cnt0, turn0, losses):
    """Rows (use_loss_ts, use_corr, use_ind_teacher, turn_on_teacher, cnt, avg_loss_ins) after each step of
    forward_train, the gates being those handed to that step's loss."""
    avg, cnt, turn, rows = avg0, cnt0, turn0, []
    for loss in losses:
        g = (avg < 0.3, avg < 0.2 and use_corr, use_ind_teacher and turn)
        avg = avg * 0.9 + 0.1 * float(np.float32(loss))
        if use_ind_teacher and not turn and cnt > 13000:
            turn = True
        else:
            cnt += 1
        rows.append(g + (turn, cnt, avg))
    return rows


class EmaModel(nn.Module):
    """Float32 and float16 parameters, BatchNorm and GroupNorm state and int64 counters: every kind of entry a detector's
    state dict has."""

    def __init__(self):
        super().__init__()
        self.conv = nn.Conv2d(3, 8, 3)
        self.bn = nn.BatchNorm2d(8)
        self.gn = nn.GroupNorm(2, 8)
        self.head = nn.Linear(8, 24).half()
        self.register_buffer('counter', torch.zeros(16, dtype=torch.int64))
        self.register_buffer('scale', torch.zeros(12, dtype=torch.float64))


_F32_EDGES = [0.0, -0.0, 1e-45, -1e-45, 1e-40, -2.5e-39, 1.1754942e-38, float('inf'), float('-inf'), 16777216.0,
              16777217.0, -16777215.0, 3.4028235e38, 1.0, -1.0]
_F16_EDGES = [0.0, -0.0, 6e-8, -6e-8, 3e-5, -6.1e-5, float('inf'), float('-inf'), 65504.0, -65504.0, 2048.0, 2049.0,
              1.0, -1.0]
_I64_EDGES = [0, 1, -1, 16777215, 16777216, 16777217, 16777219, -16777217, 33554435, 1000, 99, 2 ** 40 + 1, 7, 13001,
              -3, 2 ** 24 + 3]


def ema_states(seed):
    """(teacher, student) EmaModels filled with seeded values and the edge values above."""
    out = []
    for k in range(2):
        torch.manual_seed(seed * 2 + k)
        m = EmaModel()
        with torch.no_grad():
            for name, t in m.state_dict().items():
                if t.dtype == torch.int64:
                    t.copy_(torch.randint(-2 ** 25, 2 ** 25, t.shape))
                else:
                    t.copy_((torch.randn(t.shape, dtype=torch.float64) * 3).to(t.dtype))
            edges = {torch.float32: _F32_EDGES, torch.float16: _F16_EDGES}
            for name, t in m.state_dict().items():
                flat = t.view(-1)
                if t.dtype == torch.int64:
                    e = torch.tensor(_I64_EDGES[k:] + _I64_EDGES[:k])[:flat.numel()]
                elif t.dtype in edges:
                    e = torch.tensor(edges[t.dtype][k:] + edges[t.dtype][:k], dtype=t.dtype)[:flat.numel()]
                else:
                    continue
                flat[:len(e)] = e
            m.bn.num_batches_tracked.fill_(16777217 + k * 1000)
        out.append(m)
    return out[0], out[1]


# (name, use_ind_teacher, use_corr, avg_loss_ins at the start, cnt at the start, loss_ins per step): each run crosses the
# teacher's turn-on (cnt > 13000) and both thresholds of avg_loss_ins (0.3: teacher-student loss, 0.2: correspondence)
GATE_RUNS = [
    ('from_start', True, True, 2, 12990, [0.0] * 24 + [0.5, 0.9, 0.0, 0.0, 0.1, 0.0, 0.25, 0.3]),
    ('crossing', True, True, 0.3, 12998, [0.0] * 5 + [0.9, 0.0, 0.0, 0.0, 2.0, 0.0]),
    ('no_corr', True, False, 0.3, 12999, [0.0] * 4 + [0.9, 0.0, 0.0]),
    ('shared_teacher', False, True, 0.3, 12998, [0.0] * 5 + [1.0, 0.0]),
]
