"""Golden vectors for DiscoBox's independent teacher, minted from the REFERENCE's own methods (authoring container only).

``SingleStageWSInsTeacherDetector.momentum_update`` and ``SingleStageWSInsTSDetector.forward_train`` are AST-extracted
from mmdet/models/detectors/single_stage_ts.py (the module imports mmcv, so it is not imported) and run on CPU:
  (i)  ``momentum_update`` on the seeded teacher / student ``EmaModel`` states of oracle/teacher_ema.py at every momentum
       of ``MOMENTA``: float32 and float16 parameters, BatchNorm and GroupNorm state, int64 counters, with +-0,
       subnormals, +-inf and integers around 2^24;
  (ii) ``forward_train`` bound to stub modules, driven by the loss_ins sequences of ``GATE_RUNS``: per step the gates its
       loss receives, ``turn_on_teacher``, ``cnt`` and ``avg_loss_ins``.
Both are asserted equal to oracle/teacher_ema.py and written to tests/golden/teacher_ema.npz.
    python -m oracle.make_golden_teacher_ema
"""
import ast
import os
import types
from collections import OrderedDict

import numpy as np
import torch

from oracle import teacher_ema as ote

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'teacher_ema.npz')
REL = 'mmdet/models/detectors/single_stage_ts.py'


def reference_methods():
    """(momentum_update, forward_train) of the reference, compiled from its source."""
    src = open(os.path.join(REF, REL)).read()
    classes = {n.name: n for n in ast.parse(src).body if isinstance(n, ast.ClassDef)}

    def method(cls, name):
        fn = [n for n in classes[cls].body if isinstance(n, ast.FunctionDef) and n.name == name][0]
        ns = dict(torch=torch, OrderedDict=OrderedDict)
        exec(compile(ast.Module(body=[fn], type_ignores=[]), REL, 'exec'), ns)
        return ns[name]
    return (method('SingleStageWSInsTeacherDetector', 'momentum_update'),
            method('SingleStageWSInsTSDetector', 'forward_train'))


def same(a, b):
    """Bit for bit, a NaN only as a NaN."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.kind == 'f':
        nan = np.isnan(a)
        return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint8), b[~nan].view(np.uint8))
    return np.array_equal(a, b)


class _Head:
    """The head: its forward returns (cate, kernel) and its loss records the gates and returns the next loss_ins."""

    def __init__(self, losses, calls):
        self.seq, self.calls = iter(losses), calls

    def __call__(self, feats):
        return feats, feats

    def loss(self, *args, use_loss_ts, use_ind_teacher, use_corr, **kw):
        self.calls.append((use_loss_ts, use_corr, use_ind_teacher))
        return {'loss_ins': torch.tensor(next(self.seq), dtype=torch.float32)}


class _MaskFeat:
    start_level, end_level = 0, 3

    def __call__(self, feats):
        return feats[0]


def stub_detector(forward_train, use_ind_teacher, use_corr, avg0, cnt0, losses, calls):
    """A stand-in with the attributes forward_train reads (stub modules around the head's loss)."""
    x = [torch.zeros(1)] * 5
    head = _Head(losses, calls)
    teacher = types.SimpleNamespace(extract_feat=lambda img: x, bbox_head=head, mask_feat_head=_MaskFeat(),
                                    momentum_update=lambda cur, m=None: None)
    det = types.SimpleNamespace(extract_feat=lambda img: x, bbox_head=head, mask_feat_head=_MaskFeat(),
                                tsw=types.SimpleNamespace(teacher=teacher), use_ind_teacher=use_ind_teacher,
                                use_corr=use_corr, train_cfg=None, avg_loss_ins=avg0, cnt=cnt0, turn_on_teacher=False)
    return types.MethodType(forward_train, det), det


def main():
    ref_update, ref_forward = reference_methods()
    arrays = {}
    # (i) momentum_update
    for seed, m in enumerate(ote.MOMENTA):
        teacher, student = ote.ema_states(seed)
        t_in = {k: v.numpy().copy() for k, v in teacher.state_dict().items()}
        s_in = {k: v.numpy().copy() for k, v in student.state_dict().items()}
        types.MethodType(ref_update, teacher)(student, m)
        got = {k: v.numpy() for k, v in teacher.state_dict().items()}
        want = ote.ema_state(t_in, s_in, m)
        for k in got:
            assert same(got[k], want[k]), (m, k, got[k], want[k])
            arrays[f'ema{seed}/teacher/{k}'] = t_in[k]
            arrays[f'ema{seed}/student/{k}'] = s_in[k]
            arrays[f'ema{seed}/out/{k}'] = got[k]
        arrays[f'ema{seed}/momentum'] = np.float64(m)
        print('momentum', m, len(got), 'entries')
    # (ii) forward_train's control flow
    for name, ind, corr, avg0, cnt0, losses in ote.GATE_RUNS:
        calls, rows = [], []
        fwd, det = stub_detector(ref_forward, ind, corr, avg0, cnt0, losses, calls)
        for _ in losses:
            fwd(torch.zeros(1), [{}], [], [])
            rows.append(calls[-1] + (det.turn_on_teacher, det.cnt, det.avg_loss_ins))
        want = ote.gates(ind, corr, avg0, cnt0, False, losses)
        assert rows == want, (name, rows, want)
        assert any(r[0] for r in rows) and not all(r[0] for r in rows), name
        assert any(r[3] for r in rows) and not all(r[3] for r in rows) or not ind, name
        arrays[f'gates/{name}/config'] = np.array([ind, corr, cnt0], np.int64)
        arrays[f'gates/{name}/avg0'] = np.float64(avg0)
        arrays[f'gates/{name}/losses'] = np.array(losses, np.float32)
        arrays[f'gates/{name}/flags'] = np.array([r[:4] for r in rows], np.int64)
        arrays[f'gates/{name}/cnt'] = np.array([r[4] for r in rows], np.int64)
        arrays[f'gates/{name}/avg'] = np.array([r[5] for r in rows], np.float64)
        print(name, len(rows), 'steps')
    np.savez_compressed(OUT, **arrays)
    print('written', OUT, os.path.getsize(OUT), 'bytes')


if __name__ == '__main__':
    main()
