"""The momentum (EMA) update of a teacher's tensors from a student's, on the kernel of csrc/momentum_update.cu: for every
pair, in place, ``t <- fl(fl(s * (1. - m)) + fl(t * m))`` with the roundings of torch's ``cur * (1. - m) + self * m``
followed by ``load_state_dict``'s ``copy_`` (integer and bool tensors go through float32 and back), in one launch for up
to 1024 pairs.

``momentum_update_`` packs and checks the pairs on every call; ``Table`` and ``launch`` let a caller that keeps the same
tensors pack them once.  Neither allocates device memory nor synchronises the host."""
import ctypes

import numpy as np
import torch

from .. import _lib as L

DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2, torch.float64: 3, torch.int64: 4, torch.int32: 5,
          torch.int16: 6, torch.int8: 7, torch.uint8: 8, torch.bool: 9}          # bxs_ema_dtype_t


def _non_overlapping_and_dense(t):
    """Some order of the dimensions makes ``t`` contiguous (row-major, channels_last, any permutation)."""
    expect = 1
    for stride, size in sorted((st, sz) for sz, st in zip(t.shape, t.stride()) if sz != 1):
        if stride != expect:
            return False
        expect *= size
    return True


class Table:
    """The (teacher, student) pairs of one update, checked and packed as the kernel's host arrays.  A teacher tensor
    listed again with the same student tensor (tied weights under two state-dict keys) is packed once."""

    def __init__(self, teacher_tensors, student_tensors):
        teacher_tensors, student_tensors = list(teacher_tensors), list(student_tensors)
        if len(teacher_tensors) != len(student_tensors):
            raise RuntimeError(f'momentum_update_: {len(teacher_tensors)} teacher tensors but {len(student_tensors)} '
                               'student tensors')
        rows, seen, self.device = [], set(), None
        for i, (t, s) in enumerate(zip(teacher_tensors, student_tensors)):
            if not isinstance(t, torch.Tensor) or not isinstance(s, torch.Tensor):
                raise RuntimeError(f'momentum_update_: pair {i} is not a pair of tensors')
            if not (t.is_cuda and s.is_cuda):
                raise RuntimeError(f'momentum_update_: pair {i}: tensors must be CUDA tensors')
            if self.device is None:
                self.device = t.device
            if t.device != self.device or s.device != self.device:
                raise RuntimeError(f'momentum_update_: pair {i}: every tensor must be on {self.device}')
            if t.dtype != s.dtype or t.shape != s.shape or t.stride() != s.stride():
                raise RuntimeError(f'momentum_update_: pair {i}: teacher {t.dtype} {tuple(t.shape)} strides {t.stride()} '
                                   f'and student {s.dtype} {tuple(s.shape)} strides {s.stride()} differ')
            if t.dtype not in DTYPES:
                raise RuntimeError(f'momentum_update_: pair {i}: unsupported dtype {t.dtype}')
            if not _non_overlapping_and_dense(t):
                raise RuntimeError(f'momentum_update_: pair {i}: tensors must be non-overlapping and dense')
            row = (t.data_ptr(), s.data_ptr(), t.numel(), DTYPES[t.dtype])
            if row[2] == 0 or row in seen:
                continue
            seen.add(row)
            rows.append(row)
        rows = np.array(rows, dtype=np.int64).reshape(-1, 4)
        self.n = len(rows)
        self.teacher = np.ascontiguousarray(rows[:, 0])
        self.student = np.ascontiguousarray(rows[:, 1])
        self.count = np.ascontiguousarray(rows[:, 2])
        self.dtype = np.ascontiguousarray(rows[:, 3], dtype=np.int32)


def launch(table, momentum):
    """Update the tensors of ``table`` on the current stream of their device, with ``a = 1. - momentum`` and
    ``b = momentum`` computed as Python computes them."""
    if table.n == 0:
        return
    ab = (ctypes.c_double * 2)(1. - momentum, momentum)
    with torch.cuda.device(table.device):
        L.check(L.lib().bxs_momentum_update(table.teacher.ctypes.data, table.student.ctypes.data, table.count.ctypes.data,
                                            table.dtype.ctypes.data, table.n, ab, L.stream()), 'momentum_update_')


def momentum_update_(teacher_tensors, student_tensors, momentum):
    """In place, for every pair: ``teacher <- student * (1. - momentum) + teacher * momentum``, rounded as torch rounds
    that expression followed by ``teacher.copy_``.  Each pair must have the same shape, dtype, device and strides and be
    non-overlapping and dense (channels_last included); anything else, or a CPU tensor, raises ``RuntimeError`` naming
    the pair.  Overlapping teacher tensors, or a student tensor that overlaps a teacher tensor other than exactly its own,
    raise ``BoxSegError``."""
    launch(Table(teacher_tensors, student_tensors), momentum)
