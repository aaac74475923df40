"""DiscoBox's independent teacher, CPU side: (1) the oracle (oracle/teacher_ema.py) reproduces the golden vectors minted
from the reference's own ``momentum_update`` and ``forward_train`` (oracle/make_golden_teacher_ema.py); (2) the argument
checks of ``bxs_momentum_update``, none of which launches; (3) ``momentum_update``'s pairing errors are those of
``load_state_dict(strict=True)``, and the pairing cache sees every change of the tensors.  The GPU twin of this file is
tests/test_teacher_ema_gpu.py."""
import ctypes

import numpy as np
import pytest
import torch
from torch import nn

from oracle import teacher_ema as ote


def _same(a, b):
    """Bit for bit, a NaN only as a NaN."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.kind != 'f':
        return np.array_equal(a, b)
    nan = np.isnan(a)
    return np.array_equal(nan, np.isnan(b)) and np.array_equal(a[~nan].view(np.uint8), b[~nan].view(np.uint8))


def ema_case(g, i):
    """(momentum, teacher, student, out) state dicts of numpy arrays of golden case i."""
    keys = [k.split('/', 2)[2] for k in g.files if k.startswith(f'ema{i}/out/')]
    part = lambda p: {k: g[f'ema{i}/{p}/{k}'] for k in keys}               # noqa: E731
    return float(g[f'ema{i}/momentum']), part('teacher'), part('student'), part('out')


@pytest.mark.parametrize('i', range(len(ote.MOMENTA)))
def test_oracle_momentum_update_reproduces_reference_golden(golden, i):
    m, teacher, student, out = ema_case(golden('teacher_ema'), i)
    assert m == ote.MOMENTA[i]
    got = ote.ema_state(teacher, student, m)
    assert got.keys() == out.keys() and len(out) == 13
    for k in out:
        assert _same(got[k], out[k]), k


def test_golden_states_cover_their_edges(golden):
    g = golden('teacher_ema')
    _, teacher, student, _ = ema_case(g, 0)
    dtypes = {v.dtype for v in teacher.values()}
    assert {np.dtype(np.float32), np.dtype(np.float16), np.dtype(np.float64), np.dtype(np.int64)} <= dtypes
    f32 = np.concatenate([v.ravel() for v in teacher.values() if v.dtype == np.float32])
    f16 = np.concatenate([v.ravel() for v in teacher.values() if v.dtype == np.float16])
    for x in (f32, f16):
        assert np.isposinf(x).any() and np.isneginf(x).any()
        assert (np.signbit(x) & (x == 0)).any() and (~np.signbit(x) & (x == 0)).any()
        fin = np.abs(x[np.isfinite(x) & (x != 0)])
        assert (fin < np.finfo(x.dtype).tiny).any()                           # subnormals
    ints = np.concatenate([v.ravel() for v in teacher.values() if v.dtype == np.int64])
    assert (np.abs(ints) > 2 ** 24).any() and (ints == 2 ** 24 + 1).any()


@pytest.mark.parametrize('run', ote.GATE_RUNS, ids=[r[0] for r in ote.GATE_RUNS])
def test_oracle_gates_reproduce_reference_golden(golden, run):
    g = golden('teacher_ema')
    name, ind, corr, avg0, cnt0, losses = run
    rows = ote.gates(ind, corr, avg0, cnt0, False, losses)
    assert np.array_equal(np.array([r[:4] for r in rows], np.int64), g[f'gates/{name}/flags'])
    assert np.array_equal(np.array([r[4] for r in rows], np.int64), g[f'gates/{name}/cnt'])
    assert np.array_equal(np.array([r[5] for r in rows], np.float64), g[f'gates/{name}/avg'])
    flags = g[f'gates/{name}/flags']
    assert flags[:, 0].any() and not flags[:, 0].all()                         # both sides of 0.3
    if corr:
        assert flags[:, 1].any() and not flags[:, 1].all()                     # both sides of 0.2
    if ind:
        assert flags[:, 3].any() and not flags[:, 3].all()                     # the turn-on


@pytest.fixture(scope='module')
def lib():
    from boxinstseg_b200 import _lib, build
    import os
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.lib()


def _arr(ctype, vals):
    return ctypes.cast((ctype * len(vals))(*vals), ctypes.c_void_p)


def test_c_abi_argument_validation_without_gpu(lib):
    """Every check runs before any device call: the invalid tables return -1 here, and the tables without work return 0."""
    ab = _arr(ctypes.c_double, [0.001, 0.999])
    buf = (ctypes.c_float * 4096)()
    base = ctypes.addressof(buf)

    def call(ts, ss, counts, dtypes, ab=ab, n=None):
        n = len(counts) if n is None else n
        return lib.bxs_momentum_update(_arr(ctypes.c_void_p, ts), _arr(ctypes.c_void_p, ss), _arr(ctypes.c_int64, counts),
                                       _arr(ctypes.c_int32, dtypes), n, ab, None)
    t0, t1, s0, s1 = base, base + 1024, base + 2048, base + 3072
    assert call([t0], [s0], [4], [0], n=-1) == -1                               # negative n
    assert call([t0], [s0], [4], [0], ab=None) == -1                            # no scalars
    assert call([t0], [s0], [-1], [0]) == -1                                    # negative count
    assert call([t0], [s0], [4], [10]) == -1                                    # unknown dtype
    assert call([t0], [s0], [4], [-1]) == -1
    assert call([None], [s0], [4], [0]) == -1                                   # NULL region with a count
    assert call([t0], [None], [4], [0]) == -1
    assert call([t0, t0 + 12], [s0, s1], [4, 4], [0, 0]) == -1                  # teacher regions overlap by one float
    assert call([t0, t0 + 4], [s0, s1], [1, 4], [3, 0]) == -1                   # a float64 reaching into the next region
    assert call([t0, t1], [t1, s1], [4, 4], [0, 0]) == -1                       # a student is another pair's teacher
    assert call([t0, t1], [t0 + 4, s1], [4, 4], [0, 0]) == -1                   # a student half on its own teacher
    assert call([t0, t1], [t1 - 4, s1], [4, 4], [0, 0]) == -1                   # a student reaching into the next teacher
    assert lib.bxs_momentum_update(None, None, None, None, 0, ab, None) == 0    # n == 0: nothing to do
    assert call([None, None], [None, None], [0, 0], [0, 9]) == 0                # zero-element entries: no launch
    assert call([t0, t0], [s0, s1], [0, 0], [0, 0]) == 0                        # empty regions never overlap


class _Net(nn.Module):
    def __init__(self, out=5, extra=False):
        super().__init__()
        self.conv = nn.Conv2d(3, 4, 3)
        self.bn = nn.BatchNorm2d(4)
        self.block = nn.Sequential(nn.Linear(4, out))
        if extra:
            self.block.add_module('tail', nn.Linear(2, 2))
            self.register_buffer('steps', torch.zeros((), dtype=torch.int64))


def _load_error(teacher, student):
    with pytest.raises(RuntimeError) as e:
        teacher.load_state_dict(student.state_dict(), strict=True)
    return str(e.value)


@pytest.mark.parametrize('teacher, student', [
    (lambda: _Net(extra=True), lambda: _Net()),                         # missing keys
    (lambda: _Net(), lambda: _Net(extra=True)),                         # unexpected keys, in two modules
    (lambda: _Net(out=6), lambda: _Net()),                              # size mismatches
    (lambda: _Net(out=6, extra=True), lambda: _Net(out=5)),             # all three at once
], ids=['missing', 'unexpected', 'size', 'all'])
def test_pairing_errors_are_load_state_dicts(teacher, student):
    from boxinstseg_b200.models.detectors import momentum_update
    t, s = teacher(), student()
    before = {k: v.clone() for k, v in t.state_dict().items()}
    want = _load_error(t, s)
    t.load_state_dict(before)
    with pytest.raises(RuntimeError) as e:
        momentum_update(t, s, 0.999)
    assert str(e.value) == want
    assert all(torch.equal(v, before[k]) for k, v in t.state_dict().items())   # nothing was updated


def test_cpu_tensors_raise():
    from boxinstseg_b200.models.detectors import momentum_update
    from boxinstseg_b200.ops.ema import momentum_update_
    with pytest.raises(RuntimeError, match='pair 0'):
        momentum_update_([torch.zeros(3)], [torch.zeros(3)], 0.5)
    t = _Net()
    t.teacher_momentum = 0.999
    with pytest.raises(RuntimeError, match='CUDA'):
        momentum_update(t, _Net())
    with pytest.raises(RuntimeError, match='2 teacher tensors but 1'):
        momentum_update_([torch.zeros(3)] * 2, [torch.zeros(3)], 0.5)


def test_fingerprint_sees_every_change_of_the_state():
    from boxinstseg_b200.models.detectors.discobox import _fingerprint
    m = _Net()
    fp = _fingerprint(m)
    assert fp == _fingerprint(m)
    changes = [
        lambda: setattr(m.conv, 'weight', nn.Parameter(m.conv.weight.detach().clone())),     # a replaced parameter
        lambda: setattr(m.bn, 'running_mean', m.bn.running_mean.clone()),                   # a replaced buffer
        lambda: m.to(torch.float64),                                                        # .to()
        lambda: m.to(memory_format=torch.channels_last),
        lambda: m.block.add_module('more', nn.Linear(1, 1)),                                # a new module
    ]
    for change in changes:
        change()
        new = _fingerprint(m)
        assert new != fp
        fp = new
    m.bn.register_state_dict_post_hook(lambda *a: None)
    assert _fingerprint(m) is None                                                         # hooks: no caching
