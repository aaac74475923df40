"""CPU: the linear-sum-assignment core (csrc/lsap_core.cuh, the source of lsap_kernel) built for the host through
tests/host_harness/lsap_host.cpp returns scipy.optimize.linear_sum_assignment's row_ind / col_ind exactly -- ties included --
and the status the kernel reports where scipy raises.  Also the host-side argument checks of bxs_lsap_solve /
bxs_lsap_workspace_bytes and of ops.lsap, which run before any device call."""
import ctypes
import os

import numpy as np
import pytest
import torch
from scipy.optimize import linear_sum_assignment

from tests.helpers import host_twin

OK, INVALID, INFEASIBLE = 0, 1, 2


@pytest.fixture(scope='module')
def twin():
    lib = host_twin('lsap_host')

    def solve(c):
        c = np.ascontiguousarray(c)
        match = np.full(c.shape[0], -7, np.int32)
        st = lib.host_lsap_solve(c.ctypes.data_as(ctypes.c_void_p), 0 if c.dtype == np.float32 else 1, c.shape[0], c.shape[1],
                                 match.ctypes.data_as(ctypes.c_void_p))
        return st, match
    return solve


def scipy_result(c):
    """(status, row_ind, col_ind) of scipy, the status being the kernel's code for scipy's ValueError."""
    try:
        r, k = linear_sum_assignment(c)
    except ValueError as e:
        return (INVALID if 'invalid numeric entries' in str(e) else INFEASIBLE if 'infeasible' in str(e) else -1), None, None
    return OK, r, k


def assert_same(twin, c):
    want, r, k = scipy_result(c)
    st, match = twin(c)
    assert st == want, (c.shape, st, want)
    if want != OK:
        assert (match == -1).all()
        return
    rows = np.nonzero(match >= 0)[0]
    assert np.array_equal(rows, r) and np.array_equal(match[rows], k), c.shape


def seeded_matrix(rng, kind, nr, nc):
    if kind == 'normal':
        return rng.standard_normal((nr, nc)).astype(np.float32)
    if kind == 'int3':                                      # heavy ties
        return rng.integers(0, 3, (nr, nc)).astype(np.float32)
    if kind == 'zeros':
        return np.zeros((nr, nc), np.float32)
    c = rng.integers(0, 4, (nr, nc)).astype(np.float32)    # +inf entries, infeasible when a row or column is cut off
    c[rng.random((nr, nc)) < 0.3] = np.inf
    return c


@pytest.mark.parametrize('kind', ['normal', 'int3', 'zeros', 'inf'])
def test_lsap_matches_scipy(twin, kind):
    """800 seeded matrices per kind (3200 in all), shapes 1x1 .. 39x39 in both orientations."""
    rng = np.random.default_rng(['normal', 'int3', 'zeros', 'inf'].index(kind))
    shapes = set()
    for _ in range(800):
        nr, nc = (int(v) for v in rng.integers(1, 40, 2))
        shapes.add((nr > nc) - (nr < nc))
        assert_same(twin, seeded_matrix(rng, kind, nr, nc))
    assert shapes == {-1, 0, 1}


def test_lsap_float64_and_transposed(twin):
    rng = np.random.default_rng(7)
    for nr, nc in [(5, 9), (9, 5), (1, 30), (30, 1), (17, 17)]:
        c = rng.standard_normal((nr, nc))
        assert_same(twin, c)
        assert_same(twin, np.ascontiguousarray(c.T))
        assert_same(twin, np.round(c).astype(np.float64))


def test_lsap_invalid_and_infeasible(twin):
    c = np.zeros((4, 6), np.float32)
    for bad in (np.nan, -np.inf):
        for shape in [(4, 6), (6, 4), (1, 1)]:
            c = np.ones(shape, np.float32)
            c[shape[0] - 1, 0] = bad
            assert scipy_result(c)[0] == INVALID
            assert_same(twin, c)
    c = np.ones((3, 3), np.float32)
    c[1, :] = np.inf                                        # a row with no finite entry
    assert scipy_result(c)[0] == INFEASIBLE
    assert_same(twin, c)
    assert_same(twin, np.ascontiguousarray(c.T))
    c = np.full((2, 5), np.inf, np.float32)
    c[0, 0] = c[1, 0] = 1.0                                 # two rows, one reachable column
    assert scipy_result(c)[0] == INFEASIBLE
    assert_same(twin, c)


@pytest.mark.parametrize('shape', [(0, 5), (5, 0), (0, 0)])
def test_lsap_empty(twin, shape):
    c = np.zeros(shape, np.float32)
    st, match = twin(c)
    assert st == OK and match.shape == (shape[0],) and (match == -1).all()
    r, k = linear_sum_assignment(c)
    assert r.size == 0 and k.size == 0


@pytest.mark.parametrize('G', [0, 1, 7, 50, 100, 150])
def test_lsap_box2mask_costs(twin, G):
    """100 x G costs of Box2Mask's assigner config (box2mask_*.py:111-114): 2 * classification cost + 5 * BoxMatchingCost of
    sigmoid row / column profiles, in float32 as the device computes them."""
    from boxinstseg_b200.core import BoxMatchingCost, ClassificationCost
    gen = torch.Generator().manual_seed(G)
    Q, H, W, ncls = 100, 64, 80, 81
    for _ in range(5):
        cls_pred = torch.randn(Q, ncls, generator=gen)
        labels = torch.randint(0, 80, (G,), generator=gen)
        pr, pc = torch.sigmoid(torch.randn(Q, H, generator=gen) * 3), torch.sigmoid(torch.randn(Q, W, generator=gen) * 3)
        gr, gc = (torch.rand(G, H, generator=gen) > 0.6).float(), (torch.rand(G, W, generator=gen) > 0.6).float()
        cost = ClassificationCost(2.0)(cls_pred, labels) + BoxMatchingCost(5.0, pred_act=True, eps=1.0)._cost(pr, pc, gr, gc)
        assert cost.shape == (Q, G) and cost.dtype == torch.float32
        assert_same(twin, cost.numpy())


@pytest.fixture(scope='module')
def lib():
    from boxinstseg_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.lib()


def _arr(*v):
    return (ctypes.c_int64 * len(v))(*v)


def test_lsap_abi_validation(lib):
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.c_void_p(ctypes.addressof(buf))
    solve = lib.bxs_lsap_solve
    rows, cols, offs = _arr(3, 4), _arr(5, 2), _arr(0, 15)
    assert solve(p, offs, rows, cols, -1, 0, p, p, p, None) == -1
    assert solve(p, offs, rows, cols, 2, 2, p, p, p, None) == -1          # unknown dtype
    assert solve(p, offs, rows, cols, 2, -1, p, p, p, None) == -1
    assert solve(None, offs, rows, cols, 2, 0, p, p, p, None) == -1        # cost needed
    assert solve(p, None, rows, cols, 2, 0, p, p, p, None) == -1
    assert solve(p, offs, None, cols, 2, 0, p, p, p, None) == -1
    assert solve(p, offs, rows, None, 2, 0, p, p, p, None) == -1
    assert solve(p, offs, rows, cols, 2, 0, None, p, p, None) == -1       # match needed
    assert solve(p, offs, rows, cols, 2, 0, p, None, p, None) == -1       # status always needed
    assert solve(p, offs, rows, cols, 2, 0, p, p, None, None) == -1       # workspace needed
    assert solve(p, offs, _arr(3, -1), cols, 2, 0, p, p, p, None) == -1   # negative size
    assert solve(p, _arr(0, -4), rows, cols, 2, 0, p, p, p, None) == -1   # negative offset
    assert solve(p, offs, _arr(3, 1 << 31), cols, 2, 0, p, p, p, None) == -3   # beyond int32 indices
    assert solve(None, None, None, None, 0, 0, None, None, None, None) == 0   # nothing to do
    # empty problems need neither costs nor workspace (and match only when they have rows)
    assert solve(None, _arr(0, 0), _arr(0, 0), _arr(3, 0), 2, 0, None, None, None, None) == -1   # status still needed


def test_lsap_workspace_query(lib):
    ws = lib.bxs_lsap_workspace_bytes
    assert ws(_arr(0, 5), _arr(7, 0), 2) == 0
    one = ws(_arr(100), _arr(50), 1)
    assert one == ws(_arr(50), _arr(100), 1)                 # a tall problem is solved transposed
    assert one >= 8 * (50 + 2 * 100) + 4 * (3 * 100 + 50) + 150
    assert ws(_arr(100, 100, 0), _arr(50, 50, 9), 3) == 2 * one
    assert ws(None, _arr(1), 1) == 0 and ws(_arr(1), _arr(1), -1) == 0


def test_lsap_python_validation():
    from boxinstseg_b200.ops.lsap import linear_sum_assignment, solve_batched
    with pytest.raises(ValueError, match='2-D'):
        solve_batched([torch.zeros(3)])
    with pytest.raises(ValueError, match='2-D'):
        linear_sum_assignment(torch.zeros(2, 3, 4))
    with pytest.raises(RuntimeError, match='CUDA'):
        solve_batched([torch.zeros(3, 4)])
