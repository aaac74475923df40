"""CPU: the C-ABI shared library loads without a GPU and exports every symbol include/boxseg_b200.h
declares; the ctypes types read from the header are the C types; host-side argument validation works."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
c_p, c_i64, c_int, c_f = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int, ctypes.c_float


def _header():
    with open(os.path.join(ROOT, 'include', 'boxseg_b200.h')) as f:
        return re.sub(r'/\*.*?\*/', '', f.read(), flags=re.S)


def _declared():
    return sorted(set(re.findall(r'\b(bxs_\w+)\s*\(', _header())))


@pytest.fixture(scope='module')
def lib():
    from boxinstseg_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib


def test_every_declared_symbol_is_exported_and_bound(lib):
    names = _declared()
    assert len(names) >= 40
    handle = ctypes.CDLL(lib.LIB_PATH)
    missing = [n for n in names if not hasattr(handle, n)]
    assert not missing, f'declared in the header but not exported: {missing}'
    h = lib.lib()           # resolves + types every symbol
    for n in names:
        fn = getattr(h, n)
        assert fn.argtypes == lib.SIGNATURES[n] and fn.restype is lib.RESTYPES[n], n


@pytest.mark.parametrize('name, argtypes, restype', [
    ('bxs_boxinst_targets_forward', [c_p] * 13 + [c_i64] * 3 + [c_int] * 3 + [c_f, c_p], c_int),
    ('bxs_corr_retrieve', [c_p] * 19 + [c_i64] * 8 + [c_f] * 6 + [c_int] * 2 + [c_p], c_int),
    ('bxs_sigmoid_focal_loss_cells_forward', [c_p] * 7 + [c_i64] * 3 + [c_f] * 3 + [c_p], c_int),   # const float* const*
    ('bxs_lsap_workspace_bytes', [c_p, c_p, c_i64], c_i64),
    ('bxs_version', [], c_int),
    ('bxs_last_error', [], ctypes.c_char_p),
])
def test_header_signatures(name, argtypes, restype):
    from boxinstseg_b200 import _lib as lib
    assert lib.SIGNATURES[name] == argtypes and lib.RESTYPES[name] is restype


def test_every_int64_result_is_bound_as_int64():
    """A size query left at ctypes' default c_int would truncate a workspace of 2 GiB or more."""
    from boxinstseg_b200 import _lib as lib
    wide = set(re.findall(r'\bint64_t\s+(bxs_\w+)\s*\(', _header()))
    assert len(wide) >= 25
    assert {n for n, r in lib.RESTYPES.items() if r is c_i64} == wide
    assert {n for n, r in lib.RESTYPES.items() if r is c_int} == set(lib.SIGNATURES) - wide - {'bxs_last_error'}


def test_parse_header_on_text():
    from boxinstseg_b200 import _lib as lib
    text = '''/* bxs_in_a_comment(double x); */
    typedef void* bxs_stream_t;
    int64_t bxs_a(const void* const* p, int64_t n, int k, float x, bxs_stream_t s);
    int bxs_b(void);'''
    argtypes, restypes = lib.parse_header(text)
    assert argtypes == {'bxs_a': [c_p, c_i64, c_int, c_f, c_p], 'bxs_b': []}
    assert restypes == {'bxs_a': c_i64, 'bxs_b': c_int}
    with pytest.raises(TypeError):
        lib.parse_header('int bxs_c(const void* p, double x);')
    with pytest.raises(TypeError):
        lib.parse_header('double bxs_d(int n);')


def test_identity_and_no_device(lib):
    h = lib.lib()
    assert h.bxs_version() == 100
    import torch
    if not torch.cuda.is_available():
        assert h.bxs_device_sm_count() == -4          # BXS_ERR_NO_DEVICE, no crash


def test_workspace_queries_and_argument_validation_without_gpu(lib):
    h = lib.lib()
    assert h.bxs_pairwise_nlog_forward(None, None, 1, 4, 4, 3, 2, 0, None) == -1      # null pointers
    assert h.bxs_boxinst_loss_workspace_bytes(128, 200, 256) > 0
    assert h.bxs_boxinst_loss_workspace_bytes(0, 200, 256) == 0
    assert h.bxs_levelset_fused_workspace_bytes(16) > 0 and h.bxs_lcm_workspace_bytes(8, 96, 96) > 0
    assert h.bxs_mst_workspace_bytes(2, 18240, 9216) > 0 and h.bxs_refine_scratch_bytes(2, 1, 9216) > 0
    p = ctypes.cast((ctypes.c_float * 64)(), ctypes.c_void_p)
    assert h.bxs_refine_forward_grouped(*[p] * 7, None, *[p] * 6, 2, 3, 1, 16, None) == -1    # no tree_of: n must equal G
    assert h.bxs_refine_backward_feature_grouped(*[p] * 6, None, *[p] * 4, 2, 3, 1, 16, None) == -1
    assert h.bxs_refine_backward_weight_grouped(*[p] * 6, None, *[p] * 8, 2, 3, 1, 16, None) == -1


def test_ops_fail_loudly_on_cpu_tensors(lib):
    import torch
    from boxinstseg_b200.ops.pairwise import pairwise_nlog
    with pytest.raises(RuntimeError):
        pairwise_nlog(torch.zeros(1, 1, 4, 4), 3, 2)
    from boxinstseg_b200.models.losses import LevelsetLoss
    with pytest.raises(RuntimeError):
        LevelsetLoss()(torch.rand(1, 2, 4, 4), torch.rand(1, 3, 4, 4), torch.ones(1))


def test_missing_library_is_an_error(lib, monkeypatch):
    monkeypatch.setattr(lib, '_lib', None)
    monkeypatch.setattr(lib, 'LIB_PATH', '/nonexistent/libboxseg_b200.so')
    with pytest.raises(ImportError):
        lib.lib()


def test_argument_validation_of_the_f_row_entry_points(lib):
    """Host-side checks run before any launch, so they can be exercised without a GPU: null pointers and malformed tables are
    invalid arguments (-1), shapes outside the kernels' envelopes are unsupported (-3)."""
    import ctypes
    h = lib.lib()
    buf = (ctypes.c_float * 64)()
    p = ctypes.cast(buf, ctypes.c_void_p)
    off2 = ctypes.cast((ctypes.c_int64 * 3)(0, 1, 2), ctypes.c_void_p)
    lvl = ctypes.cast((ctypes.c_int64 * 2)(0, 4), ctypes.c_void_p)
    assert h.bxs_fcos_targets(None, p, p, off2, p, p, p, 2, 1, lvl, p, p, p, p, 1, 1, 80, None) == -1          # no points
    assert h.bxs_fcos_targets(p, p, p, off2, p, p, p, 2, 9, lvl, p, p, p, p, 1, 1, 80, None) == -3             # > 8 levels
    assert h.bxs_fcos_targets(p, p, p, off2, p, p, p, 257, 1, lvl, p, p, p, p, 1, 1, 80, None) == -3           # > 256 images
    bad = ctypes.cast((ctypes.c_int64 * 3)(0, 2, 1), ctypes.c_void_p)
    assert h.bxs_fcos_targets(p, p, p, bad, p, p, p, 2, 1, lvl, p, p, p, p, 1, 1, 80, None) == -1              # offsets decrease
    assert h.bxs_fcos_targets(p, None, None, off2, p, p, p, 2, 1, lvl, p, p, p, p, 1, 1, 80, None) == -1       # GTs without boxes
    assert h.bxs_corr_solve(None, p, 5, 7, 7, 9, 10, 1, None) == -1
    assert h.bxs_corr_solve(p, p, 5, 7, 7, 8, 10, 1, None) == -1                                               # even window
    assert h.bxs_corr_solve(p, p, 5, 16, 16, 9, 10, 1, None) == -3                                             # tables > 200 KB
    assert h.bxs_corr_transfer_workspace_bytes(5, 28, 28) == 5 * 2 * 784 * 4 and h.bxs_corr_transfer_workspace_bytes(0, 28, 28) == 0
    assert h.bxs_corr_transfer(p, p, p, p, p, p, None, 5, 7, 7, 28, 28, None) == -1                            # no workspace
    assert h.bxs_corr_transfer(p, p, p, p, p, p, p, 5, 16, 16, 28, 28, None) == -3
    assert h.bxs_meanfield_forward_inter(None, None, p, p, p, 0.5, p, p, p, p, 4, 8, 8, 3, 10, None) == -1
