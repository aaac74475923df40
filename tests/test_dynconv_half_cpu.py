"""CPU: host-side validation of the 16-bit dynamic 1x1 convolution entry points (bxs_dynconv1x1_half_*).  Every check runs
before any device call, so invalid arguments (-1) and shapes outside the 16-bit kernels' envelope (-3) are reported
without a GPU."""
import ctypes
import os

import pytest

F16, BF16 = 0, 1


@pytest.fixture(scope='module')
def lib():
    from boxinstseg_b200 import _lib, build
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib.lib()


_BUF = ctypes.create_string_buffer(256)


@pytest.fixture(scope='module')
def p():
    """A 16-byte aligned host address: the alignment check must not be what rejects a call."""
    return ctypes.c_void_p((ctypes.addressof(_BUF) + 15) & ~15)


@pytest.mark.parametrize('dt', [F16, BF16])
def test_half_forward_validation(lib, p, dt):
    fwd = lib.bxs_dynconv1x1_half_forward
    assert fwd(None, p, p, 1, 32, 64, 4, dt, None) == -1
    assert fwd(p, None, p, 1, 32, 64, 4, dt, None) == -1
    assert fwd(p, p, None, 1, 32, 64, 4, dt, None) == -1
    assert fwd(p, p, p, 0, 32, 64, 4, dt, None) == -1
    assert fwd(p, p, p, 1, 32, 64, 0, dt, None) == -1
    assert fwd(p, p, p, 1, 32, 64, 4, 2, None) == -1            # unknown dtype
    assert fwd(p, p, p, 1, 32, 64, 4, -1, None) == -1
    assert fwd(p, p, p, 1, 48, 64, 4, dt, None) == -3            # C % 32
    assert fwd(p, p, p, 1, 288, 64, 4, dt, None) == -3           # C > 256
    assert fwd(p, p, p, 1, 32, 68, 4, dt, None) == -3            # P % 8 == 4
    odd = ctypes.c_void_p(p.value + 8)
    assert fwd(odd, p, p, 1, 32, 64, 4, dt, None) == -3          # base not 16-byte aligned


@pytest.mark.parametrize('dt', [F16, BF16])
def test_half_backward_validation(lib, p, dt):
    bwd = lib.bxs_dynconv1x1_half_backward
    assert bwd(None, p, p, p, p, p, 1, 32, 64, 4, dt, None) == -1
    assert bwd(p, p, None, p, p, p, 1, 32, 64, 4, dt, None) == -1
    assert bwd(p, p, p, None, None, p, 1, 32, 64, 4, dt, None) == -1     # no gradient requested
    assert bwd(p, p, p, p, p, None, 1, 32, 64, 4, dt, None) == -1        # no workspace
    assert bwd(p, p, p, p, p, p, 1, 32, -64, 4, dt, None) == -1
    assert bwd(p, p, p, p, p, p, 1, 32, 64, 4, 7, None) == -1             # unknown dtype
    assert bwd(p, p, p, p, p, p, 1, 40, 64, 4, dt, None) == -3            # C % 32
    assert bwd(p, p, p, p, p, p, 1, 512, 64, 4, dt, None) == -3           # C > 256
    assert bwd(p, p, p, p, p, p, 1, 32, 68, 4, dt, None) == -3            # P % 8 == 4
    assert bwd(p, p, p, p, p, p, 1, 32, 64, 257, dt, None) == -3          # d/d feat needs I <= 256


def test_half_workspace_query(lib):
    ws = lib.bxs_dynconv1x1_half_backward_workspace_bytes
    for dt in (F16, BF16):
        assert ws(1, 256, 51200, 16, dt) > 0
        assert ws(2, 128, 900, 300, dt) >= 2 * 2 * 128 * 320          # at least the transposed, padded kernels
        assert ws(0, 256, 51200, 16, dt) == 0 and ws(1, 256, 0, 16, dt) == 0 and ws(1, 256, 51200, 0, dt) == 0
    assert ws(1, 256, 51200, 16, 2) == 0
