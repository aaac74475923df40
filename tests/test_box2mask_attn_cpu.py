"""CPU: Box2Mask's attention-mask oracle (oracle/box2mask_head.py) against the golden vectors minted from the reference's own
``forward_head`` / ``forward``; the C entry point bxs_box2mask_attn_mask is exported and rejects bad arguments before any
device call; the op's dtype and device errors; the head's error without the reference's modules."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import box2mask_head as ob

SEEDS = (0, 1)


def _unpack(packed, n):
    return torch.from_numpy(np.unpackbits(packed, axis=-1, count=n).astype(bool))


@pytest.mark.parametrize('seed', SEEDS)
def test_oracle_attention_lines_against_golden(golden, seed):
    g = golden('box2mask_attn')
    heads = int(g[f's{seed}_heads'])
    i = 0
    while f's{seed}_mask_pred{i}' in g:
        size = tuple(int(v) for v in g[f's{seed}_size{i}'])
        mp = torch.from_numpy(g[f's{seed}_mask_pred{i}'])
        attn = ob.attention_mask(mp, size, heads)
        assert torch.equal(attn, _unpack(g[f's{seed}_attn{i}'], size[0] * size[1]))
        if f's{seed}_given{i}' in g:
            assert torch.equal(ob.reset_full_rows(attn), _unpack(g[f's{seed}_given{i}'], size[0] * size[1]))
        i += 1
    assert i == 5


@pytest.mark.parametrize('seed', SEEDS)
def test_oracle_decoder_loop_against_golden(golden, seed):
    """The restated loop on the seeded stand-ins reproduces the reference's head outputs and the masks its layers got."""
    g = golden('box2mask_attn')
    attrs, feats = ob.standins(seed)
    m = ob.attach(torch.nn.Module(), attrs)
    with torch.no_grad():
        outs, given, _ = ob.forward(m, feats, feats[0].shape[0])
    for i, o in enumerate(outs):
        size = tuple(int(v) for v in g[f's{seed}_size{i}'])
        assert tuple(o[1].shape[-2:]) == (16, 16) and o[2].shape[-1] == size[0] * size[1]
        torch.testing.assert_close(o[1], torch.from_numpy(g[f's{seed}_mask_pred{i}']), rtol=1e-5, atol=1e-5)
        assert torch.equal(o[2], _unpack(g[f's{seed}_attn{i}'], o[2].shape[-1]))
    for i, m_ in enumerate(given):
        assert torch.equal(m_, _unpack(g[f's{seed}_given{i}'], m_.shape[-1]))


def test_reset_full_rows_semantics():
    a = torch.tensor([[[True, True, True], [True, False, True], [False, False, False]]])
    assert torch.equal(ob.reset_full_rows(a), torch.tensor([[[False, False, False], [True, False, True],
                                                             [False, False, False]]]))


@pytest.fixture(scope='module')
def lib():
    from boxinstseg_b200 import _lib, build
    import os
    if not os.path.exists(_lib.LIB_PATH):
        build.build()
    return _lib


def test_entry_point_is_exported(lib):
    assert 'bxs_box2mask_attn_mask' in lib.SIGNATURES
    assert hasattr(ctypes.CDLL(lib.LIB_PATH), 'bxs_box2mask_attn_mask')


def test_argument_validation_without_gpu(lib):
    """Every check runs before any device call: -1 for invalid arguments, -3 for shapes outside the kernel, 0 for B*Q == 0."""
    f = lib.lib().bxs_box2mask_attn_mask
    p = ctypes.cast((ctypes.c_float * 64)(), ctypes.c_void_p)
    ok = (1, 4, 16, 16, 8, 8, 8, 0, 1)                         # B, Q, H, W, h, w, heads, dtype, reset
    assert f(None, p, *ok, None) == -1
    assert f(p, None, *ok, None) == -1
    for k, bad in ((0, -1), (1, -1), (2, 0), (3, 0), (4, 0), (5, 0), (6, 0), (7, 3), (7, -1)):
        args = list(ok)
        args[k] = bad
        assert f(p, p, *args, None) == -1, (k, bad)
    assert f(None, None, 0, 4, 16, 16, 8, 8, 8, 0, 1, None) == 0           # B*Q == 0: no-op, no pointer needed
    assert f(None, None, 2, 0, 16, 16, 8, 8, 8, 2, 0, None) == 0
    assert f(p, p, 1, 4, 16, 16, 1 << 24, 1, 8, 0, 1, None) == -3         # a side >= 2^24
    assert f(p, p, 1, 4, 16, 16, 2048, 2048, 1, 1, 1, None) == -3         # a row larger than 8 CTAs of shared memory
    assert f(p, p, 1 << 40, 1 << 20, 16, 16, 8, 8, 8, 0, 1, None) == -3   # element count above INT64_MAX


def test_op_rejects_other_dtypes_and_cpu_tensors(lib):
    from boxinstseg_b200.ops.box2mask import attention_mask
    with pytest.raises(TypeError):
        attention_mask(torch.zeros(1, 2, 4, 4, dtype=torch.float64), (2, 2), 8)
    with pytest.raises(TypeError):
        attention_mask(torch.zeros(1, 2, 4, 4, dtype=torch.int32), (2, 2), 8)
    with pytest.raises(RuntimeError):
        attention_mask(torch.zeros(1, 2, 4, 4), (2, 2), 8)


def test_head_without_reference_modules_raises():
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import Box2MaskHead
    head = Box2MaskHead()
    with pytest.raises(RuntimeError, match='transformer_decoder'):
        head.forward_head(torch.zeros(4, 1, 32), torch.zeros(1, 32, 8, 8), (4, 4))
