"""The float64 logit-arg-max projection oracle (oracle.boxinst.projection_losses_logit_argmax), which the GPU tie tests
judge the BoxInst kernels against: equal to the score-based oracle where nothing ties, and on exact ties its gradient
lands on the first index of every row and column, with -0 and +0 equal."""
import numpy as np
import torch

from oracle import boxinst as ob


def _box_targets(n, h, w):
    t = torch.zeros(n, 1, h, w, dtype=torch.float64)
    for i in range(n):
        t[i, 0, i % h: h - 1, 1 + i % 3: w - 2] = 1.0
    return t


def _first_argmax_mask(x):
    """Brute force with numpy (first occurrence of the maximum, -0 == +0), independent of torch.max."""
    a = x.detach().numpy()[:, 0]
    m = np.zeros(a.shape, dtype=bool)
    for i in range(a.shape[0]):
        for y in range(a.shape[1]):
            m[i, y, int(np.argmax(a[i, y]))] = True
        for c in range(a.shape[2]):
            m[i, int(np.argmax(a[i, :, c])), c] = True
    return torch.from_numpy(m)[:, None]


def _grad(fn, x, t):
    x = x.clone().requires_grad_(True)
    out = fn(x, t)
    (g,) = torch.autograd.grad((out * torch.arange(1, out.numel() + 1, dtype=out.dtype)).sum(), x)
    return out.detach(), g


def test_untied_inputs_match_the_score_oracle():
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(4, 1, 19, 23, generator=gen, dtype=torch.float64) * 3
    t = _box_targets(4, 19, 23)
    v_new, g_new = _grad(ob.projection_losses_logit_argmax, x, t)
    v_old, g_old = _grad(lambda a, b: ob.projection_losses(a.sigmoid(), b), x, t)
    assert torch.allclose(v_new, v_old, rtol=1e-14, atol=0)
    assert torch.allclose(g_new, g_old, rtol=1e-12, atol=1e-300)
    assert torch.equal(g_new != 0, _first_argmax_mask(x))


def _tied_cases():
    gen = torch.Generator().manual_seed(1)
    up = ob.aligned_bilinear(torch.randn(3, 1, 8, 10, generator=gen) * 3, 2)        # rows 0/1 and columns 0/1 equal
    yield 'upsample', up
    yield 'fp16', (torch.randn(3, 1, 16, 40, generator=gen) * 3).half().float()
    yield 'quarter', torch.round(torch.randn(3, 1, 16, 20, generator=gen) * 8) / 4
    yield 'constant', torch.full((2, 1, 9, 12), 0.7)
    sz = -(torch.rand(2, 1, 12, 16, generator=gen) + 0.5)                          # all negative ...
    sz[0, 0, 2, 3], sz[0, 0, 2, 9] = -0.0, 0.0                                      # ... row 2: -0 before +0
    sz[1, 0, 1, 5], sz[1, 0, 10, 5] = -0.0, 0.0                                     # ... column 5: -0 above +0
    yield 'signed_zero', sz


def test_tied_inputs_send_the_gradient_to_the_first_index():
    for name, x in _tied_cases():
        x = x.double()
        t = _box_targets(x.shape[0], x.shape[2], x.shape[3])
        _, g = _grad(ob.projection_losses_logit_argmax, x, t)
        first = _first_argmax_mask(x)
        assert torch.equal(g != 0, first), name
        assert torch.equal(ob.logit_argmax_mask(x), first), name
    _, _, _, _, (_, sz) = _tied_cases()
    sz = sz.double()
    assert sz.max(dim=3)[1][0, 0, 2] == 3                 # the -0 wins its row: it comes first
    assert sz.max(dim=2)[1][1, 0, 5] == 1                 # and its column
    assert ob.logit_argmax_mask(torch.full((1, 1, 5, 7), 2.0))[0, 0].nonzero().tolist() == \
        [[0, c] for c in range(7)] + [[r, 0] for r in range(1, 5)]      # constant map: row 0 and column 0
