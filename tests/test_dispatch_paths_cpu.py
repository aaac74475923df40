"""The float64 oracle of the LCM and the mean field (oracle.levelset) pinned on the reference's own classes in the regimes
that only the less common launch paths reach: LCM dilations 1, 3 and 5 with 0 or 3 iterations on maps as small as or
smaller than the dilation and on flat image regions, and mean-field kernel sizes 1, 5 and 7 including a map smaller than
the kernel.  The vectors are minted by oracle/make_golden_dispatch_edges.py; the GPU tests of those paths
(tests/test_dispatch_paths_gpu.py) are judged against this oracle."""
import numpy as np
import pytest
import torch

from oracle import levelset as ol
from oracle.make_golden_dispatch_edges import LCM_DILATIONS, LCM_ITERS, LCM_SHAPES, MF_CASES

T = torch.from_numpy


@pytest.mark.parametrize('si', range(len(LCM_SHAPES)))
@pytest.mark.parametrize('iters', LCM_ITERS)
@pytest.mark.parametrize('d', LCM_DILATIONS)
def test_lcm_oracle_vs_reference(golden, d, iters, si):
    g = golden('dispatch_edges')
    tag = f'lcm_d{d}_i{iters}_s{si}'
    imgs, phis, box = (T(g[f'{tag}_{k}']).double() for k in ('imgs', 'phis', 'box'))
    assert tuple(imgs.shape) == LCM_SHAPES[si]
    p = phis.clone().requires_grad_(True)
    loss = ol.lcm_loss(imgs, p, box, iters, d)
    (gp,) = torch.autograd.grad(loss, p)
    refined = ol.lcm_refine(imgs, phis, iters, d)
    assert torch.allclose(loss.detach(), T(g[f'{tag}_loss']), rtol=1e-12, atol=1e-15)
    assert torch.allclose(gp, T(g[f'{tag}_g_phis']), rtol=1e-12, atol=1e-15)
    assert torch.allclose(refined, T(g[f'{tag}_refined']), rtol=1e-12, atol=1e-15)
    if iters == 0:
        assert float(loss.detach()) == 0.0 and not gp.any() and torch.equal(refined, phis)
    assert (imgs[..., -1] == 0).all()                                  # a flat (std 0) image region is part of every case


@pytest.mark.parametrize('ci', range(len(MF_CASES)))
def test_meanfield_oracle_vs_reference(golden, ci):
    g = golden('dispatch_edges')
    ks, h, w = MF_CASES[ci]
    tag = f'mf_k{ks}_c{ci}'
    fm, kr, x, t = (T(g[f'{tag}_{k}']) for k in ('feature', 'kernel', 'x', 'targets'))
    k = ol.meanfield_kernel(fm, ks, 0.5, 30.0, 2.0)
    assert k.shape == kr.shape == (1, ks * ks, h * w)
    assert torch.allclose(k, kr, rtol=1e-5, atol=1e-9)
    ps, va = ol.meanfield_forward(kr, x, t, ks, 10, 0.1)
    want = np.unpackbits(g[f'{tag}_pseudo'], axis=-1)[..., :w]
    assert np.array_equal(ps.numpy().astype(np.uint8), want)          # binary output: exact
    assert torch.equal(va, T(g[f'{tag}_valid']))
