"""Golden vectors for the LCM and mean-field regimes the other fixtures leave out, minted from the reference's own
``LCM`` / ``LocalConsistencyModule`` (mmdet/models/losses/levelset_loss.py:64-126) and ``MeanField``
(mmdet/models/dense_heads/discobox_head.py:585-651), AST-extracted like oracle/make_golden.py does.

  * LCM with dilations 1, 3 and 5 and 0 or 3 iterations, on maps larger than, equal to and smaller than the dilation
    (the replicate padding then repeats the border pixel over the whole pad), with flat zero-padded image regions where
    the neighbourhood's standard deviation is 0 and the 1e-8 term decides.  Run in float64 (the module cast with
    ``.double()``): loss, d loss / d phi and the refined map.
  * MeanField with kernel sizes 1, 5 and 7, including a 3x4 map smaller than the 7x7 kernel: the bilateral kernel,
    pseudo-labels and ``valid`` in float32, as the reference computes them.

Asserts the oracle (oracle.levelset) reproduces the reference, writes tests/golden/dispatch_edges.npz.
      python -m oracle.make_golden_dispatch_edges"""
import os

import numpy as np
import torch

from oracle import levelset as ol
from oracle.make_golden import OUT, _Registry, extract

LCM_DILATIONS = (1, 3, 5)
LCM_ITERS = (0, 3)
LCM_SHAPES = ((2, 3, 12, 13), (1, 3, 2, 3), (2, 1, 1, 7), (1, 2, 5, 5))      # (n, C, h, w)
MF_CASES = ((1, 10, 12), (5, 10, 12), (7, 10, 12), (7, 3, 4), (5, 1, 9))      # (kernel_size, h, w)
MF_CFG = dict(theta0=0.5, theta1=30, theta2=10, alpha0=2, iter=10, base=0.1)


def lcm_case(seed, n, C, h, w):
    """imgs with a zero-padded (flat) right part, phis in [0, 1), fractional box targets with an all-zero instance."""
    gen = torch.Generator().manual_seed(seed)
    imgs = torch.rand(n, C, h, w, generator=gen)
    imgs[..., (3 * w) // 4:] = 0
    phis = torch.rand(n, 1, h, w, generator=gen)
    box = (torch.rand(n, 1, h, w, generator=gen) > 0.3).float() * torch.rand(n, 1, h, w, generator=gen)
    if n > 1:
        box[-1] = 0
    return imgs, phis, box


def mf_case(seed, ks, h, w, n=4):
    gen = torch.Generator().manual_seed(seed)
    fm = torch.randn(1, 3, h, w, generator=gen)
    x = torch.rand(n, 1, h, w, generator=gen)
    t = torch.zeros(n, 1, h, w)
    t[0, 0, h // 4: h - h // 4, w // 5: w - w // 5] = 1
    t[1] = 1
    t[2, 0, h // 2, w // 2] = 1
    t[3, 0, :max(h // 2, 1), :] = 1
    return fm, x, t


def main():
    ls = extract('mmdet/models/losses/levelset_loss.py', ['LCM', 'LocalConsistencyModule'], dict(LOSSES=_Registry()))
    db = extract('mmdet/models/dense_heads/discobox_head.py', ['MeanField'])
    out = {}
    worst = 0.0
    for d in LCM_DILATIONS:
        for iters in LCM_ITERS:
            for si, (n, C, h, w) in enumerate(LCM_SHAPES):
                tag = f'lcm_d{d}_i{iters}_s{si}'
                imgs, phis, box = lcm_case(1000 * d + 10 * iters + si, n, C, h, w)
                # the reference's own LCM with its module built for (d, iters) instead of the hard-coded (2, 10)
                ls.LCM.__globals__['LocalConsistencyModule'] = \
                    lambda num_iter, dilations, d=d, iters=iters: ls.LocalConsistencyModule([d], iters).double()
                p64 = phis.double().requires_grad_(True)
                loss = ls.LCM(imgs.double(), p64, box.double())
                (g,) = torch.autograd.grad(loss, p64)
                refined = ls.LocalConsistencyModule([d], iters).double()(imgs.double(), phis.double())
                o64 = phis.double().requires_grad_(True)
                o_loss = ol.lcm_loss(imgs.double(), o64, box.double(), iters, d)
                (o_g,) = torch.autograd.grad(o_loss, o64)
                o_ref = ol.lcm_refine(imgs.double(), phis.double(), iters, d)
                for a, b in ((o_loss, loss), (o_g, g), (o_ref, refined)):
                    err = ((a.detach() - b.detach()).abs().max() / b.detach().abs().max().clamp(min=1e-30)).item()
                    worst = max(worst, err)
                    assert err <= 1e-12, f'{tag}: oracle deviates from the reference, {err:.3e}'
                out.update({f'{tag}_imgs': imgs.numpy(), f'{tag}_phis': phis.numpy(), f'{tag}_box': box.numpy(),
                            f'{tag}_loss': loss.detach().numpy(), f'{tag}_g_phis': g.numpy(),
                            f'{tag}_refined': refined.numpy()})
    ls.LCM.__globals__['LocalConsistencyModule'] = ls.LocalConsistencyModule
    print(f'LCM: {len(LCM_DILATIONS) * len(LCM_ITERS) * len(LCM_SHAPES)} cases, oracle vs reference (float64) {worst:.2e}')
    for ci, (ks, h, w) in enumerate(MF_CASES):
        tag = f'mf_k{ks}_c{ci}'
        fm, x, t = mf_case(ci, ks, h, w)
        mf = db.MeanField(fm, kernel_size=ks, **MF_CFG)
        pseudo, valid = mf(x, t)
        k = ol.meanfield_kernel(fm, ks, 0.5, 30.0, 2.0)
        kr = mf.kernel[:, 0]
        err = ((k - kr).abs() / (1e-9 / 1e-5 + kr.abs())).max().item()
        assert err <= 1e-5, f'{tag}: kernel oracle deviates from the reference, scaled err {err:.3e}'
        o_ps, o_va = ol.meanfield_forward(kr, x, t, ks, 10, 0.1)
        assert torch.equal(o_ps, pseudo) and torch.equal(o_va, valid), f'{tag}: pseudo labels must be bit-exact'
        fg = int(pseudo.sum())
        print(f'{tag}: kernel scaled err {err:.2e}, {fg} foreground pixels, valid {valid.tolist()}')
        out.update({f'{tag}_feature': fm.numpy(), f'{tag}_kernel': kr.numpy(), f'{tag}_x': x.numpy(),
                    f'{tag}_targets': t.numpy(), f'{tag}_pseudo': np.packbits(pseudo.numpy().astype(np.uint8), axis=-1),
                    f'{tag}_valid': valid.numpy()})
    np.savez_compressed(os.path.join(OUT, 'dispatch_edges.npz'), **out)
    print('written', os.path.normpath(os.path.join(OUT, 'dispatch_edges.npz')))


if __name__ == '__main__':
    main()
