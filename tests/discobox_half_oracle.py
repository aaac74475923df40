"""Float64 restatement of the DiscoBox mask loss on 16-bit predictions (ops/discobox.py, csrc/discobox_loss.cu), for the
tests.  It takes the ROUNDED scores s = torch.sigmoid(x) (and t of an independent teacher) as given and returns the
per-level sums and the gradient before its final rounding to the logits' dtype."""
import torch
import torch.nn.functional as F

from oracle import levelset as ol


def _dice(x, t):
    return 1 - 2 * (x * t).sum(1) / (((x * x).sum(1) + 1e-3) + ((t * t).sum(1) + 1e-3))


def pseudo_label(s, tg, kernels, img_inds, t=None, num_iter=10, base=0.1, kernel_size=3):
    """Mean-field pseudo-label [n,h,w] of the reference under autocast: x = (t + s) / 2 in the 16-bit dtype, then the
    float32 mean field (oracle.levelset.meanfield_forward) with the bilateral kernel of each instance's image.
    kernels: list of [1,k*k,h*w] (one per image)."""
    t = s if t is None else t
    m = ((t + s) / 2).float()
    tgf = (tg != 0).float()
    out = torch.zeros(tg.shape, dtype=torch.uint8)
    for b, k in enumerate(kernels):
        sel = img_inds == b
        if sel.any():
            p, _ = ol.meanfield_forward(k, m[sel].unsqueeze(1), tgf[sel].unsqueeze(1), kernel_size, num_iter, base)
            out[sel] = p[:, 0].to(torch.uint8)
    return out


def first_argmax(v, dim):
    """First index of the maximum along `dim` (torch.max(dim) on CUDA; documented for argmax)."""
    return torch.argmax(v, dim=dim, keepdim=True)


def disco_half_loss(s, tg, pseudo=None, g_ins=1.0, g_ts=1.0):
    """s [n,h,w]: the rounded scores (any dtype, widened exactly); tg [n,h,w] binary targets; pseudo [n,h,w] in {0,1} or
    None (no teacher-student term).  Returns float64 (num_ins, num_ts, count, g_x): num_ins = sum keep * mil,
    num_ts = sum keep * d_ts (0 without pseudo), count = sum keep, and g_x = g_s * s * (1 - s) with
    g_s = d(g_ins * num_ins + g_ts * num_ts)/ds, the row / column maxima taking their FIRST arg-max."""
    s64 = s.double().detach().requires_grad_(True)
    tgf = (tg != 0).double()
    keep = (tgf.flatten(1).sum(1) > 0).double()
    r = s64.gather(2, first_argmax(s64.detach(), 2)).squeeze(2)      # row profiles [n,h]
    c = s64.gather(1, first_argmax(s64.detach(), 1)).squeeze(1)      # column profiles [n,w]
    mil = _dice(r, tgf.amax(2)) + _dice(c, tgf.amax(1))
    num_ins = (mil * keep).sum()
    num_ts = torch.zeros((), dtype=torch.float64)
    if pseudo is not None:
        enl = F.max_pool2d(tgf.unsqueeze(1), 3, 1, 1).squeeze(1)
        d_ts = _dice((s64 * enl).flatten(1), pseudo.double().flatten(1))
        num_ts = (d_ts * keep).sum()
    (g_s,) = torch.autograd.grad(g_ins * num_ins + g_ts * num_ts, s64)
    sd = s64.detach()
    return num_ins.detach(), num_ts.detach(), keep.sum(), g_s * sd * (1 - sd)
