"""DiscoBox mask loss of one FPN level on float16 / bfloat16 mask logits (the reference trains DiscoBox under autocast,
discobox_head.py:1142): sigmoid, MIL dice (:542-562), mean-field teacher, teacher-student dice and the keep weights of
``DiscoBoxSOLOv2Head.mask_loss``, in a handful of launches (csrc/discobox_loss.cu, ``bxs_meanfield_forward_logits``).

The 16-bit predictions are read as they are: ``s = torch.sigmoid(x)`` bit for bit, the profiles' arg-max on that
rounded ``s``, every sum in float32, and the gradient rounded to the logits' dtype once, after the sigmoid backward."""
import torch

from .. import _lib as L

HALF_DTYPES = {torch.float16: 0, torch.bfloat16: 1}          # bxs_half_t


def _pseudo_label(mf, s, t, tg, img_inds):
    """Mean-field pseudo-label [n,h,w] uint8 of the 16-bit logits, with the bilateral kernel ``mf`` holds."""
    n, h, w = s.shape
    lib = L.lib()
    obj_img = None
    if mf.kernel.shape[0] > 1:
        assert img_inds is not None, 'a multi-image kernel needs img_inds'
        obj_img = img_inds.to(device=s.device, dtype=torch.int32).contiguous()
    pseudo = torch.empty((n, h, w), dtype=torch.uint8, device=s.device)
    ws = torch.empty(max(lib.bxs_meanfield_workspace_bytes(n, h, w), 1), dtype=torch.uint8, device=s.device)
    L.check(lib.bxs_meanfield_forward_logits(L.ptr(mf.kernel), L.ptr(obj_img), L.ptr(s), L.ptr(t), L.ptr(tg),
                                             HALF_DTYPES[s.dtype], mf._neglog.ctypes.data, L.ptr(pseudo), L.ptr(ws),
                                             n, h, w, mf.kernel_size, mf.iter, L.stream()), 'meanfield_forward_logits')
    return pseudo


class _DiscoBoxMaskLoss(torch.autograd.Function):
    @staticmethod
    def forward(ctx, s_logits, targets, img_inds, mf, t_logits, use_loss_ts):
        s = s_logits.contiguous()
        t = None if t_logits is None else t_logits.contiguous()
        tg = targets.contiguous()
        L.require_cuda(s, t, tg)
        n, h, w = s.shape
        lib = L.lib()
        out = torch.empty(3, dtype=torch.float32, device=s.device)
        ws = torch.empty(max(lib.bxs_discobox_loss_workspace_bytes(n, h, w), 1), dtype=torch.uint8, device=s.device)
        with torch.cuda.device(s.device):
            pseudo = _pseudo_label(mf, s, t, tg, img_inds) if use_loss_ts and n else None
            L.check(lib.bxs_discobox_loss_forward(L.ptr(s), L.ptr(tg), L.ptr(pseudo), HALF_DTYPES[s.dtype], L.ptr(ws),
                                                  L.ptr(out), n, h, w, L.stream()), 'discobox_loss_forward')
        ctx.save_for_backward(s, tg, pseudo, ws)
        return out[0], out[1], out[2]

    @staticmethod
    def backward(ctx, g_ins, g_ts, _g_count):
        s, tg, pseudo, ws = ctx.saved_tensors
        n, h, w = s.shape
        g = torch.empty_like(s)
        if n:
            g2 = torch.stack((g_ins, g_ts)).float()
            with torch.cuda.device(s.device):
                L.check(L.lib().bxs_discobox_loss_backward(L.ptr(s), L.ptr(tg), L.ptr(pseudo), HALF_DTYPES[s.dtype],
                                                           L.ptr(ws), L.ptr(g2), L.ptr(g), n, h, w, L.stream()),
                        'discobox_loss_backward')
        return g, None, None, None, None, None


def discobox_mask_loss(s_logits, targets, img_inds, mf, t_logits=None, use_loss_ts=True):
    """One level of ``DiscoBoxSOLOv2Head.mask_loss`` on 16-bit logits.

    s_logits [n,h,w] float16 or bfloat16 (the student's mask logits); targets [n,h,w] binary (uint8, or anything that
    becomes uint8 with one ``ne(0)``); img_inds [n] (image of each instance, for a multi-image ``mf``); mf: the
    ``MeanField`` whose bilateral kernels the pseudo-label uses (may be None when ``use_loss_ts`` is False); t_logits:
    independent-teacher logits of the same dtype, or None (the teacher is the student, detached).
    Returns float32 scalars (num_ins, num_ts, count) = (sum keep * mil, sum keep * d_ts, sum keep), keep = 0 for an
    all-zero target; num_ts is 0 without the teacher term.  Differentiable in ``s_logits`` only; the gradient comes back
    in its dtype."""
    if s_logits.dtype not in HALF_DTYPES:
        raise TypeError(f'discobox_mask_loss takes float16 or bfloat16 logits, not {s_logits.dtype}')
    if t_logits is not None and t_logits.dtype != s_logits.dtype:
        raise TypeError(f'teacher logits are {t_logits.dtype}, student logits {s_logits.dtype}')
    if use_loss_ts and mf is None:
        raise ValueError('the teacher-student term needs a MeanField')
    if targets.dtype != torch.uint8:
        targets = targets.ne(0).view(torch.uint8)
    if t_logits is not None:
        t_logits = t_logits.detach()
    return _DiscoBoxMaskLoss.apply(s_logits, targets, img_inds, mf, t_logits, bool(use_loss_ts))
