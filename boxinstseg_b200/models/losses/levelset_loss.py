"""``LevelsetLoss`` / ``region_levelset`` / ``length_regularization`` -- registry drop-ins for
mmdet/models/losses/levelset_loss.py:7-60, computed by libboxseg_b200 (the region energy: one cluster launch
forward, one launch backward with an analytic gradient; no [n,C,h,w] temporaries)."""
import torch
import torch.nn as nn

from ... import _lib as L
from ..builder import LOSSES, register


class _LevelsetFused(torch.autograd.Function):
    """One launch forward (a cluster of 8 CTAs per instance, the means -> energy dependency through distributed shared
    memory), one launch backward.  mode 1 = the whole assembly of box_solov2_head.py:341-360 / box2mask_head.py:305-327
    from (logits, box mask, raw targets); mode 0 = LevelsetLoss.forward / region_levelset on dense (scores2, targets,
    pixel_num)."""

    @staticmethod
    def forward(ctx, x, y, targets, pixel_num, loss_weight, mode):
        xs = x.contiguous().float()
        ys = y.contiguous().float() if y is not None else None
        t = targets.contiguous().float()
        p = pixel_num.contiguous().float() if pixel_num is not None else None
        L.require_cuda(xs, ys, t, p)
        n, C, h, w = t.shape
        assert mode != 0 or xs.shape == (n, 2, h, w)
        lib = L.lib()
        loss = torch.empty(n, dtype=torch.float32, device=t.device)
        ws = torch.empty(max(lib.bxs_levelset_fused_workspace_bytes(n), 1), dtype=torch.uint8, device=t.device)
        if n:
            with torch.cuda.device(t.device):
                L.check(lib.bxs_levelset_fused_forward(L.ptr(xs), L.ptr(ys), L.ptr(t), L.ptr(p), L.ptr(loss), L.ptr(ws), n, C, h,
                                                       w, float(loss_weight), mode, L.stream()), 'levelset_fused_forward')
        ctx.save_for_backward(xs, ys, t, ws)
        ctx.cfg = (float(loss_weight), mode)
        return loss

    @staticmethod
    def backward(ctx, g_loss):
        xs, ys, t, ws = ctx.saved_tensors
        loss_weight, mode = ctx.cfg
        n, C, h, w = t.shape
        need_x, need_t = ctx.needs_input_grad[0], ctx.needs_input_grad[2]
        gx = torch.empty_like(xs) if need_x else None
        gt = torch.empty_like(t) if need_t else None
        if n and (need_x or need_t):
            with torch.cuda.device(t.device):
                L.check(L.lib().bxs_levelset_fused_backward(L.ptr(xs), L.ptr(ys), L.ptr(t), L.ptr(ws),
                                                            L.ptr(g_loss.contiguous().float()), L.ptr(gx), L.ptr(gt), n, C, h, w,
                                                            loss_weight, mode, L.stream()), 'levelset_fused_backward')
        return gx, None, gt, None, None, None


def levelset_assembly(mask_logits, box_mask, targets, loss_weight=1.0):
    """loss [n] = LevelsetLoss(cat(s, 1 - s) * box, targets * box, clamp(sum box, 1)) with s = sigmoid(mask_logits):
    mask_logits, box_mask [n,h,w] (or [n,1,h,w]), targets [n,C,h,w] raw (NOT yet multiplied by the box mask).
    box_solov2_head.py:341-351,357-360; box2mask_head.py:305-312,322-327."""
    n, C, h, w = targets.shape
    return _LevelsetFused.apply(mask_logits.reshape(n, h, w), box_mask.reshape(n, h, w), targets, None, loss_weight, 1)


class _LengthReg(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scores):
        s = scores.contiguous().float()
        L.require_cuda(s)
        n, C, h, w = s.shape
        out = torch.empty(n, dtype=torch.float32, device=s.device)
        ws = torch.empty(max(n, 1) * 64, dtype=torch.float32, device=s.device)
        if n:
            with torch.cuda.device(s.device):
                L.check(L.lib().bxs_length_reg_forward(L.ptr(s), L.ptr(out), L.ptr(ws), n, C, h, w, L.stream()),
                        'length_reg_forward')
        ctx.save_for_backward(s)
        return out

    @staticmethod
    def backward(ctx, g_out):
        (s,) = ctx.saved_tensors
        n, C, h, w = s.shape
        g = torch.empty_like(s)
        if n:
            with torch.cuda.device(s.device):
                L.check(L.lib().bxs_length_reg_backward(L.ptr(s), L.ptr(g_out.contiguous().float()), L.ptr(g), n, C, h,
                                                        w, L.stream()), 'length_reg_backward')
        return g


class region_levelset(nn.Module):
    """mask_score [n,2,h,w], lst_target [n,C,h,w] -> energy [n] (levelset_loss.py:21-44)."""

    def forward(self, mask_score, lst_target):
        ones = torch.ones(mask_score.shape[0], dtype=torch.float32, device=mask_score.device)
        return _LevelsetFused.apply(mask_score, None, lst_target, ones, 1.0, 0)


class length_regularization(nn.Module):
    """levelset_loss.py:47-60 (defined by the reference, never called by its heads)."""

    def forward(self, mask_score):
        return _LengthReg.apply(mask_score)


@register(LOSSES)
class LevelsetLoss(nn.Module):
    def __init__(self, loss_weight=1.0):
        super().__init__()
        self.loss_weight = loss_weight

    def forward(self, mask_logits, targets, pixel_num):
        return _LevelsetFused.apply(mask_logits, None, targets, pixel_num, self.loss_weight, 0)


class _LCM(torch.autograd.Function):
    @staticmethod
    def forward(ctx, imgs, phis, box, dilation, num_iter):
        im = imgs.contiguous().float()
        ph = phis.contiguous().float()
        bx = box.contiguous().float()
        L.require_cuda(im, ph, bx)
        n, C, h, w = im.shape
        assert ph.shape == (n, 1, h, w) and bx.shape == (n, 1, h, w)
        lib = L.lib()
        out = torch.zeros(1, dtype=torch.float32, device=im.device)
        ws = torch.empty(max(lib.bxs_lcm_workspace_bytes(n, h, w), 4), dtype=torch.uint8, device=im.device)
        if n:
            with torch.cuda.device(im.device):
                L.check(lib.bxs_lcm_forward(L.ptr(im), L.ptr(ph), L.ptr(bx), L.ptr(out), L.ptr(ws), n, C, h, w,
                                            dilation, num_iter, L.stream()), 'lcm_forward')
        ctx.save_for_backward(ph, bx, ws)
        ctx.cfg = (dilation, num_iter)
        return out[0]

    @staticmethod
    def backward(ctx, g):
        ph, bx, ws = ctx.saved_tensors
        n, _, h, w = ph.shape
        gp = torch.zeros_like(ph)
        if n:
            with torch.cuda.device(ph.device):
                L.check(L.lib().bxs_lcm_backward(L.ptr(ph), L.ptr(bx), L.ptr(ws), L.ptr(g.reshape(1).contiguous().float()),
                                                 L.ptr(gp), n, h, w, ctx.cfg[0], ctx.cfg[1], L.stream()), 'lcm_backward')
        return None, gp, None, None, None


class LocalConsistencyModule(nn.Module):
    """levelset_loss.py:74-126: ``forward(imgs, masks)`` returns the masks after ``num_iter`` rounds of affinity-weighted
    neighbour averaging (dilation 2, 8 neighbours, alpha 0.3) -- the refined phi the ``LCM`` loss compares with its input.
    Runs the same kernels as ``LCM`` (bxs_lcm_forward) and reads the refined map out of their workspace; no autograd
    node (the differentiable entry point is ``LCM``, which is what Box2MaskHead.loss_single calls, box2mask_head.py:331)."""

    def __init__(self, dilations, num_iter):
        super().__init__()
        assert len(dilations) == 1, 'the reference only ever uses dilations=[2]'
        self.dilations = dilations
        self.num_iter = num_iter
        self.alpha = 0.3

    @torch.no_grad()
    def forward(self, imgs, masks):
        im = imgs.contiguous().float()
        ph = masks.contiguous().float()
        L.require_cuda(im, ph)
        n, C, h, w = im.shape
        assert ph.shape == (n, 1, h, w)
        lib = L.lib()
        out = torch.zeros(1, dtype=torch.float32, device=im.device)
        ws = torch.empty(max(lib.bxs_lcm_workspace_bytes(n, h, w), 4), dtype=torch.uint8, device=im.device)
        if n == 0:
            return ph
        with torch.cuda.device(im.device):
            L.check(lib.bxs_lcm_forward(L.ptr(im), L.ptr(ph), L.ptr(torch.ones_like(ph)), L.ptr(out), L.ptr(ws), n, C, h, w,
                                        self.dilations[0], self.num_iter, L.stream()), 'lcm_forward')
        hw = h * w
        return ws.view(torch.float32)[n * 8 * hw: n * 9 * hw].view(n, 1, h, w).clone()     # phi_T of the workspace layout


def LCM(imgs, pred_phis, box_targets):
    """local consistency loss, levelset_loss.py:64-71 (num_iter=10, dilations=[2])."""
    return _LCM.apply(imgs, pred_phis, box_targets, 2, 10)
