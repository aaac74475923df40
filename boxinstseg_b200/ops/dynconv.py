"""a2/a3/a4: dense dynamic 1x1 convolution ``out[b,i] = sum_c kernel[b,i,c] * feat[b,c]`` on Hopper wgmma.

Forward is the hand-written TMA + wgmma (TF32, FP32 accumulate in registers) kernel of libboxseg_b200.
Backward is the same machinery (bxs_dynconv1x1_backward): d/d feat = kernel^T . g_out re-uses the forward kernel with
the operand roles swapped, d/d kernel = g_out . feat^T is a split-K wgmma kernel over the pixels with an ordered
(deterministic) reduction of the partials.  Only d/d feat with more than 256 kernels per image (outside every reference
call site: the heads convolve the POSITIVE kernels of an image) goes through cuBLAS (torch.bmm).
"""
import torch

from .. import _lib as L


class _DynConv1x1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, kernels):
        f = feat.contiguous().float()
        k = kernels.contiguous().float()
        L.require_cuda(f, k)
        B, C, h, w = f.shape
        assert k.dim() == 3 and k.shape[0] == B and k.shape[2] == C, 'kernels must be [B,I,C]'
        I = k.shape[1]
        out = torch.empty((B, I, h, w), dtype=torch.float32, device=f.device)
        if B and I:
            with torch.cuda.device(f.device):
                L.check(L.lib().bxs_dynconv1x1_forward(L.ptr(f), L.ptr(k), L.ptr(out), B, C, h * w, I, L.stream()),
                        'dynconv1x1_forward')
        ctx.save_for_backward(f, k)
        return out

    @staticmethod
    def backward(ctx, g_out):
        f, k = ctx.saved_tensors
        B, C, h, w = f.shape
        I = k.shape[1]
        need_f, need_k = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (B and I) or not (need_f or need_k):
            return (torch.zeros_like(f) if need_f else None), (torch.zeros_like(k) if need_k else None)
        g = g_out.contiguous().float()
        gf = gk = None
        native_f = need_f and I <= 256
        if need_f and not native_f:
            gf = torch.bmm(k.transpose(1, 2), g.flatten(2)).view(B, C, h, w)
        if native_f or need_k:
            gf = torch.empty_like(f) if native_f else gf
            gk = torch.empty_like(k) if need_k else None
            with torch.cuda.device(f.device):
                ws = torch.empty(L.lib().bxs_dynconv1x1_backward_workspace_bytes(B, C, h * w, I), dtype=torch.uint8,
                                 device=f.device)
                L.check(L.lib().bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), L.ptr(gf) if native_f else None,
                                                        L.ptr(gk), L.ptr(ws), B, C, h * w, I, L.stream()),
                        'dynconv1x1_backward')
        return gf, gk


def dynconv1x1(feat, kernels):
    """feat [B,C,h,w], kernels [B,I,C] -> [B,I,h,w]   (C % 32 == 0, C <= 256, h*w % 4 == 0)."""
    return _DynConv1x1.apply(feat, kernels)


def solo_dynamic_conv(feature_pred, kernel_pred):
    """BoxSOLOv2 call site (box_solov2_head.py:204-211): feature_pred [B,C,h,w], kernel_pred [B,C,S,S]
    -> [B,S*S,h,w] with cell s = gy*S+gx (the reference's permute(0,2,3,1).view(-1,C) order)."""
    B, C, S, _ = kernel_pred.shape
    return dynconv1x1(feature_pred, kernel_pred.permute(0, 2, 3, 1).reshape(B, S * S, C))


def box2mask_mask_pred(mask_embed, mask_feature):
    """Box2Mask call site (box2mask_head.py:345): einsum('bqc,bchw->bqhw')."""
    return dynconv1x1(mask_feature, mask_embed)
