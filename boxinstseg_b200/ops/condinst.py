"""a1: CondInst dynamic mask head on the C ABI (replaces CondInstMaskHead.forward,
mmdet/models/dense_heads/condinst_head.py:1139-1164; differentiable wrt mask_feat and params)."""
import torch

from .. import _lib as L


class _DynamicMaskHead(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, params, coors, soi, img_inds, in_stride, factor, rel):
        feat = feat.contiguous().float()
        params = params.contiguous().float()
        L.require_cuda(feat, params, coors, soi, img_inds)
        N, P = params.shape
        B, C, h, w = feat.shape
        out = torch.empty((N, 1, factor * h, factor * w), dtype=torch.float32, device=feat.device)
        if N:
            with torch.cuda.device(feat.device):
                L.check(L.lib().bxs_condinst_head_forward(L.ptr(feat), L.ptr(params), L.ptr(coors), L.ptr(soi),
                                                          L.ptr(img_inds), L.ptr(out), N, B, C, h, w, P, in_stride,
                                                          factor, int(rel), L.stream()), 'condinst_head_forward')
        ctx.save_for_backward(feat, params, coors, soi, img_inds)
        ctx.cfg = (in_stride, factor, int(rel))
        return out

    @staticmethod
    def backward(ctx, g_out):
        feat, params, coors, soi, img_inds = ctx.saved_tensors
        in_stride, factor, rel = ctx.cfg
        N, P = params.shape
        B, C, h, w = feat.shape
        g_feat = torch.empty_like(feat)
        g_params = torch.empty_like(params)
        if N == 0:
            return g_feat.zero_(), g_params, None, None, None, None, None, None
        g_out = g_out.contiguous().float()
        lib = L.lib()
        ws = torch.empty(lib.bxs_condinst_head_workspace_bytes(N, B, h, w, P), dtype=torch.uint8, device=feat.device)
        with torch.cuda.device(feat.device):
            L.check(lib.bxs_condinst_head_backward(L.ptr(feat), L.ptr(params), L.ptr(coors), L.ptr(soi),
                                                   L.ptr(img_inds), L.ptr(g_out), L.ptr(g_feat), L.ptr(g_params),
                                                   L.ptr(ws), N, B, C, h, w, P, in_stride, factor, rel, L.stream()),
                    'condinst_head_backward')
        return g_feat, g_params, None, None, None, None, None, None


def dynamic_mask_head(feat, params, coors, level_inds, img_inds, sizes_of_interest, in_stride=8, out_stride=4,
                      channels=8, num_layers=3, rel_coors=True):
    """feat [B,C,h,w], params [N,P], coors [N,2], level_inds/img_inds [N] -> mask logits [N,1,f*h,f*w]."""
    if channels != 8 or num_layers != 3:
        raise NotImplementedError('libboxseg_b200 implements dynamic_channels=8, dynamic_convs=3 '
                                  '(every CondInst/BoxInst config of the reference)')
    if feat.shape[1] > 32:
        raise NotImplementedError('mask_feat channels > 32')
    dev = feat.device
    soi = sizes_of_interest.to(device=dev, dtype=torch.float32)[level_inds.long()].contiguous() if rel_coors else None
    coors = coors.to(device=dev, dtype=torch.float32).contiguous() if rel_coors else None
    img32 = img_inds.to(device=dev, dtype=torch.int32).contiguous()
    return _DynamicMaskHead.apply(feat, params, coors, soi, img32, in_stride, in_stride // out_stride, rel_coors)


def paste_masks(mask_logits, factor, img_shape, ori_shape=None):
    """The mask lines of CondInstMaskHead.simple_test (condinst_head.py:1261-1281) in one pass: mask_logits [n,1,h,w] ->
    bool [n, H, W] = aligned_bilinear(sigmoid(mask_logits), factor)[:, :, :H_img, :W_img] > 0.5, resized bilinearly
    (align_corners=False) to ``ori_shape[:2]`` before the threshold when ``ori_shape`` is given (``rescale=True``)."""
    n, _, h, w = mask_logits.shape
    logits = mask_logits.detach().float().contiguous()
    L.require_cuda(logits)
    H_img, W_img = [int(v) for v in img_shape[:2]]
    H, W = [int(v) for v in ori_shape[:2]] if ori_shape is not None else (H_img, W_img)
    out = torch.empty((n, H, W), dtype=torch.bool, device=logits.device)
    with torch.cuda.device(logits.device):
        L.check(L.lib().bxs_condinst_paste_masks(L.ptr(logits), n, h, w, int(factor), H_img, W_img, H, W,
                                                 int(ori_shape is not None), L.ptr(out), L.stream()), 'condinst_paste_masks')
    return out
