"""a4: Box2Mask's cross-attention mask (box2mask_head.py:346-355, and the reset of the forward loop, :397) as one launch of
``bxs_box2mask_attn_mask`` (csrc/box2mask_attn.cu)."""
import torch

from .. import _lib as L

_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}        # bxs_attn_dtype_t


def attention_mask(mask_pred, size, num_heads, reset_full_rows=False):
    """mask_pred [B,Q,H,W] float32 / float16 / bfloat16 CUDA -> torch.bool [B*num_heads, Q, h*w], bit for bit

        m = F.interpolate(mask_pred, size, mode='bilinear', align_corners=False)
        m = m.flatten(2).unsqueeze(1).repeat((1, num_heads, 1, 1)).flatten(0, 1)
        m = m.sigmoid() < 0.5

    with the interpolation of ``ops.resize.bilinear_resize`` and, for 16-bit inputs, torch's rounding to that dtype after
    the interpolation and after the sigmoid.  ``reset_full_rows``: a row that is all True comes back all False (what
    ``attn_mask[torch.where(attn_mask.sum(-1) == attn_mask.shape[-1])] = False`` does), without a host synchronisation.
    No autograd: the reference detaches the mask."""
    if mask_pred.dtype not in _DTYPES:
        raise TypeError(f'attention_mask: mask_pred must be float32, float16 or bfloat16, got {mask_pred.dtype}')
    x = mask_pred.detach().contiguous()
    L.require_cuda(x)
    h, w = (int(size), int(size)) if isinstance(size, int) else (int(size[0]), int(size[1]))
    B, Q, H, W = x.shape
    out = torch.empty((B * num_heads, Q, h * w), dtype=torch.bool, device=x.device)
    with torch.cuda.device(x.device):
        L.check(L.lib().bxs_box2mask_attn_mask(L.ptr(x), L.ptr(out), B, Q, H, W, h, w, num_heads, _DTYPES[x.dtype],
                                               int(bool(reset_full_rows)), L.stream()), 'box2mask_attn_mask')
    return out
