"""Dense masks of axis-aligned rectangles on the device, on the kernel of csrc/box_masks.cu: ``out[g, y, x] = (y0 <= y < y1)
and (x0 <= x < x1)`` for the rectangle ``(y0, x0, y1, x1)`` of mask g.  The rectangles are HOST arrays that travel in the
kernel parameters, so a call copies nothing to the device and never waits on it."""
import numpy as np
import torch

from .. import _lib as L

# dtype -> (element bytes, bit pattern of 1); every other dtype is written as uint8 and converted with ``.to(dtype)``
ONE_BITS = {torch.uint8: (1, 1), torch.bool: (1, 1), torch.int8: (1, 1), torch.int16: (2, 1),
            torch.float16: (2, 0x3C00), torch.bfloat16: (2, 0x3F80), torch.int32: (4, 1), torch.float32: (4, 0x3F800000)}


def rasterize(rects, sizes, dtype=torch.uint8, device=None):
    """``rects[b]``: image b's host rectangles, an integer ``[G_b, 4]`` array of ``(y0, x0, y1, x1)`` with ``0 <= y0 <= y1
    <= H_b`` and ``0 <= x0 <= x1 <= W_b``; ``sizes[b] = (H_b, W_b)`` -> the list of dense ``[G_b, H_b, W_b]`` tensors of
    ``dtype`` on the CUDA ``device`` (default: the current one), with 1 inside each rectangle and 0 elsewhere.  One launch
    chain for the whole batch on the device's current stream.  A rectangle out of that order raises ``BoxSegError``."""
    device = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
    if device.type != 'cuda':
        raise RuntimeError(f'box_masks.rasterize: device must be a CUDA device, got {device}')
    dtype = torch.uint8 if dtype is None else dtype
    if len(rects) != len(sizes):
        raise ValueError(f'box_masks.rasterize: {len(rects)} rectangle arrays but {len(sizes)} sizes')
    es, one = ONE_BITS.get(dtype, ONE_BITS[torch.uint8])
    kind = dtype if dtype in ONE_BITS else torch.uint8
    table = [np.asarray(r, dtype=np.int64).reshape(-1, 4) for r in rects]
    shape = np.array([(len(r), int(h), int(w)) for r, (h, w) in zip(table, sizes)], dtype=np.int64).reshape(-1, 3)
    if any((r < np.iinfo(np.int32).min).any() or (r > np.iinfo(np.int32).max).any() for r in table):
        raise L.BoxSegError('box_masks.rasterize: invalid argument (a rectangle outside the int32 range)')
    with torch.cuda.device(device):
        outs = [torch.empty(tuple(int(v) for v in s), dtype=kind, device=device) for s in shape]
        if outs:
            flat = np.ascontiguousarray(np.concatenate(table).astype(np.int32))
            ptrs = np.array([o.data_ptr() if o.numel() else 0 for o in outs], dtype=np.uint64)
            L.check(L.lib().bxs_box_masks_rasterize(ptrs.ctypes.data, flat.ctypes.data, shape.ctypes.data, len(outs), es,
                                                    one, L.stream()), 'box_masks.rasterize')
    return outs if kind is dtype else [o.to(dtype) for o in outs]
