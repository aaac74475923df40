"""``encode_mask_results`` (mmdet/core/mask/utils.py:38-65) on the RLE kernels of csrc/mask_rle.cu: the same signature and
the same value, byte for byte, as the reference's loop of ``pycocotools.mask.encode`` calls.

Every mask of a call goes through one ``ops.mask_rle.encode`` per (device, H, W) group, in class order and then detection
order.  Host masks (numpy arrays, CPU tensors) are packed into one pinned staging buffer and uploaded to the current CUDA
device in one non-blocking copy; CUDA masks are stacked on their own device.  An entry that is already an RLE dict is
returned unchanged, so the function is idempotent."""
import numpy as np
import torch

from ..ops import mask_rle

_DTYPES = (np.dtype(np.bool_), np.dtype(np.uint8))


def _is_rle(m):
    return isinstance(m, dict) and 'size' in m and 'counts' in m


def _check(m):
    if isinstance(m, torch.Tensor):
        ok = m.dtype in (torch.bool, torch.uint8)
    else:
        m = np.asarray(m)
        ok = m.dtype in _DTYPES
    if not ok:
        raise TypeError(f'masks must be bool or uint8, got {m.dtype}')
    if m.ndim != 2:
        raise ValueError(f'a mask must be [H, W], got {tuple(m.shape)}')
    return m


def stage(ms):
    """The host 2-D masks ms, all [H, W], packed into one pinned uint8 tensor [n, H, W] (bool as 0 / 1)."""
    H, W = ms[0].shape
    staging = torch.empty((len(ms), H, W), dtype=torch.uint8, pin_memory=True)
    s = staging.numpy()
    for i, m in enumerate(ms):
        s[i] = np.asarray(m)
    return staging


def _encode_group(ms):
    """The RLE dicts of the 2-D masks ms, all of one (device, H, W)."""
    if isinstance(ms[0], torch.Tensor) and ms[0].is_cuda:
        return mask_rle.encode(torch.stack([m.view(torch.uint8) for m in ms]))
    return mask_rle.encode(stage(ms).to(torch.cuda.current_device(), non_blocking=True))


def encode_mask_results(mask_results):
    """Encode bitmap mask results to COCO RLE: a per-class list of masks -> the per-class list of their RLE dicts, or the
    tuple (cls_segms, cls_mask_scores) -> (the encoded cls_segms, cls_mask_scores).  A class entry is anything iterable over
    2-D masks: a list of numpy arrays or tensors (CPU or CUDA), or a [k, H, W] array or tensor.  Masks must be bool or
    uint8 (TypeError otherwise)."""
    if isinstance(mask_results, tuple):
        cls_segms, cls_mask_scores = mask_results
    else:
        cls_segms = mask_results
    encoded = [[] for _ in range(len(cls_segms))]
    groups = {}                                           # (device, H, W) -> [(class, slot)], [masks]
    for i in range(len(cls_segms)):
        for m in cls_segms[i]:
            if _is_rle(m):
                encoded[i].append(m)
                continue
            m = _check(m)
            dev = m.device if isinstance(m, torch.Tensor) and m.is_cuda else None
            slots, ms = groups.setdefault((dev, *m.shape), ([], []))
            slots.append((i, len(encoded[i])))
            ms.append(m)
            encoded[i].append(None)
    for slots, ms in groups.values():
        for (i, j), rle in zip(slots, _encode_group(ms)):
            encoded[i][j] = rle
    if isinstance(mask_results, tuple):
        return encoded, cls_mask_scores
    return encoded
