"""COCO RLE of instance masks on the kernels of csrc/mask_rle.cu: pycocotools' ``mask.encode`` (maskApi.c rleEncode +
rleToString), byte for byte, for a whole batch of device masks at once.

``rle_counts`` gives the uncompressed RLE on the device; ``encode`` the ``{'size', 'counts'}`` dicts of pycocotools.  A call
waits on the host at most twice: once to read the total run count, which sizes the counts exactly and bounds the characters
at 6 per run, and once (``encode``) to end the copy of the characters and their offsets to pinned host memory."""
import torch

from .. import _lib as L


def _check(masks):
    if masks.dtype not in (torch.bool, torch.uint8):
        raise TypeError(f'masks must be bool or uint8, got {masks.dtype}')
    if masks.dim() != 3:
        raise ValueError(f'masks must be [n, H, W], got {tuple(masks.shape)}')
    masks = masks.contiguous()
    L.require_cuda(masks)
    return masks.view(torch.uint8)


def _wait(*copies):
    """Non-blocking copies (dst, src) into pinned host memory, then one event wait for them."""
    for dst, src in copies:
        dst.copy_(src, non_blocking=True)
    done = torch.cuda.Event()
    done.record()
    done.synchronize()


def _counts(masks):
    """(counts int32 [R], offsets int64 [n + 1]) of dense uint8 CUDA masks, with the one host wait for R."""
    n, H, W = masks.shape
    dev = masks.device
    lib = L.lib()
    with torch.cuda.device(dev):
        ws = torch.empty(lib.bxs_mask_rle_counts_workspace_bytes(n, H, W), dtype=torch.uint8, device=dev)
        offsets = torch.empty(n + 1, dtype=torch.int64, device=dev)
        L.check(lib.bxs_mask_rle_runs(L.ptr(masks), n, H, W, L.ptr(ws), L.ptr(offsets), L.stream()), 'mask_rle_runs')
        total = torch.empty(1, dtype=torch.int64, pin_memory=True)
        _wait((total, offsets[n:]))                                            # host wait 1: R
        counts = torch.empty(int(total[0]), dtype=torch.int32, device=dev)
        L.check(lib.bxs_mask_rle_counts(L.ptr(masks), n, H, W, L.ptr(ws), L.ptr(offsets), L.ptr(counts), L.stream()),
                'mask_rle_counts')
    return counts, offsets


def rle_counts(masks):
    """(counts int32 [R], offsets int64 [n + 1]) on the device for bool or uint8 masks [n, H, W] (CUDA, any strides): mask
    k's uncompressed COCO RLE is counts[offsets[k]:offsets[k + 1]], the run lengths of its bytes in column-major order,
    starting with a run of zeros (0 when the first byte is non-zero).  A change between two non-zero values of a uint8
    mask closes a run, as in pycocotools.  One host wait (the total run count)."""
    masks = _check(masks)
    n = masks.shape[0]
    if n == 0:
        return (torch.empty(0, dtype=torch.int32, device=masks.device),
                torch.zeros(1, dtype=torch.int64, device=masks.device))
    return _counts(masks)


def encode(masks):
    """pycocotools' ``mask.encode`` of each of the bool or uint8 masks [n, H, W] (CUDA, any strides): a list of n
    ``{'size': [H, W], 'counts': bytes}``.  Two host waits whatever n is; none and no device work for n == 0."""
    masks = _check(masks)
    n, H, W = masks.shape
    if n == 0:
        return []
    counts, offsets = _counts(masks)
    R = counts.numel()
    dev = masks.device
    lib = L.lib()
    with torch.cuda.device(dev):
        ws = torch.empty(lib.bxs_mask_rle_strings_workspace_bytes(n, R), dtype=torch.uint8, device=dev)
        chars = torch.empty(6 * R, dtype=torch.uint8, device=dev)
        char_off = torch.empty(n + 1, dtype=torch.int64, device=dev)
        L.check(lib.bxs_mask_rle_strings(L.ptr(counts), L.ptr(offsets), n, R, L.ptr(ws), L.ptr(chars), L.ptr(char_off),
                                         L.stream()), 'mask_rle_strings')
        host_chars = torch.empty(6 * R, dtype=torch.uint8, pin_memory=True)
        host_off = torch.empty(n + 1, dtype=torch.int64, pin_memory=True)
        _wait((host_chars, chars), (host_off, char_off))                       # host wait 2: the strings
    o = host_off.tolist()
    buf = host_chars.numpy()[:o[n]].tobytes()
    size = [int(H), int(W)]
    return [{'size': list(size), 'counts': buf[o[k]:o[k + 1]]} for k in range(n)]
