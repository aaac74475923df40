"""pycocotools' mask ``encode`` and ``decode`` restated in numpy (maskApi.c: rleEncode + rleToString, rleFrString +
rleDecode; _mask.pyx: encode, decode).  mmdet's ``encode_mask_results`` (mmdet/core/mask/utils.py:38-65) binds
``mask_util`` to this module in oracle/make_golden_mask_rle.py.

The encoding rules are restated from maskApi.c; this restatement has not been run against a build of pycocotools.  The GPU
tests cross-check against ``pycocotools.mask`` wherever it can be imported."""
import numpy as np


def _to_string(cnts):
    """rleToString: count i is written as x = cnts[i], minus cnts[i - 2] when i > 2; 5 bits per character, low bits
    first, 0x20 while more follow, + 48."""
    x = cnts.astype(np.int64)
    x[3:] -= cnts[1:-2].astype(np.int64)
    chars = np.zeros((len(x), 7), np.uint8)
    n = np.zeros(len(x), np.int64)
    live = np.ones(len(x), bool)
    for r in range(7):
        c = x & 0x1f
        x = x >> 5                                            # arithmetic, as on C's long
        more = np.where(c & 0x10, x != -1, x != 0)
        chars[:, r] = (c | np.where(more, 0x20, 0)) + 48
        n += live
        live &= more
    assert not live.any()
    return chars[np.arange(7)[None, :] < n[:, None]].tobytes()


def counts(T):
    """rleEncode of one mask's bytes T in the order they are given: the lengths of the runs of equal bytes, starting from a
    previous byte of 0 (a first count of 0 when T[0] != 0); [0] for no bytes."""
    T = np.asarray(T, np.uint8).reshape(-1)
    b = np.flatnonzero(T != np.concatenate(([0], T[:-1]))) if T.size else np.zeros(0, np.int64)
    return np.diff(np.concatenate((b, [T.size])), prepend=0).astype(np.uint32)


def encode(bimask):
    """_mask.encode: a uint8 [h, w, n] Fortran-contiguous array -> n dicts {'size': [h, w], 'counts': bytes}."""
    if not isinstance(bimask, np.ndarray) or bimask.dtype != np.uint8 or bimask.ndim != 3 \
            or not bimask.flags.f_contiguous:
        raise ValueError('ndarray is not Fortran contiguous uint8 [h, w, n]')
    h, w, n = bimask.shape
    flat = bimask.reshape(-1, order='F')                     # memory order: a view
    a = h * w
    return [{'size': [h, w], 'counts': _to_string(counts(flat[i * a:(i + 1) * a]))} for i in range(n)]


def from_string(s):
    """rleFrString: the counts of a string written by rleToString."""
    out = []
    v = np.frombuffer(s, np.uint8).astype(np.int64) - 48
    p = 0
    while p < len(v):
        x = k = 0
        more = True
        while more:
            c = int(v[p])
            x |= (c & 0x1f) << 5 * k
            more = bool(c & 0x20)
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << 5 * k
        if len(out) > 2:
            x += out[-2]
        out.append(x)
    return np.array(out, np.uint32)


def decode(rle):
    """mask.decode of one dict: uint8 [h, w], runs alternating 0 and 1 from 0."""
    h, w = rle['size']
    c = from_string(rle['counts'])
    flat = np.repeat(np.arange(len(c)) % 2, c).astype(np.uint8)
    return flat.reshape(w, h).T
