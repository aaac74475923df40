"""``BoxMasks``: the ground-truth masks of box supervision kept as what they are, one axis-aligned rectangle per instance.

BoxLevelSet, DiscoBox and Box2Mask train on masks that are their boxes (``GenerateBoxMask``,
mmdet/datasets/pipelines/loading.py:647-668).  ``BitmapMasks`` carries them as a uint8 ``[G, H, W]`` host array through
every transform, the dataloader's pickles and a blocking host-to-device copy in the training step.  Every transform those
pipelines apply keeps a rectangle a rectangle: nearest-neighbour resizing maps each axis through a non-decreasing index
map, flipping mirrors it, cropping, padding and expanding offset or clip it.  So ``BoxMasks`` keeps int64 ``[G, 4]``
half-open rectangles ``(y0, x0, y1, x1)`` and writes the bytes only when asked: ``to_tensor`` on a CUDA device is one
kernel (``ops.box_masks.rasterize``), ``masks`` / ``to_ndarray`` build the host array.

Each method returns what ``BitmapMasks``' does on the materialised array, the same shape and the same bits, including
its quirks: ``crop`` at the image's edge declares a size of 1 while the slice is empty (the array then holds no mask),
and an empty ``BitmapMasks`` is uint8 ``[0, h, w]``.  What does not keep rectangles (any interpolation but 'nearest', a
``pad_val`` other than 0, ``translate``, ``shear``, ``rotate``, ``crop_and_resize``, arguments outside the shapes the
transforms produce) materialises the array and defers to ``BitmapMasks``, which needs mmdet.  With mmdet importable
``BoxMasks`` subclasses its ``BitmapMasks``, so the pipeline's ``isinstance`` checks keep passing."""
import numpy as np
import torch

try:                                            # pragma: no cover - mmdet is absent in this image
    from mmdet.core.mask.structures import BitmapMasks as _Base
    HAVE_MMDET = True
except Exception:                               # noqa: BLE001
    _Base = object
    HAVE_MMDET = False


def rescale_size(old_size, scale):
    """mmcv's ``rescale_size((w, h), scale)`` (mmcv/image/geometric.py): ``(new_w, new_h)`` for a float or int scale
    factor, or for a tuple the largest size within (long edge, short edge) keeping the aspect ratio, rounded as
    ``int(x * s + 0.5)``."""
    w, h = old_size
    if isinstance(scale, (float, int)):
        if scale <= 0:
            raise ValueError(f'Invalid scale {scale}, must be positive.')
        factor = scale
    elif isinstance(scale, tuple):
        factor = min(max(scale) / max(h, w), min(scale) / min(h, w))
    else:
        raise TypeError(f'Scale must be a number or tuple of int, but got {type(scale)}')
    return int(w * float(factor) + 0.5), int(h * float(factor) + 0.5)


def nearest_map(src, dst):
    """The source index of each of ``dst`` destination indices under OpenCV's ``INTER_NEAREST`` resize of an axis of
    ``src`` (resizeNN in imgproc/src/resize.cpp): ``min(floor(d * (1. / (dst / src))), src - 1)`` in float64."""
    ifx = 1. / (float(dst) / float(src))
    return np.minimum(np.floor(np.arange(dst, dtype=np.float64) * ifx).astype(np.int64), src - 1)


def _map_ranges(lo, hi, src, dst):
    """The destination range [d0, d1) whose source indices fall in [lo, hi), for int64 arrays ``lo``, ``hi``: the map is
    non-decreasing, so it is one contiguous range."""
    m = nearest_map(src, dst)
    return np.searchsorted(m, lo, 'left'), np.searchsorted(m, hi, 'left')


class BoxMasks(_Base):
    """G masks of ``height x width`` that are rectangles: int64 ``rects [G, 4]`` of half-open ``(y0, x0, y1, x1)``.  A
    rectangle with ``y1 <= y0`` or ``x1 <= x0`` is an empty mask; rectangles are clipped to the image and empty ones are
    stored as zeros, so equal masks have equal rectangles."""

    def __init__(self, rects, height, width):
        r = np.asarray(rects, dtype=np.int64).reshape(-1, 4)
        r = np.stack([np.clip(r[:, 0], 0, height), np.clip(r[:, 1], 0, width), np.clip(r[:, 2], 0, height),
                      np.clip(r[:, 3], 0, width)], axis=1)
        r[(r[:, 2] <= r[:, 0]) | (r[:, 3] <= r[:, 1])] = 0
        self.rects = r
        self.height = height
        self.width = width
        self._masks = None

    # ---------------------------------------------------------------------------------------------------- the array
    @property
    def masks(self):
        """The uint8 ``[G, height, width]`` array, built on first use and kept (read-only: it is derived from ``rects``)."""
        if self._masks is None:
            m = np.zeros((len(self.rects), self.height, self.width), dtype=np.uint8)
            for g, (y0, x0, y1, x1) in enumerate(self.rects):
                m[g, y0:y1, x0:x1] = 1
            m.flags.writeable = False
            self._masks = m
        return self._masks

    def to_ndarray(self):
        return self.masks

    def to_tensor(self, dtype, device):
        """``torch.tensor(self.to_ndarray(), dtype=dtype, device=device)``; on a CUDA device written by one kernel from the
        rectangles, without a host array, a host-to-device copy or a host wait."""
        device = torch.device(device)
        if device.type == 'cuda':
            from ..ops.box_masks import rasterize
            return rasterize([self.rects], [(self.height, self.width)], dtype, device)[0]
        return torch.tensor(self.to_ndarray(), dtype=dtype, device=device)

    def _bitmap(self):
        if not HAVE_MMDET:
            raise NotImplementedError('BoxMasks: this transform does not keep rectangles, and deferring it to '
                                      "BitmapMasks needs mmdet")
        return _Base(self.to_ndarray().copy(), self.height, self.width)

    # ------------------------------------------------------------------------------------------------- containers
    def __reduce__(self):
        return BoxMasks, (self.rects, self.height, self.width)

    def __getitem__(self, index):
        return BoxMasks(self.rects[index].reshape(-1, 4), self.height, self.width)

    def __iter__(self):
        return iter(self.masks)

    def __len__(self):
        return len(self.rects)

    def __repr__(self):
        return f'{self.__class__.__name__}(num_masks={len(self)}, height={self.height}, width={self.width})'

    @property
    def areas(self):
        """The pixel count of each mask, in ``BitmapMasks.areas``' dtype (numpy's sum of uint8: uint64)."""
        r = self.rects
        return ((r[:, 2] - r[:, 0]) * (r[:, 3] - r[:, 1])).astype(np.uint64)

    def get_bboxes(self):
        """float32 ``[G, 4]`` ``(x0, y0, x1, y1)`` of each mask's pixels (exclusive ends), zeros for an empty mask."""
        return self.rects[:, [1, 0, 3, 2]].astype(np.float32)

    # ------------------------------------------------------------------------------------------------- transforms
    def resize(self, out_shape, interpolation='nearest'):
        h, w = out_shape
        if len(self) and (interpolation != 'nearest' or int(h) <= 0 or int(w) <= 0):
            return self._bitmap().resize(out_shape, interpolation)
        r = self.rects
        if len(self):
            y0, y1 = _map_ranges(r[:, 0], r[:, 2], self.height, int(h))
            x0, x1 = _map_ranges(r[:, 1], r[:, 3], self.width, int(w))
            r = np.stack([y0, x0, y1, x1], axis=1)
        return BoxMasks(r, h, w)

    def rescale(self, scale, interpolation='nearest'):
        new_w, new_h = rescale_size((self.width, self.height), scale)
        if len(self) and (interpolation != 'nearest' or new_h <= 0 or new_w <= 0):
            return self._bitmap().rescale(scale, interpolation)
        return self.resize((new_h, new_w))

    def flip(self, flip_direction='horizontal'):
        assert flip_direction in ('horizontal', 'vertical', 'diagonal')
        y0, x0, y1, x1 = self.rects.T
        H, W = self.height, self.width
        if flip_direction in ('vertical', 'diagonal'):
            y0, y1 = H - y1, H - y0
        if flip_direction in ('horizontal', 'diagonal'):
            x0, x1 = W - x1, W - x0
        return BoxMasks(np.stack([y0, x0, y1, x1], axis=1), H, W)

    def pad(self, out_shape, pad_val=0):
        h, w = out_shape
        if len(self) and (pad_val != 0 or h < self.height or w < self.width):
            return self._bitmap().pad(out_shape, pad_val)
        return BoxMasks(self.rects, h, w)

    def crop(self, bbox):
        assert isinstance(bbox, np.ndarray)
        assert bbox.ndim == 1
        if len(self) and not np.issubdtype(bbox.dtype, np.integer):
            return self._bitmap().crop(bbox)
        bbox = bbox.copy()
        bbox[0::2] = np.clip(bbox[0::2], 0, self.width)
        bbox[1::2] = np.clip(bbox[1::2], 0, self.height)
        x1, y1, x2, y2 = bbox
        w = np.maximum(x2 - x1, 1)
        h = np.maximum(y2 - y1, 1)
        # BitmapMasks slices masks[:, y1:y1 + h, x1:x1 + w] and reshapes it to (-1, h, w): a slice that starts at the
        # image's edge is empty, and the reshape turns it into no mask at all
        if y1 >= self.height or x1 >= self.width:
            return BoxMasks(np.zeros((0, 4), np.int64), h, w)
        r = self.rects - np.array([y1, x1, y1, x1], dtype=np.int64)
        return BoxMasks(r, h, w)

    def expand(self, expanded_h, expanded_w, top, left):
        if len(self) and not (0 <= top and top + self.height <= expanded_h and 0 <= left
                              and left + self.width <= expanded_w):
            return self._bitmap().expand(expanded_h, expanded_w, top, left)
        r = self.rects + np.array([top, left, top, left], dtype=np.int64)
        return BoxMasks(r, expanded_h, expanded_w)

    def crop_and_resize(self, bboxes, out_shape, inds, device='cpu', interpolation='bilinear', binarize=True):
        return self._bitmap().crop_and_resize(bboxes, out_shape, inds, device, interpolation, binarize)

    def translate(self, out_shape, offset, direction='horizontal', fill_val=0, interpolation='bilinear'):
        return self._bitmap().translate(out_shape, offset, direction, fill_val, interpolation)

    def shear(self, out_shape, magnitude, direction='horizontal', border_value=0, interpolation='bilinear'):
        return self._bitmap().shear(out_shape, magnitude, direction, border_value, interpolation)

    def rotate(self, out_shape, angle, center=None, scale=1.0, fill_val=0):
        return self._bitmap().rotate(out_shape, angle, center, scale, fill_val)
