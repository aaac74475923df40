"""``GenerateBoxMask`` (mmdet/datasets/pipelines/loading.py:647-668) producing ``BoxMasks``."""
import numpy as np

from ..core.box_masks import BoxMasks


def _python_slice(start, stop, n):
    """numpy's ``a[start:stop]`` on an axis of length n as the range [lo, hi): negative bounds count from the end, and
    both are then clipped to [0, n] (``slice.indices``)."""
    start = np.clip(np.where(start < 0, start + n, start), 0, n)
    stop = np.clip(np.where(stop < 0, stop + n, stop), 0, n)
    return start, stop


class GenerateBoxMask:
    """The ground-truth masks of box supervision: mask i is ``masks[i, ry0:ry1 + 1, rx0:rx1 + 1] = 1`` of an image-sized
    array, with ``(rx0, ry0, rx1, ry1) = gt_bboxes[i].round().astype(int)`` (numpy's round: half to even) and numpy's
    slicing rules.  It builds ``BoxMasks`` of those rectangles, equal to the reference's ``BitmapMasks`` in every
    method, without the array, and appends 'gt_masks' to ``results['mask_fields']``."""

    def __init__(self):
        pass

    def _generate_mask_from_box(self, results):
        boxes = np.asarray(results['gt_bboxes']).round().astype(int).reshape(-1, 4)
        h, w = results['img'].shape[:2]
        y0, y1 = _python_slice(boxes[:, 1], boxes[:, 3] + 1, h)
        x0, x1 = _python_slice(boxes[:, 0], boxes[:, 2] + 1, w)
        results['gt_masks'] = BoxMasks(np.stack([y0, x0, y1, x1], axis=1), h, w)
        results['mask_fields'].append('gt_masks')
        return results

    def __call__(self, results):
        return self._generate_mask_from_box(results)

    def __repr__(self):
        return self.__class__.__name__ + '()'
