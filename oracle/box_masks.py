"""numpy restatement of the box-mask data pipeline on dense arrays: GenerateBoxMask (mmdet/datasets/pipelines/loading.py:
647-668) and the BitmapMasks methods the box-supervised configs use (mmdet/core/mask/structures.py:193-545).

mmcv is not installed here, so ``rescale_size``, ``imrescale``, ``imresize``, ``imflip`` and ``impad`` (mmcv 1.x,
mmcv/image/geometric.py) are RESTATED from mmcv's source, not run.  ``imresize`` with 'nearest' is OpenCV's
``cv2.resize(INTER_NEAREST)``; ``resize_nearest`` restates it (resizeNN in imgproc/src/resize.cpp) for machines without
cv2, and ``imresize`` uses the real cv2 where it imports.

Chains: a chain is ``[('generate', boxes, h, w), op, ...]`` with ops ``('rescale', scale)``, ``('resize', (h, w))``,
``('flip', direction)``, ``('crop', [x1, y1, x2, y2])``, ``('pad', (h, w))``, ``('expand', (eh, ew, top, left))``,
``('index', inds)`` and ``('filter', min_wh)`` (FilterAnnotations on ``get_bboxes()``); ``apply`` runs one op on any
object with BitmapMasks' interface, so the same chain drives the reference, this restatement and ``BoxMasks``."""
import numpy as np

try:
    import cv2
except ImportError:                              # pragma: no cover
    cv2 = None


# ------------------------------------------------------------------------------------------- mmcv, restated
def rescale_size(old_size, scale):
    w, h = old_size
    if isinstance(scale, (float, int)):
        assert scale > 0
        s = scale
    else:
        s = min(max(scale) / max(h, w), min(scale) / min(h, w))
    return int(w * float(s) + 0.5), int(h * float(s) + 0.5)


def resize_nearest(img, size):
    """cv2.resize(img, size=(w, h), interpolation=INTER_NEAREST), restated: destination d reads source
    min(floor(d * (1 / (dst / src))), src - 1) on each axis."""
    w, h = size
    sh, sw = img.shape[:2]
    ys = [min(int(np.floor(y * (1. / (h / sh)))), sh - 1) for y in range(h)]
    xs = [min(int(np.floor(x * (1. / (w / sw)))), sw - 1) for x in range(w)]
    return img[np.array(ys, dtype=np.int64)][:, np.array(xs, dtype=np.int64)]


def imresize(img, size, interpolation='nearest'):
    assert interpolation == 'nearest'
    if cv2 is not None:
        return cv2.resize(img, size, interpolation=cv2.INTER_NEAREST)
    return resize_nearest(img, size)


def imrescale(img, scale, interpolation='nearest'):
    h, w = img.shape[:2]
    return imresize(img, rescale_size((w, h), scale), interpolation)


def imflip(img, direction='horizontal'):
    axes = {'horizontal': 1, 'vertical': 0, 'diagonal': (0, 1)}[direction]
    return np.flip(img, axis=axes)


def impad(img, shape, pad_val=0):
    assert shape[0] >= img.shape[0] and shape[1] >= img.shape[1]
    out = np.full((shape[0], shape[1]), pad_val, dtype=img.dtype)
    out[:img.shape[0], :img.shape[1]] = img
    return out


# ------------------------------------------------------------------------------------------- the pipeline, restated
def generate_box_mask(gt_bboxes, h, w):
    """uint8 [G, h, w]: mask i is 1 on [ry0:ry1 + 1, rx0:rx1 + 1] of the rounded (half to even) box, numpy slicing."""
    boxes = np.asarray(gt_bboxes).round().astype(int)
    m = np.zeros((len(boxes), h, w), dtype=np.uint8)
    for i, (rx0, ry0, rx1, ry1) in enumerate(boxes):
        m[i, ry0:ry1 + 1, rx0:rx1 + 1] = 1
    return Bitmap(m, h, w)


class Bitmap:
    """BitmapMasks' behaviour on a dense uint8 [G, H, W] array."""

    def __init__(self, masks, height, width):
        self.height, self.width = height, width
        if len(masks) == 0:
            self.masks = np.empty((0, height, width), dtype=np.uint8)
        else:
            self.masks = np.asarray(masks).reshape(-1, height, width)    # an empty slice reshapes to no mask at all

    def __len__(self):
        return len(self.masks)

    def __getitem__(self, index):
        return Bitmap(self.masks[index].reshape(-1, self.height, self.width), self.height, self.width)

    def rescale(self, scale, interpolation='nearest'):
        if len(self) == 0:
            w, h = rescale_size((self.width, self.height), scale)
            return Bitmap(np.empty((0, h, w), np.uint8), h, w)
        out = np.stack([imrescale(m, scale, interpolation) for m in self.masks])
        return Bitmap(out, *out.shape[1:])

    def resize(self, out_shape, interpolation='nearest'):
        if len(self) == 0:
            return Bitmap(np.empty((0, *out_shape), np.uint8), *out_shape)
        return Bitmap(np.stack([imresize(m, out_shape[::-1], interpolation) for m in self.masks]), *out_shape)

    def flip(self, flip_direction='horizontal'):
        if len(self) == 0:
            return Bitmap(self.masks, self.height, self.width)
        return Bitmap(np.stack([imflip(m, flip_direction) for m in self.masks]), self.height, self.width)

    def pad(self, out_shape, pad_val=0):
        if len(self) == 0:
            return Bitmap(np.empty((0, *out_shape), np.uint8), *out_shape)
        return Bitmap(np.stack([impad(m, out_shape, pad_val) for m in self.masks]), *out_shape)

    def crop(self, bbox):
        bbox = bbox.copy()
        bbox[0::2] = np.clip(bbox[0::2], 0, self.width)
        bbox[1::2] = np.clip(bbox[1::2], 0, self.height)
        x1, y1, x2, y2 = bbox
        w, h = np.maximum(x2 - x1, 1), np.maximum(y2 - y1, 1)
        if len(self) == 0:
            return Bitmap(np.empty((0, h, w), np.uint8), h, w)
        return Bitmap(self.masks[:, y1:y1 + h, x1:x1 + w], h, w)

    def expand(self, expanded_h, expanded_w, top, left):
        out = np.zeros((len(self), expanded_h, expanded_w), np.uint8)
        if len(self):
            out[:, top:top + self.height, left:left + self.width] = self.masks
        return Bitmap(out, expanded_h, expanded_w)

    @property
    def areas(self):
        return self.masks.sum((1, 2))

    def to_ndarray(self):
        return self.masks

    def get_bboxes(self):
        out = np.zeros((len(self), 4), dtype=np.float32)
        for i, m in enumerate(self.masks):
            ys, xs = np.nonzero(m.any(1))[0], np.nonzero(m.any(0))[0]
            if len(xs) and len(ys):
                out[i] = (xs[0], ys[0], xs[-1] + 1, ys[-1] + 1)
        return out


# ------------------------------------------------------------------------------------------- chains
def apply(m, op):
    kind, arg = op[0], op[1]
    if kind == 'rescale':
        return m.rescale(tuple(arg) if isinstance(arg, (list, tuple)) else arg)
    if kind == 'resize':
        return m.resize(tuple(arg))
    if kind == 'flip':
        return m.flip(arg)
    if kind == 'crop':
        return m.crop(np.asarray(arg, dtype=np.int64))
    if kind == 'pad':
        return m.pad(tuple(arg))
    if kind == 'expand':
        return m.expand(*arg)
    if kind == 'index':
        return m[np.asarray(arg)]
    if kind == 'filter':                                         # FilterAnnotations(min_gt_bbox_wh) on get_bboxes()
        b = m.get_bboxes()
        return m[((b[:, 2] - b[:, 0]) > arg) & ((b[:, 3] - b[:, 1]) > arg)]
    raise ValueError(kind)


def _boxes(rng, G, h, w, special=True):
    """float32 [G, 4] xyxy boxes: ordinary ones, and (with ``special``) half-integer corners, boxes partly or wholly
    outside the image, negative corners, one-pixel and whole-image boxes."""
    x = np.sort(rng.uniform(-0.2 * w, 1.2 * w, (G, 2)), 1)
    y = np.sort(rng.uniform(-0.2 * h, 1.2 * h, (G, 2)), 1)
    b = np.stack([x[:, 0], y[:, 0], x[:, 1], y[:, 1]], 1)
    if special:
        for i in range(G):
            k = rng.integers(0, 6)
            if k == 0:
                b[i] = np.floor(b[i]) + 0.5                      # rounding ties
            elif k == 1:
                b[i] = (0, 0, w - 1, h - 1) if rng.integers(2) else (-0.5, -0.5, w - 0.5, h - 0.5)
            elif k == 2:
                c = rng.integers(0, [w, h])
                b[i] = (c[0], c[1], c[0], c[1])                  # one pixel
            elif k == 3:
                b[i] = (rng.uniform(-3 * w, -1), rng.uniform(-h, h), rng.uniform(-w, w), rng.uniform(-h, 2 * h))
    return b.astype(np.float32)


def random_chain(rng, max_side=40, max_g=6):
    """A short random chain over small images: every op, arguments at and past the edges the transforms produce."""
    h, w = (int(v) for v in rng.integers(1, max_side + 1, 2))
    G = int(rng.integers(0, max_g + 1))
    chain = [('generate', _boxes(rng, G, h, w), h, w)]
    for _ in range(int(rng.integers(1, 6))):
        k = rng.integers(0, 8)
        if k == 0:
            chain.append(('rescale', float(rng.choice([0.1, 0.25, 0.5, 0.75, 1.0, 1.3, 2.0, 3.0, rng.uniform(0.2, 2.5)]))))
        elif k == 1:
            chain.append(('rescale', tuple(int(v) for v in rng.integers(1, 2 * max_side, 2))))
        elif k == 2:
            chain.append(('resize', tuple(int(v) for v in rng.integers(1, 2 * max_side, 2))))
        elif k == 3:
            chain.append(('flip', str(rng.choice(['horizontal', 'vertical', 'diagonal']))))
        elif k == 4:
            x1, y1 = (int(v) for v in rng.integers(-5, max_side + 5, 2))
            chain.append(('crop', [x1, y1, x1 + int(rng.integers(-3, max_side)), y1 + int(rng.integers(-3, max_side))]))
        elif k == 5:
            chain.append(('pad', None))                          # resolved to a size at or past the current one
        elif k == 6:
            chain.append(('expand', None))
        else:
            chain.append(('index', None))
    return chain


def resolve(op, m, rng):
    """Fill in the arguments of a 'pad', 'expand' or 'index' op that depend on the masks it applies to; a 'rescale' that
    would reach a size of 0 (where cv2 raises) becomes a rescale by 1."""
    if op[0] == 'rescale' and 0 in rescale_size((m.width, m.height), op[1]):
        return ('rescale', 1.0)
    if op[0] == 'pad' and op[1] is None:
        return ('pad', (int(m.height + rng.integers(0, 9)), int(m.width + rng.integers(0, 9))))
    if op[0] == 'expand' and op[1] is None:
        eh, ew = int(m.height + rng.integers(0, 9)), int(m.width + rng.integers(0, 9))
        return ('expand', (eh, ew, int(rng.integers(0, eh - m.height + 1)), int(rng.integers(0, ew - m.width + 1))))
    if op[0] == 'index' and op[1] is None:
        n = len(m)
        k = rng.integers(0, 3)
        if k == 0:
            return ('index', rng.random(n) < 0.6)                # bool, as FilterAnnotations / RandomCrop
        if k == 1:
            return ('index', rng.integers(0, max(n, 1), int(rng.integers(0, 4))) if n else np.zeros(0, np.int64))
        return ('index', np.arange(n)[::-1].copy())
    return op


def run_chain(chain, make, rng=None):
    """The masks after each step of ``chain``, built with ``make(boxes, h, w)``; ops with unresolved arguments are
    resolved against the masks they apply to.  Returns (steps, resolved chain)."""
    rng = rng or np.random.default_rng(0)
    _, boxes, h, w = chain[0]
    m = make(boxes, h, w)
    steps, done = [m], [chain[0]]
    for op in chain[1:]:
        op = resolve(op, m, rng)
        m = apply(m, op)
        steps.append(m)
        done.append(op)
    return steps, done
