"""The instance-output tail of ``MaskFormer.simple_test`` (mmdet/models/detectors/maskformer.py:156-177), the one
``Box2Mask`` inherits, restated with ``bbox2result`` (mmdet/core/bbox/transforms.py:116-133) and plain ``.cpu().numpy()``
copies: one per mask, as the reference makes them.  Its contract is the reference's values; it makes no promise about how
often the host waits.  ``ins_results`` comes from ``MaskFormerFusionHead.simple_test`` (oracle/box2mask_infer.py restates
it), on CPU or CUDA."""
import numpy as np
import torch


def bbox2result(bboxes, labels, num_classes):
    """Per class the float rows of ``bboxes [n, 5]`` whose label is that class, in detection order; one separate
    float32 ``[0, 5]`` array per class when ``n == 0``."""
    if bboxes.shape[0] == 0:
        return [np.zeros((0, 5), dtype=np.float32) for _ in range(num_classes)]
    if isinstance(bboxes, torch.Tensor):
        bboxes, labels = bboxes.detach().cpu().numpy(), labels.detach().cpu().numpy()
    return [bboxes[labels == c, :] for c in range(num_classes)]


def maskformer_simple_test_tail(ins_results, num_things_classes):
    """Per image ``(bbox_results, mask_results)`` of the list of ``(labels [n], bboxes [n, 5], masks [n, H, W])``:
    ``mask_results[c]`` holds the numpy masks labelled ``c`` in detection order."""
    out = []
    for labels, bboxes, masks in ins_results:
        bbox_results = bbox2result(bboxes, labels, num_things_classes)
        mask_results = [[] for _ in range(num_things_classes)]
        for j, label in enumerate(labels):
            mask_results[label].append(masks[j].detach().cpu().numpy())
        out.append((bbox_results, mask_results))
    return out


def assert_same(got, want, what=''):
    """Two per-image lists of ``(bbox_results, mask_results)`` equal element for element: list lengths, array types,
    dtypes, shapes, per-class order and every bit of every value."""
    assert len(got) == len(want), what
    for b, ((gb, gm), (wb, wm)) in enumerate(zip(got, want)):
        assert type(gb) is list and type(gm) is list and len(gb) == len(wb) and len(gm) == len(wm), (what, b)
        pairs = list(zip(gb, wb)) + [(x, y) for gc, wc in zip(gm, wm) for x, y in zip(gc, wc)]
        assert [len(c) for c in gm] == [len(c) for c in wm], (what, b)
        for x, y in pairs:
            assert type(x) is np.ndarray and x.dtype == y.dtype and x.shape == y.shape, (what, b, x.dtype, y.dtype)
            assert x.tobytes() == y.tobytes(), (what, b)
