"""``MaskFormer.simple_test`` (mmdet/models/detectors/maskformer.py:111-177) and ``Box2Mask``, which inherits it
(mmdet/models/detectors/box2mask.py), with one host wait per call instead of one blocking copy per mask.

The reference's tail turns each image's ``ins_results`` into ``bbox2result``'s per-class boxes and per-class numpy masks,
with a pageable ``.cpu()`` per mask.  ``format_instance_results`` instead enqueues, for every image with detections, one
non-blocking copy of its masks and one of a packed byte table of its boxes and labels, both to pinned host memory; one
event wait then ends the device work of the whole call, and the per-class split runs on the host.  Images without
detections do no device work.  The returned masks are views of one host tensor per image: a mask kept alive keeps its whole
image's buffer alive.  Every call allocates its own buffers, so a later call never writes into an earlier call's results."""
import numpy as np
import torch

from ..builder import HEADS, register


def _stage(labels, bboxes, masks):
    """Enqueue one image's copies on the current stream of the masks' device: (pinned masks, pinned table, box dtype).
    Each row of the table is a label as int64 followed by its box's bytes, so that both start at an offset their types
    can be viewed at."""
    if masks.dtype not in (torch.bool, torch.uint8):
        raise TypeError(f'masks must be bool or uint8, got {masks.dtype}')
    if not masks.is_cuda:
        raise RuntimeError(f'format_instance_results expects CUDA tensors, got masks on {masks.device}')
    masks = masks.detach().contiguous()
    boxes = bboxes.detach().contiguous()
    with torch.cuda.device(masks.device):
        label_bytes = labels.detach().to(torch.int64).contiguous()[:, None].view(torch.uint8)
        table = torch.cat([label_bytes, boxes.view(torch.uint8)], 1)
        host_masks = torch.empty(masks.shape, dtype=masks.dtype, pin_memory=True)
        host_table = torch.empty(table.shape, dtype=torch.uint8, pin_memory=True)
        host_masks.copy_(masks, non_blocking=True)
        host_table.copy_(table, non_blocking=True)
    return host_masks, host_table, boxes.dtype


def _split(staged, num_classes):
    """(bbox_results, mask_results) of one image from its host copies, after the wait."""
    mask_results = [[] for _ in range(num_classes)]
    if staged is None:
        return [np.zeros((0, 5), dtype=np.float32) for _ in range(num_classes)], mask_results
    host_masks, host_table, dtype = staged
    n = host_table.shape[0]
    labels = host_table[:, :8].reshape(-1).view(torch.int64).tolist()
    boxes = host_table[:, 8:].reshape(-1).view(dtype).view(n, -1).numpy()
    masks = host_masks.numpy()
    rows = [[] for _ in range(num_classes)]
    for j, label in enumerate(labels):
        mask_results[label].append(masks[j])           # the reference's list indexing, its IndexError included
        if label >= 0:
            rows[label].append(j)                      # bbox2result's ``labels == i`` never matches a negative label
    empty = boxes[:0]
    return [boxes.take(r, 0) if r else empty.copy() for r in rows], mask_results


def format_instance_results(ins_results_list, num_things_classes):
    """The reference's ``MaskFormer.simple_test`` tail for each image's ``ins_results``: per image ``(bbox_results,
    mask_results)``.

    ``ins_results_list`` holds one ``(labels int64 [n], bboxes float32 [n, 5], masks bool [n, H, W])`` per image, as
    ``MaskFormerFusionHead.simple_test`` returns it, on CUDA.  ``bbox_results`` is ``bbox2result``'s value: for ``n == 0``
    a separate ``np.zeros((0, 5), np.float32)`` per class, otherwise each class's box rows in detection order, in the
    boxes' dtype.  ``mask_results[c]`` holds class ``c``'s masks as numpy ``[H, W]`` arrays (the masks' dtype) in
    detection order.

    The masks of one image are views of one pinned host tensor that holds all ``n`` of them: a mask kept alive keeps that
    whole buffer alive, and page-locked.  A caller that keeps a few masks for long should copy them.  Masks that are neither
    bool nor uint8 raise ``TypeError`` and CPU tensors ``RuntimeError``, unless ``n == 0``.  Non-contiguous masks are made
    dense on the device first."""
    staged, devices = [], []
    for labels, bboxes, masks in ins_results_list:
        if bboxes.shape[0] == 0:
            staged.append(None)
            continue
        staged.append(_stage(labels, bboxes, masks))
        if masks.device not in devices:
            devices.append(masks.device)
    for dev in devices:                                # one device in practice: the one host wait of the call
        with torch.cuda.device(dev):
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
    return [_split(s, num_things_classes) for s in staged]


@register(HEADS, partial=True)
class MaskFormer:
    """mmdet/models/detectors/maskformer.py: the reference's detector with ``simple_test``'s result formatting on one
    host wait.  Uses the detector's ``extract_feat``, ``panoptic_head``, ``panoptic_fusion_head``, ``num_things_classes``
    and ``num_stuff_classes``."""

    def simple_test(self, imgs, img_metas, **kwargs):
        """The reference's signature, call order and return value: with ``num_stuff_classes == 0`` (every Box2Mask
        config) one ``(bbox_results, mask_results)`` per image."""
        feats = self.extract_feat(imgs)
        mask_cls_results, mask_pred_results = self.panoptic_head.simple_test(feats, img_metas, **kwargs)
        results = self.panoptic_fusion_head.simple_test(mask_cls_results, mask_pred_results, img_metas, **kwargs)
        for res in results:
            if 'pan_results' in res:
                res['pan_results'] = res['pan_results'].detach().cpu().numpy()
        ins = [res for res in results if 'ins_results' in res]
        for res, out in zip(ins, format_instance_results([res['ins_results'] for res in ins], self.num_things_classes)):
            res['ins_results'] = out
        for res in results:
            assert 'sem_results' not in res, 'semantic segmentation results are not supported yet'
        if self.num_stuff_classes == 0:
            results = [res['ins_results'] for res in results]
        return results


@register(HEADS, partial=True)
class Box2Mask(MaskFormer):
    """mmdet/models/detectors/box2mask.py: ``MaskFormer`` under Box2Mask's name, ``simple_test`` on one host wait."""
