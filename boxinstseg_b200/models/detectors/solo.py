"""``format_results`` of the SOLOv2-family detectors -- ``SingleStageBoxInsDetector`` (mmdet/models/detectors/
single_stage_boxseg.py:75-90, BoxLevelSet) and ``SingleStageWSInsDetector`` (single_stage_ts.py:88-103, DiscoBoxSOLOv2),
whose two copies are the same function -- with one host wait per image instead of up to nine per detection; and
BoxLevelSet's ``simple_test`` (single_stage_boxseg.py:64-73) on ``BoxSOLOv2Head.simple_test``, which convolves only the
candidate grid cells instead of all of them.

Per image: one ``bxs_mask_extents`` call gives every mask's area and box; the masks and one packed float64 table of labels,
scores, areas and boxes are copied to pinned host memory without blocking, and one event wait ends the device work.  The
per-class split then runs on the host.  ``n == 0`` does no device work.  The returned masks are views of one host tensor per
image: a mask kept alive keeps its whole image's buffer alive."""
import numpy as np
import torch

from ...ops import solo_seg as S
from ..builder import HEADS, register
from ..dense_heads.mask_loss_heads import BoxSOLOv2Head

_BOX = [3, 4, 5, 6, 1]          # columns of the packed table that make a bbox row: x0, y0, x1, y1, score


def format_results(results, num_classes):
    """The reference's ``format_results(results)`` with ``self.bbox_head.num_classes = num_classes``:
    ``(bbox_results, (mask_results, score_results))``, per class in detection order the CPU masks (the masks' dtype), the
    0-d CPU scores (the scores' dtype) and a float64 [k, 5] array of [x_min, y_min, x_max + 1, y_max + 1, score];
    ``np.zeros((0, 5))`` for a class without detections.  Detections whose mask has no set pixel are dropped."""
    mask_results = [[] for _ in range(num_classes)]
    score_results = [[] for _ in range(num_classes)]
    rows = [[] for _ in range(num_classes)]
    labels, scores, masks = results.labels, results.scores, results.masks
    if len(labels) > 0:
        if masks.dtype not in (torch.bool, torch.uint8):
            raise TypeError(f'masks must be bool or uint8, got {masks.dtype}')
        masks = masks.contiguous()
        area, box = S.mask_extents(masks)                                       # raises for CPU tensors, as every op does
        with torch.cuda.device(masks.device):
            table = torch.cat([labels[:, None].double(), scores[:, None].double(), area[:, None].double(), box.double()], 1)
            host_masks = torch.empty(masks.shape, dtype=masks.dtype, pin_memory=True)
            host_table = torch.empty(table.shape, dtype=table.dtype, pin_memory=True)
            host_masks.copy_(masks, non_blocking=True)
            host_table.copy_(table, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
            done.synchronize()                                                  # the one host wait
        t = host_table.numpy()
        host_scores = host_table[:, 1].to(scores.dtype)                        # exact: the table holds them in float64
        for i in np.flatnonzero(t[:, 2] > 0):
            c = int(t[i, 0])
            mask_results[c].append(host_masks[i])
            score_results[c].append(host_scores[i])
            rows[c].append(i)
        bbox_results = [t[r][:, _BOX] if r else np.zeros((0, 5)) for r in rows]
    else:
        bbox_results = [np.zeros((0, 5)) for _ in range(num_classes)]
    return bbox_results, (mask_results, score_results)


class _FormatResults:
    def format_results(self, results):
        return format_results(results, self.bbox_head.num_classes)


@register(HEADS, partial=True)
class BoxLevelSet(_FormatResults):
    """mmdet/models/detectors/boxlevelset.py: the reference's detector with ``format_results`` on one host wait and
    ``simple_test`` on the candidate cells."""

    def simple_test(self, img, img_meta, rescale=False):
        """The reference's ``simple_test``: per image ``format_results`` of the head's results.  With this package's
        ``BoxSOLOv2Head`` the results come from ``bbox_head.simple_test`` -- bit for bit those of ``get_seg`` on
        ``bbox_head(x, eval=True)``, without the dense [B, S^2, h, w] predictions of every level; any other head runs the
        reference's lines."""
        x = self.extract_feat(img)
        if isinstance(self.bbox_head, BoxSOLOv2Head):
            results_list = self.bbox_head.simple_test(x, img_meta, rescale=rescale, cfg=self.test_cfg)
        else:
            outs = self.bbox_head(x, eval=True)
            results_list = self.bbox_head.get_seg(*(tuple(outs) + (img_meta, self.test_cfg, rescale)))
        return [self.format_results(results) for results in results_list]
