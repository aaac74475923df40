"""``format_results`` of the SOLOv2-family detectors restated line by line: ``SingleStageBoxInsDetector.format_results``
(mmdet/models/detectors/single_stage_boxseg.py:75-90) and ``SingleStageWSInsDetector.format_results`` (single_stage_ts.py:
88-103), which are the same function.  ``num_classes`` stands for ``self.bbox_head.num_classes``.  Pinned to the reference's
own function by tests/golden/solo_format.npz (oracle/make_golden_solo_format.py)."""
import numpy as np
import torch


def format_results(results, num_classes):
    bbox_results = [[] for _ in range(num_classes)]
    mask_results = [[] for _ in range(num_classes)]
    score_results = [[] for _ in range(num_classes)]

    for cate_label, cate_score, seg_mask in zip(results.labels, results.scores, results.masks):
        if seg_mask.sum() > 0:
            mask_results[cate_label].append(seg_mask.cpu())
            score_results[cate_label].append(cate_score.cpu())
            ys, xs = torch.where(seg_mask)
            min_x, min_y = xs.min().cpu().data.numpy(), ys.min().cpu().data.numpy()
            max_x, max_y = xs.max().cpu().data.numpy(), ys.max().cpu().data.numpy()
            bbox_results[cate_label].append([min_x, min_y, max_x + 1, max_y + 1, cate_score.cpu().data.numpy()])

    bbox_results = [np.array(bbox_result) if len(bbox_result) > 0 else np.zeros((0, 5)) for bbox_result in bbox_results]
    return bbox_results, (mask_results, score_results)
