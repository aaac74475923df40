"""CPU: the registered BoxLevelSet answers the reference's ``simple_test`` (single_stage_boxseg.py:64), and runs the
reference's lines for a head that is not this package's BoxSOLOv2Head."""
import inspect
import types

import numpy as np
import pytest
import torch


def test_box_level_set_simple_test_signature():
    from boxinstseg_b200.models import HEADS
    det = HEADS.get('BoxLevelSet')
    assert det is not None and callable(getattr(det, 'simple_test', None))
    # single_stage_boxseg.py:64: def simple_test(self, img, img_meta, rescale=False)
    params = list(inspect.signature(det.simple_test).parameters.values())
    assert [p.name for p in params] == ['self', 'img', 'img_meta', 'rescale']
    assert params[-1].default is False
    assert all(p.kind == p.POSITIONAL_OR_KEYWORD for p in params)


def test_head_simple_test_signature():
    from boxinstseg_b200.models import HEADS
    params = inspect.signature(HEADS.get('BoxSOLOv2Head').simple_test).parameters
    assert list(params)[:4] == ['self', 'feats', 'img_metas', 'rescale'] and params['rescale'].default is False
    assert params['cfg'].default is None


def test_other_heads_run_the_reference_lines():
    """A head that is not BoxSOLOv2Head: ``bbox_head(x, eval=True)``, ``get_seg(*outs, img_meta, test_cfg, rescale)``, then
    ``format_results`` per image (empty results need no device)."""
    from boxinstseg_b200.models import HEADS
    calls = []

    class Head:
        num_classes = 3

        def __call__(self, x, eval=False):
            calls.append(('forward', x, eval))
            return ('seg', 'cate', 'lst')

        def get_seg(self, *args):
            calls.append(('get_seg',) + args)
            empty = dict(labels=torch.zeros(0, dtype=torch.int64), scores=torch.zeros(0), masks=torch.zeros(0, 4, 5))
            return [types.SimpleNamespace(**empty) for _ in args[3]]

    det = HEADS.get('BoxLevelSet')()
    det.bbox_head, det.test_cfg = Head(), dict(score_thr=0.1)
    det.extract_feat = lambda img: ('feats', img)
    metas = [dict(img_shape=(4, 5, 3))] * 2
    out = det.simple_test('img', metas, rescale=True)
    assert calls == [('forward', ('feats', 'img'), True), ('get_seg', 'seg', 'cate', 'lst', metas, det.test_cfg, True)]
    assert len(out) == 2
    for bbox, (masks, scores) in out:
        assert len(bbox) == len(masks) == len(scores) == 3
        assert all(isinstance(b, np.ndarray) and b.shape == (0, 5) for b in bbox)
        assert all(m == [] for m in masks) and all(s == [] for s in scores)


def test_head_simple_test_needs_the_towers():
    from boxinstseg_b200.models import build_head
    head = build_head(dict(type='BoxSOLOv2Head', num_classes=80, num_grids=[40, 36, 24, 16, 12]))
    with pytest.raises(RuntimeError, match='simple_test'):
        head.simple_test([torch.zeros(1, 8, 4, 4)] * 5, [dict(img_shape=(16, 16, 3))], cfg=dict(score_thr=0.1))
