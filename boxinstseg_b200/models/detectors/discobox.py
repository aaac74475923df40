"""f3: the teacher-student glue of ``DiscoBoxSOLOv2`` (mmdet/models/detectors/discobox.py), whose training step is
``SingleStageWSInsTSDetector.forward_train`` with the independent teacher's ``momentum_update``
(mmdet/models/detectors/single_stage_ts.py:118-131, 179-237), without the reference's per-step costs:

* ``momentum_update`` is the teacher's method as a function: the two models' ``state_dict()`` entries paired by key, the
  reference's errors for missing, unexpected and mis-shaped keys, then ONE ``momentum_update_`` call (csrc/momentum_update.cu)
  instead of two multiplies, one add and one ``copy_`` per entry.  The pairing is cached per (teacher, student) and used
  only while neither model's tensors changed: a replaced parameter or buffer, a ``.to()`` or a changed module tree packs
  the pairs again from fresh ``state_dict()`` walks.
* ``forward_train`` keeps the reference's signature, call order and results, but ``avg_loss_ins`` lives on the device as a
  float64 0-d tensor, updated as ``avg * 0.9 + 0.1 * loss_ins.double()`` (Python's float arithmetic, bit for bit).  Its
  value is copied without blocking to pinned memory behind an event, and the next step reads it through that event just
  before the gates need it: the host never waits on the queued work of the current step.  ``DiscoBoxSOLOv2.avg_loss_ins``
  stays a readable and assignable Python number (reading it waits on the event).
"""
import weakref

import torch
from torch import nn

from ...ops import ema
from ..builder import HEADS, register
from .solo import _FormatResults

# teacher -> (weak reference to the student, fingerprints of both, ema.Table); only a module whose state_dict() the
# fingerprint pins (no state-dict hooks, no extra state) is cached
_PAIRS = weakref.WeakKeyDictionary()


def _fingerprint(model):
    """Everything ``model.state_dict()`` is made of -- module names, each parameter's and persistent buffer's address,
    dtype, shape and strides -- or None when a hook or an extra state could change it behind these."""
    out = []
    for name, m in model.named_modules():
        if m._state_dict_hooks or m._state_dict_pre_hooks or \
                type(m).get_extra_state is not nn.Module.get_extra_state:
            return None
        out.append(name)
        for d in (m._parameters, m._buffers):
            for k, t in d.items():
                if t is not None and k not in m._non_persistent_buffers_set:
                    out.append((k, t.data_ptr(), t.dtype, t.shape, t.stride()))
    return out


def _load_errors(teacher, mine, cur):
    """The message ``teacher.load_state_dict(cur, strict=True)`` raises, in its order, or None when it would load."""
    missing = [k for k in mine if k not in cur]
    sizes = [f'size mismatch for {k}: copying a param with shape {cur[k].shape} from checkpoint, the shape in current '
             f'model is {mine[k].shape}.' for k in mine if k in cur and cur[k].shape != mine[k].shape]
    order = {}                                       # module prefixes in load_state_dict's walk

    def walk(m, prefix):
        order.setdefault(prefix, len(order))
        for n, child in m._modules.items():
            if child is not None:
                walk(child, prefix + n + '.')
    walk(teacher, '')

    def owner(key):                                  # the module whose strict check reports an unexpected key
        m, prefix, parts = teacher, '', key.split('.')
        while len(parts) > 1 and m._modules.get(parts[0]) is not None:
            m, prefix, parts = m._modules[parts[0]], prefix + parts[0] + '.', parts[1:]
        return order[prefix]
    unexpected = sorted((k for k in cur if k not in mine), key=owner)      # stable: the student's order within a module
    msgs = []
    if missing:
        msgs.append('Missing key(s) in state_dict: {}. '.format(', '.join(f'"{k}"' for k in missing)))
    if unexpected:
        msgs.append('Unexpected key(s) in state_dict: {}. '.format(', '.join(f'"{k}"' for k in unexpected)))
    msgs += sizes
    if not msgs:
        return None
    return 'Error(s) in loading state_dict for {}:\n\t{}'.format(teacher.__class__.__name__, '\n\t'.join(msgs))


def _pairs(teacher, cur_model):
    fp = (_fingerprint(teacher), _fingerprint(cur_model))
    hit = _PAIRS.get(teacher)
    if hit is not None and hit[0]() is cur_model and hit[1] == fp:
        return hit[2]
    cur, mine = cur_model.state_dict(), teacher.state_dict()
    err = _load_errors(teacher, mine, cur)
    if err is not None:
        raise RuntimeError(err)
    table = ema.Table([mine[k] for k in cur], [cur[k] for k in cur])
    if fp[0] is not None and fp[1] is not None:
        _PAIRS[teacher] = (weakref.ref(cur_model), fp, table)
    else:
        _PAIRS.pop(teacher, None)
    return table


def momentum_update(teacher, cur_model, teacher_momentum=None):
    """single_stage_ts.py:118-131, ``teacher.momentum_update(cur_model, teacher_momentum)``: every entry of the teacher's
    state becomes ``cur * (1. - m) + self * m`` rounded as the reference rounds it (integer entries through float32), in
    one launch.  ``teacher_momentum=None`` reads ``teacher.teacher_momentum``.  Raises the ``RuntimeError`` of
    ``load_state_dict(strict=True)`` when the keys or shapes of the two states differ."""
    if teacher_momentum is None:
        teacher_momentum = teacher.teacher_momentum
    ema.launch(_pairs(teacher, cur_model), teacher_momentum)


def _avg_read(det):
    """``det.avg_loss_ins`` as a Python number: after a step, the value that step left, through its event."""
    d = det.__dict__
    if d.get('_bxs_avg_event') is not None:
        d['_bxs_avg_event'].synchronize()
        return d['_bxs_avg_host'].item()
    return d.get('_bxs_avg_value', 2)


def _avg_write(det, value):
    det.__dict__['_bxs_avg_value'] = value
    det.__dict__['_bxs_avg_event'] = None
    det.__dict__['_bxs_avg_device'] = None


def _avg_update(det, loss_ins):
    """``avg = avg * 0.9 + 0.1 * loss_ins`` in float64 on loss_ins's device, then a non-blocking copy to pinned memory
    and an event for the next read."""
    d = det.__dict__
    dev = loss_ins.device
    with torch.cuda.device(dev):
        prev = d.get('_bxs_avg_device')
        if prev is None or prev.device != dev:
            prev = torch.full((), _avg_read(det), dtype=torch.float64, device=dev)
        avg = prev * 0.9 + 0.1 * loss_ins.detach().double().reshape(())
        if d.get('_bxs_avg_host') is None:
            d['_bxs_avg_host'] = torch.empty((), dtype=torch.float64, pin_memory=True)
            d['_bxs_avg_ready'] = torch.cuda.Event()
        d['_bxs_avg_host'].copy_(avg, non_blocking=True)
        d['_bxs_avg_ready'].record(torch.cuda.current_stream(dev))
    d['_bxs_avg_device'] = avg
    d['_bxs_avg_event'] = d['_bxs_avg_ready']


def forward_train(det, img, img_metas, gt_bboxes, gt_labels, gt_bboxes_ignore=None, gt_masks=None):
    """single_stage_ts.py:179-237 on the attributes of ``SingleStageWSInsTSDetector`` (``extract_feat``, ``bbox_head``,
    ``mask_feat_head``, ``tsw``, ``use_ind_teacher``, ``use_corr``, ``train_cfg``, ``cnt``, ``turn_on_teacher``), with both
    teacher updates on ``momentum_update`` and ``avg_loss_ins`` kept on the device (see the module's docstring)."""
    if det.turn_on_teacher and det.use_ind_teacher:
        momentum_update(det.tsw.teacher, det)

    student_x = det.extract_feat(img)
    student_outs = det.bbox_head(student_x)
    _, s_kernel_preds = student_outs

    with torch.no_grad():
        if det.turn_on_teacher and det.use_ind_teacher:
            teacher_x = det.tsw.teacher.extract_feat(img)
            teacher_outs = det.tsw.teacher.bbox_head(teacher_x)
            _, t_kernel_preds = teacher_outs

    s_mask_feat_pred = det.mask_feat_head(student_x[det.mask_feat_head.start_level:det.mask_feat_head.end_level + 1])
    if det.turn_on_teacher and det.use_ind_teacher:
        with torch.no_grad():
            t_mask_feat_pred = det.tsw.teacher.mask_feat_head(
                teacher_x[det.tsw.teacher.mask_feat_head.start_level:det.tsw.teacher.mask_feat_head.end_level + 1])
    else:
        teacher_x = student_x

    if det.turn_on_teacher and det.use_ind_teacher:
        loss_inputs = student_outs + (t_kernel_preds, s_mask_feat_pred, t_mask_feat_pred, gt_bboxes, gt_labels, gt_masks,
                                      img_metas, det.train_cfg)
    else:
        loss_inputs = student_outs + (None, s_mask_feat_pred, None, gt_bboxes, gt_labels, gt_masks, img_metas,
                                      det.train_cfg)

    avg = _avg_read(det)                             # the previous step's value: its event, not this step's work
    losses = det.bbox_head.loss(
        *loss_inputs,
        img=img,
        gt_bboxes_ignore=gt_bboxes_ignore,
        use_loss_ts=avg < 0.3,
        use_ind_teacher=det.use_ind_teacher and det.turn_on_teacher,
        use_corr=avg < 0.2 and det.use_corr,
        s_feat=student_x[det.mask_feat_head.start_level:det.mask_feat_head.end_level + 1],
        t_feat=teacher_x[det.mask_feat_head.start_level:det.mask_feat_head.end_level + 1])

    _avg_update(det, losses['loss_ins'])
    if det.use_ind_teacher and not det.turn_on_teacher and det.cnt > 13000:
        momentum_update(det.tsw.teacher, det, 0)
        det.turn_on_teacher = True
        print("Turn on teacher.")
    else:
        det.cnt += 1
    return losses


@register(HEADS, partial=True)
class DiscoBoxSOLOv2(_FormatResults):
    """mmdet/models/detectors/discobox.py: the reference's detector with ``format_results`` on one host wait, the
    teacher's momentum update in one launch and ``avg_loss_ins`` read one step late through an event."""

    avg_loss_ins = property(_avg_read, _avg_write, doc='single_stage_ts.py:161, 230: the running mean of loss_ins.')

    def forward_train(self, img, img_metas, gt_bboxes, gt_labels, gt_bboxes_ignore=None, gt_masks=None):
        return forward_train(self, img, img_metas, gt_bboxes, gt_labels, gt_bboxes_ignore, gt_masks)
