"""Fused BoxInst mask-loss operators (SURVEY.md section 8 rows a5, a6+a7+a8) on the C ABI.

``boxinst_targets``  replaces CondInstMaskHead.get_targets / get_bitmasks_from_boxes
                     (mmdet/models/dense_heads/condinst_head.py:1345-1448), entirely on the GPU.
``boxinst_mask_loss`` replaces the arithmetic of CondInstMaskHead.loss (:1288-1343).

Neither function synchronises the host with the device.
"""
from dataclasses import dataclass
from typing import List, Optional

import numpy as np
import torch

from .. import _lib as L


@dataclass
class BoxInstTargets:
    edge_bits: Optional[torch.Tensor]   # uint8 [B,H,W]; bit c <=> similarity[c] >= thresh (size 3 only)
    similarity: Optional[torch.Tensor]  # float32 [B,k*k-1,H,W] (only when requested)
    rects: torch.Tensor                 # int32 [G,4] (j0,j1,i0,i1), inclusive, in loss-grid coordinates
    gt_img: torch.Tensor                # int32 [G] image of each GT
    num_gts: List[int]                  # per image
    lab: torch.Tensor                   # float32 [B,3,H,W]
    valid: torch.Tensor                 # uint8 [B,H,W]

    def bitmasks(self):
        """Dense float bitmasks, list of [G_i,H,W] -- API parity with the reference's `bitmasks`."""
        G = self.rects.shape[0]
        H, W = self.valid.shape[-2:]
        out = torch.empty((G, H, W), dtype=torch.float32, device=self.rects.device)
        if G:
            with torch.cuda.device(out.device):
                L.check(L.lib().bxs_boxinst_bitmasks(L.ptr(self.rects), L.ptr(out), G, H, W, L.stream()),
                        'boxinst_bitmasks')
        return list(torch.split(out, self.num_gts))


def _norm_cfg(img_metas):
    cfg = img_metas[0]['img_norm_cfg']
    mean = np.ascontiguousarray(np.asarray(cfg['mean'], dtype=np.float32).reshape(3))
    std = np.ascontiguousarray(np.asarray(cfg['std'], dtype=np.float32).reshape(3))
    to_rgb = bool(cfg.get('to_rgb', True))
    for m in img_metas[1:]:
        c = m['img_norm_cfg']
        if not (np.allclose(np.asarray(c['mean'], np.float32), mean) and np.allclose(np.asarray(c['std'], np.float32), std)
                and bool(c.get('to_rgb', True)) == to_rgb):
            raise NotImplementedError('per-image normalisation constants are not supported')
    if not to_rgb:
        # get_original_image (condinst_head.py:176-186) always hands true RGB to rgb2lab: tensor2imgs(to_rgb=...) followed
        # by the [::-1] flip.  The LAB kernel reads channel 0 as R, so a BGR-ordered tensor (caffe-style configs) would be
        # silently mis-coloured; all shipped BoxInst configs use to_rgb=True.
        raise NotImplementedError('img_norm_cfg.to_rgb=False (BGR input tensors) is not supported by the LAB kernel')
    return mean, std


def boxinst_targets(img, img_metas, gt_bboxes, stride=4, pairwise_size=3, pairwise_dilation=2,
                    pairwise_color_thresh=0.3, bottom_pixels_removed=10, want_similarity=False):
    """img [B,3,Hp,Wp] normalised RGB (float32, CUDA); gt_bboxes list of [G_i,4] xyxy."""
    img = img.contiguous()
    L.require_cuda(img)
    if img.dtype != torch.float32:
        img = img.float()
    B, _, Hp, Wp = img.shape
    assert Hp % stride == 0 and Wp % stride == 0, 'padded image must be divisible by the loss stride'
    H, W = Hp // stride, Wp // stride
    dev = img.device
    hw = np.zeros((B, 2), dtype=np.int32)
    removed = np.zeros(B, dtype=np.int32)
    for i, m in enumerate(img_metas):
        ih, iw = m['img_shape'][:2]
        hw[i] = (ih, iw)
        removed[i] = int(bottom_pixels_removed * float(ih) / float(m['ori_shape'][0]))
    mean, std = _norm_cfg(img_metas)
    lab = torch.empty((B, 3, H, W), dtype=torch.float32, device=dev)
    valid = torch.empty((B, H, W), dtype=torch.uint8, device=dev)
    K = pairwise_size * pairwise_size - 1
    sim = torch.empty((B, K, H, W), dtype=torch.float32, device=dev) if (want_similarity or pairwise_size != 3) else None
    bits = torch.empty((B, H, W), dtype=torch.uint8, device=dev) if pairwise_size == 3 else None
    num_gts = [int(b.shape[0]) for b in gt_bboxes]
    G = sum(num_gts)
    boxes = (torch.cat([b.reshape(-1, 4) for b in gt_bboxes]) if G else torch.zeros((0, 4), device=dev)).to(
        device=dev, dtype=torch.float32).contiguous()
    rects = torch.empty((G, 4), dtype=torch.int32, device=dev)
    gt_img = torch.empty(G, dtype=torch.int32, device=dev)
    ng = np.asarray(num_gts, dtype=np.int32)
    with torch.cuda.device(dev):
        # metadata by value: no host-to-device copies, capturable
        L.check(L.lib().bxs_boxinst_targets_forward(
            L.ptr(img), L.ptr(boxes), hw.ctypes.data, removed.ctypes.data, ng.ctypes.data, mean.ctypes.data,
            std.ctypes.data, L.ptr(lab), L.ptr(valid), L.ptr(sim), L.ptr(bits), L.ptr(rects), L.ptr(gt_img), B, Hp, Wp,
            stride, pairwise_size, pairwise_dilation, float(pairwise_color_thresh), L.stream()), 'boxinst_targets')
    return BoxInstTargets(bits, sim, rects, gt_img, num_gts, lab, valid)


# Scheduler state of the single-pass kernel (work-item counter, per-instance completion counters, finalize ticket,
# fixed-point loss sums): zero before first use, left zero by every call that runs to completion, owned by ONE stream
# at a time.  Pools of slots are created per device outside any graph capture; eager calls take the slot of their
# stream, every captured call site takes a slot of its own (a captured graph may be replayed on any stream,
# concurrently with eager work).  A pool is zero-filled on the stream that creates it; other streams wait on the
# pool's creation event before their first use.  When the pool runs dry an eager call simply adds another pool; a
# capturing call falls back to a graph-private state that is re-zeroed by a memset node at every replay.
_SCHED_SLOTS = 256
_SCHED = {}     # device index -> dict(pools=[tensor [slots, words]], events=[Event], by_stream={}, next=int, seen=set())


def _sched_new_pool(st, words, device):
    st['pools'].append(torch.zeros((_SCHED_SLOTS, words), dtype=torch.int32, device=device))
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream(device))
    st['events'].append(ev)


def _sched_slot(st, slot):
    return st['pools'][slot // _SCHED_SLOTS][slot % _SCHED_SLOTS]


def _sched_state(device):
    words = max(int(L.lib().bxs_boxinst_loss_fused_sched_bytes()), 16) // 4
    capturing = torch.cuda.is_current_stream_capturing()
    st = _SCHED.get(device.index)
    if st is None:
        if capturing:           # first use ever is inside a capture: a graph-private, memset-initialised state
            return torch.zeros(words, dtype=torch.int32, device=device)
        st = dict(pools=[], events=[], by_stream={}, next=0, seen=set())
        _sched_new_pool(st, words, device)
        _SCHED[device.index] = st
    cur = torch.cuda.current_stream(device)
    if capturing:
        if st['next'] >= _SCHED_SLOTS * len(st['pools']):
            return torch.zeros(words, dtype=torch.int32, device=device)
        slot, st['next'] = st['next'], st['next'] + 1
        return _sched_slot(st, slot)
    key = cur.cuda_stream
    slot = st['by_stream'].get(key)
    if slot is None:
        if st['next'] >= _SCHED_SLOTS * len(st['pools']):
            _sched_new_pool(st, words, device)
        slot, st['next'] = st['next'], st['next'] + 1
        st['by_stream'][key] = slot
    pool = slot // _SCHED_SLOTS
    if (key, pool) not in st['seen']:       # first use of this pool on this stream: its zero fill must have completed
        cur.wait_event(st['events'][pool])
        st['seen'].add((key, pool))
    return _sched_slot(st, slot)


def boxinst_loss_plan(targets, gt_inds, H, W, pairwise_dilation=2):
    """Work plan of the single-pass loss kernel for one (targets, instance->GT assignment) pair: item descriptors in
    queue order + the logit-independent weight total of condinst_head.py:1318-1319.  Index work on the targets only;
    build it where the targets are built and pass it to `boxinst_mask_loss(plan=...)` (without it the loss call
    builds one itself, two small extra launches).  Returns None outside the single-pass envelope."""
    inst_gt = gt_inds if (gt_inds.dtype == torch.int32 and gt_inds.is_contiguous()) else gt_inds.to(torch.int32).contiguous()
    N = int(inst_gt.numel())
    lib = L.lib()
    if targets.edge_bits is None or N == 0 or not lib.bxs_boxinst_loss_fused_supported(N, H, W, pairwise_dilation):
        return None
    dev = targets.edge_bits.device
    plan = torch.empty(lib.bxs_boxinst_loss_plan_bytes(N, H, W, pairwise_dilation), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        L.check(lib.bxs_boxinst_loss_plan(L.ptr(targets.edge_bits), L.ptr(targets.rects), L.ptr(inst_gt), L.ptr(targets.gt_img),
                                          L.ptr(plan), N, H, W, pairwise_dilation, L.stream()), 'boxinst_loss_plan')
    return plan


class _BoxInstMaskLoss(torch.autograd.Function):
    """Two schedules of the same arithmetic.  When a gradient is wanted and the shape is inside the single-pass
    envelope, forward runs `bxs_boxinst_loss_fused_forward` (logits read once, gradient written once) and backward
    only converts for upstream gradients != 1; otherwise the two-call kernels (forward, then backward re-reading
    the logits) are used.  A second backward through the same node (retain_graph) always takes the two-call
    kernels, because the single-pass gradient buffer is converted in place."""

    @staticmethod
    def forward(ctx, mask_logits, edge_bits, rects, inst_gt, gt_img, iter_buf, warmup_iters, dilation, plan=None):
        logits = L.dense_aligned(mask_logits)       # float4 / bulk-copy reads: one schedule whatever view the caller holds
        L.require_cuda(logits, edge_bits, rects, inst_gt, gt_img, iter_buf)
        N, _, H, W = logits.shape
        lib = L.lib()
        dev = logits.device
        out = torch.empty(4, dtype=torch.float32, device=dev)
        fused = bool(ctx.needs_input_grad[0] and N > 0 and lib.bxs_boxinst_loss_fused_supported(N, H, W, dilation))
        ctx.fused, ctx.dilation, ctx.calls = fused, dilation, 0
        ctx.set_materialize_grads(False)          # no zero-fill kernels for unused / non-differentiable outputs
        with torch.cuda.device(dev):
            if fused:
                ws = torch.empty(lib.bxs_boxinst_loss_fused_workspace_bytes(N, H, W), dtype=torch.uint8, device=dev)
                g_logits = torch.empty_like(logits)
                sched = _sched_state(dev)
                if plan is not None:
                    rc = lib.bxs_boxinst_loss_fused_forward_planned(L.ptr(logits), L.ptr(edge_bits), L.ptr(plan), L.ptr(iter_buf),
                                                                    float(warmup_iters), L.ptr(ws), L.ptr(sched), L.ptr(out),
                                                                    L.ptr(g_logits), N, H, W, dilation, L.stream())
                else:
                    rc = lib.bxs_boxinst_loss_fused_forward(L.ptr(logits), L.ptr(edge_bits), L.ptr(rects), L.ptr(inst_gt),
                                                            L.ptr(gt_img), L.ptr(iter_buf), float(warmup_iters), L.ptr(ws),
                                                            L.ptr(sched), L.ptr(out), L.ptr(g_logits), N, H, W, dilation, L.stream())
                if rc != 0:
                    sched.zero_()        # a failed launch may leave the counters dirty: never reuse them as they are
                L.check(rc, 'boxinst_loss_fused_forward')
            else:
                g_logits = None
                ws = torch.empty(lib.bxs_boxinst_loss_workspace_bytes(N, H, W), dtype=torch.uint8, device=dev)
                L.check(lib.bxs_boxinst_loss_forward(L.ptr(logits), L.ptr(edge_bits), L.ptr(rects), L.ptr(inst_gt),
                                                     L.ptr(gt_img), L.ptr(iter_buf), float(warmup_iters), L.ptr(ws),
                                                     L.ptr(out), N, H, W, dilation, L.stream()), 'boxinst_loss_forward')
        # the gradient buffer rides along as a saved tensor (not a ctx attribute): autograd releases saved tensors right
        # after backward returns, so AccumulateGrad sees a sole owner and adopts the buffer instead of cloning 26 MB
        if g_logits is None:
            ctx.save_for_backward(logits, edge_bits, rects, inst_gt, gt_img, ws, iter_buf)
        else:
            ctx.save_for_backward(logits, edge_bits, rects, inst_gt, gt_img, ws, iter_buf, g_logits)
        ctx.warmup_iters = float(warmup_iters)
        aux = out[2:]
        ctx.mark_non_differentiable(aux)
        return out[0], out[1], aux

    @staticmethod
    def backward(ctx, g_prj, g_pair, _g_aux):
        saved = ctx.saved_tensors
        logits, edge_bits, rects, inst_gt, gt_img, ws, iter_buf = saved[:7]
        N, _, H, W = logits.shape
        lib = L.lib()
        ctx.calls += 1
        if g_prj is None and g_pair is None:
            return (None,) * 9
        zero = None
        if g_prj is None or g_pair is None:
            zero = torch.zeros((), dtype=torch.float32, device=logits.device)
        g_prj = zero if g_prj is None else g_prj.reshape(()).to(torch.float32)
        g_pair = zero if g_pair is None else g_pair.reshape(()).to(torch.float32)
        with torch.cuda.device(logits.device):
            if ctx.fused and ctx.calls == 1:
                g_logits = saved[7]
                del saved
                L.check(lib.bxs_boxinst_loss_fused_backward(L.ptr(ws), L.ptr(g_prj), L.ptr(g_pair), L.ptr(g_logits), N, H, W,
                                                            L.stream()), 'boxinst_loss_fused_backward')
                return g_logits, None, None, None, None, None, None, None, None
            if ctx.fused:       # the in-place buffer is spent: recompute with the two-call kernels
                ws = torch.empty(lib.bxs_boxinst_loss_workspace_bytes(N, H, W), dtype=torch.uint8, device=logits.device)
                tmp = torch.empty(4, dtype=torch.float32, device=logits.device)
                L.check(lib.bxs_boxinst_loss_forward(L.ptr(logits), L.ptr(edge_bits), L.ptr(rects), L.ptr(inst_gt),
                                                     L.ptr(gt_img), L.ptr(iter_buf), ctx.warmup_iters, L.ptr(ws),
                                                     L.ptr(tmp), N, H, W, ctx.dilation, L.stream()), 'boxinst_loss_forward')
            g = torch.stack([g_prj, g_pair])
            g_logits = torch.empty_like(logits)
            L.check(lib.bxs_boxinst_loss_backward(L.ptr(logits), L.ptr(edge_bits), L.ptr(rects), L.ptr(inst_gt),
                                                  L.ptr(gt_img), L.ptr(ws), L.ptr(g), L.ptr(g_logits), N, H, W,
                                                  ctx.dilation, L.stream()), 'boxinst_loss_backward')
        return g_logits, None, None, None, None, None, None, None, None


def boxinst_mask_loss(mask_logits, targets: BoxInstTargets, gt_inds, iter_buf, warmup_iters=10000,
                      pairwise_dilation=2, plan=None):
    """(loss_prj, loss_pairwise) for mask_logits [N,1,H,W] float32; gt_inds [N] indexes the
    concatenated GT list (as in condinst_head.py:1302,1316).  Requires pairwise_size == 3.
    `plan`: optional result of `boxinst_loss_plan(targets, gt_inds, H, W, dilation)` for the same arguments."""
    if targets.edge_bits is None:
        raise NotImplementedError('the fused loss is specialised to pairwise_size == 3')
    if mask_logits.dtype != torch.float32:
        mask_logits = mask_logits.float()        # @force_fp32(apply_to=('mask_logits',)), :1288
    inst_gt = gt_inds if (gt_inds.dtype == torch.int32 and gt_inds.is_contiguous()) else gt_inds.to(torch.int32).contiguous()
    prj, pair, _ = _BoxInstMaskLoss.apply(mask_logits, targets.edge_bits, targets.rects, inst_gt, targets.gt_img,
                                          iter_buf, warmup_iters, pairwise_dilation, plan)
    return prj, pair
