"""a2/a3/a4: dense dynamic 1x1 convolution ``out[b,i] = sum_c kernel[b,i,c] * feat[b,c]`` on Hopper wgmma.

Forward is the hand-written TMA + wgmma (TF32, FP32 accumulate in registers) kernel of libboxseg_b200.
Backward is the same machinery (bxs_dynconv1x1_backward): d/d feat = kernel^T . g_out re-uses the forward kernel with
the operand roles swapped, d/d kernel = g_out . feat^T is a split-K wgmma kernel over the pixels with an ordered
(deterministic) reduction of the partials.  Only d/d feat with more than 256 kernels per image (outside every reference
call site: the heads convolve the POSITIVE kernels of an image) goes through cuBLAS (torch.bmm).

FP16 / BF16 operands run the 16-bit kernels (bxs_dynconv1x1_half_*: FP32 accumulation, result and gradients in the
operand dtype), and under ``torch.autocast('cuda')`` both operands are cast to the autocast dtype first, as autocast does
for the ``F.conv2d`` this op replaces.
"""
import ctypes

import torch

from .. import _lib as L
from .resize import bilinear_resize

_HALF = {torch.float16: 0, torch.bfloat16: 1}          # bxs_half_t
_AUTOCAST_ELIGIBLE = (torch.float32, torch.float16, torch.bfloat16)


def _half_native(f):
    """Inside the envelope of the 16-bit kernels: C % 32 == 0, C <= 256, h*w % 8 == 0 (the operands are 16-byte aligned
    by the time they get here: L.dense_aligned)."""
    B, C, h, w = f.shape
    return C % 32 == 0 and C <= 256 and (h * w) % 8 == 0


def _forward(f, k):
    B, C, h, w = f.shape
    I = k.shape[1]
    out = torch.empty((B, I, h, w), dtype=f.dtype, device=f.device)
    if B and I:
        with torch.cuda.device(f.device):
            if f.dtype == torch.float32:
                L.check(L.lib().bxs_dynconv1x1_forward(L.ptr(f), L.ptr(k), L.ptr(out), B, C, h * w, I, L.stream()),
                        'dynconv1x1_forward')
            else:
                L.check(L.lib().bxs_dynconv1x1_half_forward(L.ptr(f), L.ptr(k), L.ptr(out), B, C, h * w, I, _HALF[f.dtype],
                                                            L.stream()), 'dynconv1x1_half_forward')
    return out


def _backward(f, k, g, need_f, need_k):
    B, C, h, w = f.shape
    I = k.shape[1]
    gf = gk = None
    native_f = need_f and I <= 256
    if need_f and not native_f:
        gf = torch.bmm(k.transpose(1, 2), g.flatten(2)).view(B, C, h, w)
    if native_f or need_k:
        gf = torch.empty_like(f) if native_f else gf
        gk = torch.empty_like(k) if need_k else None
        with torch.cuda.device(f.device):
            if f.dtype == torch.float32:
                ws = torch.empty(L.lib().bxs_dynconv1x1_backward_workspace_bytes(B, C, h * w, I), dtype=torch.uint8,
                                 device=f.device)
                L.check(L.lib().bxs_dynconv1x1_backward(L.ptr(f), L.ptr(k), L.ptr(g), L.ptr(gf) if native_f else None,
                                                        L.ptr(gk), L.ptr(ws), B, C, h * w, I, L.stream()),
                        'dynconv1x1_backward')
            else:
                dt = _HALF[f.dtype]
                ws = torch.empty(L.lib().bxs_dynconv1x1_half_backward_workspace_bytes(B, C, h * w, I, dt),
                                 dtype=torch.uint8, device=f.device)
                L.check(L.lib().bxs_dynconv1x1_half_backward(L.ptr(f), L.ptr(k), L.ptr(g),
                                                             L.ptr(gf) if native_f else None, L.ptr(gk), L.ptr(ws), B, C,
                                                             h * w, I, dt, L.stream()), 'dynconv1x1_half_backward')
    return gf, gk


class _DynConv1x1(torch.autograd.Function):
    @staticmethod
    def forward(ctx, feat, kernels):
        half = feat.dtype == kernels.dtype and feat.dtype in _HALF
        # TMA tensor maps: dense and 16-byte aligned, whatever view the caller holds
        f = L.dense_aligned(feat if half else feat.float())
        k = L.dense_aligned(kernels if half else kernels.float())
        L.require_cuda(f, k)
        B, C, h, w = f.shape
        assert k.dim() == 3 and k.shape[0] == B and k.shape[2] == C, 'kernels must be [B,I,C]'
        ctx.save_for_backward(f, k)
        if half and not _half_native(f):                # outside the 16-bit envelope: the FP32 kernels on promoted copies
            return _forward(f.float(), k.float()).to(f.dtype)
        return _forward(f, k)

    @staticmethod
    def backward(ctx, g_out):
        f, k = ctx.saved_tensors
        B, C, h, w = f.shape
        I = k.shape[1]
        need_f, need_k = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if not (B and I) or not (need_f or need_k):
            return (torch.zeros_like(f) if need_f else None), (torch.zeros_like(k) if need_k else None)
        g = L.dense_aligned(g_out.to(f.dtype))
        if f.dtype != torch.float32 and not _half_native(f):
            gf, gk = _backward(f.float(), k.float(), g.float(), need_f, need_k)
            return (None if gf is None else gf.to(f.dtype)), (None if gk is None else gk.to(f.dtype))
        return _backward(f, k, g, need_f, need_k)


def dynconv1x1(feat, kernels):
    """feat [B,C,h,w], kernels [B,I,C] -> [B,I,h,w]   (C % 32 == 0, C <= 256, h*w % 4 == 0).

    The dtype rules of the ``F.conv2d`` / ``einsum`` it replaces:
      * both operands float32: TF32 kernels, float32 result and gradients;
      * both float16 or both bfloat16: 16-bit kernels (FP32 accumulation), result and gradients in that dtype
        (outside their envelope -- h*w % 8 != 0 -- the float32 kernels on promoted copies, rounded back);
      * inside ``torch.autocast('cuda')``: both operands are cast to the autocast dtype first, then the above; gradients
        reach float32 leaves in float32 through autograd's cast;
      * any other mix: both promoted to float32.
    """
    if torch.is_autocast_enabled('cuda'):
        dt = torch.get_autocast_dtype('cuda')
        cast = lambda t: t.to(dt) if t.is_cuda and t.dtype in _AUTOCAST_ELIGIBLE else t    # noqa: E731
        with torch.autocast('cuda', enabled=False):
            return _DynConv1x1.apply(cast(feat), cast(kernels))
    return _DynConv1x1.apply(feat, kernels)


def solo_dynamic_conv(feature_pred, kernel_pred):
    """BoxSOLOv2 call site (box_solov2_head.py:204-211): feature_pred [B,C,h,w], kernel_pred [B,C,S,S]
    -> [B,S*S,h,w] with cell s = gy*S+gx (the reference's permute(0,2,3,1).view(-1,C) order)."""
    B, C, S, _ = kernel_pred.shape
    return dynconv1x1(feature_pred, kernel_pred.permute(0, 2, 3, 1).reshape(B, S * S, C))


def _i64(vals):
    return (ctypes.c_int64 * len(vals))(*vals)


def _ptrs(tensors):
    return (ctypes.c_void_p * len(tensors))(*[None if t is None else t.data_ptr() for t in tensors])


class _SoloCells(torch.autograd.Function):
    """Levels -> positive rows on bxs_dynconv1x1_cells_*.  Inputs: the plan (host lists), the device cell list, then the
    operands and the raw kernel grids."""

    @staticmethod
    def forward(ctx, plan, cells, *tensors):
        level_op, counts = plan
        n_ops = len(tensors) - len(level_op)
        ops, kerns = tensors[:n_ops], tensors[n_ops:]
        B, C = ops[0].shape[:2]
        outs = [ops[o].new_empty((sum(n), ops[o].shape[2], ops[o].shape[3])) for o, n in zip(level_op, counts)]
        ctx.save_for_backward(cells, *tensors)
        ctx.plan = plan
        args = (_i64([o.shape[2] * o.shape[3] for o in ops]), _ptrs(kerns), _i64([k.shape[-1] for k in kerns]),
                _i64(level_op), _i64([c for n in counts for c in n]))
        ctx.args = args
        flat = args[-1]
        with torch.cuda.device(ops[0].device):
            ws = torch.empty(L.lib().bxs_dynconv1x1_cells_forward_workspace_bytes(flat, len(kerns), B, C), dtype=torch.uint8,
                             device=ops[0].device)
            L.check(L.lib().bxs_dynconv1x1_cells_forward(_ptrs(ops), args[0], args[1], args[2], args[3], flat, L.ptr(cells),
                                                         _ptrs(outs), L.ptr(ws), len(kerns), n_ops, B, C, L.stream()),
                    'dynconv1x1_cells_forward')
        return tuple(outs)

    @staticmethod
    def backward(ctx, *g_outs):
        cells, *tensors = ctx.saved_tensors
        level_op, counts = ctx.plan
        n_ops = len(tensors) - len(level_op)
        ops, kerns = tensors[:n_ops], tensors[n_ops:]
        B, C = ops[0].shape[:2]
        need_op = any(ctx.needs_input_grad[2:2 + n_ops])
        need_k = any(ctx.needs_input_grad[2 + n_ops:])
        g = [torch.zeros((sum(n),) + ops[o].shape[2:], device=ops[0].device) if t is None else L.dense_aligned(t.float())
             for t, o, n in zip(g_outs, level_op, counts)]
        g_ops = [torch.empty_like(o) for o in ops] if need_op else None
        g_k = [torch.empty_like(k) for k in kerns] if need_k else None
        sizes, kp, grid, lop, flat = ctx.args
        lib = L.lib()
        with torch.cuda.device(ops[0].device):
            ws = torch.empty(lib.bxs_dynconv1x1_cells_backward_workspace_bytes(sizes, grid, lop, flat, len(kerns), n_ops, B, C),
                             dtype=torch.uint8, device=ops[0].device)
            call = lambda gop, gk: lib.bxs_dynconv1x1_cells_backward(      # noqa: E731
                _ptrs(ops), sizes, kp, grid, lop, flat, L.ptr(cells), _ptrs(g), gop, gk, L.ptr(ws), len(kerns), n_ops, B, C,
                L.stream())
            if need_op and _cells_widest_problem(level_op, counts) > 256:
                # more than 256 kernels in a problem: d/d operand through cuBLAS, as dynconv1x1 does beyond 256 kernels
                g_ops = _cells_operand_grad_mm(ops, kerns, cells, g, level_op, counts)
                rc = call(None, _ptrs(g_k)) if need_k else 0
            else:
                rc = call(_ptrs(g_ops) if need_op else None, _ptrs(g_k) if need_k else None)
            L.check(rc, 'dynconv1x1_cells_backward')
        return (None, None, *(g_ops if need_op else [None] * n_ops), *(g_k if need_k else [None] * len(kerns)))


def _cells_widest_problem(level_op, counts):
    """Kernels of the widest (operand, image) problem, each level's count padded to 32: what the d/d operand kernel reduces
    over (cells_kp in csrc/dynconv_wgmma.cu), and what limits it to 256."""
    widest = 0
    for o in set(level_op):
        per_image = zip(*[n for n, lo in zip(counts, level_op) if lo == o])
        widest = max([widest] + [sum((c + 31) & ~31 for c in image) for image in per_image])
    return widest


def _cells_operand_grad_mm(ops, kerns, cells, g, level_op, counts):
    g_ops = [torch.zeros_like(o) for o in ops]
    start = 0
    for l, (o, n) in enumerate(zip(level_op, counts)):
        C = kerns[l].shape[1]
        row = 0
        for b, nb in enumerate(n):
            if nb:
                k = kerns[l][b].reshape(C, -1)[:, cells[start:start + nb].long()]
                g_ops[o][b] += (k @ g[l][row:row + nb].flatten(1)).view_as(g_ops[o][b])
            start, row = start + nb, row + nb
    return g_ops


CELLS_MAX_IMAGES = 16      # images of one bxs_dynconv1x1_cells_* or bxs_disco_cells_* call (their problem tables)


def _image_groups(B):
    """[b0, b1) ranges of at most CELLS_MAX_IMAGES images covering the batch in order."""
    return [(b0, min(b0 + CELLS_MAX_IMAGES, B)) for b0 in range(0, max(B, 1), CELLS_MAX_IMAGES)]


def solo_cells_conv(feature_pred, kernel_preds, cells, out_sizes):
    """The positive rows of BoxSOLOv2's per-level dynamic convolution (box_solov2_head.py:204-216, indexed as :317-320).

    feature_pred [B,C,h,w]; kernel_preds: per level the raw grid [B,C,S,S] (as ``solo_kernel`` produces it); cells: per level
    a list of B int tensors, the ascending positive cells (gy*S + gx) of each image; out_sizes: per level (h_l, w_l).
    Returns per level [n_l, h_l, w_l] = interpolate(conv2d(feature_pred, cells), (h_l, w_l), bilinear)[positives], images
    in order: the reference's rows.  The resize is applied to the operand instead of the result (both are linear and
    per channel): levels of feature_pred's own size convolve it directly, every other size convolves one
    ``bilinear_resize`` of it, shared by the consecutive levels of that size.  All levels and images run in one launch
    (TF32 operands, FP32 accumulation); a batch of more than 16 images runs one launch per group of 16 and concatenates
    each level's rows in image order.  Other dtypes are promoted to float32.  Differentiable with respect to
    feature_pred and kernel_preds; gradients are deterministic.  C % 32 == 0, C <= 256, h_l*w_l % 4 == 0."""
    f = L.dense_aligned(feature_pred.float())
    L.require_cuda(f)
    sizes = [(int(s[0]), int(s[1])) for s in out_sizes]
    level_op, op_sizes = [], []
    for s in sizes:
        if not op_sizes or op_sizes[-1] != s:
            op_sizes.append(s)
        level_op.append(len(op_sizes) - 1)
    ops = [f if s == tuple(f.shape[-2:]) else bilinear_resize(f, s) for s in op_sizes]
    kerns = [k.contiguous().float() for k in kernel_preds]
    groups = []
    for b0, b1 in _image_groups(f.shape[0]):
        counts = [[int(c.numel()) for c in lvl[b0:b1]] for lvl in cells]
        flat = [c.reshape(-1) for lvl in cells for c in lvl[b0:b1]]
        flat = torch.cat(flat).to(device=f.device, dtype=torch.int32) if flat else f.new_zeros(0, dtype=torch.int32)
        whole = b1 - b0 == f.shape[0]
        groups.append(_SoloCells.apply((level_op, counts), flat, *[t if whole else t[b0:b1] for t in ops + kerns]))
    if len(groups) == 1:
        return list(groups[0])
    return [torch.cat(rows, 0) for rows in zip(*groups)]        # the level rows are image-major: groups in image order


_PACK_DTYPE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


class _DiscoPack(torch.autograd.Function):
    """Raw kernel grids -> packed [B,I_pad,C] rows (bxs_disco_cells_pack); backward: bxs_disco_cells_unpack_grad."""

    @staticmethod
    def forward(ctx, counts, I_pad, cells, *grids):
        B, C = grids[0].shape[:2]
        args = (_i64([g.shape[-1] for g in grids]), _i64(counts), L.ptr(cells), cells.numel(), len(grids), B, C, I_pad,
                _PACK_DTYPE[grids[0].dtype])
        packed = grids[0].new_empty((B, I_pad, C))
        with torch.cuda.device(cells.device):
            L.check(L.lib().bxs_disco_cells_pack(_ptrs(grids), args[0], args[1], args[2], args[3], L.ptr(packed), None,
                                                 *args[4:], L.stream()), 'disco_cells_pack')
        ctx.save_for_backward(cells)
        ctx.args = args
        ctx.shapes = [g.shape for g in grids]
        return packed

    @staticmethod
    def backward(ctx, g_packed):
        (cells,) = ctx.saved_tensors
        grid, counts, _, n_cells, n_levels, B, C, I_pad, dt = ctx.args
        g = L.dense_aligned(g_packed.to(next(k for k, v in _PACK_DTYPE.items() if v == dt)))
        g_grids = [g.new_empty(s) for s in ctx.shapes]
        with torch.cuda.device(g.device):
            L.check(L.lib().bxs_disco_cells_unpack_grad(L.ptr(g), grid, counts, L.ptr(cells), n_cells, _ptrs(g_grids),
                                                        n_levels, B, C, I_pad, dt, L.stream()), 'disco_cells_unpack_grad')
        return (None, None, None, *g_grids)


def disco_cells_conv(ins_pred, kernel_preds_raw, grid_orders):
    """Every (level, image) dynamic convolution of DiscoBox (discobox_head.py:1180-1246) in ONE ``dynconv1x1`` call.

    ins_pred [B,C,h,w]; kernel_preds_raw: per level the raw grid [B,C,S,S]; grid_orders: per level a list of B int tensors,
    the covered cells (gy*S + gx) of each image in the target builder's order, repeats included.  Every level convolves the
    same ``ins_pred[b]``, so the kernels of all levels of image b are packed, in the grids' dtype, into one [B,I_pad,C]
    operand (``bxs_disco_cells_pack``, one call per group of at most 16 images; I_pad the largest per-image total of the
    whole batch, zero rows past an image's own) and convolved by ``dynconv1x1`` under its dtype and autocast rules.
    Returns (per level [n_l,h,w] or None for a level without cells, per level the int64 image of each row or None): the
    rows the reference concatenates.  Differentiable with respect to ins_pred and kernel_preds_raw; d/d kernel_preds_raw
    sums repeated cells in row order (``bxs_disco_cells_unpack_grad``), bit-identical from run to run.  The
    per-(level, image) counts are the cell tensors' shapes: nothing is read back."""
    B = ins_pred.shape[0]
    n_lv = len(kernel_preds_raw)
    counts = [int(grid_orders[l][b].numel()) for l in range(n_lv) for b in range(B)]
    totals = [sum(counts[l * B + b] for l in range(n_lv)) for b in range(B)]
    I_pad = max(totals)
    dev = ins_pred.device
    if I_pad == 0:
        return [None] * n_lv, [None] * n_lv
    dt = kernel_preds_raw[0].dtype if kernel_preds_raw[0].dtype in _PACK_DTYPE else torch.float32
    grids = [L.dense_aligned(k.to(dt)) for k in kernel_preds_raw]
    L.require_cuda(*grids)
    packs = []
    for b0, b1 in _image_groups(B):
        cells = torch.cat([grid_orders[l][b].reshape(-1) for l in range(n_lv) for b in range(b0, b1)]).to(dev, torch.int32)
        g_counts = [counts[l * B + b] for l in range(n_lv) for b in range(b0, b1)]
        whole = b1 - b0 == B
        packs.append(_DiscoPack.apply(g_counts, I_pad, cells, *[g if whole else g[b0:b1] for g in grids]))
    packed = packs[0] if len(packs) == 1 else torch.cat(packs, 0)                      # [B,I_pad,C]
    rows = dynconv1x1(ins_pred, packed)                                              # [B,I_pad,h,w]
    preds, img_inds = [], []
    row0 = [0] * B
    for l in range(n_lv):
        n = counts[l * B:(l + 1) * B]
        if not sum(n):
            preds.append(None)
            img_inds.append(None)
            continue
        preds.append(torch.cat([rows[b, row0[b]:row0[b] + n[b]] for b in range(B) if n[b]], 0))
        img_inds.append(torch.cat([torch.full((n[b],), b, dtype=torch.int64, device=dev) for b in range(B) if n[b]]))
        row0 = [r + c for r, c in zip(row0, n)]
    return preds, img_inds


def box2mask_mask_pred(mask_embed, mask_feature):
    """Box2Mask call site (box2mask_head.py:345): einsum('bqc,bchw->bqhw')."""
    return dynconv1x1(mask_feature, mask_embed)
