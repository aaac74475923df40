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


PACK_MAX_IMAGES = 16       # images of one bxs_disco_cells_pack call (its problem table)
PACK_MAX_ROWS = 2048       # rows per image of one bxs_disco_cells_pack call (the unpack's row links in shared memory)
PACK_MAX_GRID = 64         # S of a grid the pack takes (the unpack's list heads in shared memory)
_PACK_DTYPE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


class _CellPack(torch.autograd.Function):
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


_DiscoPack = _CellPack          # its name while DiscoBox was its only user


def _image_groups(B):
    """[b0, b1) ranges of at most PACK_MAX_IMAGES images covering the batch in order."""
    return [(b0, min(b0 + PACK_MAX_IMAGES, B)) for b0 in range(0, max(B, 1), PACK_MAX_IMAGES)]


def row_chunks(seg_counts):
    """Splits the rows of a pack into calls of at most PACK_MAX_ROWS rows per image.  seg_counts[l][b]: the rows of
    segment (level l, image b); image b's rows are those of its segments (0, b), (1, b), ... in turn.  Returns one
    (I_pad, counts, pieces) per call: I_pad its largest row count of an image, counts[l * B + b] the rows of segment (l, b)
    it takes, and per segment part it takes, level-major then image-major, (l, b, j, n, r): rows j .. j + n of segment
    (l, b) are its rows r .. r + n of image b."""
    n_lv, B = len(seg_counts), len(seg_counts[0])
    totals = [sum(seg_counts[l][b] for l in range(n_lv)) for b in range(B)]
    chunks = []
    for lo in range(0, max(max(totals), 1), PACK_MAX_ROWS):
        hi = lo + PACK_MAX_ROWS
        counts, pieces, q = [], [], [0] * B
        for l in range(n_lv):
            for b in range(B):
                a, e = max(q[b], lo), min(q[b] + seg_counts[l][b], hi)
                counts.append(max(0, e - a))
                if e > a:
                    pieces.append((l, b, a - q[b], e - a, a - lo))
                q[b] += seg_counts[l][b]
        chunks.append((max(min(t, hi) - lo for t in totals), counts, pieces))
    return chunks


def cells_conv(operand, grids, cells):
    """The dynamic convolution of some grid cells of every level with one operand.

    operand [B,C,h,w]; grids: per level the raw kernel grid [B,C,S,S] (S <= 64), all of one dtype (float32, float16 or
    bfloat16); cells: per level a list of B int tensors, the cells (gy*S + gx) of each image in any order, repeats allowed.
    Returns per level [n_l,h,w]: the rows of image 0, then image 1, ..., each image's in the order of its cells.
    The kernels of all levels of image b are packed, in the grids' dtype, into the rows of one [B,I_pad,C] operand
    (``bxs_disco_cells_pack``: one call per group of at most 16 images and chunk of at most 2048 rows per image, the chunks
    side by side; I_pad the largest per-image total of the batch, zero rows past an image's own), convolved by one
    ``dynconv1x1`` call under its dtype and autocast rules, and the level rows are taken out of the [B,I_pad,h,w] result by
    one ``index_select``.  Differentiable with respect to operand and grids; d/d grids sums repeated cells in row order
    (``bxs_disco_cells_unpack_grad``) and is 0 at every cell not named, bit-identical from run to run.  The counts are the
    cell tensors' shapes: nothing is read back and nothing is copied to the device but the cells."""
    big = [g.shape[-1] for g in grids if g.shape[-1] > PACK_MAX_GRID]
    if big:
        raise NotImplementedError(f'cells_conv: kernel grids of at most {PACK_MAX_GRID} x {PACK_MAX_GRID} cells, got '
                                  f'{big[0]} x {big[0]}')
    grids = [L.dense_aligned(g) for g in grids]
    L.require_cuda(*grids)
    B, dev = operand.shape[0], operand.device
    seg_counts = [[int(c.numel()) for c in lvl] for lvl in cells]
    packs, pieces, col = [], [], 0
    for I_pad, counts, parts in row_chunks(seg_counts):
        group_packs = []
        for b0, b1 in _image_groups(B):
            flat = [cells[l][b].reshape(-1)[j:j + n] for l, b, j, n, _ in parts if b0 <= b < b1]
            flat = torch.cat(flat).to(dev, torch.int32) if flat else torch.zeros(0, dtype=torch.int32, device=dev)
            g_counts = [counts[l * B + b] for l in range(len(grids)) for b in range(b0, b1)]
            whole = b1 - b0 == B
            group_packs.append(_CellPack.apply(g_counts, I_pad, flat, *[g if whole else g[b0:b1] for g in grids]))
        packs.append(group_packs[0] if len(group_packs) == 1 else torch.cat(group_packs, 0))
        pieces += [(l, b, j, n, col + r) for l, b, j, n, r in parts]
        col += I_pad
    packed = packs[0] if len(packs) == 1 else torch.cat(packs, 1)                       # [B,I_pad,C]
    rows = dynconv1x1(operand, packed)                                                # [B,I_pad,h,w]
    pieces.sort()                                                                     # level, image, row of the segment
    index = [torch.arange(b * col + r, b * col + r + n, device=dev) for _, b, _, n, r in pieces]
    index = torch.cat(index) if index else torch.zeros(0, dtype=torch.int64, device=dev)
    return list(rows.reshape((-1,) + rows.shape[2:]).index_select(0, index).split([sum(n) for n in seg_counts]))


def solo_cells_conv(feature_pred, kernel_preds, cells, out_sizes):
    """The positive rows of BoxSOLOv2's per-level dynamic convolution (box_solov2_head.py:204-216, indexed as :317-320).

    feature_pred [B,C,h,w]; kernel_preds: per level the raw grid [B,C,S,S] (as ``solo_kernel`` produces it); cells: per level
    a list of B int tensors, the ascending positive cells (gy*S + gx) of each image; out_sizes: per level (h_l, w_l).
    Returns per level [n_l, h_l, w_l] = interpolate(conv2d(feature_pred, cells), (h_l, w_l), bilinear)[positives], images
    in order: the reference's rows.  The resize is applied to the operand instead of the result (both are linear and
    per channel): levels of feature_pred's own size convolve it directly, every other size convolves one
    ``bilinear_resize`` of it, and each run of consecutive levels of one size is one ``cells_conv`` call, so each operand is
    read once per image for all its levels.  TF32 operands and FP32 accumulation whatever the autocast state: other dtypes
    are promoted to float32.  Differentiable with respect to feature_pred and kernel_preds; gradients are deterministic.
    C % 32 == 0, C <= 256, h_l*w_l % 4 == 0; a grid larger than 64 x 64 cells raises NotImplementedError."""
    sizes = [(int(s[0]), int(s[1])) for s in out_sizes]
    rows, l0 = [], 0
    with torch.autocast('cuda', enabled=False):
        f = L.dense_aligned(feature_pred.float())
        L.require_cuda(f)
        for l1 in range(1, len(sizes) + 1):
            if l1 == len(sizes) or sizes[l1] != sizes[l0]:
                op = f if sizes[l0] == tuple(f.shape[-2:]) else bilinear_resize(f, sizes[l0])
                rows += cells_conv(op, [k.float() for k in kernel_preds[l0:l1]], cells[l0:l1])
                l0 = l1
    return rows


def disco_cells_conv(ins_pred, kernel_preds_raw, grid_orders):
    """Every (level, image) dynamic convolution of DiscoBox (discobox_head.py:1180-1246) in ONE ``cells_conv`` call.

    ins_pred [B,C,h,w]; kernel_preds_raw: per level the raw grid [B,C,S,S]; grid_orders: per level a list of B int tensors,
    the covered cells (gy*S + gx) of each image in the target builder's order, repeats included.  Every level convolves the
    same ``ins_pred[b]``, so the kernels of all levels are packed in the grids' dtype (float32 for any other) and convolved
    by ``dynconv1x1`` under its dtype and autocast rules.  Returns (per level [n_l,h,w] or None for a level without cells,
    per level the int64 image of each row or None): the rows the reference concatenates.  Differentiable with respect to
    ins_pred and kernel_preds_raw; d/d kernel_preds_raw sums repeated cells in row order, bit-identical from run to run.
    The per-(level, image) counts are the cell tensors' shapes: nothing is read back."""
    B, n_lv = ins_pred.shape[0], len(kernel_preds_raw)
    counts = [[int(grid_orders[l][b].numel()) for b in range(B)] for l in range(n_lv)]
    if not any(map(any, counts)):
        return [None] * n_lv, [None] * n_lv
    dt = kernel_preds_raw[0].dtype if kernel_preds_raw[0].dtype in _PACK_DTYPE else torch.float32
    rows = cells_conv(ins_pred, [k.to(dt) for k in kernel_preds_raw], grid_orders)
    preds, img_inds = [], []
    for r, n in zip(rows, counts):
        if not sum(n):
            preds.append(None)
            img_inds.append(None)
            continue
        preds.append(r)
        img_inds.append(torch.cat([torch.full((c,), b, dtype=torch.int64, device=ins_pred.device) for b, c in enumerate(n)
                                   if c]))
    return preds, img_inds


def box2mask_mask_pred(mask_embed, mask_feature):
    """Box2Mask call site (box2mask_head.py:345): einsum('bqc,bchw->bqhw')."""
    return dynconv1x1(mask_feature, mask_embed)
