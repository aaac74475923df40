"""Oracle (test infrastructure only) for the BoxInst / CondInst rows of SURVEY.md section 8:
a1 (dynamic mask head), a5 (colour-similarity + box bitmask targets), a6 (projection
term), a7 (pairwise -log P(same label)), a8 (weighted reduction).

Independent restatement in plain torch-on-CPU; works in float32 or float64 (pass
float64 tensors to get the high-precision truth).  Never imported by the product.
"""
import math

import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------------------
# neighbourhood enumeration
# ----------------------------------------------------------------------------------------
def neighbour_offsets(size, dilation):
    """(dy, dx) of the k*k-1 neighbours, row-major, centre skipped.

    Follows mmdet/ops/pairwise/csrc/pairwise/pairwise.cu:77,87-90 (dy outer, dx inner)
    which equals the F.unfold order of mmdet/models/dense_heads/condinst_head.py:190-217.
    """
    r = (size // 2) * dilation
    offs = []
    for dy in range(-r, r + 1, dilation):
        for dx in range(-r, r + 1, dilation):
            if dy == 0 and dx == 0:
                continue
            offs.append((dy, dx))
    return offs


def _shifted(x, dy, dx, fill=0.0):
    """y[..., i, j] = x[..., i+dy, j+dx], `fill` where that falls outside the map."""
    h, w = x.shape[-2:]
    out = torch.full_like(x, fill)
    ys0, ys1 = max(0, -dy), min(h, h - dy)
    xs0, xs1 = max(0, -dx), min(w, w - dx)
    if ys0 < ys1 and xs0 < xs1:
        out[..., ys0:ys1, xs0:xs1] = x[..., ys0 + dy:ys1 + dy, xs0 + dx:xs1 + dx]
    return out


def _inside(h, w, dy, dx, like):
    m = torch.zeros(h, w, dtype=like.dtype, device=like.device)
    ys0, ys1 = max(0, -dy), min(h, h - dy)
    xs0, xs1 = max(0, -dx), min(w, w - dx)
    if ys0 < ys1 and xs0 < xs1:
        m[ys0:ys1, xs0:xs1] = 1
    return m


# ----------------------------------------------------------------------------------------
# a7: pairwise term
# ----------------------------------------------------------------------------------------
def pairwise_nlog(logits, size, dilation):
    """-log( s_p s_q + (1-s_p)(1-s_q) ) for every pixel p and neighbour q.

    logits [B,1,H,W] -> [B,k*k-1,H,W].  An out-of-image neighbour contributes log-prob 0
    for both classes, so the entry is -log(s_p + (1-s_p)) = 0.
    Follows pairwise.cu:38-50,68-104 and its twin compute_pairwise_term
    (condinst_head.py:86-114).
    """
    assert logits.dim() == 4 and logits.size(1) == 1
    x = logits[:, 0]
    h, w = x.shape[-2:]
    lfg = F.logsigmoid(x)
    lbg = F.logsigmoid(-x)
    outs = []
    for dy, dx in neighbour_offsets(size, dilation):
        both_fg = lfg + _shifted(lfg, dy, dx, 0.0)
        both_bg = lbg + _shifted(lbg, dy, dx, 0.0)
        outs.append(-torch.logaddexp(both_fg, both_bg))
    return torch.stack(outs, dim=1)


# ----------------------------------------------------------------------------------------
# a6: projection term
# ----------------------------------------------------------------------------------------
def dice_1d(x, t, eps=1e-5):
    """1 - 2<x,t>/(|x|^2+|t|^2+eps) per row of [n, L].  condinst_head.py:117-131."""
    x = x.flatten(1)
    t = t.flatten(1)
    return 1.0 - 2.0 * (x * t).sum(1) / ((x * x).sum(1) + (t * t).sum(1) + eps)


def projection_losses(scores, targets, eps=1e-5):
    """Per-instance projection loss [n] (sum of the two axis terms).

    scores/targets [n,1,H,W].  condinst_head.py:134-143 (BoxInst, then .mean()) and
    mmdet/models/losses/box_projection_loss.py:18-42 (BoxLevelset/Box2Mask, x loss_weight).
    """
    # .max(dim)[0] (not amax): like the reference the gradient goes to ONE arg-max element
    col_s, col_t = scores.max(dim=2)[0], targets.max(dim=2)[0]     # profile over columns
    row_s, row_t = scores.max(dim=3)[0], targets.max(dim=3)[0]     # profile over rows
    return dice_1d(row_s, row_t, eps) + dice_1d(col_s, col_t, eps)


def projection_losses_logit_argmax(logits, targets, eps=1e-5):
    """Per-instance projection loss [n] with the positions chosen on the LOGITS, in float64.

    This is what the BoxInst kernels compute (DESIGN section 4, note (i)): the row / column
    arg-max of the logits by torch.max(dim) -- the first index on exact ties, -0 equal to +0 --
    then the sigmoid at those positions.  ``projection_losses(sigmoid(x))`` picks its positions
    among the scores instead, which differ where the sigmoid saturates, so it cannot judge them.
    """
    x = logits.to(torch.float64)
    t = targets.to(torch.float64)
    s = torch.sigmoid(x)
    row_s = s.gather(3, x.max(dim=3, keepdim=True)[1]).squeeze(3)   # [n,1,H]
    col_s = s.gather(2, x.max(dim=2, keepdim=True)[1]).squeeze(2)   # [n,1,W]
    return dice_1d(row_s, t.amax(dim=3), eps) + dice_1d(col_s, t.amax(dim=2), eps)


def logit_argmax_mask(logits):
    """bool [n,1,H,W]: the elements that are the first row or column arg-max of ``logits``
    (torch.max(dim)); the only places the projection term sends a gradient."""
    n, c, h, w = logits.shape
    m = torch.zeros(n, c, h, w, dtype=torch.bool, device=logits.device)
    m.scatter_(3, logits.max(dim=3, keepdim=True)[1], True)
    m.scatter_(2, logits.max(dim=2, keepdim=True)[1], True)
    return m


# ----------------------------------------------------------------------------------------
# a5: targets
# ----------------------------------------------------------------------------------------
_XYZ_FROM_RGB = np.array([[0.412453, 0.357580, 0.180423],
                          [0.212671, 0.715160, 0.072169],
                          [0.019334, 0.119193, 0.950227]], dtype=np.float64)
_D65_2DEG = np.array([0.95047, 1.0, 1.08883], dtype=np.float64)


def rgb2lab_u8(rgb_u8):
    """uint8 [H,W,3] RGB -> float64 [H,W,3] CIE-LAB (D65, 2 degree observer).

    Restates scikit-image ``color.rgb2lab`` (third-party, called at condinst_head.py:1413):
    /255, sRGB inverse companding (0.04045, 12.92, 1.055, 2.4), XYZ matrix, divide by
    the white point, f(t)=cbrt(t) if t>0.008856 else 7.787 t + 16/116,
    L=116 fy-16, a=500(fx-fy), b=200(fy-fz).
    """
    v = np.asarray(rgb_u8, dtype=np.float64) / 255.0
    lin = np.where(v > 0.04045, np.power((v + 0.055) / 1.055, 2.4), v / 12.92)
    xyz = lin @ _XYZ_FROM_RGB.T
    xyz = xyz / _D65_2DEG
    f = np.where(xyz > 0.008856, np.cbrt(xyz), 7.787 * xyz + 16.0 / 116.0)
    fx, fy, fz = f[..., 0], f[..., 1], f[..., 2]
    return np.stack([116.0 * fy - 16.0, 500.0 * (fx - fy), 200.0 * (fy - fz)], axis=-1)


def denormalise_to_u8(img, mean, std):
    """Normalised float32 [3,h,w] (RGB order) -> uint8 [3,h,w] RGB.

    Restates mmcv ``tensor2imgs``/``imdenormalize`` as used at condinst_head.py:170-186:
    float32 multiply by std, float32 add of mean (two separately rounded operations, as
    OpenCV's multiply/add do for a 32F image and a non-integer scalar), ``astype(uint8)``
    (truncation); the BGR flip and the flip back at :183 cancel.
    """
    x = img.detach().to(torch.float32).cpu().numpy()
    m = np.asarray(mean, dtype=np.float32).reshape(3, 1, 1)
    s = np.asarray(std, dtype=np.float32).reshape(3, 1, 1)
    y = (x * s).astype(np.float32) + m
    y = np.clip(np.trunc(y), 0, 255)
    return torch.from_numpy(y.astype(np.uint8))


def colour_similarity(lab, valid, size, dilation):
    """lab [3,H,W], valid [H,W] -> [k*k-1,H,W]:  exp(-|lab_p-lab_q|_2/2) * valid[q].

    Out-of-image q: LAB treated as 0 in the difference and valid as 0.
    condinst_head.py:220-246.
    """
    outs = []
    for dy, dx in neighbour_offsets(size, dilation):
        d = lab - _shifted(lab, dy, dx, 0.0)
        sim = torch.exp(-0.5 * torch.sqrt((d * d).sum(0)))
        outs.append(sim * _shifted(valid, dy, dx, 0.0))
    return torch.stack(outs, 0)


def box_bitmask(box, h_full, w_full, stride):
    """[h_full/stride, w_full/stride] float mask of the centre-sampled box.

    full[int(y1):int(y2)+1, int(x1):int(x2)+1] = 1 then [s//2::s, s//2::s]
    (condinst_head.py:1426-1432).  Python slicing semantics (negative / overshooting
    indices) are kept by rasterising exactly that way.
    """
    full = torch.zeros(h_full, w_full, dtype=torch.float32)
    x1, y1, x2, y2 = (float(v) for v in box)
    full[int(y1):int(y2) + 1, int(x1):int(x2) + 1] = 1.0
    st = stride // 2
    return full[st::stride, st::stride].clone()


def boxinst_targets(img, img_metas, gt_bboxes, stride=4, size=3, dilation=2,
                    bottom_pixels_removed=10):
    """Per-image similarity [B,k*k-1,H,W] (float32) and per-GT bitmasks (list of [G_i,H,W]).

    condinst_head.py:1345-1448 (get_targets + get_bitmasks_from_boxes) without the G-fold
    duplication of the similarity (every GT of an image shares one map).
    """
    B, _, hp, wp = img.shape
    assert hp % stride == 0 and wp % stride == 0
    st = stride // 2
    sims, bitmasks = [], []
    for i in range(B):
        meta = img_metas[i]
        ih, iw = meta['img_shape'][:2]
        valid = torch.ones(ih, iw, dtype=torch.float32)
        removed = int(bottom_pixels_removed * float(ih) / float(meta['ori_shape'][0]))
        if removed > 0:
            valid[-removed:, :] = 0
        valid = F.pad(valid, (0, wp - iw, 0, hp - ih))
        cfg = meta['img_norm_cfg']
        rgb = denormalise_to_u8(img[i, :, :ih, :iw], cfg['mean'], cfg['std']).float()
        rgb = F.pad(rgb, (0, wp - iw, 0, hp - ih))
        small = F.avg_pool2d(rgb[None], stride, stride)[0]
        small_u8 = small.to(torch.uint8).permute(1, 2, 0).numpy()
        lab = torch.from_numpy(rgb2lab_u8(small_u8)).to(torch.float32).permute(2, 0, 1)
        sims.append(colour_similarity(lab, valid[st::stride, st::stride], size, dilation))
        bitmasks.append(torch.stack([box_bitmask(b, hp, wp, stride) for b in gt_bboxes[i]])
                        if len(gt_bboxes[i]) else torch.zeros(0, hp // stride, wp // stride))
    return torch.stack(sims), bitmasks


# ----------------------------------------------------------------------------------------
# a6+a7+a8: the BoxInst mask loss
# ----------------------------------------------------------------------------------------
def boxinst_mask_loss(mask_logits, sim_per_inst, bitmask_per_inst, size=3, dilation=2,
                      colour_thresh=0.3, warmup_factor=1.0):
    """(loss_prj, loss_pairwise) of CondInstMaskHead.loss, condinst_head.py:1288-1343.

    mask_logits [N,1,H,W]; sim_per_inst [N,k*k-1,H,W]; bitmask_per_inst [N,1,H,W].
    """
    scores = mask_logits.sigmoid()
    loss_prj = projection_losses(scores, bitmask_per_inst).mean()
    pl = pairwise_nlog(mask_logits, size, dilation)
    wgt = (sim_per_inst >= colour_thresh).to(pl.dtype) * bitmask_per_inst.to(pl.dtype)
    loss_pair = (pl * wgt).sum() / wgt.sum().clamp(min=1.0) * warmup_factor
    return loss_prj, loss_pair


# ----------------------------------------------------------------------------------------
# a1: CondInst dynamic mask head
# ----------------------------------------------------------------------------------------
def aligned_bilinear(t, factor):
    """condinst_head.py:146-167 restated as an explicit gather-lerp.

    out[Y,X] = bilerp(t_pad, (Y - f//2)/f, (X - f//2)/f) for Y,X >= f//2 with t_pad the
    map extended by one replicated row/column; rows/cols < f//2 replicate index f//2.
    """
    if factor == 1:
        return t
    n, c, h, w = t.shape
    f = factor
    ys = (torch.arange(f * h, dtype=t.dtype) - f // 2).clamp(min=0) / f
    xs = (torch.arange(f * w, dtype=t.dtype) - f // 2).clamp(min=0) / f
    y0 = ys.floor().long()
    x0 = xs.floor().long()
    wy = (ys - y0).view(1, 1, -1, 1)
    wx = (xs - x0).view(1, 1, 1, -1)
    y1 = (y0 + 1).clamp(max=h - 1)
    x1 = (x0 + 1).clamp(max=w - 1)
    y0 = y0.clamp(max=h - 1)
    x0 = x0.clamp(max=w - 1)
    top = t[:, :, y0][:, :, :, x0] * (1 - wx) + t[:, :, y0][:, :, :, x1] * wx
    bot = t[:, :, y1][:, :, :, x0] * (1 - wx) + t[:, :, y1][:, :, :, x1] * wx
    return top * (1 - wy) + bot * wy


def condinst_mask_head(feat, params, coors, level_inds, img_inds, in_stride=8, out_stride=4,
                       sizes_of_interest=(64, 128, 256, 512, 1024), channels=8, rel_coors=True):
    """Dynamic 3-layer 1x1 FCN per instance + x(in_stride/out_stride) aligned upsample.

    feat [B,Cin,h,w]; params [N, P] laid out [W1|W2|W3|b1|b2|b3]; coors [N,2] (x,y);
    returns [N,1,f*h,f*w].  condinst_head.py:1120-1164.
    """
    n = params.size(0)
    _, cin, h, w = feat.shape
    x = feat[img_inds]
    if rel_coors:
        xs = torch.arange(w, dtype=feat.dtype) * in_stride + in_stride // 2
        ys = torch.arange(h, dtype=feat.dtype) * in_stride + in_stride // 2
        soi = torch.tensor(sizes_of_interest, dtype=feat.dtype)[level_inds].view(n, 1, 1)
        relx = (coors[:, 0].view(n, 1, 1) - xs.view(1, 1, w)).expand(n, h, w) / soi
        rely = (coors[:, 1].view(n, 1, 1) - ys.view(1, h, 1)).expand(n, h, w) / soi
        x = torch.cat([relx[:, None], rely[:, None], x], dim=1)
        cin = cin + 2
    sizes = [cin * channels, channels * channels, channels, channels, channels, 1]
    w1, w2, w3, b1, b2, b3 = torch.split(params, sizes, dim=1)
    x = x.flatten(2)                                                  # [N, cin, hw]
    x = torch.relu(torch.bmm(w1.reshape(n, channels, cin), x) + b1[:, :, None])
    x = torch.relu(torch.bmm(w2.reshape(n, channels, channels), x) + b2[:, :, None])
    x = torch.bmm(w3.reshape(n, 1, channels), x) + b3[:, :, None]
    return aligned_bilinear(x.view(n, 1, h, w), in_stride // out_stride)


# ----------------------------------------------------------------------------------------
# f2: CondInstMaskHead.training_sample, topk_per_img branch (condinst_head.py:1166-1232), restated with the same loops
# ----------------------------------------------------------------------------------------
def training_sample_topk(cls_scores, centerness, img_inds, gt_inds, topk_per_img):
    """cls_scores [P,C], centerness [P] (positives only, logits), img_inds / gt_inds [P] -> sampled indices into the
    positives, in the reference's order: images ascending, unique GT indices ascending, torch.topk order inside a GT that
    has more than inst_per_gt = max(int(topk / #GTs), 1) positives, original order otherwise."""
    out = []
    inst = torch.arange(cls_scores.shape[0])
    for img_id in range(int(img_inds.max()) + 1 if img_inds.numel() else 0):
        m = img_inds == img_id
        if not m.any():
            continue
        g = gt_inds[m]
        ids = inst[m]
        uniq = g.unique()
        per_gt = max(int(topk_per_img / uniq.numel()), 1)
        for gi in uniq:
            gm = g == gi
            sel = ids[gm]
            if sel.numel() > per_gt:
                sc = cls_scores[m][gm].sigmoid().max(dim=1)[0] * centerness[m][gm].sigmoid()
                sel = sel[sc.topk(per_gt, dim=0)[1]]
            out.append(sel)
    return torch.cat(out) if out else inst[:0]
