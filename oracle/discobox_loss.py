"""Restatement of ``DiscoBoxSOLOv2Head.loss`` (mmdet/models/dense_heads/discobox_head.py:1142-1360) without the
correspondence branch (``use_corr=False``): the SOLO targets of every image (``solov2_target_single``), the kernels of the
covered cells gathered by ``grid_order`` and one convolution per (level, image) with objects, the host loops over levels and
images, one mean field per image, the MIL and teacher-student dice losses and the category focal loss on the permuted and
concatenated logits (the torch form, ``py_sigmoid_focal_loss``).  Plain torch, on CPU or CUDA tensors."""
import torch
import torch.nn.functional as F

from oracle import levelset as ol
from oracle import solo_targets as ost
from oracle.solo_head import py_sigmoid_focal_loss

# the head's defaults (discobox_head.py:662-666, 703-719) and the DiscoBox config's loss_ts / loss_cate
CFG = dict(scale_ranges=((8, 32), (16, 64), (32, 128), (64, 256), (128, 512)), strides=(8, 8, 16, 32, 32), sigma=0.2,
           ins_loss_weight=1.0, ts_loss_weight=1.0, mf=dict(alpha0=2.0, theta0=0.5, theta1=30.0, kernel_size=3, base=0.10,
                                                             iter=10),
           focal=(2.0, 0.25, 1.0))


def dice_loss(x, t):
    """:542-550, in its own order of additions (float32, as there)."""
    x = x.contiguous().view(x.size(0), -1).float()
    t = t.contiguous().view(t.size(0), -1).float()
    return 1 - (2 * (x * t).sum(1)) / (((x * x).sum(1) + 0.001) + ((t * t).sum(1) + 0.001))


def mil_loss(x, t):
    """:552-562."""
    return dice_loss(x.max(2)[0], t.max(2)[0]) + dice_loss(x.max(1)[0], t.max(1)[0])


def conv2d(feat_img, kernels):
    """:1214-1219: feat_img [C,h,w], kernels [C,I] -> [I,h,w]."""
    C, I = kernels.shape
    return F.conv2d(feat_img[None], kernels.permute(1, 0).view(I, -1, 1, 1), stride=1)[0]


def loss(cate_preds, s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list, gt_label_list,
         gt_mask_list, img, seg_num_grids, num_classes, use_loss_ts=False, use_ind_teacher=False, cfg=CFG, conv=conv2d):
    """gt_mask_list: per image uint8 NUMPY [G,H,W].  ``conv`` computes one (level, image) convolution (default: F.conv2d).
    Returns dict(loss_ins, loss_ts, loss_cate, loss_corr) as the reference does with use_corr=False."""
    fsize = tuple(s_ins_pred.shape[-2:])
    dev = s_ins_pred.device
    tg = [ost.disco_target_single(b.cpu(), l.cpu(), m, fsize, cfg['scale_ranges'], cfg['strides'], seg_num_grids,
                                  cfg['sigma'], num_classes, best=False)
          for b, l, m in zip(gt_bbox_list, gt_label_list, gt_mask_list)]
    L_, B = len(seg_num_grids), len(tg)
    ins_labels = [torch.cat([tg[b][0][lv] for b in range(B)], 0).to(dev) for lv in range(L_)]
    s_list, t_list, img_list = [], [], []
    for lv in range(L_):                                                                    # :1206-1246
        s_b, t_b, i_b = [], [], []
        for b in range(B):
            order = torch.as_tensor(tg[b][3][lv], dtype=torch.int64, device=dev)
            if order.numel() == 0:
                continue
            C = s_kernel_preds_raw[lv].shape[1]
            s_b.append(conv(s_ins_pred[b], s_kernel_preds_raw[lv][b].reshape(C, -1)[:, order]))
            if use_ind_teacher:
                t_b.append(conv(t_ins_pred[b], t_kernel_preds_raw[lv][b].reshape(C, -1)[:, order]))
            i_b.append(torch.ones(order.numel(), device=dev) * b)
        s_list.append(torch.cat(s_b, 0) if s_b else None)
        t_list.append(torch.cat(t_b, 0) if t_b else None)
        img_list.append(torch.cat(i_b, 0) if i_b else None)
    color_feats = F.interpolate(img, fsize, mode='bilinear', align_corners=True)          # :1201
    mf = cfg['mf']
    kernels = [ol.meanfield_kernel(color_feats[b:b + 1], mf['kernel_size'], mf['theta0'], mf['theta1'], mf['alpha0'])
               for b in range(B)]
    loss_ins, loss_ts = [], []
    for s_in, t_in, img_inds, target in zip(s_list, t_list, img_list, ins_labels):          # :1271-1300
        if s_in is None:
            continue
        s = torch.sigmoid(s_in)
        t = torch.sigmoid(t_in) if use_ind_teacher else s
        keep = torch.tensor([bool(x.sum()) for x in target], device=dev)
        if keep.sum() == 0:
            continue
        s, t, img_inds, target = s[keep], t[keep], img_inds[keep], target[keep]
        loss_ins.append(mil_loss(s, target))
        if use_loss_ts:
            enlarged = F.max_pool2d(target.float()[:, None], kernel_size=3, stride=1, padding=1)[:, 0].byte()
            for b in range(B):
                sel = img_inds == b
                if sel.sum() > 0:
                    x = ((t[sel][:, None] + s[sel][:, None]) / 2).float()
                    pseudo, _ = ol.meanfield_forward(kernels[b].to(x.dtype), x, target[sel][:, None].to(x.dtype),
                                                     mf['kernel_size'], mf['iter'], mf['base'])
                    loss_ts.append(dice_loss(s[sel] * enlarged[sel], pseudo))
    zero = color_feats.new_zeros(())
    l_ins = torch.cat(loss_ins).mean() * cfg['ins_loss_weight'] if loss_ins else zero
    l_ts = torch.cat(loss_ts).mean() * cfg['ts_loss_weight'] if (use_loss_ts and loss_ts) else zero
    cate_labels = torch.cat([torch.cat([tg[b][1][lv].flatten() for b in range(B)]) for lv in range(L_)]).to(dev)
    num_ins = torch.cat([torch.cat([tg[b][2][lv].flatten() for b in range(B)]) for lv in range(L_)]).sum()
    C = cate_preds[0].shape[1]
    flat = torch.cat([p.permute(0, 2, 3, 1).reshape(-1, C) for p in cate_preds]).float()   # :1348-1355
    onehot = F.one_hot(cate_labels, C + 1)[:, :C]
    gamma, alpha, weight = cfg['focal']
    l_cate = py_sigmoid_focal_loss(flat, onehot, gamma, alpha, float(num_ins) + 1, weight)
    return dict(loss_ins=l_ins, loss_ts=l_ts, loss_cate=l_cate, loss_corr=zero)
