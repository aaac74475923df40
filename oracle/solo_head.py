"""BoxSOLOv2Head's training ``forward`` and ``loss`` (mmdet/models/dense_heads/box_solov2_head.py:179-388) restated line by
line, and seeded stand-in towers with the reference constructor's channel plan (:62-157), shared by the tests and
tools/bench_solo_head.py.

The restatement keeps what the package's head replaces: the dense ``F.conv2d(groups=B)`` over every grid cell and its
``F.interpolate`` (:204-216), boolean indexing, image / level-set targets repeated per instance (:294-320), and the focal
loss as torch lines (``py_sigmoid_focal_loss`` + ``weight_reduce_loss``, mmdet/models/losses/focal_loss.py, utils.py).  The
per-level mask-loss lines (:334-367) are restated too; the target builder, the MST / tree filter and the two loss modules
come from ``cpu_parts`` (CPU oracles: pinned to the reference's own methods by tests/golden/solo_head.npz, minted by
oracle/make_golden_solo_head.py) or ``gpu_parts`` (the package's CUDA pieces)."""
import math
import types

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F


def _conv_module(cin, cout, norm):
    """mmcv ConvModule(3x3, padding 1): conv (no bias under a norm) -> GN(32) -> ReLU."""
    if norm:
        return nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1, bias=False), nn.GroupNorm(32, cout), nn.ReLU())
    return nn.Sequential(nn.Conv2d(cin, cout, 3, padding=1), nn.ReLU())


def attach_towers(head, in_channels, seg_feat_channels, num_classes, stacked_convs=4, seed=0):
    """Adds ``_init_layers``'s modules to ``head`` (the config's norm_cfg=None for feature_convs, GN(32) for the kernel and
    category towers), initialised from ``seed`` (torch's default init, the category bias at prior 0.01)."""
    with torch.random.fork_rng(devices=[]):
        torch.manual_seed(seed)
        feature_convs = nn.ModuleList()
        for i in range(4):
            seq = nn.Sequential()
            if i == 0:
                seq.add_module('conv0', _conv_module(in_channels, seg_feat_channels, False))
            for j in range(i):
                cin = (in_channels + 2 if i == 3 else in_channels) if j == 0 else seg_feat_channels
                seq.add_module(f'conv{j}', _conv_module(cin, seg_feat_channels, False))
                seq.add_module(f'upsample{j}', nn.Upsample(scale_factor=2, mode='bilinear', align_corners=False))
            feature_convs.append(seq)
        kernel_convs = nn.ModuleList(_conv_module(in_channels + 2 if i == 0 else seg_feat_channels, seg_feat_channels, True)
                                     for i in range(stacked_convs))
        cate_convs = nn.ModuleList(_conv_module(in_channels if i == 0 else seg_feat_channels, seg_feat_channels, True)
                                   for i in range(stacked_convs))
        solo_cate = nn.Conv2d(seg_feat_channels, num_classes, 3, padding=1)
        nn.init.constant_(solo_cate.bias, -math.log((1 - 0.01) / 0.01))
        solo_kernel = nn.Conv2d(seg_feat_channels, seg_feat_channels, 1)
        solo_mask = nn.Conv2d(seg_feat_channels, seg_feat_channels, 1)
        levelset_bottom = nn.Conv2d(seg_feat_channels, 5, 3, padding=1)
    head.feature_convs, head.kernel_convs, head.cate_convs = feature_convs, kernel_convs, cate_convs
    head.solo_cate, head.solo_kernel, head.solo_mask, head.levelset_bottom = solo_cate, solo_kernel, solo_mask, levelset_bottom
    return head


def _coord(x):
    x_range = torch.linspace(-1, 1, x.shape[-1], device=x.device)
    y_range = torch.linspace(-1, 1, x.shape[-2], device=x.device)
    y, xx = torch.meshgrid(y_range, x_range, indexing='ij')
    return torch.cat([xx.expand([x.shape[0], 1, -1, -1]), y.expand([x.shape[0], 1, -1, -1])], 1)


def forward_single(head, x, idx, eval=False):                                 # :226-260
    kernel_feat = torch.cat([x, _coord(x)], 1)
    cate_feat = x
    for i, layer in enumerate(head.kernel_convs):
        if i == head.cate_down_pos:
            kernel_feat = F.interpolate(kernel_feat, size=head.seg_num_grids[idx], mode='bilinear')
        kernel_feat = layer(kernel_feat)
    kernel_pred = head.solo_kernel(kernel_feat)
    for i, layer in enumerate(head.cate_convs):
        if i == head.cate_down_pos:
            cate_feat = F.interpolate(cate_feat, size=head.seg_num_grids[idx], mode='bilinear')
        cate_feat = layer(cate_feat)
    cate_pred = head.solo_cate(cate_feat)
    if eval:
        cate_pred = cate_pred.sigmoid()
        local_max = F.max_pool2d(cate_pred, (2, 2), stride=1, padding=1)
        keep_mask = local_max[:, :, :-1, :-1] == cate_pred
        cate_pred = (cate_pred * keep_mask).permute(0, 2, 3, 1)
    return kernel_pred, cate_pred


def forward(head, feats, eval=False):                                         # :179-217
    feats = [feat.float() for feat in feats]
    new_feats = (F.interpolate(feats[0], scale_factor=0.5, mode='bilinear'), feats[1], feats[2], feats[3],
                 F.interpolate(feats[4], size=feats[3].shape[-2:], mode='bilinear'))          # split_feats, :219-224
    featmap_sizes = [f.size()[-2:] for f in new_feats]
    kernel_pred, cate_pred = zip(*[forward_single(head, x, i, eval) for i, x in enumerate(new_feats)])
    coord_feat = _coord(feats[-2])
    fa = head.feature_convs[0](feats[0])
    for i in range(1, 3):
        fa = fa + head.feature_convs[i](feats[i])
    fa = fa + head.feature_convs[3](torch.cat([feats[3], coord_feat], 1))
    feature_pred = head.solo_mask(fa)
    levelset_feats = head.levelset_bottom(feature_pred)
    N, c, h, w = feature_pred.shape
    feature_pred = feature_pred.view(-1, h, w).unsqueeze(0)
    ins_pred = []
    for i in range(len(kernel_pred)):
        kernel = kernel_pred[i].permute(0, 2, 3, 1).contiguous().view(-1, c).unsqueeze(-1).unsqueeze(-1)
        ins_i = F.conv2d(feature_pred, kernel, groups=N).view(N, head.seg_num_grids[i] ** 2, h, w)
        if not eval:
            ins_i = F.interpolate(ins_i, size=(featmap_sizes[i][0] * 2, featmap_sizes[i][1] * 2), mode='bilinear')
        else:
            ins_i = ins_i.sigmoid()
        ins_pred.append(ins_i)
    return ins_pred, list(cate_pred), levelset_feats


def py_sigmoid_focal_loss(pred, target, gamma, alpha, avg_factor, loss_weight):
    """FocalLoss(use_sigmoid=True).forward on one-hot targets (focal_loss.py:35-57, 225-240) + weight_reduce_loss with
    reduction 'mean' (utils.py): loss_weight * sum / (avg_factor + eps)."""
    pred_sigmoid = pred.sigmoid()
    target = target.type_as(pred)
    pt = (1 - pred_sigmoid) * target + pred_sigmoid * (1 - target)
    focal_weight = (alpha * target + (1 - alpha) * (1 - target)) * pt.pow(gamma)
    loss = F.binary_cross_entropy_with_logits(pred, target, reduction='none') * focal_weight
    return loss_weight * (loss.sum() / (avg_factor + torch.finfo(torch.float32).eps))


def gpu_parts(head):
    """The pieces ``loss`` calls, as the package provides them on the GPU: device grid targets, the package's MST / tree
    filter and loss modules (each pinned against the reference by its own tests)."""
    from boxinstseg_b200.models.dense_heads.solo_targets import solo_target_single

    def targets(b, l, m, norm_img, lst, featmap_sizes):
        return solo_target_single(b, l, m, norm_img, lst, featmap_sizes, head.scale_ranges, head.strides, head.seg_num_grids,
                                  head.sigma, head.num_classes)
    return types.SimpleNamespace(targets=targets, mst=head.mst, tree_filter=head.tree_filter, loss_boxpro=head.loss_boxpro,
                                 loss_levelset=head.loss_levelset)


def cpu_parts(head, boxpro_weight=3.0, levelset_weight=1.0):
    """The same pieces as CPU oracles: the host target builder (numpy masks, scipy, cv2; oracle/solo_targets.py), the
    Kruskal MST and tree filter of oracle/tree.py, and the restated projection / level-set losses."""
    from oracle import boxinst as ob
    from oracle import levelset as ol
    from oracle import solo_targets as ost
    from oracle import tree as ot

    def targets(b, l, m, norm_img, lst, featmap_sizes):
        return ost.solo_target_single(b, l, m, norm_img, lst, featmap_sizes, head.scale_ranges, head.strides,
                                      head.seg_num_grids, head.sigma, head.num_classes)
    return types.SimpleNamespace(targets=targets, mst=lambda fm: ot.mst(fm.detach()), tree_filter=ot.tree_filter,
                                 loss_boxpro=lambda s, b: boxpro_weight * ob.projection_losses(s, b),
                                 loss_levelset=lambda phi, t, pix: ol.levelset_loss(phi, t, pix, levelset_weight))


def loss(head, ins_preds, cate_preds, levelset_feats, gt_bbox_list, gt_label_list, gt_mask_list, img, gamma=2.0, alpha=0.25,
         loss_weight=1.0, parts=None):                                        # :262-388
    """The reference's ``loss`` lines; ``parts`` (default ``gpu_parts(head)``) supplies the target builder, MST, tree filter
    and the two mask-loss modules."""
    parts = parts or gpu_parts(head)
    featmap_sizes = [featmap.size()[-2:] for featmap in ins_preds]
    per_img = [parts.targets(b, l, m, img[i], levelset_feats[i], featmap_sizes)
               for i, (b, l, m) in enumerate(zip(gt_bbox_list, gt_label_list, gt_mask_list))]
    ins_label_list, cate_label_list, ins_ind_label_list, scale_img_list, scale_lst_list = zip(*per_img)
    lv_ind = list(zip(*ins_ind_label_list))
    ins_labels = [torch.cat([a[i] for a, i in zip(lv, ind)], 0) for lv, ind in zip(zip(*ins_label_list), lv_ind)]
    img_target = [torch.cat([s.repeat(a[i].shape[0], 1, 1, 1) for a, i, s in zip(lv, ind, si)], 0)
                  for lv, ind, si in zip(zip(*ins_label_list), lv_ind, zip(*scale_img_list))]
    lst_target = [torch.cat([s.expand(a[i].shape[0], s.shape[-3], s.shape[-2], s.shape[-1]) for a, i, s in zip(lv, ind, sl)], 0)
                  for lv, ind, sl in zip(zip(*ins_label_list), lv_ind, zip(*scale_lst_list))]
    ins_pos = [torch.cat([p[i] for p, i in zip(pl, ind)], 0) for pl, ind in zip(ins_preds, lv_ind)]
    num_ins = torch.cat([torch.cat([i.flatten() for i in ind]) for ind in lv_ind]).int().sum()
    loss_project, loss_levelset = [], []
    for ins_pred, box_mask, img_t, lst_t in zip(ins_pos, ins_labels, img_target, lst_target):    # :334-364
        if ins_pred.size()[0] == 0:
            continue
        mask_pred = torch.sigmoid(ins_pred.unsqueeze(dim=1))
        box = box_mask.unsqueeze(dim=1).to(dtype=mask_pred.dtype)
        loss_project.append(parts.loss_boxpro(mask_pred, box))
        phi = torch.cat((mask_pred, 1.0 - mask_pred), dim=1) * box
        pixel_num = torch.clamp(box.sum((1, 2, 3)), min=1)
        loss_img = parts.loss_levelset(phi, img_t * box, pixel_num) * 0.05
        f_img = parts.tree_filter(mask_pred, img_t, parts.mst(img_t))
        f_lst = parts.tree_filter(f_img, lst_t, parts.mst(lst_t), low_tree=False)
        loss_feat = parts.loss_levelset(phi, torch.cat((f_img, f_lst), dim=1) * box, pixel_num) * 5.0
        loss_levelset.append(loss_img + loss_feat)
    flatten_cate_labels = torch.cat([torch.cat([c.flatten() for c in lv]) for lv in zip(*cate_label_list)])
    flatten_cate_preds = torch.cat([c.permute(0, 2, 3, 1).reshape(-1, head.num_classes) for c in cate_preds])
    target = F.one_hot(flatten_cate_labels, num_classes=head.num_classes + 1)[:, :head.num_classes]
    loss_cate = py_sigmoid_focal_loss(flatten_cate_preds, target, gamma, alpha, num_ins + 1, loss_weight)
    return dict(loss_boxpro=torch.cat(loss_project).mean(), loss_levelset=torch.cat(loss_levelset).mean(), loss_cate=loss_cate)


def golden_case(seed=0, B=2, H=128, W=160, C=64, gts=3, mask_sizes=None):
    """The seeded case of tests/golden/solo_head.npz on the CPU: (head with stand-in towers, FPN inputs P2..P6, images,
    boxes, labels, box-shaped uint8 masks as numpy arrays).  ``mask_sizes[b]``: the (H_b, W_b) of image b's masks (mmdet pads
    an image's masks to that image's own pad shape, not to the batch's)."""
    from boxinstseg_b200.models import build_head
    gen = torch.Generator().manual_seed(seed)
    head = attach_towers(build_head(dict(GOLDEN_HEAD, in_channels=C, seg_feat_channels=C)), C, C, 80, seed=seed)
    feats = [torch.randn(B, C, -(-H // s), -(-W // s), generator=gen) for s in (4, 8, 16, 32, 64)]
    img = torch.randn(B, 3, H, W, generator=gen)
    bboxes, labels, masks = [], [], []
    for b in range(B):
        hb, wb = mask_sizes[b] if mask_sizes else (H, W)
        wh = 12 + torch.rand(gts, 2, generator=gen) * torch.tensor([wb - 16.0, hb - 16.0]) * 0.7
        x1 = torch.rand(gts, generator=gen) * (wb - 2 - wh[:, 0])
        y1 = torch.rand(gts, generator=gen) * (hb - 2 - wh[:, 1])
        bx = torch.stack([x1, y1, x1 + wh[:, 0], y1 + wh[:, 1]], 1)
        m = np.zeros((gts, hb, wb), np.uint8)
        for g, (a, c, d, e) in enumerate(bx.tolist()):
            m[g, int(c):int(e) + 1, int(a):int(d) + 1] = 1
        bboxes.append(bx)
        labels.append(torch.randint(0, 80, (gts,), generator=gen))
        masks.append(m)
    return head, feats, img, bboxes, labels, masks


# configs/boxlevelset/box_levelset_coco_r50_fpn_3x.py:17-33
GOLDEN_HEAD = dict(type='BoxSOLOv2Head', num_classes=80, stacked_convs=4, strides=[8, 8, 16, 32, 32],
                   scale_ranges=((1, 96), (48, 192), (96, 384), (192, 768), (384, 2048)), sigma=0.2,
                   num_grids=[40, 36, 24, 16, 12], cate_down_pos=0,
                   loss_cate=dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0))
