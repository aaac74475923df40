"""Box2MaskHead's training ``loss`` / ``loss_single`` / ``get_targets`` (mmdet/models/dense_heads/box2mask_head.py:135-335)
restated line by line, shared by the tests, oracle/make_golden_box2mask_loss.py and tools/bench_box2mask_loss.py.

The restatement keeps what the package's head replaces: one Hungarian matching per (layer, image) on the host with scipy
(mask_hungarian_assigner.py:113-132) and MaskPseudoSampler's boolean bookkeeping (mask_pseudo_sampler.py), the
classification loss as torch lines (``F.cross_entropy(weight=class_weight, reduction='none')`` + ``weight_reduce_loss``,
cross_entropy_loss.py, utils.py), boolean indexing of the matched rows, ``mask_weights.sum(dim=1).cpu()`` and the image
targets and trees repeated per matched query.  The cost matrix, the MST / tree filter and the mask-loss modules come from
``cpu_parts`` (CPU oracles; the cost on the up-sampled prediction as the reference computes it) or ``gpu_parts`` (the
package's CUDA pieces; the cost from the low-resolution profiles)."""
import types

import torch
import torch.nn.functional as F
from scipy.optimize import linear_sum_assignment

FLT_EPS = torch.finfo(torch.float32).eps


def upsampled_cost(cls_score, mask_pred, gt_labels, gt_masks, cls_weight=2.0, dice_weight=5.0, eps=1.0):
    """:157-161 + mask_hungarian_assigner.py:92-111 with ClassificationCost and BoxMatchingCost(pred_act=True) on the
    prediction up-sampled to the ground truths' size (match_cost.py:174-193, 381-425)."""
    mask_pred = F.interpolate(mask_pred.unsqueeze(1), gt_masks.shape[-2:], mode='bilinear', align_corners=False).sigmoid()
    gt = gt_masks.unsqueeze(1).float()

    def dice(a, b):
        a, b = a.flatten(1), b.flatten(1)
        return 1 - (2 * a @ b.t() + eps) / (a.pow(2).sum(1)[:, None] + b.pow(2).sum(1)[None, :] + eps)
    box = dice(mask_pred.max(dim=3, keepdim=True)[0], gt.max(dim=3, keepdim=True)[0]) + \
        dice(mask_pred.max(dim=2, keepdim=True)[0], gt.max(dim=2, keepdim=True)[0])
    return -cls_score.softmax(-1)[:, gt_labels] * cls_weight + box * dice_weight


def cpu_parts(loss_box_weight=5.0, loss_mask_weight=1.0):
    """CPU oracles: the up-sampled cost, the Kruskal MST and tree filter of oracle/tree.py, the restated projection,
    level-set and LCM losses."""
    from oracle import boxinst as ob
    from oracle import levelset as ol
    from oracle import tree as ot
    return types.SimpleNamespace(
        cost=upsampled_cost, mst=lambda fm: ot.mst(fm.detach()), tree_filter=ot.tree_filter,
        loss_box=lambda s, b: loss_box_weight * ob.projection_losses(s, b),
        loss_mask=lambda phi, t, pix: ol.levelset_loss(phi, t, pix, loss_mask_weight), lcm=ol.lcm_loss)


def gpu_parts(head):
    """The same pieces as the package provides them on the GPU (each pinned against the reference by its own tests): the
    assigner's cost from the low-resolution profiles, the MST / tree filter, the loss modules and the LCM kernel."""
    from boxinstseg_b200.models.losses import LCM
    return types.SimpleNamespace(
        cost=lambda c, m, l, g: head.hungarian.cost_matrix(c, m, l, g, lowres=True), mst=head.mst,
        tree_filter=head.tree_filter, loss_box=head.loss_box, loss_mask=head.loss_mask, lcm=LCM)


def _scale_target(t, size=(96, 96)):                                             # mmdet/models/utils/misc.py:75-86
    return F.interpolate(t.unsqueeze(1) if t.dim() == 3 else t, size=size, mode='bilinear', align_corners=False)


def get_target_single(parts, num_queries, num_classes, cls_score, mask_pred, gt_labels, gt_masks):    # :152-189
    """(labels, label_weights, mask_targets, mask_weights, pos_inds, neg_inds) with scipy and MaskPseudoSampler.sample."""
    dev = mask_pred.device
    gt_inds = torch.zeros(mask_pred.shape[0], dtype=torch.long, device=dev)
    if gt_labels.shape[0] and mask_pred.shape[0]:
        cost = parts.cost(cls_score, mask_pred, gt_labels, gt_masks).detach().cpu()
        r, c = linear_sum_assignment(cost)
        gt_inds[torch.from_numpy(r).to(dev)] = torch.from_numpy(c).to(dev) + 1
    pos_inds = torch.nonzero(gt_inds > 0, as_tuple=False).squeeze(-1).unique()
    neg_inds = torch.nonzero(gt_inds == 0, as_tuple=False).squeeze(-1).unique()
    pos_assigned_gt_inds = gt_inds[pos_inds] - 1
    labels = gt_labels.new_full((num_queries,), num_classes, dtype=torch.long)
    labels[pos_inds] = gt_labels[pos_assigned_gt_inds].long()
    label_weights = gt_labels.new_ones((num_queries,))
    mask_targets = gt_masks.unsqueeze(1)[pos_assigned_gt_inds]
    mask_weights = mask_pred.new_zeros((num_queries,))
    mask_weights[pos_inds] = 1.0
    return labels, label_weights, mask_targets, mask_weights, pos_inds, neg_inds


def get_targets(parts, num_queries, num_classes, cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list):
    """:135-149"""
    out = list(zip(*[get_target_single(parts, num_queries, num_classes, c, m, l, g)
                     for c, m, l, g in zip(cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list)]))
    return (*[list(o) for o in out[:4]], sum(i.numel() for i in out[4]), sum(i.numel() for i in out[5]))


def cross_entropy_loss(cls_scores, labels, label_weights, class_weight, loss_weight, avg_factor):
    """CrossEntropyLoss(use_sigmoid=False, reduction='mean').forward (cross_entropy_loss.py:12-60, 257-300) +
    weight_reduce_loss (utils.py:30-59)."""
    loss = F.cross_entropy(cls_scores, labels, weight=class_weight, reduction='none', ignore_index=-100)
    loss = loss * label_weights.float()
    return loss_weight * (loss.sum() / (avg_factor + FLT_EPS))


def loss_single(parts, num_queries, num_classes, class_weight, cls_loss_weight, cls_scores, mask_preds, lst_feat,
                gt_labels_list, gt_masks_list, norm_img):                                                    # :224-335
    """(loss_cls, loss_project, loss_levelset) of one decoder layer."""
    pred_shape = mask_preds.shape[-2:]
    norm_img = F.interpolate(norm_img, pred_shape, mode='bilinear', align_corners=False)
    lst_feat = F.interpolate(lst_feat, pred_shape, mode='bilinear', align_corners=False)
    num_imgs = cls_scores.size(0)
    (labels_list, label_weights_list, mask_targets_list, mask_weights_list, _, _) = get_targets(
        parts, num_queries, num_classes, [cls_scores[i] for i in range(num_imgs)], [mask_preds[i] for i in range(num_imgs)],
        gt_labels_list, gt_masks_list)
    labels = torch.stack(labels_list, dim=0).flatten(0, 1)
    label_weights = torch.stack(label_weights_list, dim=0).flatten(0, 1)
    mask_targets = torch.cat(mask_targets_list, dim=0)
    mask_weights = torch.stack(mask_weights_list, dim=0)
    cw = cls_scores.new_tensor(class_weight)
    loss_cls = cross_entropy_loss(cls_scores.flatten(0, 1), labels, label_weights, cw, cls_loss_weight, cw[labels].sum())
    mask_preds = mask_preds[mask_weights > 0]
    if mask_targets.shape[0] == 0:
        return loss_cls, mask_preds.sum(), mask_preds.sum()
    scale_img, scale_feat = _scale_target(norm_img), _scale_target(lst_feat)
    norm_img_tree, lst_feat_tree = parts.mst(scale_img), parts.mst(scale_feat)
    repeat = [int(v) for v in mask_weights.sum(dim=1).cpu().numpy().tolist()]
    keep = [i for i in range(num_imgs) if repeat[i]]
    img_targets = torch.cat([norm_img[i:i + 1].repeat(repeat[i], 1, 1, 1) for i in keep], 0)
    lst_targets = torch.cat([lst_feat[i:i + 1].repeat(repeat[i], 1, 1, 1) for i in keep], 0)
    img_tree = torch.cat([norm_img_tree[i:i + 1].repeat(repeat[i], 1, 1) for i in keep], 0)
    feat_tree = torch.cat([lst_feat_tree[i:i + 1].repeat(repeat[i], 1, 1) for i in keep], 0)
    box = F.interpolate(mask_targets.to(mask_preds.dtype), pred_shape, mode='bilinear', align_corners=False)
    s = torch.sigmoid(mask_preds.unsqueeze(dim=1))
    loss_project = parts.loss_box(s, box).mean()
    phi = torch.cat((s, 1.0 - s), dim=1) * box
    pixel_num = torch.clamp(box.sum((1, 2, 3)), min=1)
    loss_img = parts.loss_mask(phi, img_targets * box, pixel_num).mean() * 0.05
    img_targets, lst_targets, s96 = _scale_target(img_targets), _scale_target(lst_targets), _scale_target(s)
    f_img = parts.tree_filter(s96, img_targets, img_tree)
    f_lst = parts.tree_filter(f_img, lst_targets, feat_tree, low_tree=False)
    deep = torch.cat((F.interpolate(f_img, pred_shape, mode='bilinear', align_corners=False),
                      F.interpolate(f_lst, pred_shape, mode='bilinear', align_corners=False)), dim=1) * box
    loss_feat = parts.loss_mask(phi, deep, pixel_num).mean() * 5.0
    loss_lcm = 0.2 * parts.lcm(img_targets, s96, _scale_target(box))
    return loss_cls, loss_project, loss_img + loss_feat + loss_lcm


def loss(parts, num_queries, num_classes, class_weight, cls_loss_weight, all_cls_scores, all_mask_preds, all_lst_feats,
         gt_labels_list, gt_masks_list, norm_img):                                                           # :192-221
    """The reference's dict, with ``all_cls_scores`` / ``all_mask_preds`` promoted to float32 (``@force_fp32``)."""
    outs = [loss_single(parts, num_queries, num_classes, class_weight, cls_loss_weight, c.float(), m.float(), f,
                        gt_labels_list, gt_masks_list, norm_img)
            for c, m, f in zip(all_cls_scores, all_mask_preds, all_lst_feats)]
    d = dict(loss_cls=outs[-1][0], loss_project=outs[-1][1], loss_levelset=outs[-1][2])
    for i, (c, p, s) in enumerate(outs[:-1]):
        d[f'd{i}.loss_cls'], d[f'd{i}.loss_project'], d[f'd{i}.loss_levelset'] = c, p, s
    return d


def assignments(parts, cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list):
    """The matched ground truth of every query (-1: none) per image, scipy on ``parts.cost``."""
    out = []
    for c, m, l, g in zip(cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list):
        match = torch.full((m.shape[0],), -1, dtype=torch.long)
        if l.shape[0]:
            r, k = linear_sum_assignment(parts.cost(c, m, l, g).detach().cpu())
            match[torch.from_numpy(r)] = torch.from_numpy(k)
        out.append(match)
    return out


def golden_case(seed=0, B=2, gts=(3, 0), Q=8, num_classes=4, layers=3, pred=96, mask=192, margin=6.0):
    """The seeded case of tests/golden/box2mask_loss.npz (CPU tensors): (all_cls_scores, all_mask_preds, all_lst_feats,
    gt_labels_list, gt_masks_list, norm_img).  Layer l plants ground truth g on query perm_l[g]: a box-shaped logit map
    (+margin inside, -margin outside) and a class logit of +margin, so that every matching is unique by a clear margin; the
    other queries are small noise.  The default prediction size is the trees' 96x96, so no map the MSTs are built on is an
    up-sampled one: bilinear up-sampling makes linear ramps whose neighbouring differences tie, and a tie lets two
    implementations of the resize that differ in the last bit pick different, equally minimal trees."""
    gen = torch.Generator().manual_seed(seed)
    K = num_classes + 1
    gt_labels, gt_masks, boxes = [], [], []
    for G in gts:
        m = torch.zeros(G, mask, mask, dtype=torch.long)
        bx = []
        for g in range(G):
            y0, x0 = (int(v) for v in torch.randint(0, mask // 2, (2,), generator=gen))
            hh, ww = (int(v) for v in torch.randint(mask // 6, mask // 2, (2,), generator=gen))
            m[g, y0:y0 + hh, x0:x0 + ww] = 1
            bx.append((y0, x0, hh, ww))
        gt_masks.append(m)
        gt_labels.append(torch.randint(0, num_classes, (G,), generator=gen))
        boxes.append(bx)
    cls_all, mask_all, lst_all = [], [], []
    f = pred / mask
    for _ in range(layers):
        cls = torch.randn(B, Q, K, generator=gen) * 0.5
        mp = torch.randn(B, Q, pred, pred, generator=gen) * 0.5 - margin
        for b in range(B):
            perm = torch.randperm(Q, generator=gen)
            for g, (y0, x0, hh, ww) in enumerate(boxes[b][:Q]):
                q = int(perm[g])
                mp[b, q, int(y0 * f):int((y0 + hh) * f), int(x0 * f):int((x0 + ww) * f)] += 2 * margin
                cls[b, q, int(gt_labels[b][g])] += margin
        cls_all.append(cls)
        mask_all.append(mp)
        lst_all.append(torch.randn(B, 1, pred, pred, generator=gen))
    norm_img = F.interpolate(torch.randn(B, 3, 8, 8, generator=gen), (mask, mask), mode='bilinear', align_corners=False) + \
        0.05 * torch.randn(B, 3, mask, mask, generator=gen)
    return cls_all, mask_all, lst_all, gt_labels, gt_masks, norm_img


# configs/box2mask/box2mask_r50_lsj_8x2_50e_coco.py:92-97, 110-114
GOLDEN_NUM_CLASSES = 4
GOLDEN_CLASS_WEIGHT = [1.0] * GOLDEN_NUM_CLASSES + [0.1]
ASSIGNER = dict(type='MaskHungarianAssigner', cls_cost=dict(type='ClassificationCost', weight=2.0),
                dice_cost=dict(type='BoxMatchingCost', weight=5.0, pred_act=True, eps=1.0))
