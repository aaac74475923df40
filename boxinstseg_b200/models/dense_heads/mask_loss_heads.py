"""Mask-loss assembly of the three SOLO/Mask2Former-style heads (SURVEY.md section 8 row a17) and their
dynamic-conv call sites (a2-a4), on the kernels of libboxseg_b200:

  ``BoxSOLOv2Head``       mmdet/models/dense_heads/box_solov2_head.py:204-217 (dynamic conv), :334-367 (loss)
  ``DiscoBoxSOLOv2Head``  mmdet/models/dense_heads/discobox_head.py:1206-1300 (per-image conv, MIL dice, mean-field teacher)
  ``Box2MaskHead``        mmdet/models/dense_heads/box2mask_head.py:338-359 (mask_pred einsum), :269-335 (loss_single)

The mask-loss hot path and its immediate callers are implemented here: the SOLO target builders live in
``solo_targets.py`` / ``disco_targets.py`` (f2), the Hungarian front half in ``core/assigner.py`` (f1), DiscoBox's
cross-image correspondence loss in ``disco_corr.py`` (f4; ``DiscoBoxSOLOv2Head.corr_inputs / corr_loss``).  The conv towers,
category losses and inference are out of scope (SURVEY 2.1 row 3): the classes keep the reference's registry names and accept (and store) the reference's constructor kwargs so
the configs build, and expose the hot-path pieces as methods with the tensors the reference passes between
its own lines.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ...ops.box2mask import attention_mask
from ...ops.discobox import HALF_DTYPES, discobox_mask_loss
from ...ops.dynconv import box2mask_mask_pred, dynconv1x1, solo_cells_conv, solo_dynamic_conv
from ...ops.lsap import solve_batched
from ...ops.resize import bilinear_resize, scale_target as _scale_target   # a18: F.interpolate / _scale_target as kernels
from ...ops._streams import Forked, run_concurrently
from ...ops.tree_filter import MinimumSpanningTree, TreeFilter2D
from ..builder import HEADS, build_loss, register
from ..losses import LCM, levelset_assembly, mil_loss
from .meanfield import MeanField


def _phi_and_pixels(mask_pred, box_mask):
    """cat(s, 1-s) * box ; clamp(sum box, 1)  (box_solov2_head.py:341-349, box2mask_head.py:305-310)."""
    phi = torch.cat((mask_pred, 1.0 - mask_pred), dim=1) * box_mask
    pix = box_mask.sum((1, 2, 3)).clamp(min=1)
    return phi, pix


@register(HEADS, partial=True)
class BoxSOLOv2Head(nn.Module):
    """BoxLevelset head: mask-loss path only."""

    def __init__(self, num_classes=80, in_channels=256, loss_boxpro=None, loss_levelset=None, **cfg):
        super().__init__()
        self.num_classes = num_classes
        self.in_channels = in_channels
        self.cfg = cfg
        self.loss_boxpro = build_loss(loss_boxpro or dict(type='BoxProjectionLoss', loss_weight=3.0))
        self.loss_levelset = build_loss(loss_levelset or dict(type='LevelsetLoss', loss_weight=1.0))
        self.mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
        self.tree_filter = TreeFilter2D()

    # a2 -- box_solov2_head.py:204-217
    def dynamic_conv(self, feature_pred, kernel_pred, out_size=None, cells=None):
        """feature_pred [B,C,h,w], kernel_pred [B,C,S,S] -> [B,S*S,h',w'].  ``cells`` (list of per-image ascending index
        tensors) restricts the convolution to the positive grid cells the loss will index (:317-320), which is
        what the training loss needs, and returns the per-image list of [n_b,h',w'] rows (``solo_cells_conv``: one launch,
        the resize applied to feature_pred); without it all S*S cells are computed as the reference does."""
        if cells is not None:
            size = tuple(out_size) if out_size is not None else tuple(feature_pred.shape[-2:])
            rows = solo_cells_conv(feature_pred, [kernel_pred], [cells], [size])[0]
            return list(rows.split([int(c.numel()) for c in cells]))
        ins = solo_dynamic_conv(feature_pred, kernel_pred)
        if out_size is not None:
            ins = bilinear_resize(ins, out_size)          # :213, align_corners=False
        return ins

    # a17 -- box_solov2_head.py:334-367
    def mask_loss(self, ins_preds, ins_labels, img_targets, lst_targets, shared_trees=True, inst_imgs=None):
        """Per level lists: ins_pred [n,h,w] logits, ins_label [n,h,w] box masks, and either
          * img_target [n,3,h,w], lst_target [n,5,h,w] per INSTANCE (the reference's tensors, :296-305), or
          * with ``inst_imgs`` (list of int tensors [n], image of each instance): img_target [B,3,h,w],
            lst_target [B,5,h,w] per IMAGE -- the trees, their BFS orders, edge weights and normalisers are then
            built once per image and shared by its instances (``tree_of``), with no host synchronisation at all.
        ``shared_trees`` (per-instance inputs only): identical rows are detected and their MSTs shared; the reference
        rebuilds identical trees per instance (:300-305,353).  Same losses either way.
        Per level: one sigmoid, BoxProjectionLoss, ONE launch per level-set term (sigmoid / cat / * box / clamp inside,
        ``levelset_assembly``), two tree filters."""
        w_ls = self.loss_levelset.loss_weight

        def level(lvl, ins_pred, box_mask, img_t, lst_t):
            mask_pred = torch.sigmoid(ins_pred.unsqueeze(1))
            box = box_mask.unsqueeze(1).to(mask_pred.dtype)
            l_prj = self.loss_boxpro(mask_pred, box)
            if inst_imgs is not None:
                ii = inst_imgs[lvl]
                img_inst = img_t.index_select(0, ii.long())
                # the second tree and its BFS order do not depend on the first filter: build them on the side stream meanwhile
                lst = Forked(lambda: self._tree_and_order(lst_t, mask_pred.shape, None), mask_pred.device)
                f_img = self.tree_filter(mask_pred, img_t, self.mst(img_t), tree_of=ii)
                lst_tree, lst_order = lst.join()
                f_lst = self.tree_filter(f_img, lst_t, lst_tree, low_tree=False, tree_of=ii, order=lst_order)
            else:
                img_inst = img_t
                lst = Forked(lambda: self._tree_and_order(lst_t, mask_pred.shape, shared_trees), mask_pred.device)
                f_img = self.tree_filter(mask_pred, img_t, self._mst(img_t, shared_trees))
                lst_tree, lst_order = lst.join()
                f_lst = self.tree_filter(f_img, lst_t, lst_tree, low_tree=False, order=lst_order)
            loss_img = levelset_assembly(ins_pred, box, img_inst, w_ls) * 0.05             # :341-351
            loss_feat = levelset_assembly(ins_pred, box, torch.cat((f_img, f_lst), dim=1), w_ls) * 5.0   # :357-360
            return l_prj, loss_img + loss_feat

        # the FPN levels are independent (a tree filter is a dependent-level walk on ~20 CTAs): one lane stream per level
        work = [(lvl, a, b, c, d) for lvl, (a, b, c, d) in enumerate(zip(ins_preds, ins_labels, img_targets, lst_targets))
                if a.size(0) > 0]
        dev = work[0][1].device if work else None
        outs = run_concurrently([lambda w=w: level(*w) for w in work], dev) if work else []
        loss_project, loss_levelset = [o[0] for o in outs], [o[1] for o in outs]
        return dict(loss_boxpro=torch.cat(loss_project).mean(), loss_levelset=torch.cat(loss_levelset).mean())

    def _tree_and_order(self, guide, shape, shared):
        """MST of ``guide`` (shared across identical rows when ``shared`` is not None) and the BFS order the filter will use."""
        tree = self.mst(guide) if shared is None else self._mst(guide, shared)
        return tree, self.tree_filter.order(tree, shape)

    def _mst(self, guide, shared):
        if not shared or guide.size(0) == 1:
            return self.mst(guide)
        with torch.no_grad():
            flat = guide.flatten(1)
            new = torch.ones(guide.size(0), dtype=torch.bool, device=guide.device)
            new[1:] = (flat[1:] != flat[:-1]).any(1)           # instances arrive grouped by image (:296-305)
            group = torch.cumsum(new.long(), 0) - 1
            uniq = guide[new]
        return self.mst(uniq)[group]


@register(HEADS, partial=True)
class DiscoBoxSOLOv2Head(nn.Module):
    """DiscoBox head: the mask-loss path (a3, a16, a17) and, with a ``loss_corr`` config (discobox_head.py:720-749), the
    semantic-correspondence loss on top of it (f4: ``corr_loss``, models/dense_heads/disco_corr.py)."""

    def __init__(self, num_classes=80, in_channels=256, loss_ins=None, loss_ts=None, loss_corr=None, **cfg):
        super().__init__()
        self.num_classes = num_classes
        self.in_channels = in_channels
        self.cfg = cfg
        loss_ins = loss_ins or dict(loss_weight=1.0)
        loss_ts = loss_ts or dict(loss_weight=1.0, alpha0=2.0, theta0=0.5, theta1=30.0, theta2=20.0, kernel=3, base=0.10,
                                  max_iter=10)
        self.ins_loss_weight = loss_ins['loss_weight']
        self.ts_loss_weight = loss_ts['loss_weight']
        self.alpha0, self.theta0, self.theta1 = loss_ts['alpha0'], loss_ts['theta0'], loss_ts['theta1']
        self.theta2 = loss_ts.get('theta2', 10)
        self.mkernel, self.crf_base, self.crf_max_iter = loss_ts['kernel'], loss_ts['base'], loss_ts['max_iter']
        self._bxs_post_init()
        if loss_corr is not None:
            from .disco_corr import DiscoCorr
            self.corr = DiscoCorr(num_classes, loss_corr)

    def _bxs_post_init(self):
        """Also runs after the REFERENCE class's ``__init__`` when mmdet is importable (``register(partial=True)``): the
        correspondence state is then rebuilt from the attributes that constructor leaves behind (:720-749)."""
        self.corr = None
        solver, queues = getattr(self, 'semantic_corr_solver', None), getattr(self, 'object_queues', None)
        if solver is None or queues is None:
            return
        from .disco_corr import DiscoCorr
        self.corr = DiscoCorr(self.num_classes, dict(
            loss_weight=self.corr_loss_weight, corr_exp=solver.exp, corr_eps=solver.eps,
            gaussian_filter_size=solver.gaussian_filter_size, low_score=solver.low_score, corr_num_iter=solver.num_iter,
            corr_num_smooth_iter=solver.num_smooth_iter, dist_kernel=solver.dist_kernel,
            obj_bank=dict(len_object_queues=queues.len_queue, fg_iou_thresh=queues.fg_iou_thresh,
                          bg_iou_thresh=queues.bg_iou_thresh, ratio_range=queues.ratio_range,
                          appear_thresh=queues.appear_thresh, max_retrieval_objs=queues.max_retrieval_objs,
                          feat_height=self.corr_feat_height, feat_width=self.corr_feat_width,
                          mask_height=self.corr_mask_height, mask_width=self.corr_mask_width, min_size=self.objbank_min_size)))

    # f4 -- discobox_head.py:1013-1139, 1311-1337
    def corr_loss_levels(self, s_ins_pred_list, t_ins_pred_list, img_ind_list, ins_labels, kernel_label_list, s_feat, t_feat,
                         color_feats, use_ind_teacher=False, gamma=0.01):
        """The part of ``corr_loss`` after the dynamic convolutions (per-level lists as ``mask_loss`` takes them, plus the
        class of every object and the student / teacher feature maps [B,C,H,W]).  Returns (loss_corr * weight,
        mean of the correspondence-aware teacher-student dice terms) -- what ``loss`` adds to ``loss_corr`` / ``loss_ts``
        (:1329-1337).  Stateful: the object bank of ``self.corr`` is updated.  No host synchronisation (after one eager call,
        which allocates the bank, it can be captured in a CUDA graph)."""
        if self.corr is None:
            raise RuntimeError('DiscoBoxSOLOv2Head was built without loss_corr')
        mf = MeanField(color_feats, alpha0=self.alpha0, theta0=self.theta0, theta1=self.theta1, theta2=self.theta2,
                       iter=self.crf_max_iter, kernel_size=self.mkernel, base=self.crf_base, gamma=gamma)
        loss, per_level = self.corr.levels_masked(s_ins_pred_list, t_ins_pred_list or [None] * len(s_ins_pred_list),
                                                  img_ind_list, ins_labels, kernel_label_list, s_feat, t_feat, mf,
                                                  use_ind_teacher)
        if per_level:                                   # the mean over the objects with a non-empty target
            total = sum(ts.sum() for ts, _ in per_level)
            count = sum(valid.sum() for _, valid in per_level)
            ts_mean = total / count.clamp(min=1)
        else:
            ts_mean = loss.new_zeros(())
        return loss * self.corr.corr_loss_weight, ts_mean

    def _grid_cfg(self):
        """(scale_ranges, strides, seg_num_grids, sigma): attributes when the reference constructor ran (:690-700), else the
        construction kwargs with the reference's defaults (:662-666)."""
        get = lambda name, key, default: getattr(self, name, None) if getattr(self, name, None) is not None else self.cfg.get(key, default)
        return (get('scale_ranges', 'scale_ranges', ((8, 32), (16, 64), (32, 128), (64, 256), (128, 512))),
                get('strides', 'strides', (4, 8, 16, 32, 64)), get('seg_num_grids', 'num_grids', None), get('sigma', 'sigma', 0.2))

    # f2 + a3 -- discobox_head.py:917-1003 (identical in loss(), :1161-1260, with the other target builder)
    def corr_inputs(self, s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list, gt_label_list, gt_mask_list,
                    use_ind_teacher=False, best=True, conv=None):
        """From the raw head outputs to the per-level lists of ``mask_loss`` / ``corr_loss_levels``: SOLO targets of every image
        (``best_target_single`` for corr_loss, ``solov2_target_single`` with ``best=False``), the dynamic kernels of the covered
        cells gathered by ``grid_order``, one dynamic convolution per (level, image) with objects (a3: the wgmma kernel).
        ``*_kernel_preds_raw``: per level [B,C,g,g]; ``*_ins_pred`` [B,C,H,W]; ``gt_mask_list``: per image uint8 [G,H',W'] device
        tensors.  Returns (s_ins_pred_list, t_ins_pred_list, img_ind_list, ins_labels, kernel_label_list) with None for a level
        without objects.  Plain torch around ``conv`` (default: ``self.dynamic_conv``)."""
        from .disco_targets import disco_target_single
        conv = conv or self.dynamic_conv
        scale_ranges, strides, grids, sigma = self._grid_cfg()
        fsize = tuple(s_ins_pred.shape[-2:])
        per_img = [disco_target_single(b, l, m, fsize, scale_ranges, strides, grids, sigma, self.num_classes, best=best)
                   for b, l, m in zip(gt_bbox_list, gt_label_list, gt_mask_list)]
        L_, B = len(grids), len(per_img)
        ins_labels = [torch.cat([per_img[b][0][lv] for b in range(B)], 0) for lv in range(L_)]
        klabels = [torch.cat([per_img[b][1][lv].reshape(-1)[per_img[b][3][lv]] for b in range(B)], 0) for lv in range(L_)]
        s_list, t_list, img_list = [], [], []
        for lv in range(L_):
            s_lv, t_lv, i_lv = [], [], []
            for b in range(B):
                order = per_img[b][3][lv]
                if order.numel() == 0:
                    continue
                sk = s_kernel_preds_raw[lv][b].reshape(s_kernel_preds_raw[lv].shape[1], -1)[:, order]       # [C,I]
                s_lv.append(conv(s_ins_pred[b], sk))
                if use_ind_teacher:
                    tk = t_kernel_preds_raw[lv][b].reshape(t_kernel_preds_raw[lv].shape[1], -1)[:, order]
                    t_lv.append(conv(t_ins_pred[b], tk))
                i_lv.append(torch.full((order.numel(),), b, dtype=torch.int64, device=s_ins_pred.device))
            s_list.append(torch.cat(s_lv, 0) if s_lv else None)
            t_list.append(torch.cat(t_lv, 0) if t_lv else None)
            img_list.append(torch.cat(i_lv, 0) if i_lv else None)
        return s_list, t_list, img_list, ins_labels, klabels

    # f4 -- discobox_head.py:900-1139, the reference's signature
    def corr_loss(self, cate_preds, s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list, gt_label_list,
                  gt_mask_list, mean_fields, img_metas, cfg, img=None, gt_bboxes_ignore=None, use_loss_ts=False,
                  use_ind_teacher=False, s_feat=None, t_feat=None):
        """Returns (corr_loss / (num + 1e-4), [per-level dice terms]) like the reference.  ``mean_fields``: the reference passes
        one module per image; here ONE mean field over the batch is built from ``img`` (only ``gamma`` is read from the list)."""
        if self.corr is None:
            raise RuntimeError('DiscoBoxSOLOv2Head was built without loss_corr')
        s_list, t_list, img_list, ins_labels, klabels = self.corr_inputs(
            s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list, gt_label_list, gt_mask_list,
            use_ind_teacher=use_ind_teacher, best=True)
        color_feats = bilinear_resize(img, tuple(s_ins_pred.shape[-2:]), align_corners=True)                    # :957-958
        gamma = mean_fields[0].gamma if mean_fields else 0.01
        mf = MeanField(color_feats, alpha0=self.alpha0, theta0=self.theta0, theta1=self.theta1, theta2=self.theta2,
                       iter=self.crf_max_iter, kernel_size=self.mkernel, base=self.crf_base, gamma=gamma)
        return self.corr.levels(s_list, t_list, img_list, ins_labels, klabels, s_feat, t_feat, mf, use_ind_teacher)

    # a3 -- discobox_head.py:1206-1246
    @staticmethod
    def dynamic_conv(mask_feat_img, kernels):
        """mask_feat_img [C,h,w] of ONE image, kernels [C,I] (as gathered by grid_order, :1180-1185) -> [I,h,w]."""
        return dynconv1x1(mask_feat_img[None], kernels.t()[None].contiguous())[0]

    # a17 -- discobox_head.py:1266-1300, 1302-1339 (without corr_loss)
    def mask_loss(self, s_ins_pred_list, ins_labels, img_ind_list, color_feats, t_ins_pred_list=None, use_loss_ts=True):
        """Per level: s_ins_pred [n,h,w] logits, ins_label [n,h,w] box masks, img_inds [n];
        color_feats [B,3,h,w] = image resized with align_corners=True (:1201).
        No host synchronisation and no boolean indexing: instances with an all-zero target (removed by the reference,
        :1283-1287) stay in the batch with weight 0 -- the mean over the kept instances is a weighted mean -- and ONE
        mean-field module holds the bilateral kernels of all images (``obj_img`` picks the image of each object).
        A level whose student logits (and independent-teacher logits, if any) are float16 or bfloat16 -- the reference's
        autocast training -- runs ``ops.discobox.discobox_mask_loss`` on them as they are; any other level, float32
        included, the composition of ``_mask_loss_level_eager``.  The dtype of the input decides, not the autocast state."""
        mf = MeanField(color_feats, alpha0=self.alpha0, theta0=self.theta0, theta1=self.theta1, theta2=self.theta2,
                       iter=self.crf_max_iter, kernel_size=self.mkernel, base=self.crf_base) if use_loss_ts else None
        t_list = t_ins_pred_list if t_ins_pred_list is not None else s_ins_pred_list
        num_ins, num_ts, den = [], [], []
        for s_in, t_in, img_inds, target in zip(s_ins_pred_list, t_list, img_ind_list, ins_labels):
            if s_in is None or s_in.shape[0] == 0:
                continue
            t_ind = t_in if t_ins_pred_list is not None else None
            if s_in.dtype in HALF_DTYPES and (t_ind is None or t_ind.dtype == s_in.dtype):
                n_ins, n_ts, cnt = discobox_mask_loss(s_in, target, img_inds, mf, t_ind, use_loss_ts)
            else:
                n_ins, n_ts, cnt = self._mask_loss_level_eager(s_in, t_ind, img_inds, target, mf, use_loss_ts)
            num_ins.append(n_ins)
            den.append(cnt)
            if use_loss_ts:
                num_ts.append(n_ts)
        zero = color_feats.new_zeros(())
        if not num_ins:
            return dict(loss_ins=zero, loss_ts=zero)
        count = torch.stack(den).sum().clamp(min=1.0)
        l_ins = torch.stack(num_ins).sum() / count * self.ins_loss_weight
        l_ts = torch.stack(num_ts).sum() / count * self.ts_loss_weight if (use_loss_ts and num_ts) else zero
        return dict(loss_ins=l_ins, loss_ts=l_ts)

    @staticmethod
    def _mask_loss_level_eager(s_in, t_in, img_inds, target, mf, use_loss_ts):
        """One level of ``mask_loss`` as a composition of torch ops and the float32 kernels (projection loss, mean field):
        (sum keep * mil, sum keep * d_ts or None, sum keep).  ``t_in``: independent-teacher logits or None."""
        target = target.float()
        keep = (target.flatten(1).sum(1) > 0).float()            # all-zero targets carry weight 0 (:1283-1287)
        s = torch.sigmoid(s_in)
        t = s if t_in is None else torch.sigmoid(t_in)
        n_ins = (mil_loss(None, s, s, target) * keep).sum()
        cnt = keep.sum()
        n_ts = None
        if use_loss_ts:
            enlarged = F.max_pool2d(target.unsqueeze(1), kernel_size=3, stride=1, padding=1).squeeze(1)
            pseudo, _ = mf(((t + s) / 2).unsqueeze(1), target.unsqueeze(1), obj_img=img_inds)
            n_ts = (_disco_dice(s * enlarged, pseudo) * keep).sum()
        return n_ins, n_ts, cnt


def _disco_dice(x, t):
    """dice_loss of discobox_head.py:542-550 on full maps (plain reductions; the profiles are the MIL part)."""
    x, t = x.flatten(1).float(), t.flatten(1).float()
    return 1 - 2 * (x * t).sum(1) / ((x * x).sum(1) + 0.001 + (t * t).sum(1) + 0.001)


@register(HEADS, partial=True)
class Box2MaskHead(nn.Module):
    """Box2Mask head: mask-loss path only."""

    def __init__(self, in_channels=None, feat_channels=256, out_channels=256, num_things_classes=80, num_stuff_classes=0,
                 num_queries=100, loss_box=None, loss_mask=None, train_cfg=None, **cfg):
        super().__init__()
        self.num_queries = num_queries
        self.num_classes = num_things_classes + num_stuff_classes
        self.train_cfg = train_cfg
        self.cfg = cfg
        self.loss_box = build_loss(loss_box or dict(type='BoxProjectionLoss', loss_weight=5.0))
        self.loss_mask = build_loss(loss_mask or dict(type='LevelsetLoss', loss_weight=1.0))
        self.mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
        self.tree_filter = TreeFilter2D()
        self._bxs_post_init()

    def _bxs_post_init(self):
        """Also runs after the REFERENCE class's ``__init__`` when mmdet is importable: the matcher of ``get_targets`` is
        this package's MaskHungarianAssigner, built from the same ``train_cfg['assigner']`` (box2mask_head.py:95-97)."""
        from ...core.assigner import MaskHungarianAssigner      # core imports models.builder: not at module level
        cfg = (getattr(self, 'train_cfg', None) or {}).get('assigner')
        self.hungarian = MaskHungarianAssigner(**{k: v for k, v in cfg.items() if k != 'type'}) if cfg else None
        self.lsap_status = None

    # f1 -- box2mask_head.py:135-189 (get_targets + _get_target_single with MaskPseudoSampler), the reference's signature
    @torch.no_grad()
    def get_targets(self, cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list, img_metas):
        """Classification and mask targets of one decoder layer for all images: (labels_list, label_weights_list,
        mask_targets_list, mask_weights_list, num_total_pos, num_total_neg), as the reference returns them.
        cls_scores_list[b] [Q,C+1], mask_preds_list[b] [Q,h,w] (low resolution: the assigner's BoxMatchingCost upsamples it
        virtually to the ground truths' size), gt_labels_list[b] [G_b], gt_masks_list[b] [G_b,H,W].
        The cost matrices of all images are matched in ONE launch and nothing is read back to the host: the call runs under
        torch.cuda.set_sync_debug_mode('error') and can be captured in a CUDA graph.  Every size comes from the shapes:
        min(Q, G_b) positives per image, in ascending query order, pos_assigned_gt_inds = match[pos_inds].
        An image whose cost matrix holds a NaN (NaN predictions) cannot raise without a synchronisation: its queries come
        back as background (labels = num_classes, mask_weights = 0), its min(Q, G_b) mask_targets rows are placeholders,
        and ``self.lsap_status`` (int32 [B] on the device, 1 for such an image, else 0) keeps the per-image status."""
        if self.hungarian is None:
            raise RuntimeError('Box2MaskHead.get_targets needs train_cfg with an assigner')
        Q = self.num_queries
        costs = []
        for cls_score, mask_pred, gt_labels, gt_masks in zip(cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list):
            if gt_labels.shape[0] and mask_pred.shape[0]:
                costs.append(self.hungarian.cost_matrix(cls_score, mask_pred, gt_labels, gt_masks, lowres=True))
            else:
                costs.append(mask_pred.new_zeros((mask_pred.shape[0], gt_labels.shape[0])))
        matches, self.lsap_status = solve_batched(costs)
        labels_list, label_weights_list, mask_targets_list, mask_weights_list = [], [], [], []
        num_total_pos = num_total_neg = 0
        for match, mask_pred, gt_labels, gt_masks in zip(matches, mask_preds_list, gt_labels_list, gt_masks_list):
            m = match.long()
            pos = m >= 0
            k = min(mask_pred.shape[0], gt_labels.shape[0])
            pos_inds = torch.nonzero_static(pos, size=k, fill_value=0).squeeze(1)
            pos_gt = m[pos_inds].clamp(min=0)
            if gt_labels.shape[0]:
                labels = torch.where(pos, gt_labels[m.clamp(min=0)].long(), self.num_classes)
            else:
                labels = gt_labels.new_full((Q,), self.num_classes, dtype=torch.long)
            labels_list.append(labels)
            label_weights_list.append(gt_labels.new_ones((Q,)))
            mask_targets_list.append(gt_masks.unsqueeze(1)[pos_gt])
            mask_weights_list.append(pos.to(mask_pred.dtype))
            num_total_pos += k
            num_total_neg += mask_pred.shape[0] - k
        return labels_list, label_weights_list, mask_targets_list, mask_weights_list, num_total_pos, num_total_neg

    # a4 -- box2mask_head.py:343-345
    @staticmethod
    def mask_pred(mask_embed, mask_feature):
        return box2mask_mask_pred(mask_embed, mask_feature)

    # a4 -- box2mask_head.py:338-359, the reference's signature
    def forward_head(self, decoder_out, mask_feature, attn_mask_target_size):
        """(cls_pred, mask_pred, attn_mask, levelset_feat) after one decoder layer, as the reference returns them.
        ``mask_pred`` is the wgmma dynamic convolution (``mask_pred``: TF32 for float32 operands, the operand dtype under
        autocast); ``attn_mask`` [B*num_heads, Q, h*w] bool is ``ops.box2mask.attention_mask`` of it, bit for bit the
        reference's interpolate / repeat / sigmoid / compare lines on the same ``mask_pred``."""
        return self._forward_head(decoder_out, mask_feature, attn_mask_target_size, reset_full_rows=False)

    def _forward_head(self, decoder_out, mask_feature, attn_mask_target_size, reset_full_rows):
        missing = [n for n in ('transformer_decoder', 'cls_embed', 'mask_embed', 'levelset_bottom', 'num_heads')
                   if not hasattr(self, n)]
        if missing:
            raise RuntimeError('Box2MaskHead.forward_head needs the modules the reference constructor builds (mmdet '
                               f'installed); this head has no {", ".join(missing)}')
        decoder_out = self.transformer_decoder.post_norm(decoder_out).transpose(0, 1)
        cls_pred = self.cls_embed(decoder_out)
        mask_embed = self.mask_embed(decoder_out)
        mask_pred = self.mask_pred(mask_embed, mask_feature)
        attn_mask = attention_mask(mask_pred, attn_mask_target_size, self.num_heads, reset_full_rows=reset_full_rows)
        levelset_feat = self.levelset_bottom(mask_feature)
        return cls_pred, mask_pred, attn_mask, levelset_feat

    # box2mask_head.py:361-419, the reference's signature
    def forward(self, feats, img_metas):
        """(cls_pred_list, mask_pred_list, lst_feat_list) of the query-feature head and every decoder layer, as the reference
        computes them.  The mask a decoder layer receives comes out of the attention-mask kernel with its all-True rows
        already cleared (the reference clears them with a ``torch.where``, :397, one host synchronisation per layer), so
        nothing here synchronises with the host: after one eager call the forward can be captured in a CUDA graph."""
        batch_size = len(img_metas)
        mask_features, multi_scale_memorys = self.pixel_decoder(feats)
        decoder_inputs, decoder_positional_encodings = [], []
        for i in range(self.num_transformer_feat_level):
            decoder_input = self.decoder_input_projs[i](multi_scale_memorys[i])
            decoder_input = decoder_input.flatten(2).permute(2, 0, 1)
            decoder_input = decoder_input + self.level_embed.weight[i].view(1, 1, -1)
            mask = decoder_input.new_zeros((batch_size, ) + multi_scale_memorys[i].shape[-2:], dtype=torch.bool)
            decoder_positional_encoding = self.decoder_positional_encoding(mask).flatten(2).permute(2, 0, 1)
            decoder_inputs.append(decoder_input)
            decoder_positional_encodings.append(decoder_positional_encoding)
        query_feat = self.query_feat.weight.unsqueeze(1).repeat((1, batch_size, 1))
        query_embed = self.query_embed.weight.unsqueeze(1).repeat((1, batch_size, 1))

        cls_pred, mask_pred, attn_mask, lst_feat = self._forward_head(query_feat, mask_features,
                                                                      multi_scale_memorys[0].shape[-2:], True)
        cls_pred_list, mask_pred_list, lst_feat_list = [cls_pred], [mask_pred], [lst_feat]
        for i in range(self.num_transformer_decoder_layers):
            level_idx = i % self.num_transformer_feat_level
            query_feat = self.transformer_decoder.layers[i](
                query=query_feat, key=decoder_inputs[level_idx], value=decoder_inputs[level_idx], query_pos=query_embed,
                key_pos=decoder_positional_encodings[level_idx], attn_masks=[attn_mask, None],
                query_key_padding_mask=None, key_padding_mask=None)
            cls_pred, mask_pred, attn_mask, lst_feat = self._forward_head(
                query_feat, mask_features, multi_scale_memorys[(i + 1) % self.num_transformer_feat_level].shape[-2:], True)
            cls_pred_list.append(cls_pred)
            mask_pred_list.append(mask_pred)
            lst_feat_list.append(lst_feat)
        return cls_pred_list, mask_pred_list, lst_feat_list

    # a17 -- box2mask_head.py:229-233, 269-335
    def mask_loss_single(self, mask_preds, mask_targets, num_per_img, norm_img, lst_feat, trees=None):
        """mask_preds [n,h,w] matched logits (images concatenated), mask_targets [n,H,W] box masks,
        num_per_img: list of matched queries per image; norm_img [B,3,*,*], lst_feat [B,1,*,*].
        ``trees`` (optional): the ``image_trees`` of this batch -- the image MST at 96x96 does not depend on the decoder
        layer, the reference rebuilds it in each of its 10 loss_single calls (:269-272).
        Every resize is the bilinear kernel of ops.resize (a18), the two level-set terms are one launch each (a17), the
        trees / orders / edge weights / normalisers exist once per image (``tree_of``); no host synchronisation."""
        pred_shape = mask_preds.shape[-2:]
        norm_img = bilinear_resize(norm_img, pred_shape)              # :232-233
        lst_feat = bilinear_resize(lst_feat, pred_shape)
        if mask_preds.shape[0] == 0:                                  # zero match (:264-268)
            return mask_preds.sum(), mask_preds.sum()
        dev = mask_preds.device
        img96_b, lst96_b = _scale_target(norm_img), _scale_target(lst_feat)       # per IMAGE, :269-272
        img_tree = trees if trees is not None else self.mst(img96_b)
        # the second tree and its BFS order depend on nothing computed below: side stream, joined before the second filter
        def second_tree():
            tree = self.mst(lst96_b)
            return tree, self.tree_filter.order(tree, lst96_b.shape)

        lst = Forked(second_tree, lst96_b.device)
        # instance -> image, built from device-side fills only (host ints in, no copy: CUDA-graph capturable)
        tree_of = torch.cat([torch.full((int(c),), i, device=dev, dtype=torch.int32) for i, c in enumerate(num_per_img)])
        box = bilinear_resize(mask_targets.unsqueeze(1).to(mask_preds.dtype), pred_shape)   # :300
        s = torch.sigmoid(mask_preds.unsqueeze(1))
        loss_project = self.loss_box(s, box).mean()
        w_ls = self.loss_mask.loss_weight
        loss_img = levelset_assembly(mask_preds, box, norm_img.index_select(0, tree_of.long()), w_ls).mean() * 0.05   # :305-312
        s96 = _scale_target(s)
        f_img = self.tree_filter(s96, img96_b, img_tree, tree_of=tree_of)                  # :315-322
        lst_tree, lst_order = lst.join()
        f_lst = self.tree_filter(f_img, lst96_b, lst_tree, low_tree=False, tree_of=tree_of, order=lst_order)
        deep = torch.cat((bilinear_resize(f_img, pred_shape), bilinear_resize(f_lst, pred_shape)), dim=1)   # :323-324
        loss_feat = levelset_assembly(mask_preds, box, deep, w_ls).mean() * 5.0            # :325-327
        loss_lcm = 0.2 * LCM(img96_b.index_select(0, tree_of.long()), s96, _scale_target(box))   # :329-331
        return loss_project, loss_img + loss_feat + loss_lcm

    def mask_loss_layers(self, mask_preds_per_layer, mask_targets, num_per_img, norm_img, lst_feat, trees=None):
        """``mask_loss_single`` of every decoder layer (the reference's ``multi_apply(self.loss_single, ...)`` over the layers,
        box2mask_head.py:214-227): the layers are independent, so each one runs on its own lane stream.  ``mask_preds_per_layer``
        : list of [n,h,w] tensors or of callables producing them (e.g. the layer's einsum + matching, run inside the lane).
        Returns the list of (loss_project, loss_levelset) pairs."""
        if trees is None:
            first = mask_preds_per_layer[0]
            shape = (first() if callable(first) else first).shape[-2:]
            trees = self.image_trees(norm_img, shape)

        def layer(mp):
            mp = mp() if callable(mp) else mp
            return self.mask_loss_single(mp, mask_targets, num_per_img, norm_img, lst_feat, trees=trees)

        return run_concurrently([lambda mp=mp: layer(mp) for mp in mask_preds_per_layer], norm_img.device)

    def image_trees(self, norm_img, pred_shape):
        """MST of every image at 96x96 (box2mask_head.py:232,269-272): identical for all decoder layers of a step."""
        with torch.no_grad():
            return self.mst(_scale_target(bilinear_resize(norm_img, pred_shape)))
