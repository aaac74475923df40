"""Mask-loss assembly of the three SOLO/Mask2Former-style heads (SURVEY.md section 8 row a17) and their
dynamic-conv call sites (a2-a4), on the kernels of libboxseg_b200:

  ``BoxSOLOv2Head``       mmdet/models/dense_heads/box_solov2_head.py:204-217 (dynamic conv), :334-367 (loss)
  ``DiscoBoxSOLOv2Head``  mmdet/models/dense_heads/discobox_head.py:1206-1300 (per-image conv, MIL dice, mean-field teacher)
  ``Box2MaskHead``        mmdet/models/dense_heads/box2mask_head.py:338-359 (mask_pred einsum), :192-335 (loss, loss_single)

The mask-loss hot path and its immediate callers are implemented here: the SOLO target builders live in
``solo_targets.py`` / ``disco_targets.py`` (f2), the Hungarian front half in ``core/assigner.py`` (f1), DiscoBox's
cross-image correspondence loss in ``disco_corr.py`` (f4; ``DiscoBoxSOLOv2Head.corr_inputs / corr_loss``).  The conv towers
and category losses are out of scope (SURVEY 2.1 row 3); SOLOv2 inference (``get_seg`` of the two SOLOv2 heads) is in
``solo_seg.py``.  The classes keep the reference's registry names and accept (and store) the reference's constructor kwargs so
the configs build, and expose the hot-path pieces as methods with the tensors the reference passes between
its own lines.
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from ...ops.box2mask import attention_mask
from ...ops.discobox import HALF_DTYPES, discobox_mask_loss
from ...ops.dynconv import box2mask_mask_pred, disco_cells_conv, dynconv1x1, solo_cells_conv, solo_dynamic_conv
from ...ops.focal import sigmoid_focal_loss_levels
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


class SoloLevelPred:
    """One level of ``BoxSOLOv2Head.forward``'s training ``ins_pred``, not computed: the reference tensor is
    ``interpolate(conv2d(feature_pred, kernel_pred cells, groups=B), out_size, bilinear)`` [B,S*S,*out_size]
    (box_solov2_head.py:204-216).  ``shape`` / ``size()`` report that tensor's shape, ``dense()`` computes it."""

    def __init__(self, feature_pred, kernel_pred, out_size):
        self.feature_pred, self.kernel_pred, self.out_size = feature_pred, kernel_pred, tuple(int(s) for s in out_size)

    @property
    def shape(self):
        B, _, S, _ = self.kernel_pred.shape
        return torch.Size((B, S * S) + self.out_size)

    def size(self, dim=None):
        return self.shape if dim is None else self.shape[dim]

    def dense(self):
        return bilinear_resize(solo_dynamic_conv(self.feature_pred, self.kernel_pred), self.out_size)


class SoloInsPreds(list):
    """``BoxSOLOv2Head.forward``'s training ``ins_preds``: one ``SoloLevelPred`` per level, all of one ``feature_pred``.
    ``BoxSOLOv2Head.loss`` convolves only the positive cells of it; the reference's ``loss`` reads nothing but
    ``featmap.size()[-2:]`` from its ``ins_preds`` (:281)."""

    @property
    def feature_pred(self):
        return self[0].feature_pred


def _coord_feat(x):
    """The two coordinate channels of box_solov2_head.py:190-196, 230-235: x then y, linspace(-1, 1) each."""
    x_range = torch.linspace(-1, 1, x.shape[-1], device=x.device)
    y_range = torch.linspace(-1, 1, x.shape[-2], device=x.device)
    y, xx = torch.meshgrid(y_range, x_range, indexing='ij')
    return torch.cat([xx.expand([x.shape[0], 1, -1, -1]), y.expand([x.shape[0], 1, -1, -1])], 1)


_SOLO_TOWERS = ('feature_convs', 'kernel_convs', 'cate_convs', 'solo_kernel', 'solo_cate', 'solo_mask', 'levelset_bottom')


@register(HEADS, partial=True)
class BoxSOLOv2Head(nn.Module):
    """BoxLevelset head: ``forward`` / ``loss`` with the reference's signatures on the positive grid cells only, and the
    mask-loss path (``mask_loss``, ``dynamic_conv``).  The conv towers are the reference constructor's modules (mmdet
    installed, or attached by the caller); the standalone constructor builds only the losses."""

    def __init__(self, num_classes=80, in_channels=256, loss_cate=None, loss_boxpro=None, loss_levelset=None,
                 num_grids=None, strides=(4, 8, 16, 32, 64),
                 scale_ranges=((8, 32), (16, 64), (32, 128), (64, 256), (128, 512)), sigma=0.2, cate_down_pos=0, **cfg):
        super().__init__()
        self.num_classes = num_classes
        self.cate_out_channels = num_classes
        self.in_channels = in_channels
        self.seg_num_grids, self.strides, self.scale_ranges, self.sigma = num_grids, strides, scale_ranges, sigma
        self.cate_down_pos = cate_down_pos
        self.cfg = cfg
        self.loss_cate_cfg = loss_cate or dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0)
        self.loss_boxpro = build_loss(loss_boxpro or dict(type='BoxProjectionLoss', loss_weight=3.0))
        self.loss_levelset = build_loss(loss_levelset or dict(type='LevelsetLoss', loss_weight=1.0))
        self.mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
        self.tree_filter = TreeFilter2D()
        self._bxs_post_init()

    def _bxs_post_init(self):
        """Also runs after the REFERENCE class's ``__init__`` when mmdet is importable: the focal parameters are then read
        from the FocalLoss module it built (``self.loss_cate``)."""
        ref = getattr(self, 'loss_cate', None)
        if isinstance(ref, nn.Module):
            cfg = dict(use_sigmoid=ref.use_sigmoid, gamma=ref.gamma, alpha=ref.alpha, reduction=ref.reduction,
                       loss_weight=ref.loss_weight, activated=getattr(ref, 'activated', False))
        else:
            cfg = self.loss_cate_cfg
        if not cfg.get('use_sigmoid', True) or cfg.get('activated', False) or cfg.get('reduction', 'mean') != 'mean':
            raise NotImplementedError('BoxSOLOv2Head: the category loss is the sigmoid focal loss on logits with reduction '
                                      f"'mean' only, got {cfg}")
        self.focal = (float(cfg.get('gamma', 2.0)), float(cfg.get('alpha', 0.25)), float(cfg.get('loss_weight', 1.0)))

    # box_solov2_head.py:179-217, the reference's signature
    def forward(self, feats, eval=False):
        """(ins_preds, cate_preds, levelset_feats) as the reference returns them, with one difference in training: ``ins_preds``
        is a ``SoloInsPreds`` -- feature_pred, the raw kernel grids and the output sizes -- instead of the dense
        [B,S*S,h,w] predictions, which ``loss`` never needs (it convolves the positive cells only).  ``eval=True``: the
        reference's outputs, the sigmoid of the dense convolution (wgmma) and the local-max-masked category scores."""
        kernel_pred, cate_pred, featmap_sizes, feature_pred = self._towers(feats, eval, 'forward')
        levelset_feats = self.levelset_bottom(feature_pred)
        if eval:
            return [torch.sigmoid(self.dynamic_conv(feature_pred, k)) for k in kernel_pred], list(cate_pred), levelset_feats
        ins_pred = SoloInsPreds(SoloLevelPred(feature_pred, k, (2 * s[0], 2 * s[1])) for k, s in zip(kernel_pred, featmap_sizes))
        return ins_pred, list(cate_pred), levelset_feats

    # box_solov2_head.py:181-202, the lines forward and simple_test share
    def _towers(self, feats, eval, caller):
        """(kernel_pred, cate_pred, featmap_sizes, feature_pred): the per-level raw kernel grids and category outputs of
        ``forward_single`` and the mask features, everything ``forward`` computes before the dynamic convolution."""
        missing = [n for n in _SOLO_TOWERS if not hasattr(self, n)]
        if missing:
            raise RuntimeError(f'BoxSOLOv2Head.{caller} needs the modules the reference constructor builds (mmdet '
                               f'installed); this head has no {", ".join(missing)}')
        feats = [feat.float() for feat in feats]
        new_feats = self.split_feats(feats)
        featmap_sizes = [featmap.size()[-2:] for featmap in new_feats]
        kernel_pred, cate_pred = zip(*[self.forward_single(x, i, eval=eval) for i, x in enumerate(new_feats)])
        coord_feat = _coord_feat(feats[-2])
        feature_add_all_level = self.feature_convs[0](feats[0])
        for i in range(1, 3):
            feature_add_all_level = feature_add_all_level + self.feature_convs[i](feats[i])
        feature_add_all_level = feature_add_all_level + self.feature_convs[3](torch.cat([feats[3], coord_feat], 1))
        return kernel_pred, cate_pred, featmap_sizes, self.solo_mask(feature_add_all_level)

    def simple_test(self, feats, img_metas, rescale=False, cfg=None):
        """``get_seg(*forward(feats, eval=True), img_metas, cfg, rescale)`` without the dense predictions: the towers run as
        ``forward(eval=True)`` runs them (``levelset_bottom``, which ``get_seg`` never reads, is skipped), and only the
        distinct cells whose category score passes ``score_thr`` are convolved, each once (``solo_seg.candidate_sources``).
        Masks, labels and scores equal that expression's bit for bit, in float32, under float16 and under bfloat16 autocast.
        ``cfg``: the test config (``score_thr``, ``mask_thr``, ``nms_pre``, ``max_per_img``, ``kernel``, ``sigma``,
        ``filter_thr``); ``None`` reads ``self.test_cfg``.  ``rescale`` is accepted and, as in ``get_seg``, not used: the
        masks are pasted at each image's ``ori_shape``.  Two host reads per call: the candidate counts and the kept counts."""
        from .solo_seg import box_solov2_cells_get_seg
        if cfg is None:
            cfg = getattr(self, 'test_cfg', None)
            if cfg is None:
                raise ValueError('BoxSOLOv2Head.simple_test needs a test config: pass cfg or set the head\'s test_cfg')
        with torch.no_grad():
            kernel_pred, cate_pred, _, feature_pred = self._towers(feats, True, 'simple_test')
            return box_solov2_cells_get_seg(list(cate_pred), list(kernel_pred), feature_pred, self.strides, img_metas, cfg)

    # box_solov2_head.py:219-224
    @staticmethod
    def split_feats(feats):
        return (F.interpolate(feats[0], scale_factor=0.5, mode='bilinear'), feats[1], feats[2], feats[3],
                F.interpolate(feats[4], size=feats[3].shape[-2:], mode='bilinear'))

    # box_solov2_head.py:226-260
    def forward_single(self, x, idx, eval=False):
        kernel_feat = torch.cat([x, _coord_feat(x)], 1)
        cate_feat = x
        for i, kernel_layer in enumerate(self.kernel_convs):
            if i == self.cate_down_pos:
                kernel_feat = F.interpolate(kernel_feat, size=self.seg_num_grids[idx], mode='bilinear')
            kernel_feat = kernel_layer(kernel_feat)
        kernel_pred = self.solo_kernel(kernel_feat)
        for i, cate_layer in enumerate(self.cate_convs):
            if i == self.cate_down_pos:
                cate_feat = F.interpolate(cate_feat, size=self.seg_num_grids[idx], mode='bilinear')
            cate_feat = cate_layer(cate_feat)
        cate_pred = self.solo_cate(cate_feat)
        if eval:
            cate_pred = cate_pred.sigmoid()
            local_max = F.max_pool2d(cate_pred, (2, 2), stride=1, padding=1)
            cate_pred = (cate_pred * (local_max[:, :, :-1, :-1] == cate_pred)).permute(0, 2, 3, 1)
        return kernel_pred, cate_pred

    # box_solov2_head.py:262-388, the reference's signature
    def loss(self, ins_preds, cate_preds, levelset_feats, gt_bbox_list, gt_label_list, gt_mask_list, img, img_metas, cfg,
             gt_bboxes_ignore=None):
        """dict(loss_boxpro, loss_levelset, loss_cate) as the reference computes them.  ``ins_preds``: ``forward``'s
        ``SoloInsPreds`` (only the positive cells are convolved, ``solo_cells_conv``: one pack, convolution and row gather
        per run of levels of one size) or the reference's dense per-level [B,S*S,h,w] tensors (their positive rows are
        gathered).  ``gt_mask_list``: per image uint8 [G,H,W] tensors, or anything with mmdet's
        ``to_tensor(dtype, device)`` (BitmapMasks).
        The grid targets are built on the device (``solo_grid_targets``), the image and level-set targets stay per image (the
        trees are shared by its instances), ``loss_cate`` is ``sigmoid_focal_loss_levels`` on the [B,C,S,S] maps as they lie.
        ONE read back to the host: the positive count of every (level, image).
        A batch without any positive (the reference raises at :366) gives zero ``loss_boxpro`` / ``loss_levelset`` attached
        to the graph, and ``loss_cate`` over the all-background labels."""
        from .solo_targets import solo_grid_targets
        grids = list(self.seg_num_grids)
        n_lv, B = len(grids), len(gt_label_list)
        dev = levelset_feats.device
        sizes = [tuple(int(s) for s in p.size()[-2:]) for p in ins_preds]
        masks = [(m if torch.is_tensor(m) else m.to_tensor(dtype=torch.uint8, device=dev)).to(dev, torch.uint8)
                 for m in gt_mask_list]
        per_img = [solo_grid_targets(b, l, m, sizes, self.scale_ranges, self.strides, grids, self.sigma, self.num_classes,
                                     dense=False) for b, l, m in zip(gt_bbox_list, gt_label_list, masks)]
        ind = [torch.stack([per_img[b][2][lv] for b in range(B)]) for lv in range(n_lv)]            # [B,S^2] bool
        counts = torch.cat([i.sum(1) for i in ind])
        counts_host = counts.tolist()                                        # the one host read: n of every (level, image)
        n = [sum(counts_host[lv * B:(lv + 1) * B]) for lv in range(n_lv)]
        flat = torch.nonzero_static(torch.cat([i.flatten() for i in ind]), size=sum(n)).squeeze(1)
        avg_factor = counts.sum() + 1                                        # num_ins + 1 (:329, 383), on the device
        cate_labels = [torch.stack([per_img[b][1][lv] for b in range(B)]) for lv in range(n_lv)]
        loss_cate = sigmoid_focal_loss_levels(cate_preds, cate_labels, avg_factor, *self.focal)
        if sum(n) == 0:
            # 0 whatever the leaves hold (0 * Inf would be NaN), with zero gradients to every leaf
            off = torch.zeros((), dtype=torch.bool, device=dev)
            zero = sum(p.reshape(-1)[:1].sum().where(off, 0.) for p in self._graph_leaves(ins_preds, levelset_feats))
            return dict(loss_boxpro=zero, loss_levelset=zero.clone(), loss_cate=loss_cate)

        # ascending positives, level-major then image-major: the rows of the reference's boolean indexing (:294-320)
        local, start = [], 0
        for lv, S in enumerate(grids):
            local.append(flat[start:start + n[lv]] - B * sum(s * s for s in grids[:lv]))    # b * S^2 + cell
            start += n[lv]
        inst_imgs = [(loc // (S * S)).to(torch.int32) for loc, S in zip(local, grids)]
        cells = [loc % (S * S) for loc, S in zip(local, grids)]
        ins_labels = [self._box_mask_rows(per_img, lv, loc, grids[lv], sizes[lv], gt_label_list, dev)
                      for lv, loc in enumerate(local)]
        resized = {}
        for s in sizes:                                                      # :412-415, per image
            if s not in resized:
                resized[s] = (bilinear_resize(img.float(), s), bilinear_resize(levelset_feats, s))
        if isinstance(ins_preds, SoloInsPreds):
            per_level_cells = [list(c.split(counts_host[lv * B:(lv + 1) * B])) for lv, c in enumerate(cells)]
            rows = solo_cells_conv(ins_preds.feature_pred, [p.kernel_pred for p in ins_preds], per_level_cells, sizes)
        else:
            rows = [p.reshape((-1,) + tuple(p.shape[2:])).index_select(0, loc) for p, loc in zip(ins_preds, local)]
        out = self.mask_loss(rows, ins_labels, [resized[s][0] for s in sizes], [resized[s][1] for s in sizes],
                             inst_imgs=inst_imgs)
        return dict(loss_boxpro=out['loss_boxpro'], loss_levelset=out['loss_levelset'], loss_cate=loss_cate)

    # box_solov2_head.py:475-590, the reference's signature
    def get_seg(self, seg_preds, cate_preds, levelset_feats, img_metas, cfg, rescale=None):
        """Per image the reference's ``InstanceData`` (mmdet's when importable, else a namespace of the ``img_meta`` fields)
        with ``masks`` bool [n, H_ori, W_ori], ``labels`` int64 and ``scores``: ``seg_preds`` / ``cate_preds`` as
        ``forward(eval=True)`` returns them, every image of the batch at once (``solo_seg.box_solov2_get_seg``: each
        distinct candidate row read in place once, Matrix NMS and the mask paste on the GPU, two host reads per call).  Where
        Matrix NMS keeps nothing the reference raises (``F.interpolate`` of an empty batch); this returns ``empty_results``."""
        from .solo_seg import box_solov2_get_seg
        with torch.no_grad():
            return box_solov2_get_seg(seg_preds, cate_preds, self.strides, img_metas, cfg)

    @staticmethod
    def _box_mask_rows(per_img, lv, loc, S, size, gt_label_list, dev):
        """[n, h, w] uint8 box-mask targets of a level's positives: ``small[winner[cell]]`` of their image placed top-left
        (:459-466).  Each image's masks have their own size (mmdet pads them to the image's own pad shape), so every image's
        rescaled masks are placed on a level-sized canvas before the rows are gathered."""
        B, (h, w) = len(per_img), size
        smalls = [per_img[b][0][lv][1] for b in range(B) if len(gt_label_list[b])]
        if not smalls or loc.numel() == 0:
            return torch.zeros((loc.numel(), h, w), dtype=torch.uint8, device=dev)
        first = [sum(len(g) for g in gt_label_list[:b]) for b in range(B)]                  # ground truths before image b
        winner = torch.stack([per_img[b][0][lv][0] + first[b] for b in range(B)])           # into the images' concatenation
        canvas = torch.zeros((sum(s.shape[0] for s in smalls), h, w), dtype=torch.uint8, device=dev)
        g0 = 0
        for s in smalls:
            sh, sw = min(h, s.shape[1]), min(w, s.shape[2])
            canvas[g0:g0 + s.shape[0], :sh, :sw] = s[:, :sh, :sw]
            g0 += s.shape[0]
        return canvas[winner.flatten()[loc]]

    @staticmethod
    def _graph_leaves(ins_preds, levelset_feats):
        if isinstance(ins_preds, SoloInsPreds):
            return [ins_preds.feature_pred, levelset_feats] + [p.kernel_pred for p in ins_preds]
        return [levelset_feats] + list(ins_preds)

    # a2 -- box_solov2_head.py:204-217
    def dynamic_conv(self, feature_pred, kernel_pred, out_size=None, cells=None):
        """feature_pred [B,C,h,w], kernel_pred [B,C,S,S] -> [B,S*S,h',w'].  ``cells`` (list of per-image ascending index
        tensors) restricts the convolution to the positive grid cells the loss will index (:317-320), which is
        what the training loss needs, and returns the per-image list of [n_b,h',w'] rows (``solo_cells_conv``: one pack,
        convolution and row gather, the resize applied to feature_pred); without it all S*S cells are computed as the
        reference does."""
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

    def __init__(self, num_classes=80, in_channels=256, loss_ins=None, loss_ts=None, loss_corr=None, loss_cate=None, **cfg):
        super().__init__()
        self.num_classes = num_classes
        self.cate_out_channels = num_classes
        self.in_channels = in_channels
        self.cfg = cfg
        self.loss_cate = dict(loss_cate or dict(type='FocalLoss', use_sigmoid=True, gamma=2.0, alpha=0.25, loss_weight=1.0))
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
        correspondence state is then rebuilt from the attributes that constructor leaves behind (:720-749), and the focal
        parameters are read from the FocalLoss module it built.  Never raises: a ``loss_cate`` outside the envelope is
        recorded, and ``loss`` then defers to the reference or raises."""
        from .condinst_box_head import _loss_cfg
        kind, c = _loss_cfg(getattr(self, 'loss_cate', None), 'FocalLoss')
        if kind != 'FocalLoss' or not c.get('use_sigmoid', True) or c.get('activated', False) or c.get('reduction', 'mean') != 'mean':
            self.focal = f'loss_cate {kind} {c}'
        else:
            self.focal = (float(c.get('gamma', 2.0)), float(c.get('alpha', 0.25)), float(c.get('loss_weight', 1.0)))
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
        without objects.  Without ``conv``, every level and image of a network is one ``disco_cells_conv`` call (one
        dense wgmma launch on the packed kernels, the same values as one call per (level, image)); a given ``conv``
        (mask_feat_img [C,h,w], kernels [C,I]) -> [I,h,w] runs once per (level, image) with objects, in plain torch."""
        return self._corr_inputs(s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list, gt_label_list,
                                 gt_mask_list, use_ind_teacher, best, conv)[0]

    def _corr_inputs(self, s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list, gt_label_list,
                     gt_mask_list, use_ind_teacher, best, conv):
        """``corr_inputs`` and the per-image targets it was built from (``disco_target_single``'s four lists per image)."""
        from .disco_targets import disco_target_single
        scale_ranges, strides, grids, sigma = self._grid_cfg()
        fsize = tuple(s_ins_pred.shape[-2:])
        per_img = [disco_target_single(b, l, m, fsize, scale_ranges, strides, grids, sigma, self.num_classes, best=best)
                   for b, l, m in zip(gt_bbox_list, gt_label_list, gt_mask_list)]
        L_, B = len(grids), len(per_img)
        ins_labels = [torch.cat([per_img[b][0][lv] for b in range(B)], 0) for lv in range(L_)]
        klabels = [torch.cat([per_img[b][1][lv].reshape(-1)[per_img[b][3][lv]] for b in range(B)], 0) for lv in range(L_)]
        if conv is None:
            orders = [[per_img[b][3][lv] for b in range(B)] for lv in range(L_)]
            s_list, img_list = disco_cells_conv(s_ins_pred, s_kernel_preds_raw, orders)
            t_list = disco_cells_conv(t_ins_pred, t_kernel_preds_raw, orders)[0] if use_ind_teacher else [None] * L_
            return (s_list, t_list, img_list, ins_labels, klabels), per_img
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
        return (s_list, t_list, img_list, ins_labels, klabels), per_img

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

    # discobox_head.py:1142-1360, the reference's signature
    def loss(self, cate_preds, s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list, gt_label_list,
             gt_mask_list, img_metas, cfg, img=None, gt_bboxes_ignore=None, use_loss_ts=False, use_ind_teacher=False,
             use_corr=False, s_feat=None, t_feat=None):
        """dict(loss_ins, loss_ts, loss_cate, loss_corr) as the reference computes them.  ``gt_mask_list``: per image uint8
        [G,H,W] device tensors, or anything with mmdet's ``to_tensor(dtype, device)`` (BitmapMasks).

        The SOLO targets are built on the device (``solov2_target_single``'s lists; their per-(level, image) cell counts are
        the one host read), every level's and image's dynamic convolution of a network is one ``disco_cells_conv`` call, the
        mask losses run as ``mask_loss`` (one mean field over the batch), ``loss_cate`` is the focal kernel on the [B,C,S,S]
        levels as they lie with ``avg_factor = num_ins + 1`` on the device, and with ``use_loss_ts and use_corr`` the
        correspondence loss is ``corr_loss_levels`` on the ``best_target_single`` targets, its dice terms joining
        ``loss_ts``.  No loss value is read back to the host.  Autocast is the caller's: under ``torch.autocast('cuda')`` the
        convolutions take the autocast dtype, as the reference's ``@autocast()`` does.  Only the student receives gradients
        (the teacher's grids and mask features are detached); the teacher is convolved only with ``use_ind_teacher``.
        Where the reference returns ``torch.zeros(1)`` (no instance with a non-empty target) this returns a 0-d zero."""
        if isinstance(self.focal, str):
            ref = getattr(type(self), '_bxs_reference_class', None)
            if ref is not None:
                return ref.loss(self, cate_preds, s_kernel_preds_raw, t_kernel_preds_raw, s_ins_pred, t_ins_pred, gt_bbox_list,
                                gt_label_list, gt_mask_list, img_metas, cfg, img, gt_bboxes_ignore, use_loss_ts,
                                use_ind_teacher, use_corr, s_feat, t_feat)
            raise NotImplementedError(f'DiscoBoxSOLOv2Head.loss: unsupported {self.focal}')
        dev = s_ins_pred.device
        masks = [(m if torch.is_tensor(m) else m.to_tensor(dtype=torch.uint8, device=dev)).to(dev, torch.uint8)
                 for m in gt_mask_list]
        t_kern = [k.detach() for k in t_kernel_preds_raw] if use_ind_teacher else None
        t_ins = t_ins_pred.detach() if use_ind_teacher else None
        (s_list, t_list, img_list, ins_labels, _), per_img = self._corr_inputs(
            s_kernel_preds_raw, t_kern, s_ins_pred, t_ins, gt_bbox_list, gt_label_list, masks, use_ind_teacher, False, None)
        color_feats = bilinear_resize(img, tuple(s_ins_pred.shape[-2:]), align_corners=True)             # :1201
        out = self.mask_loss(s_list, ins_labels, img_list, color_feats, t_list if use_ind_teacher else None, use_loss_ts)
        loss_ins, loss_ts = out['loss_ins'], out['loss_ts']
        zero = color_feats.new_zeros(())
        if use_loss_ts and use_corr:                                                                       # :1309-1337
            c_s, c_t, c_img, c_lab, c_kl = self.corr_inputs(s_kernel_preds_raw, t_kern, s_ins_pred, t_ins, gt_bbox_list,
                                                            gt_label_list, masks, use_ind_teacher=use_ind_teacher, best=True)
            loss_corr, corr_ts = self.corr_loss_levels(c_s, c_t, c_img, c_lab, c_kl, s_feat[0], t_feat[0], color_feats,
                                                       use_ind_teacher)
            kept = sum(((t.flatten(1) != 0).any(1).sum() for s, t in zip(s_list, ins_labels) if s is not None), zero)
            loss_ts = torch.where(kept > 0, loss_ts + corr_ts * self.ts_loss_weight, zero)    # only with terms of its own
        else:
            loss_corr = zero
        B, n_lv = len(per_img), len(cate_preds)
        cate_labels = [torch.stack([per_img[b][1][lv] for b in range(B)]) for lv in range(n_lv)]
        num_ins = torch.stack([per_img[b][2][lv].sum() for b in range(B) for lv in range(n_lv)]).sum()
        loss_cate = sigmoid_focal_loss_levels(cate_preds, cate_labels, num_ins + 1, *self.focal)
        return dict(loss_ins=loss_ins, loss_ts=loss_ts, loss_cate=loss_cate, loss_corr=loss_corr)

    # discobox_head.py:1531-1660, the reference's signature
    def get_seg(self, cate_preds, kernel_preds, seg_pred, img_metas, cfg, rescale=None, img=None):
        """Per image the reference's ``InstanceData`` with ``masks`` bool [n, H_ori, W_ori], ``labels`` int64 and ``scores``,
        every image of the batch at once under float16 autocast, as the reference's ``@autocast()`` get_seg_single runs:
        each distinct candidate cell of ``kernel_preds`` is convolved with ``seg_pred`` once (``bxs_disco_cells_pack`` +
        ``dynconv1x1``), then the statistics, Matrix NMS and the mask paste on the GPU, two host reads per call
        (``solo_seg.discobox_get_seg``)."""
        from .solo_seg import discobox_get_seg
        with torch.no_grad():
            return discobox_get_seg(cate_preds, kernel_preds, seg_pred, self._grid_cfg()[1], img_metas, cfg)

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
    """Box2Mask head: ``forward`` / ``loss`` / ``loss_single`` with the reference's signatures, and the mask-loss path
    (``mask_loss_single``, ``mask_loss_layers``).  The decoder modules are the reference constructor's (mmdet installed, or
    attached by the caller); the standalone constructor builds only the losses and the matcher."""

    def __init__(self, in_channels=None, feat_channels=256, out_channels=256, num_things_classes=80, num_stuff_classes=0,
                 num_queries=100, loss_cls=None, loss_box=None, loss_mask=None, train_cfg=None, **cfg):
        super().__init__()
        self.num_queries = num_queries
        self.num_classes = num_things_classes + num_stuff_classes
        self.train_cfg = train_cfg
        self.cfg = cfg
        # configs/box2mask/box2mask_r50_lsj_8x2_50e_coco.py:92-97
        self.loss_cls_cfg = loss_cls or dict(type='CrossEntropyLoss', use_sigmoid=False, loss_weight=2.0, reduction='mean',
                                             class_weight=[1.0] * self.num_classes + [0.1])
        self.loss_box = build_loss(loss_box or dict(type='BoxProjectionLoss', loss_weight=5.0))
        self.loss_mask = build_loss(loss_mask or dict(type='LevelsetLoss', loss_weight=1.0))
        self.mst = MinimumSpanningTree(TreeFilter2D.norm2_distance)
        self.tree_filter = TreeFilter2D()
        self._bxs_post_init()

    def _bxs_post_init(self):
        """Also runs after the REFERENCE class's ``__init__`` when mmdet is importable: the matcher of ``get_targets`` is
        this package's MaskHungarianAssigner, built from the same ``train_cfg['assigner']`` (box2mask_head.py:95-97), and the
        classification loss is read from the CrossEntropyLoss module and ``class_weight`` that constructor built (:99-100)."""
        from ...core.assigner import MaskHungarianAssigner      # core imports models.builder: not at module level
        cfg = (getattr(self, 'train_cfg', None) or {}).get('assigner')
        self.hungarian = MaskHungarianAssigner(**{k: v for k, v in cfg.items() if k != 'type'}) if cfg else None
        self.lsap_status = None
        ref = getattr(self, 'loss_cls', None)
        if isinstance(ref, nn.Module):
            cls_cfg = dict(use_sigmoid=ref.use_sigmoid, use_mask=getattr(ref, 'use_mask', False), reduction=ref.reduction,
                           loss_weight=ref.loss_weight, avg_non_ignore=getattr(ref, 'avg_non_ignore', False),
                           class_weight=getattr(self, 'class_weight', ref.class_weight))
        else:
            cls_cfg = self.loss_cls_cfg
        if (cls_cfg.get('use_sigmoid', False) or cls_cfg.get('use_mask', False) or cls_cfg.get('reduction', 'mean') != 'mean'
                or cls_cfg.get('avg_non_ignore', False)):
            raise NotImplementedError('Box2MaskHead: the classification loss is the softmax cross-entropy with reduction '
                                      f"'mean' only, got {cls_cfg}")
        cw = cls_cfg.get('class_weight')
        self.cls_loss_weight = float(cls_cfg.get('loss_weight', 1.0))
        self.cls_class_weight = None if cw is None else [float(v) for v in cw]
        self._class_weight_on = {}                               # device -> [K] tensor, copied once per device

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
        costs = self._costs(cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list)
        matches, self.lsap_status = solve_batched(costs)
        return self._targets_of_matches(matches, mask_preds_list, gt_labels_list, gt_masks_list)[0]

    # f1 -- get_targets of every decoder layer (box2mask_head.py:203-205, 238-241), the matching in one launch
    @torch.no_grad()
    def get_targets_layers(self, all_cls_scores, all_mask_preds, gt_labels_list, gt_masks_list, img_metas):
        """``get_targets`` of every decoder layer: a list with one 6-tuple per layer, each bit for bit what
        ``get_targets(all_cls_scores[l], all_mask_preds[l], ...)`` returns.  all_cls_scores[l] [B,Q,C+1] (or a list of
        per-image tensors), all_mask_preds[l] [B,Q,h,w] likewise.  The L*B cost matrices are matched in ONE launch, whose
        problems (one dependent chain on one warp each) run side by side; nothing is read back to the host.
        ``self.lsap_status`` becomes int32 [L, B]."""
        return self._targets_layers(all_cls_scores, all_mask_preds, gt_labels_list, gt_masks_list)[0]

    def _targets_layers(self, all_cls_scores, all_mask_preds, gt_labels_list, gt_masks_list):
        """(per-layer 6-tuples of ``get_targets``, per-layer lists of the images' positive query indices)."""
        n_layers, B = len(all_cls_scores), len(gt_labels_list)
        costs = []
        for cls_scores, mask_preds in zip(all_cls_scores, all_mask_preds):
            costs += self._costs([cls_scores[b] for b in range(B)], [mask_preds[b] for b in range(B)], gt_labels_list,
                                 gt_masks_list)
        matches, status = solve_batched(costs)
        self.lsap_status = status.view(n_layers, B)
        out = [self._targets_of_matches(matches[l * B:(l + 1) * B], [mask_preds[b] for b in range(B)], gt_labels_list,
                                        gt_masks_list) for l, mask_preds in enumerate(all_mask_preds)]
        return [o[0] for o in out], [o[1] for o in out]

    def _costs(self, cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list):
        """The [Q, G_b] cost matrix of every image (mask_hungarian_assigner.py:92-111 on the low-resolution prediction)."""
        if self.hungarian is None:
            raise RuntimeError('Box2MaskHead.get_targets needs train_cfg with an assigner')
        costs = []
        for cls_score, mask_pred, gt_labels, gt_masks in zip(cls_scores_list, mask_preds_list, gt_labels_list, gt_masks_list):
            if gt_labels.shape[0] and mask_pred.shape[0]:
                costs.append(self.hungarian.cost_matrix(cls_score, mask_pred, gt_labels, gt_masks, lowres=True))
            else:
                costs.append(mask_pred.new_zeros((mask_pred.shape[0], gt_labels.shape[0])))
        return costs

    def _targets_of_matches(self, matches, mask_preds_list, gt_labels_list, gt_masks_list):
        """(``get_targets``' 6-tuple, the positive query indices of every image) from one layer's matches."""
        Q = self.num_queries
        labels_list, label_weights_list, mask_targets_list, mask_weights_list, pos_inds_list = [], [], [], [], []
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
            pos_inds_list.append(pos_inds)
            num_total_pos += k
            num_total_neg += mask_pred.shape[0] - k
        return ((labels_list, label_weights_list, mask_targets_list, mask_weights_list, num_total_pos, num_total_neg),
                pos_inds_list)

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

    # box2mask_head.py:445-459, the reference's signature
    def simple_test(self, feats, img_metas, **kwargs):
        """(mask_cls [B,Q,K+1], mask_pred [B,Q,h,w]) of the last decoder layer.  Unlike the reference, the mask predictions
        stay at the mask-feature resolution: MaskFormerFusionHead.simple_test upsamples them to batch_input_shape inside
        its paste.  ``ops.resize.bilinear_resize(mask_pred, batch_input_shape)`` gives the reference's tensor bit for bit."""
        all_cls_scores, all_mask_preds, _ = self(feats, img_metas)
        return all_cls_scores[-1], all_mask_preds[-1]

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
        ``mask_targets`` and ``lst_feat``: one tensor for every layer, or a list with one per layer (each decoder layer has
        its own matching and its own level-set feature, :203-205).  Returns the list of (loss_project, loss_levelset) pairs."""
        n_layers = len(mask_preds_per_layer)
        targets = list(mask_targets) if isinstance(mask_targets, (list, tuple)) else [mask_targets] * n_layers
        lst_feats = list(lst_feat) if isinstance(lst_feat, (list, tuple)) else [lst_feat] * n_layers
        if trees is None:
            first = mask_preds_per_layer[0]
            shape = (first() if callable(first) else first).shape[-2:]
            trees = self.image_trees(norm_img, shape)

        def layer(mp, tg, lf):
            mp = mp() if callable(mp) else mp
            return self.mask_loss_single(mp, tg, num_per_img, norm_img, lf, trees=trees)

        return run_concurrently([lambda w=w: layer(*w) for w in zip(mask_preds_per_layer, targets, lst_feats)],
                                norm_img.device)

    def _class_weight(self, device):
        """The class weights as a [K] float32 tensor on ``device`` (copied once per device, so that later calls read nothing
        from the host and can be captured in a CUDA graph), or None."""
        if self.cls_class_weight is None:
            return None
        cw = self._class_weight_on.get(device)
        if cw is None:
            cw = self._class_weight_on[device] = torch.tensor(self.cls_class_weight, dtype=torch.float32, device=device)
        return cw

    # box2mask_head.py:192-221, the reference's signature
    def loss(self, all_cls_scores, all_mask_preds, all_lst_feats, gt_labels_list, gt_masks_list, img_metas, norm_img):
        """The reference's dict: ``loss_cls``, ``loss_project``, ``loss_levelset`` of the last decoder layer, then
        ``d{i}.loss_*`` of the others.  all_cls_scores[l] [B,Q,C+1], all_mask_preds[l] [B,Q,h,w] (promoted to float32, the
        reference's ``@force_fp32``), all_lst_feats[l] [B,1,h',w'] (each layer its own), gt_labels_list[b] [G_b],
        gt_masks_list[b] [G_b,H,W], norm_img [B,3,H,W].
        Every layer is matched in ONE launch (``get_targets_layers``), ``loss_cls`` of every layer is ONE kernel
        (``softmax_cross_entropy_layers``), the matched rows are gathered with the min(Q, G_b) positive indices per image (known
        from the shapes), the image trees are built once, and the mask losses of the layers run on lane streams.  Nothing is
        read back to the host: after one eager call the loss can be captured in a CUDA graph.
        An image whose costs hold a NaN cannot raise without a host read (the reference raises from scipy): its layer's
        ``loss_cls`` is NaN and ``self.lsap_status[l, b]`` is non-zero.  A batch without ground truth gives zero
        ``loss_project`` / ``loss_levelset`` attached to the graph (the reference's sum over no rows)."""
        losses_cls, losses_project, losses_levelset = self._loss_layers(all_cls_scores, all_mask_preds, all_lst_feats,
                                                                        gt_labels_list, gt_masks_list, norm_img)
        loss_dict = dict(loss_cls=losses_cls[-1], loss_project=losses_project[-1], loss_levelset=losses_levelset[-1])
        for i, (c, p, s) in enumerate(zip(losses_cls[:-1], losses_project[:-1], losses_levelset[:-1])):
            loss_dict[f'd{i}.loss_cls'] = c
            loss_dict[f'd{i}.loss_project'] = p
            loss_dict[f'd{i}.loss_levelset'] = s
        return loss_dict

    # box2mask_head.py:224-335, the reference's signature
    def loss_single(self, cls_scores, mask_preds, lst_feat, gt_labels_list, gt_masks_list, img_metas, norm_img):
        """(loss_cls, loss_project, loss_levelset) of one decoder layer, as the reference returns them (``loss`` of one
        layer)."""
        c, p, s = self._loss_layers([cls_scores], [mask_preds], [lst_feat], gt_labels_list, gt_masks_list, norm_img)
        return c[0], p[0], s[0]

    def _loss_layers(self, all_cls_scores, all_mask_preds, all_lst_feats, gt_labels_list, gt_masks_list, norm_img):
        """Lists of loss_cls, loss_project, loss_levelset, one entry per decoder layer."""
        from ...ops.cross_entropy import softmax_cross_entropy_layers
        cls_scores = [c.float() for c in all_cls_scores]
        mask_preds = [m.float() for m in all_mask_preds]
        lst_feats = [f.float() for f in all_lst_feats]
        n_layers, B = len(cls_scores), len(gt_labels_list)
        dev = cls_scores[0].device
        with torch.no_grad():
            targets, pos_inds = self._targets_layers(cls_scores, mask_preds, gt_labels_list, gt_masks_list)
        labels = torch.stack([torch.stack(t[0]) for t in targets])                              # [L,B,Q]
        losses_cls = softmax_cross_entropy_layers(cls_scores, labels, self._class_weight(dev), self.cls_loss_weight)
        failed = (self.lsap_status != 0).any(1)                 # a layer with an unmatched (NaN) image: loss_cls is NaN
        losses_cls = torch.where(failed, torch.full_like(losses_cls, float('nan')), losses_cls)
        losses_cls = list(losses_cls.unbind(0))
        num_per_img = [min(mask_preds[0].shape[1], int(g.shape[0])) for g in gt_labels_list]       # from the shapes
        if sum(num_per_img) == 0:                               # zero match (:262-267): sums over no rows, on the graph
            zeros = [m[:0].sum() for m in mask_preds]
            return losses_cls, zeros, [z.clone() for z in zeros]
        rows = [torch.cat([mp[b].index_select(0, pos_inds[l][b]) for b in range(B)])
                for l, mp in enumerate(mask_preds)]                                                 # mask_preds[weights > 0]
        mask_targets = [torch.cat(t[2]).squeeze(1) for t in targets]
        pairs = self.mask_loss_layers(rows, mask_targets, num_per_img, norm_img.float(), lst_feats,
                                      trees=self.image_trees(norm_img.float(), mask_preds[0].shape[-2:]))
        return losses_cls, [p[0] for p in pairs], [p[1] for p in pairs]

    def image_trees(self, norm_img, pred_shape):
        """MST of every image at 96x96 (box2mask_head.py:232,269-272): identical for all decoder layers of a step."""
        with torch.no_grad():
            return self.mst(_scale_target(bilinear_resize(norm_img, pred_shape)))
