"""bench.py --config C | D | E: the mask-loss steps of the other three box-supervised methods of BASELINE.json
(configs[2..4]) on the synthetic shapes of SURVEY.md section 8d.  Imported by bench.py; prints nothing itself.

  C  DiscoBox R-50 800x1024      mask_feat [2,256,200,256], 16 positive kernels / image -> per-image dynamic conv (a3,
                                  wgmma) -> MIL dice + mean-field teacher + dice (a6, a16, a17), fwd + bwd wrt mask_feat
                                  and the kernels.                                   discobox_head.py:1206-1300
  D  BoxLevelset R-50 800x1024   5 levels x 16 instances (8 / image) at 200x256, 200x256, 100x128, 50x64, 50x64:
                                  projection + two level-set terms + two tree filters per level (a6, a9, a12-a15, a17),
                                  fwd + bwd wrt the mask logits and the level-set features.   box_solov2_head.py:334-367
  E  Box2Mask 1024x1024, 1 img   mask_pred = einsum(100 queries, [256,256,256] feature) (a4, wgmma), 8 matched queries,
                                  10 decoder layers: projection + level-set + tree filter at 96x96 + LCM (a6, a9, a11-a15,
                                  a17, a18), fwd + bwd wrt the mask feature, the queries and the level-set feature.
                                                                                      box2mask_head.py:229-359

Each `build_*` returns (step_fn, info): step_fn() runs ONE forward + backward; info carries images per step, the
algorithmic bytes of the step (SURVEY 8d formulas, spelled out in `algo`) and what the gradients are taken of.
`reference_step_*` restates the reference's own eager path around the reference's compiled tree_filter_cuda
(oracle/_ref, built by oracle/Makefile) for the gpu_reference leg.
"""
import glob
import importlib.util
import os

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.abspath(__file__))
HP, WP = 800, 1024
LEVELS_D = [(200, 256), (200, 256), (100, 128), (50, 64), (50, 64)]


def _image_and_boxes(seed, b_img, hp=HP, wp=WP, gts=8):
    from tests.helpers import normalise, synth_boxes, synth_image
    gen = torch.Generator().manual_seed(seed)
    imgs = torch.stack([normalise(synth_image(gen, hp, wp, 160, 3.0)) for _ in range(b_img)])
    boxes = [synth_boxes(gen, gts, hp, wp) for _ in range(b_img)]
    return gen, imgs, boxes


def _box_masks(boxes, h, w, hp, wp, dev):
    """[G,h,w] float box masks rasterised at the map's stride (centre sampling, as get_bitmasks_from_boxes does)."""
    sy, sx = hp / h, wp / w
    ys = (torch.arange(h, device=dev).float() + 0.5) * sy
    xs = (torch.arange(w, device=dev).float() + 0.5) * sx
    b = boxes.to(dev)
    my = (ys[None, :] >= b[:, 1, None]) & (ys[None, :] <= b[:, 3, None])
    mx = (xs[None, :] >= b[:, 0, None]) & (xs[None, :] <= b[:, 2, None])
    return (my[:, :, None] & mx[:, None, :]).float()


# ------------------------------------------------------------------------------------------------------------------
# config D: BoxLevelset
# ------------------------------------------------------------------------------------------------------------------
def build_D(dev, seed):
    from boxinstseg_b200.models import build_head
    from boxinstseg_b200.ops.resize import bilinear_resize
    gen, imgs, boxes = _image_and_boxes(seed, 2)
    imgs = imgs.to(dev)
    head = build_head(dict(type='BoxSOLOv2Head', num_classes=80, in_channels=256,
                           loss_boxpro=dict(type='BoxProjectionLoss', loss_weight=3.0),
                           loss_levelset=dict(type='LevelsetLoss', loss_weight=1.0)))
    inst_img = torch.arange(2, device=dev, dtype=torch.int32).repeat_interleave(8)          # 8 instances / image / level
    g = torch.Generator(device=dev).manual_seed(seed)
    preds, labels, img_t, lst_t = [], [], [], []
    for (h, w) in LEVELS_D:
        preds.append((torch.randn(16, h, w, device=dev, generator=g) * 2).requires_grad_(True))
        labels.append(torch.cat([_box_masks(b, h, w, HP, WP, dev) for b in boxes]))
        img_t.append(bilinear_resize(imgs, (h, w)))                                            # box_solov2_head.py:412-415
        lst_t.append(torch.randn(2, 5, h, w, device=dev, generator=g).requires_grad_(True))
    inst = [inst_img] * len(LEVELS_D)
    leaves = preds + lst_t

    def step():
        out = head.mask_loss(preds, labels, img_t, lst_t, inst_imgs=inst)
        grads = torch.autograd.grad(out['loss_boxpro'] + out['loss_levelset'], leaves)
        return out, grads

    byts = 0
    for (h, w) in LEVELS_D:
        n, V = 16, h * w
        byts += 3 * n * V * 4                                   # projection: read scores + targets, write grad
        for C in (3, 2):
            byts += 2 * (2 + C) * n * V * 4 + 2 * n * V * 4     # level set: 2 passes over (S0,S1,T) + grad write
        byts += 2 * 3 * 4 * n * V * (2 * 1 * 4 + 28)            # tree filter: 2 filters x (fwd, bwd feature, bwd weight~) x 4 passes
    info = dict(images=2, algo_bytes=byts,
                algo='per level: projection 3nV4 + level set sum_C[2(2+C)nV4 + 2nV4] + tree filter 2 filters x 3 x 4 passes x '
                     'nV(2C4+28) (SURVEY 8d; dependency-latency kernels: an HBM LOWER bound)',
                grads='d/d mask logits (5 levels) and d/d level-set features',
                workload='BoxLevelset R-50 mask loss fwd+bwd (config D): 2 img x 8 inst x 5 levels at 200x256,200x256,100x128,'
                         '50x64,50x64; projection + 2 level-set terms + 2 tree filters per level',
                data=dict(preds=preds, labels=labels, img_t=img_t, lst_t=lst_t, inst=inst_img))
    return step, info


# ------------------------------------------------------------------------------------------------------------------
# config E: Box2Mask
# ------------------------------------------------------------------------------------------------------------------
def build_E(dev, seed, layers=10, matched=8):
    from boxinstseg_b200.models import build_head
    gen, imgs, boxes = _image_and_boxes(seed, 1, 1024, 1024)
    imgs = imgs.to(dev)
    head = build_head(dict(type='Box2MaskHead', num_queries=100,
                           loss_box=dict(type='BoxProjectionLoss', loss_weight=5.0),
                           loss_mask=dict(type='LevelsetLoss', loss_weight=1.0)))
    g = torch.Generator(device=dev).manual_seed(seed)
    feat = torch.randn(1, 256, 256, 256, device=dev, generator=g).requires_grad_(True)
    embeds = [(torch.randn(1, 100, 256, device=dev, generator=g) * 0.05).requires_grad_(True) for _ in range(layers)]
    lst = torch.randn(1, 1, 256, 256, device=dev, generator=g).requires_grad_(True)
    sel = torch.arange(0, 100, 100 // matched, device=dev)[:matched]                       # the Hungarian-matched queries
    targets = _box_masks(boxes[0][:matched], 1024, 1024, 1024, 1024, dev)
    leaves = [feat, lst] + embeds

    def step():
        trees = head.image_trees(imgs, (256, 256))                                          # once per step, shared by the layers
        # box2mask_head.py:343-345 + matching, then loss_single, per decoder layer (multi_apply over the layers, :214-227)
        pairs = head.mask_loss_layers([lambda e=e: head.mask_pred(e, feat)[0].index_select(0, sel) for e in embeds], targets,
                                      [matched], imgs, lst, trees=trees)
        total = sum(lp + lm for lp, lm in pairs)
        return total, torch.autograd.grad(total, leaves)

    n, V, V96 = matched, 256 * 256, 96 * 96
    per_layer = (256 * V * 4 + 100 * V * 4) * 3                                             # a4 fwd + 2 bwd GEMMs: feature + output streams
    per_layer += 3 * n * V * 4 + sum(2 * (2 + C) * n * V * 4 + 2 * n * V * 4 for C in (3, 2))
    per_layer += 2 * 3 * 4 * n * V96 * (2 * 4 + 28) + 10 * 2 * n * V96 * 10 * 4
    info = dict(images=1, algo_bytes=layers * per_layer,
                algo='per decoder layer: einsum 3 x (256+100)V4 + projection 3nV4 + level set + tree filter at 96x96 + LCM '
                     '10 it x 2 x nV96 x 10 x 4 (SURVEY 8d)',
                grads='d/d mask feature, d/d 10 x query embeddings, d/d level-set feature',
                workload=f'Box2Mask mask loss fwd+bwd (config E): 1 img 1024x1024, {layers} decoder layers x ({matched} matched of 100 '
                         'queries): einsum + projection + level set + tree filter/LCM at 96x96',
                data=dict(feat=feat, embeds=embeds, lst=lst, sel=sel, targets=targets, imgs=imgs))
    return step, info


# ------------------------------------------------------------------------------------------------------------------
# config C: DiscoBox
# ------------------------------------------------------------------------------------------------------------------
def build_C(dev, seed, kernels_per_img=16):
    from boxinstseg_b200.models import build_head
    from boxinstseg_b200.ops.resize import bilinear_resize
    gen, imgs, boxes = _image_and_boxes(seed, 2, gts=kernels_per_img)
    imgs = imgs.to(dev)
    head = build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=80, in_channels=256))
    g = torch.Generator(device=dev).manual_seed(seed)
    feat = torch.randn(2, 256, 200, 256, device=dev, generator=g).requires_grad_(True)
    kern = (torch.randn(2, 256, kernels_per_img, device=dev, generator=g) * 0.05).requires_grad_(True)
    labels = torch.cat([_box_masks(b, 200, 256, HP, WP, dev) for b in boxes])
    img_inds = torch.arange(2, device=dev, dtype=torch.int32).repeat_interleave(kernels_per_img)
    color = bilinear_resize(imgs, (200, 256), align_corners=True)                           # discobox_head.py:1201

    def step():
        pred = torch.cat([head.dynamic_conv(feat[b], kern[b]) for b in range(2)])          # :1206-1220, per image
        out = head.mask_loss([pred], [labels], [img_inds], color)
        return out, torch.autograd.grad(out['loss_ins'] + out['loss_ts'], [feat, kern])

    n, V = 2 * kernels_per_img, 200 * 256
    byts = 2 * 3 * (256 * V * 4 + kernels_per_img * V * 4) + 2 * 3 * n * V * 4 + (10 * 2 * n * V * 4 * 2 + 2 * 9 * V * 4)
    info = dict(images=2, algo_bytes=byts,
                algo='dynamic conv 3 x (256+I)V4 per image + MIL/dice 2 x 3nV4 + mean field 10(2nV4*2)+9V4 per image (SURVEY 8d)',
                grads='d/d mask_feat, d/d kernels',
                workload=f'DiscoBox R-50 mask loss fwd+bwd (config C): 2 img, mask_feat [2,256,200,256], {kernels_per_img} positive '
                         'kernels/img: dynamic conv + MIL dice + mean-field teacher (10 it) + dice',
                data=dict(feat=feat, kern=kern, labels=labels, img_inds=img_inds, color=color))
    return step, info


BUILDERS = dict(C=build_C, D=build_D, E=build_E)


# ------------------------------------------------------------------------------------------------------------------
# gpu_reference: the reference's eager path around its own compiled tree_filter_cuda (baseline only)
# ------------------------------------------------------------------------------------------------------------------
def _load_ref(name):
    hits = glob.glob(os.path.join(ROOT, 'oracle', '_ref', name + '*.so'))
    if not hits:
        return None
    spec = importlib.util.spec_from_file_location(name, hits[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


class _RefTree:
    """MinimumSpanningTree + TreeFilter2D exactly as mmdet/ops/tree_filter/modules/tree_filter.py:9-150 composes them, on the
    reference's compiled kernels (functions/mst.py, bfs.py, refine.py restated as one autograd Function)."""

    def __init__(self, ext):
        self.ext = ext
        ext_ = ext

        class Refine(torch.autograd.Function):                       # functions/refine.py:9-41
            @staticmethod
            def forward(ctx, feature_in, edge_weight, idx, par, chd, low_tree):
                out, aggr, aggr_up, wsum, wsum_up = ext_.refine_forward(feature_in, edge_weight, idx, par, chd)
                ctx.save_for_backward(feature_in, edge_weight, idx, par, chd, out, aggr, aggr_up, wsum, wsum_up)
                ctx.low_tree = low_tree
                return out

            @staticmethod
            def backward(ctx, g):
                saved = ctx.saved_tensors
                gf = ext_.refine_backward_feature(*saved, g.contiguous())
                gw = None if ctx.low_tree else ext_.refine_backward_weight(*saved, g.contiguous())
                return gf, gw, None, None, None, None
        self.refine = Refine.apply

    def mst(self, fm):                                                # tree_filter.py:9-62
        b, _, h, w = fm.shape
        with torch.no_grad():
            ids = torch.arange(h * w, dtype=torch.int32, device=fm.device).view(h, w)
            index = torch.cat((torch.stack((ids[:-1], ids[1:]), 2).reshape(-1, 2),
                               torch.stack((ids[:, :-1], ids[:, 1:]), 2).reshape(-1, 2))).unsqueeze(0).expand(b, -1, -1).contiguous()
            d = lambda a, c: ((a - c) ** 2).sum(1)   # noqa: E731
            weight = torch.cat((d(fm[:, :, :-1], fm[:, :, 1:]).reshape(b, -1), d(fm[:, :, :, :-1], fm[:, :, :, 1:]).reshape(b, -1)), 1) + 1
            return self.ext.mst_forward(index, weight.contiguous(), h * w)

    def filter(self, feature_in, embed_in, tree, low_tree=True, sigma=0.02):      # tree_filter.py:91-150
        shape = feature_in.shape
        idx, par, chd = self.ext.bfs_forward(tree, 4)
        b, c = embed_in.shape[:2]
        flat = embed_in.reshape(b, c, -1)
        src = torch.gather(flat, 2, idx.long().unsqueeze(1).expand(-1, c, -1))
        dst = torch.gather(src, 2, par.long().unsqueeze(1).expand(-1, c, -1))
        dist = ((src - dst) ** 2).sum(1)
        ew = torch.exp(-dist / sigma) if low_tree else torch.exp(-dist)
        return self.refine(feature_in.reshape(shape[0], shape[1], -1).contiguous(), ew, idx, par, chd, low_tree).reshape(shape)


def _ref_levelset(phi, target, pix, w=1.0):                            # levelset_loss.py:13-44
    n, c = target.shape[:2]
    energy = 0
    for k in range(2):
        s = phi[:, k:k + 1]
        mean = (s * target).sum((2, 3)) / s.sum((2, 3)).clamp(min=1e-5)
        energy = energy + (((target - mean[:, :, None, None]) ** 2) * s).sum((1, 2, 3))
    return w * energy / c / pix


def _ref_projection(s, m, w, eps=1e-5):                               # box_projection_loss.py:11-42
    def dice(a, b):
        a, b = a.flatten(1), b.flatten(1)
        return 1 - 2 * (a * b).sum(1) / ((a * a).sum(1) + (b * b).sum(1) + eps)
    return w * (dice(s.amax(2), m.amax(2)) + dice(s.amax(3), m.amax(3)))


def reference_step_D(info):
    """BoxSOLOv2Head.loss per level as the reference runs it (box_solov2_head.py:334-367): per-INSTANCE image / feature
    targets, trees rebuilt per instance, eager elementwise chains, its own tree_filter_cuda kernels."""
    ext = _load_ref('tree_filter_cuda_ref')
    if ext is None:
        return None
    rt = _RefTree(ext)
    d = info['data']
    ii = d['inst'].long()
    leaves = d['preds'] + d['lst_t']

    def step():
        lp, ll = [], []
        for ins_pred, box, img_b, lst_b in zip(d['preds'], d['labels'], d['img_t'], d['lst_t']):
            img_t, lst_t = img_b[ii], lst_b[ii]                       # the reference's per-instance copies (:296-305)
            s = torch.sigmoid(ins_pred.unsqueeze(1))
            b = box.unsqueeze(1)
            lp.append(_ref_projection(s, b, 3.0))
            phi = torch.cat((s, 1 - s), 1) * b
            pix = b.sum((1, 2, 3)).clamp(min=1)
            l_img = _ref_levelset(phi, img_t * b, pix) * 0.05
            f1 = rt.filter(s, img_t, rt.mst(img_t))
            f2 = rt.filter(f1, lst_t, rt.mst(lst_t), low_tree=False)
            ll.append(l_img + _ref_levelset(phi, torch.cat((f1, f2), 1) * b, pix) * 5.0)
        loss = torch.cat(lp).mean() + torch.cat(ll).mean()
        return loss, torch.autograd.grad(loss, leaves)
    return step


def _ref_lcm(imgs, phi, box, dilation=2, iters=10):                   # levelset_loss.py:64-126
    def nbrs(x):
        p = F.pad(x, (dilation,) * 4, mode='replicate')
        h, w = x.shape[-2:]
        return torch.stack([p[:, :, dilation + dy * dilation: dilation + dy * dilation + h, dilation + dx * dilation: dilation + dx * dilation + w]
                            for dy, dx in [(-1, -1), (-1, 0), (-1, 1), (0, -1), (0, 1), (1, -1), (1, 0), (1, 1)]], 2)
    nb = nbrs(imgs)
    aff = -(((nb - imgs.unsqueeze(2)).abs() / (nb.std(2, keepdim=True) + 1e-8) / 0.3) ** 2).mean(1, keepdim=True)
    aff = torch.softmax(aff, 2)
    cur = phi
    for _ in range(iters):
        cur = (nbrs(cur) * aff).sum(2)
    return ((cur - phi).abs() * box).sum() / box.sum().clamp(min=1)


def reference_step_E(info, layers=10):
    """Box2MaskHead.forward_head + loss_single (box2mask_head.py:229-359) eager, cuBLAS einsum, ATen interpolate, the
    reference's tree_filter_cuda; trees rebuilt in every layer as the reference does."""
    ext = _load_ref('tree_filter_cuda_ref')
    if ext is None:
        return None
    rt = _RefTree(ext)
    d = info['data']
    leaves = [d['feat'], d['lst']] + d['embeds']
    interp = lambda t, s: F.interpolate(t, s, mode='bilinear', align_corners=False)   # noqa: E731

    def step():
        total = 0.0
        n = d['sel'].numel()
        for e in d['embeds'][:layers]:
            mp = torch.einsum('bqc,bchw->bqhw', e, d['feat'])[0][d['sel']]
            shape = mp.shape[-2:]
            img, lst = interp(d['imgs'], shape), interp(d['lst'], shape)
            it, lt = img.repeat(n, 1, 1, 1), lst.repeat(n, 1, 1, 1)
            box = interp(d['targets'].unsqueeze(1), shape)
            s = torch.sigmoid(mp.unsqueeze(1))
            lp = _ref_projection(s, box, 5.0).mean()
            phi = torch.cat((s, 1 - s), 1) * box
            pix = box.sum((1, 2, 3)).clamp(min=1)
            l_img = _ref_levelset(phi, it * box, pix).mean() * 0.05
            i96, l96, s96 = interp(it, (96, 96)), interp(lt, (96, 96)), interp(s, (96, 96))
            f1 = rt.filter(s96, i96, rt.mst(interp(img, (96, 96))).repeat(n, 1, 1))
            f2 = rt.filter(f1, l96, rt.mst(interp(lst, (96, 96))).repeat(n, 1, 1), low_tree=False)
            deep = torch.cat((interp(f1, shape), interp(f2, shape)), 1) * box
            l_feat = _ref_levelset(phi, deep, pix).mean() * 5.0
            total = total + lp + l_img + l_feat + 0.2 * _ref_lcm(i96, s96, interp(box, (96, 96)))
        return total, torch.autograd.grad(total, leaves)
    return step


def _ref_meanfield(color, x, targets, alpha0=2.0, theta0=0.5, theta1=30.0, base=0.1, iters=10):   # discobox_head.py:585-651
    f = color + 10
    unf = F.unfold(f, 3, padding=1).view(f.shape[0], f.shape[1], 9, *f.shape[-2:])
    d2 = ((unf - f.unsqueeze(2)) ** 2).sum(1)
    yy, xx = torch.meshgrid(torch.arange(-1., 2., device=f.device), torch.arange(-1., 2., device=f.device), indexing='ij')
    sp = (yy ** 2 + xx ** 2).reshape(1, 9, 1, 1)
    K = alpha0 * torch.exp(-d2 / (2 * theta0 ** 2) - sp / (2 * theta1 ** 2))
    x = ((x * targets) > 0.5).float() * (1 - 2 * base) + base
    U = torch.cat((1 - x, x), 1)
    n, _, h, w = U.shape
    for _ in range(iters):
        nl = F.unfold(-torch.log(U), 3, padding=1).view(n, 2, 9, h, w)
        fq = torch.exp(-(nl * K.unsqueeze(1)).sum(2))
        fq = torch.cat((fq[:, :1], fq[:, 1:] * targets), 1) + 1e-6
        fq = fq / fq.sum(1, keepdim=True)
        xq = (fq[:, 1:] > 0.5).float() * (1 - 2 * base) + base
        U = torch.cat((1 - xq, xq), 1)
    return (U[:, 1:] > 0.5).float()


def reference_step_C(info):
    """DiscoBox loss (discobox_head.py:1206-1300) eager: F.conv2d per image, MIL dice, MeanField via unfold, dice."""
    d = info['data']

    def step():
        pred = torch.cat([F.conv2d(d['feat'][b:b + 1], d['kern'][b].t()[:, :, None, None])[0] for b in range(2)])
        s = torch.sigmoid(pred)
        t = d['labels']
        l_ins = _ref_projection(s.unsqueeze(1), t.unsqueeze(1), 1.0, eps=2e-3).mean()
        enlarged = F.max_pool2d(t.unsqueeze(1), 3, 1, 1).squeeze(1)
        with torch.no_grad():
            pseudo = torch.cat([_ref_meanfield(d['color'][b:b + 1], s[d['img_inds'] == b].unsqueeze(1),
                                               t[d['img_inds'] == b].unsqueeze(1)) for b in range(2)]).squeeze(1)
        x, p = (s * enlarged).flatten(1), pseudo.flatten(1)
        l_ts = (1 - 2 * (x * p).sum(1) / ((x * x).sum(1) + 0.001 + (p * p).sum(1) + 0.001)).mean()
        loss = l_ins + l_ts
        return loss, torch.autograd.grad(loss, [d['feat'], d['kern']])
    return step


REFERENCE = dict(C=reference_step_C, D=reference_step_D, E=reference_step_E)
