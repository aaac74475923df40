"""Every op on the tensors a training loop really hands it: strided, offset, misaligned and stride-0 views, and zero-size
batches.

The kernels sit behind a C ABI that receives bare ``data_ptr()``s and assumes dense row-major tensors, several of them
8- or 16-byte aligned bases as well (vector loads, TMA tensor maps).  The only thing between a view and a kernel reading
the wrong elements is the normalisation each Python wrapper does, so this file calls every op twice -- once on fresh,
dense, aligned ("canonical") inputs, once with ONE tensor argument replaced by a view that is equal in value and laid out
differently -- and asserts what the layout contract of INTEGRATION.md promises: the same bits out, the same bits in every
gradient, dense outputs, gradients of the input's shape, and the view left untouched.

``CASES`` is the table: one entry per op with a seeded builder, the arguments to perturb, and a forward closure.  Bit
equality is the rule; an exception is an explicit ``tol`` entry of a case with its reason, never a global tolerance.
Test ids read ``op.shape-argument-kind``.

Upstream gradients: autograd casts a root ``grad_outputs`` to the output's dtype before it reaches a ``Function`` (a
float64 or 16-bit one arrives as a fresh float32 tensor), but it hands strides through unchanged, so the upstream sweep
perturbs the layout only: the same kinds, plus the stride-0 gradients ``out.sum()`` and ``out.mean()`` produce.
"""
import pytest
import torch

from tests.helpers import boxinst_case

pytestmark = pytest.mark.gpu

DEV = 'cuda'
KINDS = ('transposed', 'channels_last', 'sliced', 'batch_view', 'offset1')
G_KINDS = ('transposed', 'sliced', 'batch_view', 'offset1', 'expanded', 'sum', 'mean')
F16, BF16, F32 = torch.float16, torch.bfloat16, torch.float32


# ------------------------------------------------------------------------------------------------------------ layouts
def relayout(t, kind):
    """A tensor equal in value to ``t`` with another layout.  Every read of the result stays inside its own storage."""
    if kind == 'transposed':            # last two dims swapped in memory
        return t.transpose(-1, -2).contiguous().transpose(-1, -2)
    if kind == 'channels_last':
        return t.contiguous(memory_format=torch.channels_last)
    if kind == 'sliced':                # a [..., ::2] window of a buffer twice as wide
        big = t.new_zeros(t.shape[:-1] + (2 * t.shape[-1],))
        big[..., ::2] = t
        return big[..., ::2]
    if kind == 'batch_view':            # dense, one leading row into a larger buffer
        big = t.new_zeros((t.shape[0] + 1,) + tuple(t.shape[1:]))
        big[1:] = t
        return big[1:]
    if kind == 'offset1':               # dense and is_contiguous(), but only element-aligned
        flat = t.new_zeros(t.numel() + 1)
        flat[1:] = t.reshape(-1)
        return flat[1:].view(t.shape)
    raise ValueError(kind)


def applicable(kind, ndim):
    return ndim >= {'transposed': 2, 'channels_last': 4}.get(kind, 1) and (kind != 'channels_last' or ndim == 4)


def test_relayout_changes_layout_not_values():
    t = torch.arange(2 * 3 * 5 * 7, dtype=torch.float32, device=DEV).view(2, 3, 5, 7)
    for kind in KINDS:
        v = relayout(t, kind)
        assert torch.equal(v, t) and v.shape == t.shape
        assert not v.is_contiguous() or v.data_ptr() % 16 or kind == 'batch_view', kind
    assert relayout(t, 'offset1').is_contiguous() and relayout(t, 'offset1').data_ptr() % 16 == 4
    assert relayout(t.half(), 'offset1').data_ptr() % 16 == 2


# -------------------------------------------------------------------------------------------------------------- cases
def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(gen, *shape, dtype=F32):
    return torch.randn(*shape, generator=gen).to(dtype)


def _to_dev(x):
    if torch.is_tensor(x):
        return x.to(DEV)
    if isinstance(x, list) and x and torch.is_tensor(x[0]):
        return [t.to(DEV) for t in x]
    return x


class Case:
    """build(shape) -> dict of CPU inputs; prep(dict on the device) adds canonical derived inputs (trees, orders);
    fwd(dict) -> tuple of output tensors, the first ``n_diff`` differentiable with respect to the ``grad`` arguments;
    perturb: argument -> ndim; tol: argument -> (rtol, atol, reason), the explicit exceptions to bit equality."""

    def __init__(self, build, fwd, perturb, grad=(), n_diff=1, prep=None, shapes=('tiny', 'vec'), tol=None):
        self.build, self.fwd, self.perturb, self.grad, self.n_diff = build, fwd, perturb, tuple(grad), n_diff
        self.prep, self.shapes, self.tol = prep, shapes, tol or {}

    def inputs(self, shape):
        a = {k: _to_dev(v) for k, v in self.build(shape).items()}
        if self.prep is not None:
            self.prep(a)
        return a


CASES = {}


# ---- ops.dynconv
def _dynconv_build(dt):
    def build(shape):
        B, C, h, w, I = (2, 32, 3, 4, 5) if shape == 'tiny' else (2, 64, 8, 16, 40)     # vec: inside the 16-bit envelope
        g = _gen(11)
        return dict(feat=_randn(g, B, C, h, w, dtype=dt), kernels=_randn(g, B, I, C, dtype=dt))
    return build


def _dynconv_fwd(a):
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    return (dynconv1x1(a['feat'], a['kernels']),)


for _name, _dt in (('f32', F32), ('f16', F16), ('bf16', BF16)):
    CASES['dynconv1x1_' + _name] = Case(_dynconv_build(_dt), _dynconv_fwd, dict(feat=4, kernels=3), grad=('feat', 'kernels'))


def _solo_dynconv_build(shape):
    B, C, h, w, S = (2, 32, 4, 6, 3) if shape == 'tiny' else (2, 64, 8, 16, 6)
    g = _gen(12)
    return dict(feature_pred=_randn(g, B, C, h, w), kernel_pred=_randn(g, B, C, S, S))


def _solo_dynconv_fwd(a):
    from boxinstseg_b200.ops.dynconv import solo_dynamic_conv
    return (solo_dynamic_conv(a['feature_pred'], a['kernel_pred']),)


CASES['solo_dynamic_conv'] = Case(_solo_dynconv_build, _solo_dynconv_fwd, dict(feature_pred=4, kernel_pred=4),
                                  grad=('feature_pred', 'kernel_pred'))


def _mask_pred_build(shape):
    B, Q, C, h, w = (2, 5, 32, 4, 6) if shape == 'tiny' else (2, 40, 64, 8, 16)
    g = _gen(13)
    return dict(mask_embed=_randn(g, B, Q, C), mask_feature=_randn(g, B, C, h, w))


def _mask_pred_fwd(a):
    from boxinstseg_b200.ops.dynconv import box2mask_mask_pred
    return (box2mask_mask_pred(a['mask_embed'], a['mask_feature']),)


CASES['box2mask_mask_pred'] = Case(_mask_pred_build, _mask_pred_fwd, dict(mask_embed=3, mask_feature=4),
                                   grad=('mask_embed', 'mask_feature'))


def _cells_build(shape):
    g = _gen(14)
    if shape == 'tiny':
        return dict(feat=_randn(g, 2, 32, 8, 12), k0=_randn(g, 2, 32, 3, 3), k1=_randn(g, 2, 32, 2, 2),
                    cells=[[[0, 4, 8], [2]], [[1], [0, 3]]], sizes=[(8, 12), (4, 6)])
    return dict(feat=_randn(g, 2, 64, 16, 32), k0=_randn(g, 2, 64, 6, 6), k1=_randn(g, 2, 64, 4, 4),
                cells=[[list(range(0, 36, 2)), list(range(1, 36, 3))], [[0, 5, 10, 15], [3, 7]]], sizes=[(16, 32), (8, 16)])


def _cells_fwd(a):
    from boxinstseg_b200.ops.dynconv import solo_cells_conv
    cells = [[torch.tensor(c, dtype=torch.int64) for c in lvl] for lvl in a['cells']]
    return tuple(solo_cells_conv(a['feat'], [a['k0'], a['k1']], cells, a['sizes']))


CASES['solo_cells_conv'] = Case(_cells_build, _cells_fwd, dict(feat=4, k0=4, k1=4), grad=('feat', 'k0', 'k1'), n_diff=2)


# ---- ops.condinst / ops.resize / ops.box2mask
def _head_build(shape):
    B, C, h, w, N = (2, 8, 9, 11, 5) if shape == 'tiny' else (2, 16, 16, 32, 9)
    g = _gen(15)
    return dict(feat=_randn(g, B, C, h, w), params=_randn(g, N, (C + 2) * 8 + 64 + 8 + 8 + 8 + 1) * 0.3,
                coors=torch.rand(N, 2, generator=g) * torch.tensor([w * 8.0, h * 8.0]),
                level_inds=torch.randint(0, 5, (N,), generator=g), img_inds=torch.arange(N) * B // N,
                soi=torch.tensor([64., 128., 256., 512., 1024.]))


def _head_fwd(a):
    from boxinstseg_b200.ops.condinst import dynamic_mask_head
    return (dynamic_mask_head(a['feat'], a['params'], a['coors'], a['level_inds'], a['img_inds'], a['soi']),)


CASES['dynamic_mask_head'] = Case(_head_build, _head_fwd, dict(feat=4, params=2, coors=2, level_inds=1, img_inds=1, soi=1),
                                  grad=('feat', 'params'))


def _resize_build(shape):
    return dict(x=_randn(_gen(16), 2, 3, 9, 11), size=(13, 7)) if shape == 'tiny' else \
        dict(x=_randn(_gen(16), 2, 4, 16, 32), size=(32, 64))


def _resize_fwd(a):
    from boxinstseg_b200.ops.resize import bilinear_resize
    return (bilinear_resize(a['x'], a['size']),)


CASES['bilinear_resize'] = Case(_resize_build, _resize_fwd, dict(x=4), grad=('x',))


def _attn_build(dt):
    def build(shape):
        if shape == 'tiny':
            return dict(mask_pred=_randn(_gen(17), 2, 5, 9, 11, dtype=dt), size=(4, 6))
        return dict(mask_pred=_randn(_gen(17), 2, 8, 16, 16, dtype=dt), size=(8, 8))        # h*w % 16 == 0: 16-byte stores
    return build


def _attn_fwd(a):
    from boxinstseg_b200.ops.box2mask import attention_mask
    return (attention_mask(a['mask_pred'], a['size'], 2, reset_full_rows=True),)


for _name, _dt in (('f32', F32), ('f16', F16), ('bf16', BF16)):
    CASES['attention_mask_' + _name] = Case(_attn_build(_dt), _attn_fwd, dict(mask_pred=4), n_diff=0)


# ---- ops.boxinst
def _boxinst_build(shape):
    hp, wp = (148, 212) if shape == 'tiny' else (128, 256)          # loss grid 37x53 / 32x64
    return boxinst_case(3, 2, hp, wp, 2, 2)


def _boxinst_targets(a):
    from boxinstseg_b200.ops.boxinst import boxinst_targets
    return boxinst_targets(a['img'], a['metas'], a['gt_bboxes'], want_similarity=True)


def _boxinst_targets_fwd(a):
    t = _boxinst_targets(a)
    return (t.edge_bits, t.similarity, t.rects, t.gt_img, t.lab, t.valid, torch.cat(t.bitmasks()))


CASES['boxinst_targets'] = Case(_boxinst_build, _boxinst_targets_fwd, dict(img=4), n_diff=0)


def _boxinst_loss_fwd(planned):
    def fwd(a):
        from boxinstseg_b200.ops.boxinst import boxinst_loss_plan, boxinst_mask_loss
        t = _boxinst_targets(a)
        H, W = a['logits'].shape[-2:]
        plan = boxinst_loss_plan(t, a['gt_inds'], H, W) if planned else None
        return boxinst_mask_loss(a['logits'], t, a['gt_inds'], torch.tensor([5000.], device=DEV), plan=plan)
    return fwd


# with a gradient wanted the 32x64 grid runs the single-pass schedule, the 37x53 grid and every call without a gradient
# the two-call schedule
CASES['boxinst_mask_loss'] = Case(_boxinst_build, _boxinst_loss_fwd(False), dict(logits=4, gt_inds=1), grad=('logits',), n_diff=2)
CASES['boxinst_mask_loss_plan'] = Case(_boxinst_build, _boxinst_loss_fwd(True), dict(logits=4, gt_inds=1), grad=('logits',),
                                       n_diff=2)
CASES['boxinst_mask_loss_nograd'] = Case(_boxinst_build, _boxinst_loss_fwd(False), dict(logits=4), n_diff=0)


# ---- ops.pairwise
def _pairwise_build(shape):
    return dict(logits=_randn(_gen(18), 2, 1, 9, 11) if shape == 'tiny' else _randn(_gen(18), 2, 1, 32, 64))


def _pairwise_fwd(a):
    from boxinstseg_b200.ops.pairwise import pairwise_nlog
    return (pairwise_nlog(a['logits'], 3, 2),)


CASES['pairwise_nlog'] = Case(_pairwise_build, _pairwise_fwd, dict(logits=4), grad=('logits',))


# ---- ops.tree_filter
def _tree_build(shape):
    h, w = (9, 11) if shape == 'tiny' else (32, 48)
    g = _gen(19)
    return dict(guide=_randn(g, 2, 3, h, w), feature=_randn(g, 2, 4, h, w), embed=_randn(g, 2, 3, h, w) * 0.1,
                feature3=_randn(g, 3, 4, h, w), tree_of=torch.tensor([0, 1, 1], dtype=torch.int32),
                weight=torch.rand(2, h * w, generator=g), flat=_randn(g, 2, 4, h * w), g_out=_randn(g, 2, 4, h * w))


def _mst(guide):
    from boxinstseg_b200.ops.tree_filter.modules.tree_filter import MinimumSpanningTree, TreeFilter2D
    return MinimumSpanningTree(TreeFilter2D.norm2_distance)(guide)


def _tree_prep(a):
    from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as C
    a['tree'] = _mst(a['guide'])
    a['index'], a['parent'], a['child'] = C.bfs_forward(a['tree'], 4)
    a['out'], a['aggr'], a['aggr_up'], a['wsum'], a['wsum_up'] = C.refine_forward(a['flat'], a['weight'], a['index'], a['parent'],
                                                                                  a['child'])


def _bfs_fwd(a):
    from boxinstseg_b200.ops.tree_filter.functions.bfs import bfs
    return tuple(bfs(a['tree'], 4, 7))


def _filter_fwd(low_tree, shared):
    def fwd(a):
        from boxinstseg_b200.ops.tree_filter.modules.tree_filter import TreeFilter2D
        if shared:
            return (TreeFilter2D()(a['feature3'], a['embed'], a['tree'], low_tree, tree_of=a['tree_of']),)
        return (TreeFilter2D()(a['feature'], a['embed'], a['tree'], low_tree),)
    return fwd


def _refine(which):
    def fwd(a):
        from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as C
        order = (a['flat'], a['weight'], a['index'], a['parent'], a['child'])
        if which == 'forward':
            return tuple(C.refine_forward(*order))
        saved = (a['out'], a['aggr'], a['aggr_up'], a['wsum'], a['wsum_up'], a['g_out'])
        return (getattr(C, 'refine_backward_' + which)(*order, *saved),)
    return fwd


CASES['mst'] = Case(_tree_build, lambda a: (_mst(a['guide']),), dict(guide=4), n_diff=0)
CASES['bfs'] = Case(_tree_build, _bfs_fwd, dict(tree=3), n_diff=0, prep=_tree_prep)
CASES['tree_filter_low'] = Case(_tree_build, _filter_fwd(True, False), dict(feature=4, embed=4, tree=3),
                                grad=('feature', 'embed'), prep=_tree_prep)
CASES['tree_filter_high'] = Case(_tree_build, _filter_fwd(False, False), dict(feature=4, embed=4, tree=3),
                                 grad=('feature', 'embed'), prep=_tree_prep)
CASES['tree_filter_tree_of'] = Case(_tree_build, _filter_fwd(False, True), dict(feature3=4, embed=4, tree=3, tree_of=1),
                                    grad=('feature3', 'embed'), prep=_tree_prep)
# a sorted_index the caller rebuilt is no longer the tensor bfs_forward returned, so the wrapper re-derives the level order
# of the same tree from (index, parent): same root, same order, same bits
CASES['refine_forward'] = Case(_tree_build, _refine('forward'), dict(flat=3, weight=2, index=2, parent=2, child=3), n_diff=0,
                               prep=_tree_prep)
CASES['refine_backward_feature'] = Case(_tree_build, _refine('feature'),
                                        dict(weight=2, index=2, parent=2, child=3, wsum=2, g_out=3), n_diff=0, prep=_tree_prep)
CASES['refine_backward_weight'] = Case(_tree_build, _refine('weight'),
                                       dict(weight=2, index=2, child=3, out=3, aggr=3, aggr_up=3, wsum=2, wsum_up=2, g_out=3),
                                       n_diff=0, prep=_tree_prep)


# ---- models.losses
def _loss_build(shape):
    n, h, w = (3, 9, 11) if shape == 'tiny' else (4, 32, 64)
    g = _gen(20)
    box = torch.zeros(n, 1, h, w)
    for i in range(n):
        box[i, 0, 1 + i:h - 2, 2:w - 1 - i] = 1
    return dict(scores=torch.sigmoid(_randn(g, n, 1, h, w)), box=box, scores2=torch.softmax(_randn(g, n, 2, h, w), 1),
                targets=_randn(g, n, 4, h, w), pixel_num=box.sum((1, 2, 3)), logits=_randn(g, n, h, w),
                imgs=torch.rand(n, 3, h, w, generator=g), phis=torch.sigmoid(_randn(g, n, 1, h, w)))


def _losses():
    from boxinstseg_b200.models import losses
    from boxinstseg_b200.models.losses import box_projection_loss, levelset_loss
    return losses, box_projection_loss, levelset_loss


def _projection_fwd(a):
    _, bp, _ = _losses()
    return (bp.BoxProjectionLoss(2.0)(a['scores'], a['box']), bp.mil_loss(None, a['scores'], None, a['box']))


def _levelset_fwd(a):
    ls = _losses()[2]
    return (ls.LevelsetLoss(0.5)(a['scores2'], a['targets'], a['pixel_num']), ls.region_levelset()(a['scores2'], a['targets']))


def _assembly_fwd(a):
    return (_losses()[2].levelset_assembly(a['logits'], a['box'], a['targets'], 0.5),)


def _length_fwd(a):
    return (_losses()[2].length_regularization()(a['scores2']),)


def _lcm_fwd(a):
    ls = _losses()[2]
    return (ls.LCM(a['imgs'], a['phis'], a['box']), ls.LocalConsistencyModule([2], 10)(a['imgs'], a['phis']))


CASES['projection_losses'] = Case(_loss_build, _projection_fwd, dict(scores=4, box=4), grad=('scores',), n_diff=2)
CASES['levelset_loss'] = Case(_loss_build, _levelset_fwd, dict(scores2=4, targets=4, pixel_num=1), grad=('scores2', 'targets'),
                              n_diff=2)
CASES['levelset_assembly'] = Case(_loss_build, _assembly_fwd, dict(logits=3, box=4, targets=4), grad=('logits', 'targets'))
CASES['length_regularization'] = Case(_loss_build, _length_fwd, dict(scores2=4), grad=('scores2',))
CASES['lcm'] = Case(_loss_build, _lcm_fwd, dict(imgs=4, phis=4, box=4), grad=('phis',))


# ---- models.dense_heads.MeanField / ops.discobox
def _mf_build(shape):
    n, h, w = (4, 9, 11) if shape == 'tiny' else (4, 16, 32)
    g = _gen(21)
    tg = torch.zeros(n, 1, h, w)
    for i in range(n):
        tg[i, 0, 1 + i % 3:h - 2, 2:w - 2 - i % 3] = 1
    return dict(color=_randn(g, 2, 3, h, w), x=torch.rand(n, 1, h, w, generator=g), targets=tg,
                inter=torch.rand(n, 2, h, w, generator=g), obj_img=torch.tensor([0, 1, 0, 1], dtype=torch.int32),
                s16=_randn(g, n, h, w) * 3, t16=_randn(g, n, h, w) * 3, tg8=tg[:, 0].to(torch.uint8))


def _mean_field(color):
    from boxinstseg_b200.models.dense_heads.meanfield import MeanField
    return MeanField(color, alpha0=2.0, theta0=0.5, theta1=30.0, theta2=20.0, iter=10, kernel_size=3, base=0.1)


def _mf_fwd(inter):
    def fwd(a):
        mf = _mean_field(a['color'])
        ret, valid = mf(a['x'], a['targets'], a['inter'] if inter else None, obj_img=a['obj_img'])
        return mf.kernel, ret, valid
    return fwd


def _disco_fwd():
    def fwd(a):
        from boxinstseg_b200.ops.discobox import discobox_mask_loss
        return discobox_mask_loss(a['s16'], a['tg8'], a['obj_img'], a['mf'], a['t16'])
    return fwd


def _disco_build(dt):
    def build(shape):
        a = _mf_build(shape)
        a['s16'], a['t16'] = a['s16'].to(dt), a['t16'].to(dt)
        return a
    return build


def _disco_prep(a):
    a['mf'] = _mean_field(a['color'])


CASES['meanfield'] = Case(_mf_build, _mf_fwd(False), dict(color=4, x=4, targets=4, obj_img=1), n_diff=0)
CASES['meanfield_inter'] = Case(_mf_build, _mf_fwd(True), dict(x=4, targets=4, inter=4), n_diff=0)
for _name, _dt in (('f16', F16), ('bf16', BF16)):
    CASES['discobox_mask_loss_' + _name] = Case(_disco_build(_dt), _disco_fwd(), dict(s16=3, t16=3, tg8=3, obj_img=1),
                                                grad=('s16',), n_diff=2, prep=_disco_prep)


# ---- ops.focal / ops.cross_entropy / ops.lsap
def _focal_build(shape):
    B, C, S0, S1 = (2, 3, 5, 3) if shape == 'tiny' else (2, 16, 12, 8)
    g = _gen(22)
    return dict(p0=_randn(g, B, C, S0, S0), p1=_randn(g, B, C, S1, S1), l0=torch.randint(0, C + 1, (B, S0, S0), generator=g),
                l1=torch.randint(0, C + 1, (B, S1, S1), generator=g), avg=torch.tensor(7.0))


def _focal_fwd(a):
    from boxinstseg_b200.ops.focal import sigmoid_focal_loss_levels
    return (sigmoid_focal_loss_levels([a['p0'], a['p1']], [a['l0'], a['l1']], a['avg']),)


CASES['sigmoid_focal_loss_levels'] = Case(_focal_build, _focal_fwd, dict(p0=4, p1=4, l0=3, l1=3), grad=('p0', 'p1'))


def _ce_build(shape):
    B, Q, K = (2, 7, 5) if shape == 'tiny' else (2, 100, 81)
    g = _gen(23)
    return dict(s0=_randn(g, B, Q, K), s1=_randn(g, B, Q, K), labels=torch.randint(0, K, (2, B, Q), generator=g),
                cw=torch.cat([torch.ones(K - 1), torch.tensor([0.1])]))


def _ce_fwd(as_list):
    def fwd(a):
        from boxinstseg_b200.ops.cross_entropy import softmax_cross_entropy_layers
        labels = [a['labels'][0], a['labels'][1]] if as_list else a['labels']
        return (softmax_cross_entropy_layers([a['s0'], a['s1']], labels, a['cw'], 2.0),)
    return fwd


CASES['softmax_cross_entropy_layers'] = Case(_ce_build, _ce_fwd(False), dict(s0=3, s1=3, labels=3, cw=1), grad=('s0', 's1'))
CASES['softmax_cross_entropy_layers_list'] = Case(_ce_build, _ce_fwd(True), dict(labels=3), grad=('s0', 's1'), shapes=('tiny',))


def _lsap_build(shape):
    return dict(cost=_randn(_gen(24), 7, 5) if shape == 'tiny' else _randn(_gen(24), 40, 100))


def _lsap_fwd(a):
    from boxinstseg_b200.ops.lsap import linear_sum_assignment
    return linear_sum_assignment(a['cost'])


CASES['lsap'] = Case(_lsap_build, _lsap_fwd, dict(cost=2), n_diff=0)


# ------------------------------------------------------------------------------------------------------------- runner
def _upstream(outs, kind):
    """(what reaches backward, its canonical dense twin) for every differentiable output; None = call .sum()/.mean()."""
    gen = _gen(99)
    pairs = []
    for o in outs:
        if kind in ('sum', 'expanded'):
            dense = torch.full_like(o, 1.0 if kind == 'sum' else 0.5)
            view = None if kind == 'sum' else torch.full((), 0.5, dtype=o.dtype, device=o.device).expand(o.shape)
        elif kind == 'mean':
            dense, view = torch.full_like(o, 1.0) / o.numel(), None
        else:
            dense = torch.randn(o.shape, generator=gen).to(device=o.device, dtype=o.dtype)
            k = kind if kind is None or applicable(kind, o.dim()) else 'offset1'     # 0-/1-D losses: the kinds that exist
            view = dense if k is None else relayout(dense.reshape(1) if o.dim() == 0 else dense, k).view(o.shape)
        pairs.append((view, dense))
    return pairs


def _run(case, a, g_kind=None, canonical=True):
    leaves = {k: a[k].detach().requires_grad_(True) for k in case.grad}       # detach keeps the view's layout
    outs = tuple(case.fwd({**a, **leaves}))
    for o in outs:
        assert o.is_contiguous(), 'outputs are dense'
    grads = ()
    if leaves:
        diff = outs[:case.n_diff]
        pairs = _upstream(diff, g_kind)
        if canonical or g_kind not in ('sum', 'mean'):
            gs = [dense if canonical else view for view, dense in pairs]
            grads = torch.autograd.grad(diff, list(leaves.values()), gs, allow_unused=True)
        else:
            total = sum(o.sum() if g_kind == 'sum' else o.mean() for o in diff)
            grads = torch.autograd.grad(total, list(leaves.values()), allow_unused=True)
        for g, leaf in zip(grads, leaves.values()):
            assert g is None or g.shape == leaf.shape, 'a gradient has its input\'s shape'
    return [o.detach() for o in outs], grads


def _same(got, want, tol, what):
    assert (got is None) == (want is None), what
    if got is None:
        return
    assert got.shape == want.shape and got.dtype == want.dtype, what
    got, want = got.contiguous(), want.contiguous()
    if tol is None:
        assert torch.equal(got, want), f'{what}: {(got.double() - want.double()).abs().max().item():.3g} max abs difference'
    else:
        torch.testing.assert_close(got, want, rtol=tol[0], atol=tol[1], msg=lambda m: f'{what}: {m}')


def _compare(case, arg, ref, got):
    tol = case.tol.get(arg)
    for i, (r, g) in enumerate(zip(ref[0], got[0])):
        _same(g, r, tol, f'output {i}')
    assert len(ref[1]) == len(got[1])
    for name, r, g in zip(case.grad, ref[1], got[1]):
        _same(g, r, tol, f'd/d {name}')


_INPUT_PARAMS = [pytest.param(name, shape, arg, kind, id=f'{name}.{shape}-{arg}-{kind}')
                 for name, case in CASES.items() for shape in case.shapes for arg, ndim in case.perturb.items()
                 for kind in KINDS if applicable(kind, ndim)]


@pytest.mark.parametrize('name,shape,arg,kind', _INPUT_PARAMS)
def test_input_layout(name, shape, arg, kind):
    case = CASES[name]
    a = case.inputs(shape)
    ref = _run(case, a)
    view = relayout(a[arg], kind)
    keep = view.clone()
    if arg in ('index',):           # the level table is remembered for the tensor bfs_forward returned; a rebuilt one has none
        from boxinstseg_b200.ops.tree_filter import tree_filter_cuda as C
        assert C._recall(view) is None
    got = _run(case, {**a, arg: view})
    _compare(case, arg, ref, got)
    assert torch.equal(view, keep), 'the input is left as it was'


_UPSTREAM_PARAMS = [pytest.param(name, shape, kind, id=f'{name}.{shape}-g_out-{kind}')
                    for name, case in CASES.items() if case.grad for shape in case.shapes for kind in G_KINDS]


@pytest.mark.parametrize('name,shape,kind', _UPSTREAM_PARAMS)
def test_upstream_gradient_layout(name, shape, kind):
    case = CASES[name]
    a = case.inputs(shape)
    ref = _run(case, a, kind, canonical=True)
    got = _run(case, a, kind, canonical=False)
    _compare(case, 'g_out', ref, got)


# ---- the entry points that keep the reference's CHECK_INPUT: they refuse what the autograd-level op accepts
@pytest.mark.parametrize('kind', ['transposed', 'sliced'])
def test_pairwise_ext_refuses_strided_like_the_reference(kind):
    from boxinstseg_b200.ops.pairwise import pairwise_ext, pairwise_nlog
    x = relayout(_pairwise_build('tiny')['logits'].to(DEV), kind)
    assert not x.is_contiguous()
    with pytest.raises(RuntimeError, match='must be contiguous'):
        pairwise_ext.pairwise_nlog_forward(3, 2, x)
    out = pairwise_ext.pairwise_nlog_forward(3, 2, x.contiguous())
    with pytest.raises(RuntimeError, match='must be contiguous'):
        pairwise_ext.pairwise_nlog_backward(3, 2, x.contiguous(), out, relayout(out, kind))
    with pytest.raises(RuntimeError, match='must be a CUDA tensor'):
        pairwise_ext.pairwise_nlog_forward(3, 2, x.cpu().contiguous())
    assert torch.equal(pairwise_nlog(x, 3, 2), out)


def test_solo_cells_backward_routes_by_kernels_per_image():
    """d/d operand goes through cuBLAS exactly when an image holds more than 256 kernels of one operand (``dynconv1x1``
    decides from the shapes); an operand or upstream gradient the kernel cannot take as it is gets an aligned copy instead
    of being mistaken for that."""
    from boxinstseg_b200.ops import dynconv
    g = _gen(31)
    feat, k = _randn(g, 1, 32, 8, 8).to(DEV), _randn(g, 1, 32, 18, 18).to(DEV)
    cells = [[torch.arange(300)]]

    def grads(f, kk, g_view):
        f, kk = f.detach().requires_grad_(True), kk.detach().requires_grad_(True)
        (out,) = dynconv.solo_cells_conv(f, [kk], cells, [(8, 8)])
        return (out.detach(),) + torch.autograd.grad(out, [f, kk], g_view)

    g_out = _randn(g, 300, 8, 8).to(DEV)
    ref = grads(feat, k, g_out)
    f64 = torch.einsum('nc,chw->nhw', k[0].reshape(32, -1)[:, :300].t().double(), feat[0].double())
    torch.testing.assert_close(ref[0].double(), f64, rtol=2e-3, atol=2e-2)                 # TF32 operands
    gf64 = torch.einsum('nc,nhw->chw', k[0].reshape(32, -1)[:, :300].t().double(), g_out.double())
    torch.testing.assert_close(ref[1][0].double(), gf64, rtol=1e-4, atol=1e-3)             # the cuBLAS route, FP32
    for got in (grads(relayout(feat, 'offset1'), k, g_out), grads(feat, k, relayout(g_out, 'offset1'))):
        for r, x in zip(ref, got):
            assert torch.equal(r, x)


# ---------------------------------------------------------------------------------------------------------- zero size
# Covered elsewhere, not repeated: discobox_mask_loss (test_discobox_half_gpu), solo_cells_conv (test_solo_cells_gpu),
# the LSAP (test_lsap_gpu), the BoxInst loss and pairwise_nlog with no instance (test_boxinst_gpu).
def _zero_dynconv(dt):
    from boxinstseg_b200.ops.dynconv import dynconv1x1
    for B, I in ((2, 0), (0, 3)):
        f = torch.randn(B, 32, 4, 8, device=DEV, dtype=dt, requires_grad=True)
        k = torch.randn(B, I, 32, device=DEV, dtype=dt, requires_grad=True)
        out = dynconv1x1(f, k)
        assert out.shape == (B, I, 4, 8) and out.dtype == dt
        gf, gk = torch.autograd.grad(out.sum(), [f, k])
        assert gf.shape == f.shape and gk.shape == k.shape and not gf.any() and not gk.any()


def _zero_head():
    a = {k: _to_dev(v) for k, v in _head_build('tiny').items()}
    a.update(params=a['params'][:0], coors=a['coors'][:0], level_inds=a['level_inds'][:0], img_inds=a['img_inds'][:0])
    f, p = a['feat'].requires_grad_(True), a['params'].requires_grad_(True)
    (out,) = _head_fwd(a)
    assert out.shape == (0, 1, 18, 22) and out.dtype == F32
    gf, gp = torch.autograd.grad(out.sum(), [f, p])
    assert gf.shape == f.shape and not gf.any() and gp.shape == p.shape


def _zero_resize():
    from boxinstseg_b200.ops.resize import bilinear_resize
    x = torch.randn(0, 3, 9, 11, device=DEV, requires_grad=True)
    out = bilinear_resize(x, (13, 7))
    assert out.shape == (0, 3, 13, 7)
    assert torch.autograd.grad(out.sum(), x)[0].shape == x.shape


def _zero_attention():
    from boxinstseg_b200.ops.box2mask import attention_mask
    for B, Q in ((0, 5), (2, 0)):
        out = attention_mask(torch.randn(B, Q, 9, 11, device=DEV), (4, 6), 2, True)
        assert out.shape == (B * 2, Q, 24) and out.dtype == torch.bool


def _zero_losses():
    _, bp, ls = _losses()
    z = lambda *s: torch.zeros(*s, device=DEV, requires_grad=True)       # noqa: E731
    for fn, args in ((bp.projection_losses, (z(0, 1, 9, 11), z(0, 1, 9, 11))),
                     (ls.LevelsetLoss(), (z(0, 2, 9, 11), z(0, 4, 9, 11), z(0))),
                     (ls.levelset_assembly, (z(0, 9, 11), z(0, 9, 11), z(0, 4, 9, 11))),
                     (ls.length_regularization(), (z(0, 2, 9, 11),))):
        loss = fn(*args)
        assert loss.shape == (0,) and loss.dtype == F32
        assert torch.autograd.grad(loss.sum(), args[0])[0].shape == args[0].shape
    phis = z(0, 1, 9, 11)
    loss = ls.LCM(z(0, 3, 9, 11), phis, z(0, 1, 9, 11))
    assert loss.shape == () and loss.item() == 0.0
    assert torch.autograd.grad(loss, phis)[0].shape == phis.shape
    assert ls.LocalConsistencyModule([2], 10)(z(0, 3, 9, 11), phis).shape == (0, 1, 9, 11)


def _zero_meanfield():
    mf = _mean_field(torch.randn(2, 3, 9, 11, device=DEV))
    ret, valid = mf(torch.zeros(0, 1, 9, 11, device=DEV), torch.zeros(0, 1, 9, 11, device=DEV),
                    obj_img=torch.zeros(0, dtype=torch.int32, device=DEV))
    assert ret.shape == (0, 1, 9, 11) and valid.shape == (0,)


_ZERO = dict(dynconv1x1_f32=lambda: _zero_dynconv(F32), dynconv1x1_f16=lambda: _zero_dynconv(F16), dynamic_mask_head=_zero_head,
             bilinear_resize=_zero_resize, attention_mask=_zero_attention, losses=_zero_losses, meanfield=_zero_meanfield)


@pytest.mark.parametrize('name', list(_ZERO))
def test_zero_size(name):
    _ZERO[name]()
