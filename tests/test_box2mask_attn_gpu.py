"""GPU: Box2Mask's attention mask (ops.box2mask.attention_mask, bxs_box2mask_attn_mask) and the head that uses it.

1. The kernel is bit-exact against the composition with the same arithmetic: bilinear_resize -> (16-bit: round to the
   dtype) -> torch.sigmoid -> < 0.5 -> repeat over the heads -> the reference's reset, on config E's shapes, odd and
   up-sampling ratios, 1x1 targets, Q = 1, heads = 1, planted special values and planted rows, in all three dtypes.
2. Against torch's own F.interpolate composition (the reference's lines on the GPU), a bit may differ only where the two
   interpolations differ (FMA contraction, see test_fused_assembly_gpu.py).
3. ``Box2MaskHead.forward_head`` on seeded stand-in modules against the restated reference lines, in float32 and under
   autocast(bfloat16).
4. ``Box2MaskHead.forward`` hands every decoder layer the mask of the oracle loop, without a host synchronisation, and
   replays from a CUDA graph bit-identically."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import box2mask_head as ob
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu
DTYPES = [torch.float32, torch.float16, torch.bfloat16]
DT_IDS = ['f32', 'f16', 'bf16']


def _repeat_reset(m, heads, reset):
    m = m.flatten(2).unsqueeze(1).repeat((1, heads, 1, 1)).flatten(0, 1)
    if reset:
        m[torch.where(m.sum(-1) == m.shape[-1])] = False
    return m


def _ours_interp(mp, size):
    from boxinstseg_b200.ops.resize import bilinear_resize
    r = bilinear_resize(mp.float(), size)
    return r if mp.dtype == torch.float32 else r.to(mp.dtype)


def composition(mp, size, heads, reset):
    """The kernel's arithmetic as torch ops: the product's bilinear resize (float32, rounded for 16-bit), torch.sigmoid in
    the input dtype, the compare, the repeat and the reference's reset (box2mask_head.py:346-355, :397)."""
    return _repeat_reset(torch.sigmoid(_ours_interp(mp, size)) < 0.5, heads, reset)


def torch_lines(mp, size, heads, reset):
    """box2mask_head.py:346-355 verbatim (F.interpolate), and :397."""
    m = F.interpolate(mp, size, mode='bilinear', align_corners=False)
    m = m.flatten(2).unsqueeze(1).repeat((1, heads, 1, 1)).flatten(0, 1)
    m = m.sigmoid() < 0.5
    if reset:
        m[torch.where(m.sum(-1) == m.shape[-1])] = False
    return m


def _attn(*a, **k):
    from boxinstseg_b200.ops.box2mask import attention_mask
    return attention_mask(*a, **k)


def _logits(B, Q, H, W, dt, seed, scale=3.0):
    gen = torch.Generator(device='cuda').manual_seed(seed)
    return (torch.randn(B, Q, H, W, generator=gen, device='cuda') * scale).to(dt)


SHAPES = [  # B, Q, H, W, h, w, heads
    (1, 100, 256, 256, 32, 32, 8), (1, 100, 256, 256, 64, 64, 8), (1, 100, 256, 256, 128, 128, 8),
    (2, 100, 256, 256, 32, 32, 8), (2, 100, 256, 256, 64, 64, 8), (2, 100, 256, 256, 128, 128, 8),
    (2, 5, 37, 53, 13, 20, 8), (1, 7, 8, 8, 16, 16, 8), (2, 9, 20, 24, 1, 1, 8), (1, 1, 64, 64, 32, 32, 8),
    (2, 6, 64, 64, 16, 16, 1), (1, 3, 1, 1, 5, 3, 2), (1, 4, 16, 16, 1, 17, 3), (1, 4, 16, 16, 17, 1, 3),
]


@pytest.mark.parametrize('dt', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('shape', SHAPES, ids=lambda s: 'x'.join(map(str, s)))
def test_kernel_bit_exact_against_same_arithmetic(shape, dt):
    B, Q, H, W, h, w, heads = shape
    mp = _logits(B, Q, H, W, dt, seed=B * 1000 + h)
    if Q >= 4:       # planted rows: all True, all False, all True but one source pixel (reaches the output's (0, 0))
        mp[:, 0] = -20.0
        mp[:, 1] = 20.0
        mp[:, 2] = -20.0
        mp[:, 2, 0, 0] = 1000.0
    for reset in (False, True):
        got = _attn(mp, (h, w), heads, reset_full_rows=reset)
        assert got.dtype == torch.bool and got.shape == (B * heads, Q, h * w)
        assert torch.equal(got, composition(mp, (h, w), heads, reset)), (shape, dt, reset)
    if Q >= 4:
        rows = got.view(B, heads, Q, h * w)
        assert not rows[:, :, 0].any() and not rows[:, :, 1].any()          # the all-True row was cleared
        assert not torch.equal(got, _attn(mp, (h, w), heads))


SPECIAL = [0.0, -0.0, 2.0 ** -24, -2.0 ** -24, 1e-8, -1e-8, 1e-30, -1e-30, 5.9e-8, -5.9e-8, 1e-7, -1e-7, 3e-4, -3e-4,
           float('inf'), float('-inf'), float('nan'), 88.0, -88.0, 104.0, -104.0]


@pytest.mark.parametrize('dt', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('size', [(12, 14), (6, 7), (5, 3), (24, 28)])
def test_special_values(size, dt):
    """Signed zeros, logits whose float32 sigmoid rounds to exactly 0.5, overflow of exp, +-inf and NaN: at the identity
    size each value passes the interpolation unchanged (where no inf / NaN neighbour enters with weight 0), at the others
    it is mixed with its neighbours."""
    gen = torch.Generator(device='cuda').manual_seed(7)
    vals = torch.tensor(SPECIAL, device='cuda')
    idx = torch.randint(0, len(SPECIAL), (2, 6, 12, 14), generator=gen, device='cuda')
    mp = vals[idx].to(dt)
    mp[:, 0] = -1e-8                 # a whole row whose float32 sigmoid is exactly 0.5: all False, though every logit is < 0
    for reset in (False, True):
        assert torch.equal(_attn(mp, size, 3, reset_full_rows=reset), composition(mp, size, 3, reset)), (size, dt, reset)


@pytest.mark.parametrize('dt', DTYPES, ids=DT_IDS)
@pytest.mark.parametrize('shape', [SHAPES[0], SHAPES[2], SHAPES[6], SHAPES[7], SHAPES[8]],
                         ids=lambda s: 'x'.join(map(str, s)))
def test_against_torch_interpolate(shape, dt):
    """Bits may differ from the reference's own lines only at pixels where F.interpolate and the product's resize differ."""
    B, Q, H, W, h, w, heads = shape
    mp = _logits(B, Q, H, W, dt, seed=11 + h, scale=0.02)           # small logits: many values near the threshold
    got = _attn(mp, (h, w), heads)
    ref = torch_lines(mp, (h, w), heads, False)
    bits = torch.int32 if dt == torch.float32 else torch.int16
    ours_v = _ours_interp(mp, (h, w)).flatten(2).view(bits)
    torch_v = F.interpolate(mp, (h, w), mode='bilinear', align_corners=False).flatten(2).view(bits)
    same_v = (ours_v == torch_v).unsqueeze(1).expand(B, heads, Q, h * w).reshape(B * heads, Q, h * w)
    assert not bool(((got != ref) & same_v).any()), 'a bit differs where the interpolated values agree'
    assert same_v.float().mean() > 0.5


# ------------------------------------------------------------------------------------------------------------------------
# the head
# ------------------------------------------------------------------------------------------------------------------------
def _head(seed=0, C=256, Q=100, heads=8, feat=(64, 64), sizes=((8, 8), (16, 16), (32, 32)), layers=6):
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import Box2MaskHead
    attrs, feats = ob.standins(seed, C=C, Q=Q, num_heads=heads, num_layers=layers, feat_size=feat, sizes=sizes)
    head = ob.attach(Box2MaskHead(num_queries=Q), attrs).cuda()
    return head, [f.cuda() for f in feats]


def _reference_head_lines(head, decoder_out, mask_feature):
    """box2mask_head.py:341-345, 357 with the head's modules (the attention lines are checked separately)."""
    x = head.transformer_decoder.post_norm(decoder_out).transpose(0, 1)
    mp = torch.einsum('bqc,bchw->bqhw', head.mask_embed(x), mask_feature)
    return head.cls_embed(x), mp, head.levelset_bottom(mask_feature)


@pytest.mark.parametrize('autocast', [False, True], ids=['f32', 'autocast_bf16'])
def test_forward_head_against_reference_lines(autocast):
    head, feats = _head()
    gen = torch.Generator(device='cuda').manual_seed(3)
    with torch.no_grad():
        mask_feature = head.pixel_decoder(feats)[0]
        decoder_out = torch.randn(100, 2, 256, generator=gen, device='cuda')
        for size in ((8, 8), (16, 16), (32, 32), (13, 20)):
            with torch.autocast('cuda', dtype=torch.bfloat16, enabled=autocast):
                cls_pred, mask_pred, attn, lst = head.forward_head(decoder_out, mask_feature, size)
                cls_ref, mp_ref, lst_ref = _reference_head_lines(head, decoder_out, mask_feature)
            assert cls_pred.dtype == cls_ref.dtype and mask_pred.dtype == mp_ref.dtype == lst.dtype == lst_ref.dtype
            assert torch.equal(cls_pred, cls_ref) and torch.equal(lst, lst_ref)
            assert rel_err(mask_pred.float(), mp_ref.float()) <= (8e-3 if autocast else 1e-3)
            assert torch.equal(attn, composition(mask_pred, size, 8, False))
            rows = attn.view(2, 8, 100, -1)
            assert rows[:, :, 0].all() and not rows[:, :, 1].any()                 # the planted rows


class _Recorder(nn.Module):
    def __init__(self, layer, sink):
        super().__init__()
        self.layer, self.sink = layer, sink

    def forward(self, query, attn_masks, **kw):
        self.sink.append((query.clone(), attn_masks[0].clone()))
        return self.layer(query=query, attn_masks=attn_masks, **kw)


def test_forward_matches_oracle_loop_sync_free_and_graph_replay():
    head, feats = _head(seed=1)
    sink = []
    layers = head.transformer_decoder.layers
    head.transformer_decoder.layers = nn.ModuleList([_Recorder(l, sink) for l in layers])
    metas = [dict(), dict()]
    with torch.no_grad():
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode('error')
        try:
            cls_l, mask_l, lst_l = head.forward(feats, metas)
        finally:
            torch.cuda.set_sync_debug_mode('default')
        given = [m for _, m in sink]
        head.transformer_decoder.layers = layers
        outs, o_given, _ = ob.forward(head, feats, 2, head_fn=head.forward_head)
    assert len(given) == len(o_given) == 6 and len(cls_l) == len(outs) == 7
    for g, o in zip(given, o_given):
        assert torch.equal(g, o)
        assert not g.view(2, 8, 100, -1)[:, :, 0].any()                    # the planted all-True query was cleared
    for a, b, c, o in zip(cls_l, mask_l, lst_l, outs):
        assert torch.equal(a, o[0]) and torch.equal(b, o[1]) and torch.equal(c, o[3])

    # CUDA graph: one eager call has run; capture, replay, compare bit for bit
    head.transformer_decoder.layers = nn.ModuleList([_Recorder(l, sink) for l in layers])
    static = [f.clone() for f in feats]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(s):
        head.forward(static, metas)                                          # warm-up on the capture stream
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    sink.clear()
    with torch.no_grad(), torch.cuda.graph(graph):
        g_cls, g_mask, g_lst = head.forward(static, metas)
    g_given = [m for _, m in sink]
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(g_given, given):
        assert torch.equal(a, b)
    for a, b in zip(g_cls + g_mask + g_lst, cls_l + mask_l + lst_l):
        assert torch.equal(a, b)
