"""Restatement of Box2Mask's per-decoder-layer head (mmdet/models/dense_heads/box2mask_head.py:338-359) and of its decoder
loop (:361-419): the attention-mask lines (:346-355), the reset of the loop (:397) and the order in which the loop feeds
the masks to the decoder layers.  Plus seeded stand-in modules for the parts the reference builds from mmcv configs (pixel
decoder, transformer decoder, positional encoding), shared by oracle/make_golden_box2mask_attn.py and the tests.

Pinned against the reference's own ``forward_head`` / ``forward`` by oracle/make_golden_box2mask_attn.py."""
import torch
import torch.nn as nn
import torch.nn.functional as F


def attention_mask(mask_pred, size, num_heads):
    """:346-355 -- [B,Q,H,W] -> bool [B*num_heads, Q, h*w]: True where sigmoid(resized logit) < 0.5.  Every head of an image
    gets the same [Q, h*w] block."""
    B, Q = mask_pred.shape[:2]
    m = torch.sigmoid(F.interpolate(mask_pred, size, mode='bilinear', align_corners=False)) < 0.5
    return m.reshape(B, 1, Q, -1).expand(B, num_heads, Q, m.shape[-1] * m.shape[-2]).reshape(B * num_heads, Q, -1)


def reset_full_rows(attn_mask):
    """:397 -- a row that is all True (a query that would attend to nothing) becomes all False."""
    return attn_mask & ~attn_mask.all(-1, keepdim=True)


def forward_head(m, decoder_out, mask_feature, size):
    """:338-359 with the modules of ``m`` (post_norm, cls_embed, mask_embed, levelset_bottom, num_heads)."""
    x = m.transformer_decoder.post_norm(decoder_out).permute(1, 0, 2)
    mask_pred = (m.mask_embed(x).unsqueeze(-1).unsqueeze(-1) * mask_feature.unsqueeze(1)).sum(2)
    return m.cls_embed(x), mask_pred, attention_mask(mask_pred.detach(), size, m.num_heads), m.levelset_bottom(mask_feature)


def forward(m, feats, batch_size, head_fn=None):
    """:361-419 with the modules of ``m``; ``head_fn(decoder_out, mask_feature, size)`` (default: ``forward_head`` above) is
    the per-layer head.  Layer i (memory level i % levels) gets the mask of the head call before it with its full rows
    cleared.  Returns (the 4-tuples of the head calls, the masks the layers got, the queries they got)."""
    head_fn = head_fn or (lambda q, f, s: forward_head(m, q, f, s))
    mask_features, mems = m.pixel_decoder(feats)
    levels = m.num_transformer_feat_level
    keys, key_pos = [], []
    for i in range(levels):
        x = m.decoder_input_projs[i](mems[i]).flatten(2).permute(2, 0, 1) + m.level_embed.weight[i].view(1, 1, -1)
        pad = x.new_zeros((batch_size, ) + tuple(mems[i].shape[-2:]), dtype=torch.bool)
        keys.append(x)
        key_pos.append(m.decoder_positional_encoding(pad).flatten(2).permute(2, 0, 1))
    query = m.query_feat.weight.unsqueeze(1).repeat((1, batch_size, 1))
    query_pos = m.query_embed.weight.unsqueeze(1).repeat((1, batch_size, 1))
    outs, given, queries = [head_fn(query, mask_features, mems[0].shape[-2:])], [], []
    for i in range(m.num_transformer_decoder_layers):
        lvl = i % levels
        mask = reset_full_rows(outs[-1][2])
        given.append(mask)
        queries.append(query)
        query = m.transformer_decoder.layers[i](query=query, key=keys[lvl], value=keys[lvl], query_pos=query_pos,
                                                key_pos=key_pos[lvl], attn_masks=[mask, None])
        outs.append(head_fn(query, mask_features, mems[(i + 1) % levels].shape[-2:]))
    return outs, given, queries


# ------------------------------------------------------------------------------------------------------------------------
# seeded stand-ins for what the reference builds from mmcv configs.  Weights come from torch.Generator draws (not from
# nn.init), so they do not depend on the torch version's initialisers.
# ------------------------------------------------------------------------------------------------------------------------
def _fill(module, gen, scale):
    with torch.no_grad():
        for p in module.parameters():
            p.copy_(torch.randn(p.shape, generator=gen) * scale)
    return module


class PlantedMLP(nn.Module):
    """The 3-layer mask_embed MLP (Linear, ReLU, Linear, ReLU, Linear; :86-90) plus a fixed per-query offset, so that chosen
    queries produce chosen rows whatever the decoder does to them (with the constant channel 0 and the spike channel 1 of
    the stand-in mask features: query 0 all True, query 1 all False, query 2 all True but one pixel)."""

    def __init__(self, C, Q, gen):
        super().__init__()
        self.mlp = _fill(nn.Sequential(nn.Linear(C, C), nn.ReLU(inplace=True), nn.Linear(C, C), nn.ReLU(inplace=True),
                                       nn.Linear(C, C)), gen, C ** -0.5)
        plant = torch.zeros(Q, C)
        plant[0, 0], plant[1, 0], plant[2, 0], plant[2, 1] = -60.0, 60.0, -30.0, 400.0
        self.register_buffer('plant', plant)

    def forward(self, x):
        return self.mlp(x) + self.plant


class PixelDecoder(nn.Module):
    """feats [B,C,S,S] -> (mask_features [B,C,Hf,Wf], memories at `sizes`): channel 0 of the mask features is 1, channel 1 a
    unit spike at (1, 1), the others a small function of the input.  The memories are plain resizes of the input."""

    def __init__(self, C, feat_size, sizes, gen):
        super().__init__()
        self.proj = _fill(nn.Conv2d(C, C, 1), gen, C ** -0.5)
        self.feat_size, self.sizes = feat_size, sizes

    def forward(self, feats):
        x = feats[-1]
        f = 0.3 * torch.tanh(self.proj(F.interpolate(x, self.feat_size, mode='bilinear', align_corners=False)))
        f = torch.cat([torch.ones_like(f[:, :1]), torch.zeros_like(f[:, :1]), f[:, 2:]], 1)
        f[:, 1, 1, 1] = 1.0
        return f, [F.interpolate(x, s, mode='bilinear', align_corners=False) for s in self.sizes]


class PositionalEncoding(nn.Module):
    """mask [B,h,w] bool -> [B,C,h,w], a fixed function of the position (the reference's SinePositionalEncoding's role)."""

    def __init__(self, C):
        super().__init__()
        self.C = C

    def forward(self, mask):
        B, h, w = mask.shape
        y = torch.arange(h, device=mask.device, dtype=torch.float32).view(1, 1, h, 1)
        x = torch.arange(w, device=mask.device, dtype=torch.float32).view(1, 1, 1, w)
        k = torch.arange(self.C, device=mask.device, dtype=torch.float32).view(1, -1, 1, 1)
        return torch.sin(0.3 * (k + 1) * y / h + 0.7 * x / w + k).expand(B, self.C, h, w) * (~mask).unsqueeze(1)


class DecoderLayer(nn.Module):
    """A cross-attention stand-in that is a deterministic function of the query and of the mask it receives: every query
    moves by the mean over the heads of the keys its mask allows (all keys for an all-False row, none for an all-True one),
    so a wrong mask changes the next query."""

    def __init__(self, C, num_heads, gen):
        super().__init__()
        self.lin = _fill(nn.Linear(C, C), gen, C ** -0.5)
        self.num_heads = num_heads

    def forward(self, query, key, value, query_pos, key_pos, attn_masks, query_key_padding_mask=None, key_padding_mask=None):
        mask = attn_masks[0]
        Q, B, C = query.shape
        allowed = (~mask).view(B, self.num_heads, Q, -1).float().mean(1)                    # [B,Q,hw]
        ctx = allowed @ (value + key_pos).permute(1, 0, 2) / allowed.shape[-1]              # [B,Q,C]
        return query + torch.tanh(self.lin(ctx.permute(1, 0, 2) + query + query_pos))


class Decoder(nn.Module):
    def __init__(self, C, num_heads, num_layers, gen):
        super().__init__()
        self.post_norm = _fill(nn.LayerNorm(C), gen, 0.5)
        self.layers = nn.ModuleList([DecoderLayer(C, num_heads, gen) for _ in range(num_layers)])


def standins(seed=0, C=32, Q=8, num_classes=4, num_heads=2, num_layers=4, feat_size=(16, 16),
             sizes=((4, 4), (8, 8), (5, 7))):
    """The attributes the reference constructor leaves on the head (:57-91), built from one seed, and the input of the
    pixel decoder for two images, ``feats = [tensor [2, C, 12, 12]]``.  Returns (attributes, feats)."""
    gen = torch.Generator().manual_seed(seed)
    attrs = dict(
        num_heads=num_heads, num_queries=Q, num_transformer_feat_level=len(sizes),
        num_transformer_decoder_layers=num_layers,
        pixel_decoder=PixelDecoder(C, feat_size, sizes, gen),
        transformer_decoder=Decoder(C, num_heads, num_layers, gen),
        decoder_input_projs=nn.ModuleList([nn.Identity() for _ in sizes]),
        decoder_positional_encoding=PositionalEncoding(C),
        level_embed=_fill(nn.Embedding(len(sizes), C), gen, 0.1),
        query_embed=_fill(nn.Embedding(Q, C), gen, 1.0),
        query_feat=_fill(nn.Embedding(Q, C), gen, 1.0),
        cls_embed=_fill(nn.Linear(C, num_classes + 1), gen, C ** -0.5),
        mask_embed=PlantedMLP(C, Q, gen),
        levelset_bottom=_fill(nn.Conv2d(C, 1, 3, padding=1), gen, 0.1),
    )
    feats = [torch.randn(2, C, 12, 12, generator=gen)]
    return attrs, feats


def attach(module, attrs):
    """Sets the stand-in attributes on ``module`` (an nn.Module: submodules are registered)."""
    for k, v in attrs.items():
        setattr(module, k, v)
    return module
