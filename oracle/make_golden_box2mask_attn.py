"""Golden vectors for Box2Mask's attention mask and decoder loop, minted from the REFERENCE's own methods (authoring container
only): ``Box2MaskHead.forward_head`` and ``Box2MaskHead.forward`` are AST-extracted from
mmdet/models/dense_heads/box2mask_head.py, bound to a stand-in head carrying the seeded modules of oracle/box2mask_head.py
(LayerNorm post-norm, Linear classifier, 3-layer mask MLP with planted all-True / all-False / one-False queries, 3x3 conv,
stub pixel decoder, decoder layers that depend on the mask they get) and run on CPU.  Asserts that the oracle restatement
gives the reference's head outputs and hands every decoder layer the same mask, writes tests/golden/box2mask_attn.npz.
    python -m oracle.make_golden_box2mask_attn"""
import ast
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from oracle import box2mask_head as ob

REF = os.environ.get('BXS_REFERENCE', '/root/reference')
OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..', 'tests', 'golden', 'box2mask_attn.npz')
SEEDS = (0, 1)


def reference_head():
    src = open(os.path.join(REF, 'mmdet/models/dense_heads/box2mask_head.py')).read()
    cls = [n for n in ast.parse(src).body if isinstance(n, ast.ClassDef) and n.name == 'Box2MaskHead'][0]
    fns = [n for n in cls.body if isinstance(n, ast.FunctionDef) and n.name in ('forward_head', 'forward')]
    g = dict(torch=torch, F=F)
    exec(compile(ast.Module(body=fns, type_ignores=[]), 'box2mask_head.py', 'exec'), g)

    class RefHead(nn.Module):
        """The reference's two methods on the stand-in modules; records every head call and what each layer receives."""
        calls, given, queries = [], [], []

        def forward_head(self, decoder_out, mask_feature, size):
            out = g['forward_head'](self, decoder_out, mask_feature, size)
            self.calls.append((tuple(size), tuple(t.clone() for t in out)))     # forward clears rows of out[2] in place
            return out

        forward = g['forward']
    return RefHead


class Recorder(nn.Module):
    def __init__(self, layer, sink):
        super().__init__()
        self.layer, self.sink = layer, sink

    def forward(self, query, attn_masks, **kw):
        self.sink.given.append(attn_masks[0].clone())
        self.sink.queries.append(query)
        return self.layer(query=query, attn_masks=attn_masks, **kw)


def main():
    RefHead = reference_head()
    out = {}
    for seed in SEEDS:
        attrs, feats = ob.standins(seed)
        ref = ob.attach(RefHead(), attrs)
        ref.calls, ref.given, ref.queries = [], [], []
        layers = ref.transformer_decoder.layers
        ref.transformer_decoder.layers = nn.ModuleList([Recorder(l, ref) for l in layers])
        with torch.no_grad():
            cls_list, mask_list, lst_list = ref.forward(feats, [dict()] * feats[0].shape[0])
        ref.transformer_decoder.layers = layers
        with torch.no_grad():
            outs, given, queries = ob.forward(ref, feats, feats[0].shape[0])
        assert len(outs) == len(ref.calls) == len(cls_list) and len(given) == len(ref.given)
        for i, ((size, r), o) in enumerate(zip(ref.calls, outs)):
            assert torch.allclose(r[0], o[0], rtol=1e-5, atol=1e-5) and torch.allclose(r[1], o[1], rtol=1e-5, atol=1e-5)
            assert torch.equal(r[2], o[2]), 'oracle attention mask != reference'
            assert torch.equal(r[2], ob.attention_mask(r[1], size, ref.num_heads)), 'oracle attention lines != reference'
            assert torch.equal(r[3], o[3]) and torch.equal(r[0], cls_list[i]) and torch.equal(r[1], mask_list[i])
            rows = r[2].view(-1, ref.num_queries, r[2].shape[-1])
            assert rows[:, 0].all() and not rows[:, 1].any() and bool(((~rows[:, 2]).sum(-1) == 1).all())   # planted
            assert bool((rows[:, 3:].any(-1) & ~rows[:, 3:].all(-1)).any()), 'no mixed row'
            out[f's{seed}_size{i}'] = np.asarray(size, np.int64)
            out[f's{seed}_mask_pred{i}'] = r[1].numpy()
            out[f's{seed}_attn{i}'] = np.packbits(r[2].numpy(), axis=-1)
        for i, (rg, og, rq, oq) in enumerate(zip(ref.given, given, ref.queries, queries)):
            assert torch.equal(rg, og), 'oracle loop hands a layer another mask than the reference'
            assert torch.allclose(rq, oq, rtol=1e-5, atol=1e-5)
            assert not rg.view(-1, ref.num_queries, rg.shape[-1])[:, 0].any()          # the all-True query was cleared
            out[f's{seed}_given{i}'] = np.packbits(rg.numpy(), axis=-1)
        out[f's{seed}_heads'] = np.asarray(ref.num_heads)
    np.savez_compressed(OUT, **out)
    print('oracle == reference on', len(out), 'arrays;', os.path.getsize(OUT) // 1024, 'KiB ->', OUT)


if __name__ == '__main__':
    main()
