"""Golden vectors from the REFERENCE'S OWN CUDA extensions (oracle/_ref/*.so, built by oracle/Makefile from the reference's
mmdet/ops/pairwise and mmdet/ops/tree_filter sources, unmodified).  Needs a GPU and the built extensions; run it once where
both exist:

    python -m oracle.make_golden_ref_ext [OUT_DIR]        (default: tests/golden)

writes
  ref_ext.npz   : pairwise_nlog forward/backward, MST edge sets, refine forward/backward, and the reference's own BFS order
                  with the refine results on it -- on the inputs of tests/test_reference_ext_gpu.py;
  config_a_ref.npz : config A at full size (bench.synthetic_case(1234)) through a restatement of condinst_head.py:1288-1343
                  around the reference's pairwise op -- the losses, the gradient's norm and a seeded sample of its entries
                  (tests/test_config_a_gpu.py)."""
import glob
import importlib.util
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tests import test_reference_ext_gpu as T  # noqa: E402

DEV = T.DEV
CONFIG_A_SAMPLE = 16384


def _load(name):
    hits = glob.glob(os.path.join(ROOT, 'oracle', '_ref', name + '*.so'))
    if not hits:
        raise SystemExit(f'oracle/_ref/{name}*.so is missing: build it with `make -C oracle` where the reference exists')
    spec = importlib.util.spec_from_file_location(name, hits[0])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _np(t):
    return t.detach().cpu().numpy()


def ref_ext(pw_ext, tf_ext):
    out = {}
    for shape, k, d in T.PAIRWISE_CASES:
        key = T.case_key('pw', *shape, k, d)
        x, g = T.pairwise_inputs(shape, k)
        pw = pw_ext.pairwise_nlog_forward(k, d, x)
        gx = pw_ext.pairwise_nlog_backward(k, d, x, pw, g)
        out[key + '_shape'] = np.array(pw.shape, np.int64)
        out[key + '_fwd'] = _np(pw.flatten()[T.sample_index(pw.numel()).to(DEV)])
        out[key + '_bwd'] = _np(gx.flatten()[T.sample_index(x.numel()).to(DEV)])
    for B, C, h, w in T.MST_CASES:
        _, index, weight = T.grid_problem(B, C, h, w, seed=h)
        out[T.case_key('mst', B, C, h, w)] = _np(tf_ext.mst_forward(index.clone(), weight.clone(), h * w)).astype(np.int32)
    for B, C, h, w in T.REFINE_CASES:
        key = T.case_key('refine', B, C, h, w)
        feat, ew, idx, par, chd, gout = T.refine_inputs(B, C, h, w)
        r = tf_ext.refine_forward(feat, ew.clone(), idx.clone(), par.clone(), chd.clone())    # theirs writes entry 0 in place
        ew0 = ew.clone(); ew0[:, 0] = 0
        par0 = par.clone(); par0[:, 0] = 0
        out[key + '_out'] = _np(r[0])
        out[key + '_gfeat'] = _np(tf_ext.refine_backward_feature(feat, ew0, idx, par0, chd, r[0], r[1], r[2], r[3], r[4], gout))
        out[key + '_gweight'] = _np(tf_ext.refine_backward_weight(feat, ew0, idx, par0, chd, r[0], r[1], r[2], r[3], r[4], gout))
    tree, feat, gout, ew = T.bfs_inputs()
    ridx, rpar, rchd = tf_ext.bfs_forward(tree.clone(), 4)
    r = tf_ext.refine_forward(feat, ew.clone(), ridx.clone(), rpar.clone(), rchd.clone())
    ew0 = ew.clone(); ew0[:, 0] = 0
    par0 = rpar.clone(); par0[:, 0] = 0
    out['bfs_tree'] = _np(tree).astype(np.int32)
    out.update(bfs_idx=_np(ridx), bfs_par=_np(rpar), bfs_chd=_np(rchd))
    for i, a in enumerate(r):
        out[f'bfs_out{i}'] = _np(a)
    out['bfs_gfeat'] = _np(tf_ext.refine_backward_feature(feat, ew0, ridx, par0, rchd, r[0], r[1], r[2], r[3], r[4], gout))
    out['bfs_gweight'] = _np(tf_ext.refine_backward_weight(feat, ew0, ridx, par0, rchd, r[0], r[1], r[2], r[3], r[4], gout))
    return out


def config_a_sample_index(n):
    return T.sample_index(n, CONFIG_A_SAMPLE, seed=1234)


def config_a(pw_ext):
    import bench
    from boxinstseg_b200.ops.boxinst import boxinst_targets
    case = bench.synthetic_case(1234)
    dev = torch.device(DEV)
    t = boxinst_targets(case['img'].to(dev), case['metas'], [b.to(dev) for b in case['gt_bboxes']], want_similarity=True)

    class RefPairwise(torch.autograd.Function):            # mmdet/ops/pairwise/pairwise.py:6-26
        @staticmethod
        def forward(ctx, logits, size, dilation):
            pw = pw_ext.pairwise_nlog_forward(size, dilation, logits)
            ctx.save_for_backward(logits, pw)
            ctx.cfg = (size, dilation)
            return pw

        @staticmethod
        def backward(ctx, g):
            logits, pw = ctx.saved_tensors
            return pw_ext.pairwise_nlog_backward(ctx.cfg[0], ctx.cfg[1], logits, pw, g.contiguous()), None, None

    gi = case['gt_inds'].to(dev)
    sim = t.similarity[case['img_inds'].to(dev)]                       # the G-fold gather of condinst_head.py:1316
    bm = torch.cat(t.bitmasks())[gi][:, None]
    x = case['logits'].to(dev).requires_grad_(True)

    def dice(a, b):                                                    # condinst_head.py:117-131
        a, b = a.flatten(1), b.flatten(1)
        return 1.0 - 2.0 * (a * b).sum(1) / ((a * a).sum(1) + (b * b).sum(1) + 1e-5)

    scores = x.sigmoid()
    prj = (dice(scores.max(dim=2, keepdim=True)[0], bm.max(dim=2, keepdim=True)[0]) +
           dice(scores.max(dim=3, keepdim=True)[0], bm.max(dim=3, keepdim=True)[0])).mean()      # :134-143
    w = (sim >= 0.3).float() * bm
    pair = (RefPairwise.apply(x, 3, 2) * w).sum() / w.sum().clamp(min=1.0)                        # :1318-1332
    (g,) = torch.autograd.grad(prj + pair, x)
    sel = config_a_sample_index(g.numel())
    return dict(loss_prj=np.float64(prj.item()), loss_pairwise=np.float64(pair.item()),
                grad_norm=np.float64(g.double().norm().item()), grad_sample=_np(g.flatten()[sel.to(dev)]))


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, 'tests', 'golden')
    os.makedirs(out_dir, exist_ok=True)
    pw_ext, tf_ext = _load('pairwise_ext_ref'), _load('tree_filter_cuda_ref')
    np.savez_compressed(os.path.join(out_dir, 'ref_ext.npz'), **ref_ext(pw_ext, tf_ext))
    np.savez_compressed(os.path.join(out_dir, 'config_a_ref.npz'), **config_a(pw_ext))
    print('wrote', out_dir)


if __name__ == '__main__':
    main()
