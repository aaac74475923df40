"""GPU: ``BoxMasks.to_tensor`` and ``ops.box_masks.rasterize`` (csrc/box_masks.cu).

* ``to_tensor`` on CUDA equals ``torch.tensor(to_ndarray(), dtype, device)`` for every output type, at odd and 16-aligned
  widths, misaligned rows, G = 0, 1000 masks and H * W at the kernel's limit, without a synchronising call;
* a batch of images of different sizes in one call, and rectangle tables chunked over several launches;
* BoxSOLOv2Head.loss, DiscoBoxSOLOv2Head.loss (float16 autocast) and Box2MaskHead.loss give bit-identical losses and
  gradients from ``BoxMasks`` and from the same masks materialised as device tensors."""
import numpy as np
import pytest
import torch

from boxinstseg_b200.core import BoxMasks
from boxinstseg_b200.ops.box_masks import rasterize
from oracle import box_masks as ob

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
DTYPES = [torch.uint8, torch.bool, torch.float32, torch.float16, torch.bfloat16, torch.int64, torch.int32, torch.int16,
          torch.int8, torch.float64]


def _random(seed, G, H, W):
    rng = np.random.default_rng(seed)
    return BoxMasks(np.concatenate([rng.integers(-2, H + 2, (G, 1)), rng.integers(-2, W + 2, (G, 1)),
                                    rng.integers(-2, H + 2, (G, 1)), rng.integers(-2, W + 2, (G, 1))], 1), H, W)


def _want(m, dt):
    return torch.tensor(m.to_ndarray(), dtype=dt, device=DEV)


@pytest.mark.parametrize('dt', DTYPES)
@pytest.mark.parametrize('G, H, W', [(5, 37, 53), (7, 64, 64), (3, 1, 1), (4, 1, 97), (6, 97, 1), (0, 40, 40),
                                     (2, 0, 8), (20, 100, 136), (1000, 24, 33)])
def test_to_tensor_equals_the_host_array(dt, G, H, W):
    m = _random(G * 1000 + H, G, H, W)
    got = m.to_tensor(dt, DEV)
    assert got.dtype == dt and got.shape == (G, H, W) and got.device == torch.device(DEV)
    assert torch.equal(got, _want(m, dt))


def test_full_empty_and_edge_rectangles():
    m = BoxMasks([[0, 0, 33, 47], [0, 0, 0, 0], [32, 46, 33, 47], [0, 46, 33, 47], [32, 0, 33, 47], [5, 3, 6, 4]], 33, 47)
    for dt in DTYPES:
        assert torch.equal(m.to_tensor(dt, DEV), _want(m, dt))


@pytest.mark.parametrize('dt', [torch.uint8, torch.float16, torch.float32])
def test_misaligned_outputs(dt):
    """Rows that start at every offset from a 16-byte boundary: output views into a larger buffer."""
    rects = [np.array([[1, 2, 9, 30], [0, 0, 11, 31], [3, 17, 4, 18]])]
    for off in range(0, 16):
        buf = torch.full((off + 3 * 11 * 31 + 8,), 7, dtype=dt, device=DEV)
        want = _want(BoxMasks(rects[0], 11, 31), dt)
        from boxinstseg_b200 import _lib as L
        out = buf[off:off + 3 * 11 * 31]
        es, one = {torch.uint8: (1, 1), torch.float16: (2, 0x3C00), torch.float32: (4, 0x3F800000)}[dt]
        flat = np.ascontiguousarray(rects[0].astype(np.int32))
        sizes = np.array([[3, 11, 31]], dtype=np.int64)
        ptrs = np.array([out.data_ptr()], dtype=np.uint64)
        L.check(L.lib().bxs_box_masks_rasterize(ptrs.ctypes.data, flat.ctypes.data, sizes.ctypes.data, 1, es, one,
                                                L.stream()), 'rasterize')
        assert torch.equal(out.view(3, 11, 31), want), off
        assert (buf[:off] == 7).all() and (buf[off + 3 * 11 * 31:] == 7).all(), off


def test_no_synchronising_call():
    masks = [_random(s, 20, 800, 1216) for s in range(4)]
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode('error')
    try:
        outs = [m.to_tensor(torch.uint8, DEV) for m in masks] + [m.to_tensor(torch.bool, DEV) for m in masks]
        outs += rasterize([m.rects for m in masks], [(m.height, m.width) for m in masks], torch.float16, DEV)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    for o, m in zip(outs, masks * 3):
        assert torch.equal(o, _want(m, o.dtype))


def test_batch_of_different_sizes_in_one_call():
    masks = [_random(1, 7, 120, 97), _random(2, 0, 50, 50), _random(3, 13, 33, 200), _random(4, 2, 1, 1),
             _random(5, 5, 0, 10), _random(6, 9, 257, 31)]
    for dt in (torch.uint8, torch.bfloat16, torch.int32, torch.int64):
        outs = rasterize([m.rects for m in masks], [(m.height, m.width) for m in masks], dt, DEV)
        assert len(outs) == len(masks)
        for o, m in zip(outs, masks):
            assert torch.equal(o, _want(m, dt))


def test_tables_larger_than_one_launch_are_chunked():
    """4000 rectangles in one image (three launches of at most 1792) and 70 images (two launches of at most 64)."""
    big = _random(7, 4000, 9, 23)
    assert torch.equal(big.to_tensor(torch.uint8, DEV), _want(big, torch.uint8))
    many = [_random(100 + i, 1 + i % 40, 5 + i % 7, 3 + i % 11) for i in range(70)]
    outs = rasterize([m.rects for m in many], [(m.height, m.width) for m in many], torch.float32, DEV)
    for o, m in zip(outs, many):
        assert torch.equal(o, _want(m, torch.float32))


def test_size_near_the_limit():
    """H * W = 2^31 - 1 - 46339: one uint8 mask of 2 GB, checked against the same rectangle written by torch slicing."""
    H, W = 46340, 46339
    assert H * W < 2 ** 31 - 1
    m = BoxMasks([[3, 5, H - 2, W - 7]], H, W)
    got = m.to_tensor(torch.uint8, DEV)
    want = torch.zeros(1, H, W, dtype=torch.uint8, device=DEV)
    want[0, 3:H - 2, 5:W - 7] = 1
    assert torch.equal(got, want)
    del got, want
    from boxinstseg_b200 import _lib as L
    with pytest.raises(L.BoxSegError, match='unsupported'):
        BoxMasks([[0, 0, 1, 1]], 46341, 46341).to_tensor(torch.uint8, DEV)


# ------------------------------------------------------------------------------------------------- the heads, end to end
def _rects_of(mask):
    """The rectangle of a box-shaped host mask [H, W]."""
    ys, xs = np.nonzero(mask.any(1))[0], np.nonzero(mask.any(0))[0]
    return (ys[0], xs[0], ys[-1] + 1, xs[-1] + 1) if len(ys) else (0, 0, 0, 0)


def test_box_solov2_head_loss_from_box_masks():
    """Gradients with respect to the loss's inputs (the towers' cuDNN backward is not bitwise repeatable, the loss is)."""
    from boxinstseg_b200.models.dense_heads.mask_loss_heads import SoloInsPreds, SoloLevelPred
    from tests.test_solo_head_gpu import _case
    head, feats, img, bboxes, labels, masks = _case(3, 2, 128, 160, 64, [3, 4])
    bms = [BoxMasks([_rects_of(x) for x in m.cpu().numpy()], m.shape[1], m.shape[2]) for m in masks]
    dense = [torch.tensor(b.to_ndarray(), device=DEV) for b in bms]
    assert all(torch.equal(a, b) for a, b in zip(dense, masks))
    with torch.no_grad():
        ins, cate, lst = head(feats)

    def run(gt_masks):
        feat = ins.feature_pred.detach().clone().requires_grad_(True)
        kern = [p.kernel_pred.detach().clone().requires_grad_(True) for p in ins]
        c = [t.detach().clone().requires_grad_(True) for t in cate]
        ls = lst.detach().clone().requires_grad_(True)
        preds = SoloInsPreds(SoloLevelPred(feat, k, p.out_size) for k, p in zip(kern, ins))
        out = head.loss(preds, c, ls, bboxes, labels, gt_masks, img, None, None)
        leaves = [feat, ls] + kern + c
        grads = torch.autograd.grad(sum(out.values()), leaves, allow_unused=True)
        return out, [torch.zeros_like(x) if g is None else g for x, g in zip(leaves, grads)]

    (out_a, g_a), (out_b, g_b) = run(dense), run(bms)
    assert list(out_a) == list(out_b) and all(torch.equal(out_a[k], out_b[k]) for k in out_a)
    assert any(g.any() for g in g_a)
    assert all(torch.equal(a, b) for a, b in zip(g_a, g_b))


def test_discobox_head_loss_from_box_masks_under_autocast():
    from tests.test_discobox_loss_gpu import _gpu_case, _head, _run_loss
    inputs = list(_gpu_case(0))
    bms = [BoxMasks([_rects_of(x) for x in m.cpu().numpy()], m.shape[1], m.shape[2]) for m in inputs[7]]
    head = _head()
    runs = []
    for masks in ([torch.tensor(b.to_ndarray(), device=DEV) for b in bms], bms):
        inputs[7] = masks
        with torch.autocast('cuda', dtype=torch.float16):
            runs.append(_run_loss(head, inputs, True, False))
    (out_a, g_a), (out_b, g_b) = runs
    assert list(out_a) == list(out_b) and all(torch.equal(out_a[k], out_b[k]) for k in out_a)
    assert all(torch.equal(a, b) for a, b in zip(g_a, g_b))


def test_box2mask_head_loss_from_box_masks():
    from tests.test_box2mask_loss_gpu import _case, _head, _run
    cls, masks, lsts, labels, gts, img = _case(1, (5, 3), pred=32, mask=128)
    bms = [BoxMasks([_rects_of(x) for x in g.cpu().numpy()], g.shape[1], g.shape[2]) for g in gts]
    pad = (128, 128)
    # preprocess_panoptic_gt: gt_masks.pad(pad_shape, pad_val=0).to_tensor(dtype=torch.bool, device).long()
    ref = [torch.tensor(b.pad(pad).to_ndarray(), dtype=torch.bool, device=DEV).long() for b in bms]
    new = [b.pad(pad).to_tensor(dtype=torch.bool, device=DEV).long() for b in bms]
    assert all(torch.equal(a, b.to(DEV)) for a, b in zip(ref, gts))
    head = _head().to(DEV)
    metas = [dict() for _ in labels]
    runs = [_run(lambda c, m, f: head.loss(c, m, f, labels, g, metas, img), cls, masks, lsts) for g in (ref, new)]
    (out_a, g_a), (out_b, g_b) = runs
    assert list(out_a) == list(out_b) and all(torch.equal(out_a[k], out_b[k]) for k in out_a)
    assert all(torch.equal(a, b) for a, b in zip(g_a, g_b))


def test_golden_chains_on_the_device(golden):
    g = golden('box_masks')
    from tests.test_box_masks_cpu import _chain, make_box_masks
    for name in g['cases']:
        steps, _ = ob.run_chain(_chain(g[f'{name}/chain']), make_box_masks)
        for i, m in enumerate(steps):
            want = torch.from_numpy(g[f'{name}/{i}/masks']).to(DEV)
            got = m.to_tensor(torch.uint8, DEV)
            assert got.shape == want.shape and torch.equal(got, want), (name, i)
