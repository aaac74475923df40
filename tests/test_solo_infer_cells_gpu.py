"""BoxSOLOv2Head.simple_test and BoxLevelSet.simple_test on the GPU: the towers, then only the candidate cells convolved
(``solo_seg.candidate_sources``), against ``get_seg(*forward(feats, eval=True), ...)`` on the same towers and features --
bit for bit, in float32 and under float16 and bfloat16 autocast."""
import pytest
import torch

from oracle import solo_format as osf
from oracle.make_golden_solo_format import assert_same
from tests.test_solo_seg_gpu import _count_syncs, _quantile_thr

pytestmark = pytest.mark.gpu
DEV = 'cuda'
GRIDS = (40, 36, 24, 16, 12)
CFG = dict(mask_thr=0.55, nms_pre=500, max_per_img=100, kernel='gaussian', sigma=2.0, filter_thr=0.0)


def _head(C=64, seed=0):
    from oracle import solo_head as osh
    from boxinstseg_b200.models import build_head
    return osh.attach_towers(build_head(dict(osh.GOLDEN_HEAD, in_channels=C, seg_feat_channels=C)), C, C, 80, seed=seed).to(DEV)


def _feats(B, H=256, W=320, C=64, seed=0):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(B, C, -(-H // s), -(-W // s), generator=g).to(DEV) for s in (4, 8, 16, 32, 64)]


def _metas(B):
    shapes = [((250, 310, 3), (480, 600, 3)), ((256, 300, 3), (256, 300, 3)), ((200, 320, 3), (333, 517, 3))]
    return [dict(img_shape=shapes[b % 3][0], ori_shape=shapes[b % 3][1]) for b in range(B)]


def _cate(head, feats):
    with torch.no_grad():
        return head._towers(feats, True, 'test')[1]


def _scale_cate(head, scale):
    """Both paths read the category maps from ``forward_single``: multiply image b's by ``scale[b]`` (a [B] tensor), to
    shape the candidates image by image."""
    single = type(head).forward_single

    def forward_single(x, idx, eval=False):
        k, c = single(head, x, idx, eval=eval)
        return k, c * scale.to(c.dtype).view(-1, *[1] * (c.dim() - 1))
    head.forward_single = forward_single
    return head


def _dense(head, feats, metas, cfg):
    return head.get_seg(*head.forward(feats, eval=True), metas, cfg)


def _assert_equal(got, ref):
    assert len(got) == len(ref)
    for g, r in zip(got, ref):
        for k in ('masks', 'labels', 'scores'):
            a, b = getattr(g, k), getattr(r, k)
            assert a.dtype == b.dtype and a.shape == b.shape, (k, a.dtype, b.dtype, a.shape, b.shape)
            assert torch.equal(a, b), k


def _both(head, feats, metas, cfg, rescale=False, autocast=None):
    with torch.autocast('cuda', dtype=autocast or torch.float16, enabled=autocast is not None):
        got = head.simple_test(feats, metas, rescale, cfg=cfg)
        ref = _dense(head, feats, metas, cfg)
    _assert_equal(got, ref)
    return got


@pytest.mark.parametrize('B', [1, 2, 3])
@pytest.mark.parametrize('rescale', [False, True])
def test_equals_dense_get_seg(B, rescale):
    head, feats = _head(), _feats(B, seed=B)
    cfg = dict(CFG, score_thr=_quantile_thr(_cate(head, feats), 300 * B))
    got = _both(head, feats, _metas(B), cfg, rescale)
    assert all(len(r.scores) > 0 for r in got)
    for r, m in zip(got, _metas(B)):
        assert r.masks.dtype == torch.bool and r.masks.shape[1:] == m['ori_shape'][:2]
        assert r.labels.dtype == torch.int64 and r.scores.dtype == torch.float32


def test_test_cfg_attribute_and_missing_cfg():
    head, feats = _head(), _feats(1)
    cfg = dict(CFG, score_thr=_quantile_thr(_cate(head, feats), 200))
    with pytest.raises(ValueError):
        head.simple_test(feats, _metas(1))
    head.test_cfg = cfg
    _assert_equal(head.simple_test(feats, _metas(1)), _dense(head, feats, _metas(1), cfg))


def test_no_candidate():
    head, feats = _head(), _feats(2)
    got = _both(head, feats, _metas(2), dict(CFG, score_thr=1.0))
    assert all(len(r.scores) == 0 for r in got)


def test_nms_keeps_nothing_in_one_image():
    """Image 1's category scores scaled to a tenth: it has candidates, but every score of it ends below ``filter_thr``;
    image 0 keeps some."""
    head, feats = _head(), _feats(2, seed=5)
    _scale_cate(head, torch.tensor([1.0, 0.1], device=DEV))
    cate = _cate(head, feats)
    filter_thr = float(max(c[1].max() for c in cate)) * 1.0001
    cfg = dict(CFG, score_thr=_quantile_thr([c[1:] for c in cate], 100), filter_thr=filter_thr)
    assert sum(int((c[1] > cfg['score_thr']).sum()) for c in cate) >= 100
    got = _both(head, feats, _metas(2), cfg)
    assert len(got[0].scores) > 0 and len(got[1].scores) == 0


def test_nearly_every_cell_is_a_candidate():
    """score_thr 0: almost all 3872 cells of an image are distinct candidate rows, more than one 2048-row pack chunk.
    Then image 1's scores are zeroed, so that both chunks hold rows of image 0 only."""
    head, feats = _head(), _feats(2, seed=9)
    cate = _cate(head, feats)
    rows = sum(int((c[0] > 0).any(-1).sum()) for c in cate)
    assert rows > 3500
    got = _both(head, feats, _metas(2), dict(CFG, score_thr=0.0))
    assert all(len(r.scores) > 0 for r in got)
    _scale_cate(head, torch.tensor([1.0, 0.0], device=DEV))
    got = _both(head, feats, _metas(2), dict(CFG, score_thr=0.0))
    assert len(got[0].scores) > 0 and len(got[1].scores) == 0


def test_two_pack_image_groups():
    B = 17
    head, feats = _head(), _feats(B, H=128, W=160, seed=17)
    cfg = dict(CFG, score_thr=_quantile_thr(_cate(head, feats), 150 * B))
    metas = [dict(img_shape=(128 - b, 160 - 2 * b, 3), ori_shape=(100 + 7 * b, 90 + 11 * b, 3)) for b in range(B)]
    got = _both(head, feats, metas, cfg)
    assert sum(len(r.scores) for r in got) > 0


@pytest.mark.parametrize('dtype', [torch.float16, torch.bfloat16])
def test_autocast(dtype):
    head, feats = _head(), _feats(2, seed=3)
    with torch.autocast('cuda', dtype=dtype):
        cate = _cate(head, feats)
        assert cate[0].dtype == dtype
    cfg = dict(CFG, score_thr=_quantile_thr(cate, 500))
    got = _both(head, feats, _metas(2), cfg, autocast=dtype)
    assert all(len(r.scores) > 0 for r in got)


@pytest.mark.parametrize('K', [0, 400])
def test_at_most_two_syncs(K):
    head, feats = _head(), _feats(2)
    cfg = dict(CFG, score_thr=_quantile_thr(_cate(head, feats), K))
    head.simple_test(feats, _metas(2), cfg=cfg)                                              # warm up
    assert _count_syncs(lambda: head.simple_test(feats, _metas(2), cfg=cfg)) <= 2


def test_peak_memory_below_one_dense_prediction():
    """COCO test shape: 800 x 1344 padded input, feature_pred 200 x 336, about 100 candidates."""
    B = 2
    head, feats = _head(), _feats(B, H=800, W=1344)
    assert feats[0].shape[-2:] == (200, 336)
    cfg = dict(CFG, score_thr=_quantile_thr(_cate(head, feats), 100))
    metas = [dict(img_shape=(800, 1333, 3), ori_shape=(427, 640, 3))] * B
    head.simple_test(feats, metas, cfg=cfg)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    got = head.simple_test(feats, metas, cfg=cfg)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    dense = B * sum(s * s for s in GRIDS) * 200 * 336 * 4
    assert sum(len(r.scores) for r in got) > 0
    assert peak < dense, (peak, dense)
    _assert_equal(got, _dense(head, feats, metas, cfg))


@pytest.mark.parametrize('rescale', [False, True])
def test_box_level_set_simple_test(rescale):
    """The registered detector on a stand-in backbone against the reference's lines: forward(eval=True), get_seg,
    format_results."""
    from boxinstseg_b200.models import HEADS
    B = 2
    head, feats = _head(), _feats(B, seed=21)
    cfg = dict(CFG, score_thr=_quantile_thr(_cate(head, feats), 300))
    det = HEADS.get('BoxLevelSet')()
    img = torch.zeros(B, 3, 256, 320, device=DEV)
    det.bbox_head, det.test_cfg, det.extract_feat = head, cfg, lambda x: feats
    got = det.simple_test(img, _metas(B), rescale=rescale)
    outs = head(feats, eval=True)
    ref = [osf.format_results(r, head.num_classes) for r in head.get_seg(*(outs + (_metas(B), cfg, rescale)))]
    assert len(got) == len(ref) == B
    assert sum(len(m) for r in got for m in r[1][0]) > 0
    for g, r in zip(got, ref):
        assert_same(g, r, 'BoxLevelSet.simple_test')
