"""GPU: DiscoBox's independent teacher (csrc/momentum_update.cu, ops/ema.py, models/detectors/discobox.py).
  * ``momentum_update_`` against the reference's formula run by torch on the same CUDA tensors (``s * (1. - m) + t * m``,
    then ``t.copy_``), bit for bit through integer views (a NaN only as a NaN): every dtype at momentum 0.999, 0, 0.5 and 1,
    the golden states of the reference, DiscoBox-shaped R-50 / R-101 states, 5 000 small tensors (several launches),
    empty and one-element tensors, sizes 1-67, storage offsets 1-7, channels_last, one uint8 tensor above 2^31 elements;
  * ``momentum_update`` against the reference's method on the same models, with the turn-on copy and the cases a pairing
    cache could get wrong (a replaced parameter, a replaced buffer, ``.to()``); one launch for R-101, no synchronising call
    after the first, a CUDA graph replays to the eager result;
  * ``forward_train`` on a stand-in DiscoBox detector (tiny backbone and mask-feature head, the repo's DiscoBoxSOLOv2Head)
    against the reference's lines on a deep copy, and on stub modules against the golden gate sequences."""
import copy
import os
import sys

import numpy as np
import pytest
import torch
from torch import nn
import torch.nn.functional as F

from oracle import teacher_ema as ote

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'tools'))
from bench_teacher_ema import discobox_model, ref_momentum_update  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
MOMENTA = [0.999, 0.0, 0.5, 1.0]
ALL = [torch.float32, torch.float16, torch.bfloat16, torch.float64, torch.int64, torch.int32, torch.int16, torch.int8,
       torch.uint8, torch.bool]


def ref_update(t, s, m):
    """single_stage_ts.py:130 and load_state_dict's copy_, by torch on the same tensors."""
    t.copy_(s * (1. - m) + t * m)


_INT_VIEW = {1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}


def same(a, b):
    """Bit for bit through integer views; a NaN only has to be a NaN."""
    if a.dtype != b.dtype or a.shape != b.shape:
        return False
    if a.dtype.is_floating_point:
        na, nb = torch.isnan(a), torch.isnan(b)
        if not torch.equal(na, nb):
            return False
        v = _INT_VIEW[a.element_size()]
        return torch.equal(torch.where(na, torch.zeros_like(a), a).view(v), torch.where(nb, torch.zeros_like(b), b).view(v))
    return torch.equal(a, b)


def values(n, dtype, gen, edges=True):
    """Seeded values of every kind a state holds: normal, tiny, huge, +-0, subnormal, +-inf, NaN, integers near 2^24."""
    if dtype == torch.bool:
        return torch.rand(n, generator=gen) < 0.5
    if not dtype.is_floating_point:
        info = torch.iinfo(dtype)
        lo, hi = max(info.min, -2 ** 26), min(info.max, 2 ** 26)
        x = torch.randint(lo, hi + 1, (n,), generator=gen, dtype=torch.int64)
        if edges and n >= 8 and hi >= 2 ** 24:
            x[:8] = torch.tensor([2 ** 24 - 1, 2 ** 24, 2 ** 24 + 1, 2 ** 24 + 3, -2 ** 24 - 1, 0, -1, 1])
        return x.to(dtype)
    x = torch.randn(n, generator=gen, dtype=torch.float64) * torch.exp2(torch.randint(-30, 30, (n,), generator=gen).double())
    x = x.to(dtype)
    if edges and n >= 9:
        tiny = torch.finfo(dtype).tiny
        x[:9] = torch.tensor([0.0, -0.0, tiny / 4, -tiny / 8, float('inf'), float('-inf'), float('nan'), 1.0,
                              torch.finfo(dtype).max], dtype=torch.float64).to(dtype)
    return x


def check_pairs(ts, ss, m):
    """momentum_update_ on clones of (ts, ss) equals ref_update on other clones."""
    from boxinstseg_b200.ops.ema import momentum_update_
    a = [t.clone(memory_format=torch.preserve_format) for t in ts]
    b = [t.clone(memory_format=torch.preserve_format) for t in ts]
    momentum_update_(a, ss, m)
    for t, s in zip(b, ss):
        ref_update(t, s, m)
    torch.cuda.synchronize()
    for i, (x, y) in enumerate(zip(a, b)):
        assert same(x, y), (i, x.dtype, x.shape)


@pytest.mark.parametrize('m', MOMENTA)
@pytest.mark.parametrize('dtype', ALL, ids=str)
def test_every_dtype_against_torch(dtype, m):
    gen = torch.Generator().manual_seed(7)
    sizes = (1, 7, 16, 1000, 16385, 65536 + 13)                         # tails of the vector path, one or more chunks
    ts = [values(n, dtype, gen).to(DEV) for n in sizes]
    ss = [values(n, dtype, gen).to(DEV) for n in sizes]
    check_pairs(ts, ss, m)


@pytest.mark.parametrize('i', range(len(ote.MOMENTA)))
def test_golden_states(golden, i):
    from boxinstseg_b200.ops.ema import momentum_update_
    g = golden('teacher_ema')
    keys = [k.split('/', 2)[2] for k in g.files if k.startswith(f'ema{i}/out/')]
    m = float(g[f'ema{i}/momentum'])
    t = [torch.from_numpy(g[f'ema{i}/teacher/{k}']).to(DEV) for k in keys]
    s = [torch.from_numpy(g[f'ema{i}/student/{k}']).to(DEV) for k in keys]
    check_pairs(t, s, m)
    momentum_update_(t, s, m)
    for k, x in zip(keys, t):
        assert same(x.cpu(), torch.from_numpy(g[f'ema{i}/out/{k}'])), k


def test_small_tensors_sizes_offsets_and_layouts():
    gen = torch.Generator().manual_seed(3)
    ts, ss = [], []
    for dtype in ALL:
        for n in list(range(0, 68)):
            ts.append(values(n, dtype, gen).to(DEV))
            ss.append(values(n, dtype, gen).to(DEV))
        for off in range(1, 8):                                         # regions at every element offset
            bt, bs = values(300, dtype, gen).to(DEV), values(300, dtype, gen).to(DEV)
            ts.append(bt[off:off + 100 + off])
            ss.append(bs[8 - off:108])
        if dtype.is_floating_point:
            w = values(64 * 32 * 3 * 3, dtype, gen).to(DEV).view(64, 32, 3, 3)
            ts.append(w.to(memory_format=torch.channels_last))
            ss.append(values(w.numel(), dtype, gen).to(DEV).view(64, 32, 3, 3).to(memory_format=torch.channels_last))
    assert any(not t.is_contiguous() for t in ts)
    for m in MOMENTA:
        check_pairs(ts, ss, m)


def kernel_nodes(graph):
    """(kernel nodes, all nodes) of a graph captured with keep_graph=True: the launches the captured call enqueues.
    Launches are counted from the capture rather than with torch.profiler: in a process where other profiler sessions
    ran first (the whole GPU suite), a profile of this call was seen to record no CUDA activity at all."""
    import ctypes
    cu = ctypes.CDLL('libcuda.so.1')
    raw = ctypes.c_void_p(graph.raw_cuda_graph())
    n = ctypes.c_size_t(0)
    assert cu.cuGraphGetNodes(raw, None, ctypes.byref(n)) == 0
    nodes = (ctypes.c_void_p * n.value)()
    assert cu.cuGraphGetNodes(raw, nodes, ctypes.byref(n)) == 0
    kinds = []
    for node in nodes:
        kind = ctypes.c_int(-1)
        assert cu.cuGraphNodeGetType(ctypes.c_void_p(node), ctypes.byref(kind)) == 0
        kinds.append(kind.value)
    return sum(k == 0 for k in kinds), len(kinds)                      # 0: CU_GRAPH_NODE_TYPE_KERNEL


def small_tensors_5000():
    gen = torch.Generator().manual_seed(5)
    sizes = torch.randint(1, 68, (5000,), generator=gen).tolist()
    dts = [ALL[i % len(ALL)] for i in range(5000)]
    ts = [values(n, d, gen, edges=False).to(DEV) for n, d in zip(sizes, dts)]
    ss = [values(n, d, gen, edges=False).to(DEV) for n, d in zip(sizes, dts)]
    return ts, ss


def test_5000_small_tensors():
    ts, ss = small_tensors_5000()
    check_pairs(ts, ss, 0.999)


def test_5000_small_tensors_take_several_launches():
    """1024 entries per launch: 5 launches and nothing else.  The capture records the launches without running them."""
    from boxinstseg_b200.ops.ema import momentum_update_
    ts, ss = small_tensors_5000()
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        momentum_update_(ts, ss, 0.999)
    assert kernel_nodes(g) == (5, 5)


def test_student_aliasing_its_teacher_and_tied_weights():
    from boxinstseg_b200.ops.ema import momentum_update_
    from boxinstseg_b200._lib import BoxSegError
    gen = torch.Generator().manual_seed(9)
    t = values(1000, torch.float32, gen).to(DEV)
    want = t.clone()
    ref_update(want, want.clone(), 0.999)
    momentum_update_([t], [t], 0.999)                                   # s is t: elementwise, so well defined
    assert same(t, want)
    t, s = values(1000, torch.float32, gen).to(DEV), values(1000, torch.float32, gen).to(DEV)
    want = t.clone()
    ref_update(want, s, 0.5)
    momentum_update_([t, t], [s, s], 0.5)                               # tied weights listed twice: updated once
    assert same(t, want)
    with pytest.raises(BoxSegError):
        momentum_update_([t, t], [s, s.clone()], 0.5)                   # one teacher, two students
    with pytest.raises(RuntimeError, match='pair 1'):
        momentum_update_([t, t[::2]], [s, s[::2]], 0.5)                 # not dense
    with pytest.raises(RuntimeError, match='pair 0'):
        momentum_update_([t], [s.double()], 0.5)


def test_uint8_above_2_31_elements():
    from boxinstseg_b200.ops.ema import momentum_update_
    n = 2 ** 31 + 37
    t = torch.arange(n, device=DEV, dtype=torch.int64).remainder_(251).to(torch.uint8)
    s = torch.arange(n, device=DEV, dtype=torch.int64).remainder_(241).to(torch.uint8)
    parts = [slice(0, 2 ** 20), slice(2 ** 31 - 2 ** 19, 2 ** 31 + 2 ** 19), slice(n - 2 ** 20, n)]   # head, 2^31, tail
    want = [t[p].clone() for p in parts]
    for w, p in zip(want, parts):
        ref_update(w, s[p], 0.5)
    momentum_update_([t], [s], 0.5)
    for w, p in zip(want, parts):
        assert same(t[p], w), p


# -------------------------------------------------------------------------------------------------- DiscoBox models
def perturbed_pair(depth, seed):
    torch.manual_seed(seed)
    s = discobox_model(depth).to(DEV)
    t = copy.deepcopy(s)
    with torch.no_grad():
        for x in s.state_dict().values():
            if x.dtype.is_floating_point:
                x.add_(torch.randn_like(x) * 0.01)
            else:
                x.add_(seed + 1)
    return t, s


def assert_same_state(a, b):
    sa, sb = a.state_dict(), b.state_dict()
    assert sa.keys() == sb.keys()
    for k in sa:
        assert same(sa[k], sb[k]), k


@pytest.mark.parametrize('depth', [50, 101])
def test_discobox_states_against_reference_method(depth):
    from benchkit import syncs
    from boxinstseg_b200.models.detectors import momentum_update
    t, s = perturbed_pair(depth, 1)
    t.teacher_momentum = 0.999
    r = copy.deepcopy(t)
    for step in range(3):
        momentum_update(t, s)                                           # teacher_momentum=None reads the attribute
        ref_momentum_update(r, s, 0.999)
        assert_same_state(t, r)
        with torch.no_grad():
            for x in s.parameters():
                x.mul_(1.001)
    momentum_update(t, s, 0)                                            # the turn-on copy
    ref_momentum_update(r, s, 0)
    assert_same_state(t, r)
    assert syncs(lambda: momentum_update(t, s)) == 0
    ref_momentum_update(r, s, 0.999)
    assert_same_state(t, r)


@pytest.mark.parametrize('depth', [50, 101])
def test_discobox_state_takes_one_launch(depth):
    """The whole R-50 / R-101 state in one launch and nothing else, the pairing packed before the capture."""
    from boxinstseg_b200.models.detectors import momentum_update
    t, s = perturbed_pair(depth, 1)
    momentum_update(t, s, 0.999)
    g = torch.cuda.CUDAGraph(keep_graph=True)
    with torch.cuda.graph(g):
        momentum_update(t, s, 0.999)
    assert kernel_nodes(g) == (1, 1)


def test_pairing_cache_never_updates_a_stale_tensor():
    from boxinstseg_b200.models.detectors import momentum_update
    t, s = perturbed_pair(50, 2)
    r = copy.deepcopy(t)

    def both(m=0.999):
        momentum_update(t, s, m)
        ref_momentum_update(r, s, m)
        assert_same_state(t, r)
    both()
    s.backbone.conv1.weight = nn.Parameter(torch.randn_like(s.backbone.conv1.weight))            # student parameter
    both()
    w = nn.Parameter(t.neck.layer_blocks[0][0].weight.detach().clone())
    t.neck.layer_blocks[0][0].weight = w                                                      # teacher parameter
    r.neck.layer_blocks[0][0].weight = nn.Parameter(w.detach().clone())
    both()
    s.backbone.bn1.running_mean = torch.randn_like(s.backbone.bn1.running_mean)               # student buffer
    t.backbone.bn1.running_var = t.backbone.bn1.running_var.clone() + 1                       # teacher buffer
    r.backbone.bn1.running_var = r.backbone.bn1.running_var.clone() + 1
    both()
    t.to(torch.float64), s.to(torch.float64), r.to(torch.float64)                              # .to(): new storage
    both(0.5)
    t.to(memory_format=torch.channels_last), s.to(memory_format=torch.channels_last)
    r.to(memory_format=torch.channels_last)
    assert not s.backbone.conv1.weight.is_contiguous()
    both(0)


def test_graph_capture_replays_to_the_eager_result():
    from boxinstseg_b200.models.detectors import momentum_update
    t, s = perturbed_pair(50, 3)
    r = copy.deepcopy(t)
    momentum_update(t, s, 0.999)                                        # packs the pairs outside the capture
    ref_momentum_update(r, s, 0.999)
    snap = copy.deepcopy(t.state_dict())
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(g):
            momentum_update(t, s, 0.999)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for k, v in t.state_dict().items():                                 # capturing ran nothing
        assert same(v, snap[k]), k
    g.replay()
    torch.cuda.synchronize()
    ref_momentum_update(r, s, 0.999)
    assert_same_state(t, r)


# --------------------------------------------------------------------------------------------------- forward_train
class _Stub:
    """The stub modules of oracle/make_golden_teacher_ema.py, on the GPU: the head's loss records the gates."""

    def __init__(self, losses, calls):
        self.seq, self.calls = iter(losses), calls
        self.start_level, self.end_level = 0, 3

    def __call__(self, feats):
        return feats, feats

    def loss(self, *args, use_loss_ts, use_ind_teacher, use_corr, **kw):
        self.calls.append((use_loss_ts, use_corr, use_ind_teacher))
        return {'loss_ins': torch.tensor(next(self.seq), dtype=torch.float32, device=DEV)}


@pytest.mark.parametrize('run', ote.GATE_RUNS, ids=[r[0] for r in ote.GATE_RUNS])
def test_forward_train_gates_against_golden(golden, run):
    from boxinstseg_b200.models.detectors import DiscoBoxSOLOv2
    g = golden('teacher_ema')
    name, ind, corr, avg0, cnt0, losses = run
    calls = []
    head = _Stub(losses, calls)
    x = [torch.zeros(1, device=DEV)] * 5

    class Teacher(nn.Module):
        def __init__(self):
            super().__init__()
            self.w = nn.Parameter(torch.zeros(3, device=DEV))
            self.bbox_head, self.mask_feat_head = head, _Stub([], [])
            self.teacher_momentum = 0.999

        def extract_feat(self, img):
            return x

    class Det(DiscoBoxSOLOv2, Teacher):
        pass
    det = Det()
    det.tsw = type('W', (), {})()
    det.tsw.teacher = Teacher()
    det.use_ind_teacher, det.use_corr, det.train_cfg = ind, corr, None
    det.avg_loss_ins, det.cnt, det.turn_on_teacher = avg0, cnt0, False
    rows = []
    for _ in losses:
        det.forward_train(x[0], [{}], [], [])
        rows.append(calls[-1] + (det.turn_on_teacher, det.cnt, det.avg_loss_ins))
    assert np.array_equal(np.array([r[:4] for r in rows], np.int64), g[f'gates/{name}/flags'])
    assert np.array_equal(np.array([r[4] for r in rows], np.int64), g[f'gates/{name}/cnt'])
    assert np.array_equal(np.array([r[5] for r in rows], np.float64), g[f'gates/{name}/avg'])


def _disco_head():
    from boxinstseg_b200.models import build_head
    from oracle.make_golden_discobox_loss import CFG, GRIDS, NUM_CLASSES
    return build_head(dict(type='DiscoBoxSOLOv2Head', num_classes=NUM_CLASSES, in_channels=256, num_grids=list(GRIDS),
                           scale_ranges=CFG['scale_ranges'], strides=CFG['strides'], sigma=CFG['sigma']))


class _TinyHead(nn.Module):
    """A small forward in front of the repo's DiscoBoxSOLOv2Head.loss: per level a grid-sized category map and kernel."""

    def __init__(self, head, C=32):
        from oracle.make_golden_discobox_loss import GRIDS, NUM_CLASSES
        super().__init__()
        self.head, self.grids = head, GRIDS
        self.cate = nn.Conv2d(8, NUM_CLASSES, 3, padding=1)
        self.kernel = nn.Conv2d(8, C, 3, padding=1)

    def forward(self, feats):
        # every grid picks distinct rows and columns of the finest level: a gather whose backward is deterministic
        cate, kern = [], []
        for S in self.grids:
            i = torch.arange(S, device=feats[0].device) * feats[0].shape[-1] // S
            f = feats[0][:, :, i][:, :, :, i]
            cate.append(self.cate(f))
            kern.append(self.kernel(f))
        return cate, kern

    def loss(self, *args, **kw):
        return self.head.loss(*args, **kw)


class _MaskFeat(nn.Module):
    start_level, end_level = 0, 3

    def __init__(self, C=32):
        super().__init__()
        self.conv = nn.Conv2d(8, C, 1)

    def forward(self, feats):
        return self.conv(feats[1])


class _Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.backbone = nn.Sequential(nn.Conv2d(3, 8, 3, stride=2, padding=1), nn.BatchNorm2d(8), nn.ReLU())
        self.bbox_head = _TinyHead(_disco_head())
        self.mask_feat_head = _MaskFeat()
        self.train_cfg = None

    def extract_feat(self, img):
        x = self.backbone(img)
        return [x] + [F.avg_pool2d(x, 2 ** i) for i in range(1, 5)]


def _stand_in(cnt0, avg0):
    from boxinstseg_b200.models.detectors import DiscoBoxSOLOv2

    class Det(DiscoBoxSOLOv2, _Net):
        pass
    torch.manual_seed(0)
    det = Det().to(DEV)
    teacher = _Net().to(DEV)
    teacher.eval()
    teacher.teacher_momentum = 0.999
    det.tsw = type('W', (), {})()
    det.tsw.teacher = teacher
    det.use_ind_teacher, det.use_corr = True, False
    det.cnt, det.turn_on_teacher, det.avg_loss_ins = cnt0, False, avg0
    return det


def _ref_forward_train(self, img, img_metas, gt_bboxes, gt_labels, gt_bboxes_ignore=None, gt_masks=None):
    """single_stage_ts.py:179-237, the reference's lines (with the reference's momentum_update)."""
    if self.turn_on_teacher and self.use_ind_teacher:
        ref_momentum_update(self.tsw.teacher, self, self.tsw.teacher.teacher_momentum)
    student_x = self.extract_feat(img)
    student_outs = self.bbox_head(student_x)
    with torch.no_grad():
        if self.turn_on_teacher and self.use_ind_teacher:
            teacher_x = self.tsw.teacher.extract_feat(img)
            teacher_outs = self.tsw.teacher.bbox_head(teacher_x)
            _, t_kernel_preds = teacher_outs
    s_mask_feat_pred = self.mask_feat_head(student_x[0:4])
    if self.turn_on_teacher and self.use_ind_teacher:
        with torch.no_grad():
            t_mask_feat_pred = self.tsw.teacher.mask_feat_head(teacher_x[0:4])
    else:
        teacher_x = student_x
    if self.turn_on_teacher and self.use_ind_teacher:
        loss_inputs = student_outs + (t_kernel_preds, s_mask_feat_pred, t_mask_feat_pred, gt_bboxes, gt_labels, gt_masks,
                                      img_metas, self.train_cfg)
    else:
        loss_inputs = student_outs + (None, s_mask_feat_pred, None, gt_bboxes, gt_labels, gt_masks, img_metas, self.train_cfg)
    losses = self.bbox_head.loss(*loss_inputs, img=img, gt_bboxes_ignore=gt_bboxes_ignore,
                                 use_loss_ts=self.ref_avg < 0.3, use_ind_teacher=self.use_ind_teacher and self.turn_on_teacher,
                                 use_corr=self.ref_avg < 0.2 and self.use_corr, s_feat=student_x[0:4], t_feat=teacher_x[0:4])
    self.ref_gates = (self.ref_avg < 0.3, self.use_ind_teacher and self.turn_on_teacher)
    self.ref_avg = self.ref_avg * 0.9 + 0.1 * float(losses['loss_ins'])
    if self.use_ind_teacher and not self.turn_on_teacher and self.cnt > 13000:
        ref_momentum_update(self.tsw.teacher, self, 0)
        self.turn_on_teacher = True
    else:
        self.cnt += 1
    return losses


def test_forward_train_on_a_stand_in_detector_against_reference_lines():
    """Eight steps with an SGD step between them, across the teacher's turn-on and the 0.3 threshold of avg_loss_ins (the
    stand-in keeps use_corr off: the gates' golden test covers the 0.2 one): gates, cnt, turn_on_teacher, avg_loss_ins,
    both states and the losses equal at every step."""
    from oracle.make_golden_discobox_loss import case
    _, _, _, _, _, boxes, labels, masks, img = case(0)
    img = img.float().to(DEV)
    boxes = [b.to(DEV) for b in boxes]
    labels = [l.to(DEV) for l in labels]
    masks = [torch.from_numpy(m).to(DEV) for m in masks]
    det = _stand_in(12999, 0.3)
    ref = copy.deepcopy(det)
    ref.ref_avg = 0.3
    opt = torch.optim.SGD([p for p in det.parameters()], lr=0.01)
    ropt = torch.optim.SGD([p for p in ref.parameters()], lr=0.01)
    seen = set()
    cudnn = torch.backends.cudnn.deterministic
    torch.backends.cudnn.deterministic = True
    for step in range(8):
        if step in (2, 5):                                          # drive avg_loss_ins across 0.3 both ways
            det.avg_loss_ins = ref.ref_avg = {2: 0.1, 5: 0.6}[step]
        gates = []
        orig = det.bbox_head.head.loss

        def rec(*a, **kw):
            gates.append((kw['use_loss_ts'], kw['use_ind_teacher']))
            return orig(*a, **kw)
        det.bbox_head.head.loss = rec
        out = det.forward_train(img, [{}] * img.shape[0], boxes, labels, None, masks)
        del det.bbox_head.head.loss
        rout = _ref_forward_train(ref, img, [{}] * img.shape[0], boxes, labels, None, masks)
        assert gates[0] == ref.ref_gates
        seen.add(gates[0])
        assert (det.cnt, det.turn_on_teacher) == (ref.cnt, ref.turn_on_teacher)
        assert det.avg_loss_ins == ref.ref_avg
        assert out.keys() == rout.keys()
        for k in out:
            assert torch.equal(out[k], rout[k]), (step, k)
        assert_same_state(det.tsw.teacher, ref.tsw.teacher)
        assert_same_state(det, ref)
        for o, l in ((opt, out), (ropt, rout)):
            o.zero_grad()
            sum(v for v in l.values()).backward()
            o.step()
        assert_same_state(det, ref)
    torch.backends.cudnn.deterministic = cudnn
    assert seen == {(False, False), (True, False), (True, True), (False, True)}
    assert det.turn_on_teacher


def test_forward_train_glue_adds_no_host_sync():
    """Under sync-debug mode a step's glue adds no flagged call beyond those of the head's loss: the one event wait is on
    the previous step's avg_loss_ins."""
    import warnings
    from boxinstseg_b200.models.detectors import discobox as D
    from oracle.make_golden_discobox_loss import case
    _, _, _, _, _, boxes, labels, masks, img = case(0)
    img = img.float().to(DEV)
    boxes, labels = [b.to(DEV) for b in boxes], [l.to(DEV) for l in labels]
    masks = [torch.from_numpy(m).to(DEV) for m in masks]
    det = _stand_in(13005, 0.25)
    det.forward_train(img, [{}] * 2, boxes, labels, None, masks)      # first step: pinned buffer, pairing, turn-on
    det.forward_train(img, [{}] * 2, boxes, labels, None, masks)
    head = det.bbox_head
    metas = [{}] * 2

    def counted(fn):
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as seen:
            warnings.simplefilter('always')
            torch.cuda.set_sync_debug_mode('warn')
            try:
                fn()
            finally:
                torch.cuda.set_sync_debug_mode('default')
        return sum('called a synchronizing' in str(w.message) for w in seen)
    x = det.extract_feat(img)
    outs = head(x)
    with torch.no_grad():
        tx = det.tsw.teacher.extract_feat(img)
        t_k = det.tsw.teacher.bbox_head(tx)[1]
        t_in = det.tsw.teacher.mask_feat_head(tx[0:4])
    loss_only = counted(lambda: head.loss(*outs, t_k, det.mask_feat_head(x[0:4]), t_in, boxes, labels, masks, metas, None,
                                          img=img, use_loss_ts=True, use_ind_teacher=True, use_corr=False, s_feat=x[0:4],
                                          t_feat=tx[0:4]))
    step = counted(lambda: det.forward_train(img, metas, boxes, labels, None, masks))
    assert step == loss_only
    ev = det.__dict__['_bxs_avg_event']
    waits = []
    orig = torch.cuda.Event.synchronize

    def spy(self):
        waits.append(self is ev)
        return orig(self)
    torch.cuda.Event.synchronize = spy
    try:
        det.forward_train(img, metas, boxes, labels, None, masks)
    finally:
        torch.cuda.Event.synchronize = orig
    assert sum(waits) == 1                                           # one wait, on the event the previous step recorded
    assert D._avg_read(det) == det.avg_loss_ins
