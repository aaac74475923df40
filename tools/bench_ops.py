"""Per-operator timings on the GPU box at the shapes of SURVEY section 8d (configs C/D/E): dynamic conv (wgmma, forward and
both gradients, against cuBLAS TF32 and FP32), CondInst head, tree filter (MST / BFS / refine), level set (LevelsetLoss on
dense inputs and the fused assembly), projection, LCM, mean field, targets.  Every op is timed twice: eager (launch overhead
included) and as a CUDA-graph replay (`*_graph_us`; device time only).  Prints one JSON object."""
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402
from benchkit import graph_us, time_call  # noqa: E402

dev = torch.device('cuda:0')
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PEAK = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json')))['hbm_gbs'] if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else 3350.0   # H100 SXM data sheet


def eager_us(fn, reps=20, warm=3):
    return time_call(fn, reps=reps, warmup=warm)[0] * 1e3


def both(res, key, fn, reps=20, warm=3):
    res[key + '_us'] = eager_us(fn, reps=reps, warm=warm)
    res[key + '_graph_us'] = graph_us(fn, max(reps // 2, 3), per_graph=4)


res = {}
g = torch.Generator(device=dev).manual_seed(0)
from boxinstseg_b200.ops.dynconv import dynconv1x1  # noqa: E402
for name, (B, C, h, w, I) in dict(box2mask_E=(1, 256, 256, 256, 100), discobox_C=(1, 256, 200, 256, 16),
                                  boxsolo_D_pos100=(2, 256, 200, 256, 100), boxsolo_D_allgrid=(2, 256, 200, 256, 1600)).items():
    feats = [torch.randn(B, C, h, w, device=dev, generator=g) for _ in range(4)]       # rotation of inputs > L2
    kern = torch.randn(B, I, C, device=dev, generator=g) * 0.05
    it = [0]

    def run():
        it[0] += 1
        return dynconv1x1(feats[it[0] % 4], kern)
    us = eager_us(run)
    byts = B * (C * h * w * 4 + I * h * w * 4 + I * C * 4)
    flops = 2.0 * B * I * C * h * w
    entry = dict(us=us, algo_mb=byts / 1e6, gbs=byts / us / 1e3, frac_hbm=byts / us / 1e3 / PEAK, tflops=flops / us / 1e6)
    for tf32 in (False, True):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        entry['cublas_tf32_us' if tf32 else 'cublas_fp32_us'] = eager_us(
            lambda: torch.bmm(kern, feats[it[0] % 4].flatten(2)))
    torch.backends.cuda.matmul.allow_tf32 = False
    res['dynconv_' + name] = entry

from boxinstseg_b200.models import build_head  # noqa: E402
head = build_head(dict(type='CondInstMaskHead', in_channels=16, in_stride=8, out_stride=4, topk_per_img=64, max_proposals=-1,
                       boxinst_enabled=True)).to(dev)
feat = torch.randn(2, 16, 100, 128, device=dev, generator=g).requires_grad_(True)
params = (torch.randn(128, 233, device=dev, generator=g) * 0.3).requires_grad_(True)
coors = torch.rand(128, 2, device=dev, generator=g) * torch.tensor([1024.0, 800.0], device=dev)
levels = torch.randint(0, 5, (128,), device=dev, generator=g)
img_inds = torch.arange(128, device=dev) // 64
both(res, 'condinst_head_fwd', lambda: head(feat, params, coors, levels, img_inds))
out = head(feat, params, coors, levels, img_inds)
gout = torch.randn_like(out)
both(res, 'condinst_head_bwd', lambda: torch.autograd.grad(out, [feat, params], gout, retain_graph=True))

from boxinstseg_b200.ops.tree_filter import MinimumSpanningTree, TreeFilter2D, bfs  # noqa: E402
from boxinstseg_b200.ops.tree_filter.tree_filter_cuda import bfs_order  # noqa: E402
mst, tf = MinimumSpanningTree(TreeFilter2D.norm2_distance), TreeFilter2D()
for name, (n, h, w) in dict(levelset_D_200x256=(16, 200, 256), box2mask_E_96x96=(8, 96, 96)).items():
    guide = F.interpolate(torch.randn(n, 3, h // 8, w // 8, device=dev, generator=g), size=(h, w), mode='bilinear') + \
        0.05 * torch.randn(n, 3, h, w, device=dev, generator=g)
    feat1 = torch.rand(n, 1, h, w, device=dev, generator=g).requires_grad_(True)
    res[f'mst_{name}_us'] = eager_us(lambda: mst(guide), reps=5, warm=1)
    tree = mst(guide)
    res[f'bfs_{name}_us'] = eager_us(lambda: bfs(tree, 4), reps=5, warm=1)
    res[f'treefilter_fwd_{name}_us'] = eager_us(lambda: tf(feat1, guide, tree), reps=5, warm=1)
    o = tf(feat1, guide, tree, low_tree=False)
    res[f'treefilter_bwd_{name}_us'] = eager_us(lambda: torch.autograd.grad(o.sum(), feat1, retain_graph=True),
                                                reps=5, warm=1)
    res[f'tree_levels_{name}'] = int(bfs_order(tree, 4).num_levels.max())

from boxinstseg_b200.models.losses import LCM, LevelsetLoss, projection_losses  # noqa: E402
from boxinstseg_b200.models.losses.levelset_loss import levelset_assembly  # noqa: E402
s = torch.rand(16, 1, 200, 256, device=dev, generator=g).requires_grad_(True)
logit = torch.randn(16, 200, 256, device=dev, generator=g).requires_grad_(True)
t = torch.randn(16, 3, 200, 256, device=dev, generator=g)
m = torch.zeros(16, 1, 200, 256, device=dev)
m[:, :, 40:150, 60:200] = 1
pix = m.sum((1, 2, 3))
ls = LevelsetLoss()
both(res, 'levelset_loss_fwd_bwd', lambda: torch.autograd.grad(ls(torch.cat([s, 1 - s], 1) * m, t * m, pix).sum(), s))
both(res, 'levelset_fused_fwd_bwd', lambda: torch.autograd.grad(levelset_assembly(logit, m, t).sum(), logit))
both(res, 'projection_fwd_bwd', lambda: torch.autograd.grad(projection_losses(s, m).sum(), s))
phi = torch.rand(8, 1, 96, 96, device=dev, generator=g).requires_grad_(True)
img96 = torch.rand(8, 3, 96, 96, device=dev, generator=g)
box96 = torch.zeros(8, 1, 96, 96, device=dev)
box96[:, :, 20:70, 10:80] = 1
both(res, 'lcm_fwd_bwd', lambda: torch.autograd.grad(LCM(img96, phi, box96), phi))
from boxinstseg_b200.models.dense_heads import MeanField  # noqa: E402
cf = torch.randn(1, 3, 200, 256, device=dev, generator=g)
both(res, 'meanfield_kernel', lambda: MeanField(cf, alpha0=2, theta0=0.5, theta1=30, iter=10, base=0.1))
mf = MeanField(cf, alpha0=2, theta0=0.5, theta1=30, iter=10, base=0.1)
x = torch.rand(16, 1, 200, 256, device=dev, generator=g)
tg = torch.zeros(16, 1, 200, 256, device=dev)
tg[:, :, 30:160, 50:220] = 1
both(res, 'meanfield_10it_16obj', lambda: mf(x, tg))
from bench import synthetic_case  # noqa: E402
from boxinstseg_b200.ops.boxinst import boxinst_targets  # noqa: E402
case = synthetic_case(1234)
img = case['img'].to(dev)
boxes = [b.to(dev) for b in case['gt_bboxes']]
both(res, 'boxinst_targets', lambda: boxinst_targets(img, case['metas'], boxes))
print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}, indent=1))
