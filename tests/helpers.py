"""Shared helpers for the GPU parity tests: seeded synthetic inputs (SURVEY.md section 8d)."""
import numpy as np
import torch
import torch.nn.functional as F

MEAN = [123.675, 116.28, 103.53]
STD = [58.395, 57.12, 57.375]


def synth_image(gen, h, w, lowres=32, noise=8.0):
    """uint8-valued RGB [3,h,w] float32: low-frequency field + N(0,noise) noise."""
    coarse = torch.rand(1, 3, max(h // lowres, 2), max(w // lowres, 2), generator=gen) * 255
    img = F.interpolate(coarse, size=(h, w), mode='bilinear', align_corners=False)[0]
    return (img + torch.randn(3, h, w, generator=gen) * noise).clamp(0, 255).floor()


def normalise(raw):
    return (raw - torch.tensor(MEAN).view(3, 1, 1)) / torch.tensor(STD).view(3, 1, 1)


def make_meta(ih, iw, ori_scale=1.0):
    return dict(img_shape=(ih, iw, 3), ori_shape=(int(ih * ori_scale), int(iw * ori_scale), 3),
                img_norm_cfg=dict(mean=np.array(MEAN, dtype=np.float32), std=np.array(STD, dtype=np.float32),
                                  to_rgb=True))


def synth_boxes(gen, num, hp, wp, lo=48, hi=400):
    hi_w, hi_h = min(hi, wp - 1), min(hi, hp - 1)
    w = torch.rand(num, generator=gen) * (hi_w - min(lo, hi_w)) + min(lo, hi_w)
    h = torch.rand(num, generator=gen) * (hi_h - min(lo, hi_h)) + min(lo, hi_h)
    x1 = torch.rand(num, generator=gen) * (wp - w)
    y1 = torch.rand(num, generator=gen) * (hp - h)
    return torch.stack([x1, y1, x1 + w, y1 + h], 1).float()


def boxinst_case(seed, B, hp, wp, gts_per_img, inst_per_gt, logit_std=2.0, ragged=False, lowres=32, noise=8.0):
    """Inputs of one BoxInst mask-loss step (config A when B=2, 800x1024, 8 GT, 8 inst/GT)."""
    gen = torch.Generator().manual_seed(seed)
    imgs, metas = [], []
    for b in range(B):
        ih, iw = (hp, wp) if not (ragged and b % 2) else (hp - 8 * (b % 3 + 1), wp - 12)
        raw = synth_image(gen, ih, iw, lowres, noise)
        imgs.append(F.pad(normalise(raw), (0, wp - iw, 0, hp - ih)))
        metas.append(make_meta(ih, iw, ori_scale=1.0 if not ragged else 1.7))
    img = torch.stack(imgs)
    gt_bboxes = [synth_boxes(gen, gts_per_img, hp, wp, hi=min(400, hp // 2)) for _ in range(B)]
    gt_inds = torch.arange(B * gts_per_img).repeat_interleave(inst_per_gt)
    img_inds = gt_inds // gts_per_img
    n = gt_inds.numel()
    logits = torch.randn(n, 1, hp // 4, wp // 4, generator=gen) * logit_std
    return dict(img=img, metas=metas, gt_bboxes=gt_bboxes, gt_inds=gt_inds, img_inds=img_inds, logits=logits)


def rel_err(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def scaled_err(got, ref):
    """Element-wise: max |got - ref| / (|ref| + 1e-2 max |ref|).  Unlike ``rel_err`` a single wrong element of a large
    tensor shows: one element off by 1 % of the tensor's largest value already scores 0.5."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    if ref.numel() == 0:
        return 0.0
    floor = 1e-2 * ref.abs().max().item() + 1e-300
    return ((got - ref).abs() / (ref.abs() + floor)).max().item()


# significand bits after the point, and log2 of the smallest subnormal spacing
_HALF_BITS = {torch.float16: (10, -24), torch.bfloat16: (7, -133)}


def ulp_half(ref, dt):
    """Element-wise spacing of ``dt`` (float16 / bfloat16) at |ref|, floored at the type's smallest subnormal spacing:
    the unit in which a result rounded once to ``dt`` is judged against its float64 reference ``ref``."""
    bits, sub = _HALF_BITS[dt]
    ref = ref.detach().double().cpu()
    _, e = torch.frexp(ref)                                        # |ref| = m 2^e, m in [0.5, 1)
    ulp = torch.ldexp(torch.ones_like(ref), e - 1 - bits)
    return torch.where(ref == 0, torch.zeros_like(ref), ulp).clamp(min=2.0 ** sub)


def tied_logits(n, h, w, dt, kind, gen):
    """[n,h,w] 16-bit logits whose rounded sigmoids tie a lot: 'saturated' (every third row s == 1.0), 'quantised'
    (multiples of 1/2), 'constant', or 'boundaries' (equal maxima on both sides of every 16-row and 256-column
    boundary)."""
    x = torch.randn(n, h, w, generator=gen) * 3
    if kind == 'saturated':
        x[:, ::3] = 9.5 + torch.rand(n, len(range(0, h, 3)), w, generator=gen) * 4     # fp16 / bf16 s == 1.0
    elif kind == 'quantised':
        x = torch.round(x * 2) / 2
    elif kind == 'constant':
        x = torch.full((n, h, w), 0.375)
    elif kind == 'boundaries':
        x = torch.randn(n, h, w, generator=gen) - 4
        for y in range(15, h - 1, 16):
            x[:, y:y + 2, ::7] = 2.0
        for c in range(255, w - 1, 256):
            x[:, ::5, c:c + 2] = 2.0
    return x.to(dt)


def host_twin(name):
    """Compiles tests/host_harness/<name>.cpp -- the HOST build of the very header a kernel is made of -- with g++ and
    returns the ctypes handle (test infrastructure: lets the CPU suite check a kernel's arithmetic and indexing bit for bit
    against the oracle on a box without a GPU; the product library exports only the CUDA path)."""
    import ctypes
    import os
    import subprocess
    import tempfile
    here = os.path.dirname(os.path.abspath(__file__))
    src = os.path.join(here, 'host_harness', name + '.cpp')
    out = os.path.join(tempfile.gettempdir(), f'bxs_{name}_{os.getuid()}_{int(os.path.getmtime(src))}.so')
    core = os.path.join(here, '..', 'boxinstseg_b200', 'csrc')
    newest = max(os.path.getmtime(os.path.join(core, f)) for f in os.listdir(core) if f.endswith('.cuh'))
    if not os.path.exists(out) or os.path.getmtime(out) < max(newest, os.path.getmtime(src)):
        subprocess.run(['g++', '-O2', '-std=c++17', '-ffp-contract=off', '-fPIC', '-shared', '-x', 'c++', src, '-o', out],
                       check=True)
    return ctypes.CDLL(out)
