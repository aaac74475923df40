"""Launch paths that only large or unusual inputs select, each judged element-wise against a float64 oracle.

Several entry points choose their kernel from the input shape and the SM count:
  * LCM (lcm.cu): one CTA per instance with phi in shared memory (``lcm_fused_kernel``) when n >= 2 * SMs and
    2*h*w*4 bytes fit 200 KB, grid-wide rounds (``lcm_step_global``) otherwise;
  * mean field (meanfield.cu): compile-time 3x3 taps or generic ``kernel_size`` taps (``mf_fused_kernel<0,..>``,
    ``mf_step_global<0,..>``); per-object CTAs when n >= 2 * SMs or no workspace is given and both bit maps fit 200 KB;
  * CondInst head (condinst_head.cu): ``head_{fwd,bwd}_kernel<32>`` for 17..32 mask-feature channels; the backward splits
    each image's instances into SM-derived groups unless B*C*h*w is not a multiple of 4;
  * dense projection (projection_levelset.cu): the column maxima are taken over row segments whose height follows from
    n * w and the SM count.
Every case below restates its dispatch rule and asserts the side it lands on; the SM count is read from the library, so
the cases keep their meaning on any H100 variant.  test_profiler_sees_the_dispatched_kernel then confirms once per path,
with torch.profiler, that the rule's restatement picks the kernel that actually runs, so that a later dispatch change
cannot silently turn a case into a duplicate of another test.

Element-wise bars: ``scaled_err`` = max |got - ref| / (|ref| + 1e-2 max |ref|) over all elements.  The largest value
observed on an H100 80GB HBM3 (SXM, 132 SMs, 400 W power limit) is given next to each bar.
"""
import functools
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import boxinst as ob
from oracle import levelset as ol
from tests.helpers import scaled_err

pytestmark = pytest.mark.gpu
DEV = 'cuda:0'
FUSED_SMEM = 200 * 1024                       # kMaxFusedSmem of lcm.cu and meanfield.cu

# element-wise bars (scaled_err) and, in the comments, the largest value observed over all cases (H100 SXM, see above)
TOL_LCM_AFF = 5e-4         # affinities (see check_lcm)                  1.1e-4 (160x161)
TOL_LCM_PHI = 1e-5         # refined map phi_T                           2.0e-6
TOL_LCM_GRAD = 1e-3        # d loss / d phi_0                            4.9e-4 (3x2, d 3, 10 iterations: 18 pixels);
                           #                                             2.7e-4 on the other maps
TOL_LCM_LOSS = 2e-4        # the loss (relative)                         6.5e-5 (3x2, d 3, 10 iterations)
TOL_HEAD_OUT = 3e-5        # CondInst head logits                        7.8e-6 (config A)
TOL_HEAD_GFEAT = 3e-5      # d / d mask features                         9.4e-6 (config A)
TOL_HEAD_GPARAMS = 3e-5    # d / d dynamic parameters                    9.3e-6 (C = 32)
TOL_PRJ_GRAD = 2e-5        # dense projection d / d scores               4.7e-6
MF_MISMATCH = 2e-5         # mean field: flipped pseudo-label pixels     0 (expf differs from the CPU libm by <= 2 ulp,
                           # so exact ties may flip; the bar is the one of tests/test_losses_gpu.py)


@functools.lru_cache(maxsize=None)
def sms():
    from boxinstseg_b200 import _lib as L
    n = L.lib().bxs_device_sm_count()
    assert n > 0
    return n


def check_close(name, got, ref, tol):
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    err = scaled_err(got, ref)
    print(f'[elementwise] {name}: {err:.3e} (bar {tol:.0e})')
    assert err <= tol, (name, err)


def twice(fn):
    """fn() run twice; the two results must be bit-identical (every path here is deterministic)."""
    first, second = fn(), fn()
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    return second


# ================================================================== A. LCM
def lcm_per_instance(n, h, w):
    """bxs_lcm_forward / bxs_lcm_backward: one CTA per instance iff both phi buffers fit and n fills the SMs twice."""
    return 2 * h * w * 4 <= FUSED_SMEM and n >= 2 * sms()


def lcm_inputs(n, C, h, w, seed, fractional=True, flat=True):
    gen = torch.Generator().manual_seed(seed)
    imgs = torch.rand(n, C, h, w, generator=gen)
    phis = torch.rand(n, 1, h, w, generator=gen)
    if flat and h >= 4 and w >= 4:
        # zero-padded borders: the standard deviation is 0 and the 1e-8 term decides; with phi constant there too, deep
        # inside phi_T == phi_0 exactly, where d|x| takes sign(0) = 0
        for t, v in ((imgs, 0.0), (phis, 0.5)):
            t[..., (3 * h) // 4:, :] = v
            t[..., :, (3 * w) // 4:] = v
    if fractional:                                             # box masks bilinearly resized, as _scale_target makes them
        lo = torch.zeros(n, 1, 7, 9)
        for i in range(n):
            y0, x0 = int(torch.randint(0, 4, (1,), generator=gen)), int(torch.randint(0, 5, (1,), generator=gen))
            lo[i, 0, y0:y0 + 4, x0:x0 + 5] = 1
        box = F.interpolate(lo, size=(h, w), mode='bilinear', align_corners=False)
    else:
        box = (torch.rand(n, 1, h, w, generator=gen) > 0.4).float()
    return imgs, phis, box


def run_lcm(imgs, phis, box, d, iters, g_up=1.7):
    """(loss, d (g_up * loss) / d phi, phi_T) on the device, through _LCM and LocalConsistencyModule; run twice,
    bit-identical."""
    from boxinstseg_b200.models.losses import LocalConsistencyModule
    from boxinstseg_b200.models.losses.levelset_loss import _LCM
    im, bx = imgs.to(DEV), box.to(DEV)

    def once():
        pg = phis.to(DEV).requires_grad_(True)
        loss = _LCM.apply(im, pg, bx, d, iters)
        (g,) = torch.autograd.grad(loss * g_up, pg)
        return loss.detach(), g
    loss, g = twice(once)
    phi_t = LocalConsistencyModule(dilations=[d], num_iter=iters)(im, phis.to(DEV))
    return loss, g, phi_t


def lcm_kernel_affinity(imgs, d):
    """The float32 affinities [n,1,8,h,w] bxs_lcm_forward leaves at the head of its workspace (affinity_kernel runs
    before, and independently of, the choice of schedule)."""
    from boxinstseg_b200 import _lib as L
    n, C, h, w = imgs.shape
    im = imgs.to(DEV).contiguous()
    ones = torch.ones(n, 1, h, w, device=DEV)
    out = torch.zeros(1, device=DEV)
    lib = L.lib()
    ws = torch.empty(lib.bxs_lcm_workspace_bytes(n, h, w), dtype=torch.uint8, device=DEV)
    L.check(lib.bxs_lcm_forward(L.ptr(im), L.ptr(ones), L.ptr(ones), L.ptr(out), L.ptr(ws), n, C, h, w, d, 0, L.stream()),
            'lcm_forward')
    return ws.view(torch.float32)[:n * 8 * h * w].view(n, 1, 8, h, w).clone()


def lcm_oracle(aff, phis, box, d, iters, phi_t, g_up=1.7):
    """float64 loss, refined map and gradient of the propagation with the given affinities [n,1,8,h,w] (widened
    exactly).  d|x| = sign(x) is taken with the sign of the kernel's own phi_T - phi_0 (exact in float32): where
    |phi_T - phi_0| is within rounding of 0 the two precisions may pick different signs, which is a property of the loss,
    not an error of the kernel; those places are checked to be within rounding of 0."""
    a, b = aff.to(DEV).double(), box.to(DEV).double()
    p = phis.to(DEV).double().requires_grad_(True)
    refined = p
    for _ in range(iters):                                     # oracle.levelset.lcm_refine with these affinities
        refined = (ol._replicate_neighbours(refined, d) * a).sum(2)
    z = b.sum().clamp(min=1)
    loss = ((refined - p).abs() * b).sum() / z
    sgn = torch.sign(phi_t.double() - phis.to(DEV).double())
    (g,) = torch.autograd.grad(g_up * ((refined - p) * sgn * b).sum() / z, p)
    flip = sgn != torch.sign(refined.detach() - p.detach())
    assert ((refined.detach() - p.detach())[flip].abs() <= 1e-5).all()
    return loss.detach(), g, refined.detach()


def check_lcm(tag, imgs, phis, box, d, iters, want_per_instance):
    """The kernel's affinities against oracle.levelset.lcm_affinity, then loss, phi_T and gradient against the float64
    propagation of those affinities.  The affinity is a softmax of -z^2 with z = |dI| / std / 0.3: where the standard
    deviation of a neighbourhood is small its logits are large and float32 resolves them only to |logit| * 6e-8, which
    no kernel can beat; the propagation and its transpose, which are what the two schedules implement, are judged on
    their own."""
    n, _, h, w = phis.shape
    assert lcm_per_instance(n, h, w) == want_per_instance, (n, h, w, sms())
    loss, g, phi_t = run_lcm(imgs, phis, box, d, iters)
    aff = lcm_kernel_affinity(imgs, d)
    check_close(f'{tag} affinity', aff, ol.lcm_affinity(imgs.to(DEV).double(), d), TOL_LCM_AFF)
    o_loss, o_g, o_phi = lcm_oracle(aff, phis, box, d, iters, phi_t)
    if iters == 0:
        assert float(loss) == 0.0 and not g.any() and torch.equal(phi_t.cpu(), phis)
        return
    print(f'[elementwise] {tag} loss: {abs(float(loss) / float(o_loss) - 1):.3e} (bar {TOL_LCM_LOSS:.0e})')
    assert abs(float(loss) - float(o_loss)) <= TOL_LCM_LOSS * abs(float(o_loss)), (float(loss), float(o_loss))
    check_close(f'{tag} phi_T', phi_t, o_phi, TOL_LCM_PHI)
    check_close(f'{tag} grad', g, o_g, TOL_LCM_GRAD)


def test_lcm_cross_schedule_bit_for_bit():
    """lcm.cu: both schedules run the same per-pixel arithmetic.  K real instances with 0/1 boxes alone (grid-wide
    rounds), then scattered among all-zero-box pads up to 2 * SMs + 3 instances (one CTA per instance).  The pads add
    exact zeros to the numerator and to the integer box sum, so the gradient scale is the same float: phi_T and the
    gradient of the real instances must be bit-identical, the pads' gradient exactly 0."""
    from boxinstseg_b200.models.losses import LocalConsistencyModule
    K, h, w = 5, 96, 96
    n = 2 * sms() + 3
    imgs, phis, box = lcm_inputs(K, 3, h, w, seed=1, fractional=False)
    loss_a, g_a, phi_a = run_lcm(imgs, phis, box, 2, 10)
    assert not lcm_per_instance(K, h, w) and lcm_per_instance(n, h, w)
    gen = torch.Generator().manual_seed(2)
    pos = torch.randperm(n, generator=gen)[:K].sort()[0]
    pos[-1] = n - 1                                            # the last CTA holds a real instance
    P_imgs, P_phis, P_box = torch.rand(n, 3, h, w, generator=gen), torch.rand(n, 1, h, w, generator=gen), torch.zeros(n, 1, h, w)
    P_imgs[pos], P_phis[pos], P_box[pos] = imgs, phis, box
    loss_b, g_b, phi_b = run_lcm(P_imgs, P_phis, P_box, 2, 10)
    assert torch.equal(phi_a, phi_b[pos.to(DEV)])
    assert torch.equal(g_a, g_b[pos.to(DEV)])
    pad = torch.ones(n, dtype=torch.bool)
    pad[pos] = False
    assert (g_b[pad.to(DEV)] == 0).all()
    # the loss: per-instance sums over 1024 vs 256 threads, so rounding may differ
    print(f'[elementwise] lcm cross-schedule loss: {abs(float(loss_b) / float(loss_a) - 1):.3e} (bar 1e-6)')
    assert abs(float(loss_a) - float(loss_b)) <= 1e-6 * abs(float(loss_a)), (float(loss_a), float(loss_b))   # observed: equal
    # LocalConsistencyModule reads the same phi_T
    assert torch.equal(LocalConsistencyModule([2], 10)(imgs.to(DEV), phis.to(DEV)), phi_a)


LCM_SHAPES = [(96, 96, True), (17, 23, True), (1, 7, True), (2, 2, True),
              (160, 160, True),                                # 2*h*w*4 == 200 KB exactly: still one CTA per instance
              (160, 161, False)]                               # one column more: grid-wide even with many instances


@pytest.mark.parametrize('h,w,per_instance', LCM_SHAPES, ids=[f'{h}x{w}' for h, w, _ in LCM_SHAPES])
def test_lcm_many_instances_vs_oracle(h, w, per_instance):
    n = 2 * sms() + 3
    imgs, phis, box = lcm_inputs(n, 3, h, w, seed=h * 1000 + w)
    check_lcm(f'lcm {h}x{w} n={n}', imgs, phis, box, 2, 10, per_instance)


@pytest.mark.parametrize('iters', [0, 1, 10])
@pytest.mark.parametrize('d', [1, 2, 3])
@pytest.mark.parametrize('many', [False, True], ids=['grid', 'per_instance'])
def test_lcm_dilation_and_iterations(many, d, iters):
    """num_iter 0 (a copy on the grid-wide path, an empty loop per instance: loss and gradient exactly 0), 1 and 10;
    dilations 1-3 through _LCM and LocalConsistencyModule; a 3x2 map smaller than dilation 3 next to the 24x29 one."""
    n = 2 * sms() + 3 if many else 3
    for h, w in ((24, 29), (3, 2)):
        imgs, phis, box = lcm_inputs(n, 3, h, w, seed=d * 100 + iters + h)
        check_lcm(f'lcm {h}x{w} d={d} it={iters} n={n}', imgs, phis, box, d, iters, many)


# ================================================================== B. mean field
MF_CFG = dict(theta0=0.5, theta1=30, theta2=10, iter=10, base=0.1)


def mf_alpha0(ks):
    """DiscoBox's alpha0 = 2 at 3x3, scaled by 9 / k^2 for larger kernels.  Unscaled, 25 or 49 taps drive both energies
    past exp's float32 range: f_fg = f_bg = 1e-6 nearly everywhere, and the pseudo-label is decided by ties that even
    float32 and float64 evaluations of the oracle break differently (2.7 % of the pixels at k = 5)."""
    return 2.0 * min(1.0, 9.0 / ks ** 2)


def mf_smem(h, w):
    return 2 * ((h * w + 15) // 16) * 16


def mf_per_object(n, h, w, workspace):
    """bxs_meanfield_forward_inter / _logits: one CTA per object iff both bit maps fit and (n fills the SMs twice or
    there is no workspace)."""
    return mf_smem(h, w) <= FUSED_SMEM and (n >= 2 * sms() or not workspace)


def mf_inputs(n, h, w, seed, n_img=2):
    gen = torch.Generator().manual_seed(seed)
    fm = F.interpolate(torch.randn(n_img, 3, max(h // 8, 2), max(w // 8, 2), generator=gen), size=(h, w), mode='bilinear')
    fm = fm + torch.randn(n_img, 3, h, w, generator=gen) * 0.1
    x = torch.rand(n, 1, h, w, generator=gen)
    t = torch.zeros(n, 1, h, w)
    for i in range(n):
        y0, x0 = int(torch.randint(0, max(h // 2, 1), (1,), generator=gen)), int(torch.randint(0, max(w // 2, 1), (1,), generator=gen))
        y1 = y0 + 1 + int(torch.randint(0, h - y0, (1,), generator=gen))
        x1 = x0 + 1 + int(torch.randint(0, w - x0, (1,), generator=gen))
        t[i, 0, y0:y1, x0:x1] = 1
    obj_img = (torch.arange(n) * 7 % n_img).to(torch.int32)
    return fm, x, t, obj_img


def run_mf_inter(mf, x, t, obj_img, workspace):
    """bxs_meanfield_forward_inter on the device -> (ret, valid); run twice, bit-identical."""
    from boxinstseg_b200 import _lib as L
    n, _, h, w = x.shape
    xs, tg, oi = x.to(DEV).contiguous(), t.to(DEV).contiguous(), obj_img.to(DEV).contiguous()
    ret, valid = torch.empty_like(xs), torch.empty(n, device=DEV)
    lib = L.lib()
    ws = torch.empty(lib.bxs_meanfield_workspace_bytes(n, h, w), dtype=torch.uint8, device=DEV) if workspace else None

    def call():
        L.check(lib.bxs_meanfield_forward_inter(L.ptr(mf.kernel), L.ptr(oi), L.ptr(xs), L.ptr(tg), None, 0.0,
                                                mf._neglog.ctypes.data, L.ptr(ret), L.ptr(valid), L.ptr(ws), n, h, w,
                                                mf.kernel_size, mf.iter, L.stream()), 'meanfield_forward_inter')
        return ret.clone(), valid.clone()
    return twice(call)


def mf_oracle(kernel, x, t, obj_img, ks):
    """oracle.levelset.meanfield_forward per image, on the device in float32 (the reference's own precision)."""
    ret = torch.empty(x.shape, device=DEV)
    valid = torch.empty(x.shape[0], device=DEV)
    for b in range(kernel.shape[0]):
        sel = (obj_img == b).to(DEV)
        if sel.any():
            ret[sel], valid[sel] = ol.meanfield_forward(kernel[b:b + 1].flatten(2), x.to(DEV)[sel], t.to(DEV)[sel], ks, 10, 0.1)
    return ret, valid


MF_SHAPES = [(1, 40, 50), (3, 40, 50), (5, 40, 50), (7, 40, 50), (7, 3, 4), (1, 3, 4), (5, 1, 9),
             (5, 320, 320),                                    # 2 * 102400 bytes == 200 KB: per-object CTAs fit
             (5, 320, 321),                                    # one column more: grid-wide rounds only
             (3, 320, 320)]


@pytest.mark.parametrize('ks,h,w', MF_SHAPES, ids=[f'k{k}-{h}x{w}' for k, h, w in MF_SHAPES])
def test_meanfield_schedules_and_taps(ks, h, w):
    """Many objects with a workspace, few with a workspace, few without: bit-identical where they overlap (both schedules
    call the same mf_update), and each against the float32 oracle and the bilateral kernel against its oracle."""
    from boxinstseg_b200._lib import BoxSegError
    from boxinstseg_b200.models.dense_heads import MeanField
    n, K = 2 * sms() + 3, 5
    fm, x, t, obj_img = mf_inputs(n, h, w, seed=ks * 7 + h + w)
    mf = MeanField(fm.to(DEV), kernel_size=ks, alpha0=mf_alpha0(ks), **MF_CFG)
    k64 = ol.meanfield_kernel(fm, ks, 0.5, 30.0, mf_alpha0(ks))
    assert torch.allclose(mf.kernel.flatten(2).cpu(), k64, rtol=1e-5, atol=1e-9)
    fits = mf_smem(h, w) <= FUSED_SMEM
    runs = {}
    for tag, m, ws in (('many+ws', n, True), ('few+ws', K, True), ('few-ws', K, False)):
        per_obj = mf_per_object(m, h, w, ws)
        assert per_obj == (fits and tag != 'few+ws')
        if not ws and not fits:
            with pytest.raises(BoxSegError, match='invalid argument'):
                run_mf_inter(mf, x[:m], t[:m], obj_img[:m], ws)
            continue
        ret, valid = run_mf_inter(mf, x[:m], t[:m], obj_img[:m], ws)
        runs[tag] = (ret, valid)
    o_ret, o_valid = mf_oracle(mf.kernel, x, t, obj_img, ks)
    ret, valid = runs['many+ws']
    mism = (ret != o_ret).float().mean().item()
    print(f'[mismatch] meanfield k={ks} {h}x{w} n={n}: {mism:.2e} (bar {MF_MISMATCH:.0e})')
    assert mism <= MF_MISMATCH, mism
    assert torch.equal(valid, o_valid)
    assert 0 < int(ret.sum()) < int(t.sum())
    for tag, (r, v) in runs.items():
        assert torch.equal(r, ret[:r.shape[0]]) and torch.equal(v, valid[:v.shape[0]]), tag
    # MeanField itself: its normal route (a workspace) with many objects
    ps, va = mf(x.to(DEV), t.to(DEV), obj_img=obj_img.to(DEV))
    assert torch.equal(ps, ret) and torch.equal(va, valid)


@pytest.mark.parametrize('teacher', [False, True])
@pytest.mark.parametrize('dt', [torch.float16, torch.bfloat16])
def test_meanfield_logits_generic_taps(dt, teacher):
    """bxs_meanfield_forward_logits at kernel size 5 on all three schedules, against MeanField.forward on ((t + s) / 2)
    (bit for bit) and the float32 oracle of tests/discobox_half_oracle.pseudo_label."""
    from boxinstseg_b200 import _lib as L
    from boxinstseg_b200.models.dense_heads import MeanField
    from boxinstseg_b200.ops.discobox import HALF_DTYPES
    from tests.discobox_half_oracle import pseudo_label
    ks, h, w = 5, 48, 64
    n, K = 2 * sms() + 3, 5
    fm, _, t, obj_img = mf_inputs(n, h, w, seed=11)
    gen = torch.Generator().manual_seed(12)
    xs = (torch.randn(n, h, w, generator=gen) * 0.8).to(dt)
    xt = (torch.randn(n, h, w, generator=gen) * 0.8).to(dt) if teacher else None
    tg = t[:, 0].to(torch.uint8)
    mf = MeanField(fm.to(DEV), kernel_size=ks, alpha0=mf_alpha0(ks), **MF_CFG)
    lib = L.lib()
    outs = {}
    for tag, m, ws in (('many+ws', n, True), ('few+ws', K, True), ('few-ws', K, False)):
        s, tt, tgd, oi = xs[:m].to(DEV), None if xt is None else xt[:m].to(DEV), tg[:m].to(DEV), obj_img[:m].to(DEV)
        wsb = torch.empty(lib.bxs_meanfield_workspace_bytes(m, h, w), dtype=torch.uint8, device=DEV) if ws else None
        out = torch.empty(m, h, w, dtype=torch.uint8, device=DEV)

        def call():
            L.check(lib.bxs_meanfield_forward_logits(L.ptr(mf.kernel), L.ptr(oi), L.ptr(s), L.ptr(tt), L.ptr(tgd), HALF_DTYPES[dt],
                                                     mf._neglog.ctypes.data, L.ptr(out), L.ptr(wsb), m, h, w, ks, mf.iter,
                                                     L.stream()), 'meanfield_forward_logits')
            return (out.clone(),)
        (out,) = twice(call)
        assert mf_per_object(m, h, w, ws) == (tag != 'few+ws')
        outs[tag] = out
    ref = outs['many+ws']
    for tag, out in outs.items():
        assert torch.equal(out, ref[:out.shape[0]]), tag
    s16 = torch.sigmoid(xs.to(DEV))
    t16 = s16 if xt is None else torch.sigmoid(xt.to(DEV))
    want, _ = mf(((t16 + s16) / 2).float().unsqueeze(1), tg.to(DEV).float().unsqueeze(1), obj_img=obj_img.to(DEV))
    assert torch.equal(ref, want[:, 0].to(torch.uint8))
    kernels = [mf.kernel[b:b + 1].flatten(2).cpu() for b in range(mf.kernel.shape[0])]
    o = pseudo_label(s16.cpu(), tg, kernels, obj_img, None if xt is None else t16.cpu(), kernel_size=ks)
    mism = (ref.cpu() != o).float().mean().item()
    print(f'[mismatch] meanfield logits {dt} teacher={teacher}: {mism:.2e} (bar {MF_MISMATCH:.0e})')
    assert mism <= MF_MISMATCH and 0 < int(o.sum()) < int(tg.sum())


# ================================================================== C. CondInst dynamic mask head
def head_groups(N, B, h, w):
    """bwd_groups of condinst_head.cu: ~4 CTAs per SM, at most 8, at most ceil(N / B)."""
    tiles = -(-h // 8) * -(-w // 32)
    want = -(-4 * sms() // (tiles * B))
    return max(1, min(want, 8, -(-N // B)))


def _off_kink(pre, margin):
    """Bias shifts [N,8] that move every value of pre [N,8,m] at least `margin` away from 0: a channel that comes closer
    is shifted by minus the midpoint of the widest gap between its values near 0."""
    shift = torch.zeros(pre.shape[:2], dtype=torch.float64)
    for n, j in (pre.abs() < margin).any(2).nonzero().tolist():
        v = pre[n, j]
        v = torch.cat([v[v.abs() < 0.05], torch.tensor([-0.05, 0.05], dtype=torch.float64)]).sort()[0]
        k = int((v[1:] - v[:-1]).argmax())
        shift[n, j] = -(v[k] + v[k + 1]) / 2
    return shift


def head_problem(B, C, h, w, N, rel, seed, margin=1e-4):
    """Inputs whose layer-1 / layer-2 pre-activations all stay `margin` away from the ReLU kink (the biases of the
    channels that come closer are shifted into a gap of their values), so that float32 and float64 take the same branch
    everywhere and every gradient element can be judged."""
    gen = torch.Generator().manual_seed(seed)
    cin = C + (2 if rel else 0)
    P = cin * 8 + 64 + 8 + 8 + 8 + 1
    feat = torch.randn(B, C, h, w, generator=gen)
    params = torch.randn(N, P, generator=gen) * 0.3
    coors = torch.rand(N, 2, generator=gen) * torch.tensor([w * 8.0, h * 8.0])
    levels = torch.randint(0, 5, (N,), generator=gen)
    img_inds = torch.sort(torch.randint(0, B, (N,), generator=gen))[0]
    x = feat.double()[img_inds].flatten(2)
    if rel:                                                        # locations and relative coordinates as the head forms them
        xs = torch.arange(w, dtype=torch.float64) * 8 + 4
        ys = torch.arange(h, dtype=torch.float64) * 8 + 4
        soi = torch.tensor([64, 128, 256, 512, 1024], dtype=torch.float64)[levels].view(N, 1, 1)
        rx = ((coors[:, 0].double().view(N, 1, 1) - xs.view(1, 1, w)).expand(N, h, w) / soi).flatten(1)
        ry = ((coors[:, 1].double().view(N, 1, 1) - ys.view(1, h, 1)).expand(N, h, w) / soi).flatten(1)
        x = torch.cat([rx[:, None], ry[:, None], x], 1)
    o_b1 = cin * 8 + 64 + 8
    w1 = params[:, :cin * 8].double().view(N, 8, cin)
    w2 = params[:, cin * 8:cin * 8 + 64].double().view(N, 8, 8)

    def pre1():
        return torch.bmm(w1, x) + params[:, o_b1:o_b1 + 8].double()[:, :, None]

    def pre2():
        return torch.bmm(w2, pre1().clamp(min=0)) + params[:, o_b1 + 8:o_b1 + 16].double()[:, :, None]
    for layer, pre, off in ((1, pre1, o_b1), (2, pre2, o_b1 + 8)):
        for _ in range(3):
            v = pre()
            if not (v.abs() < margin).any():
                break
            params[:, off:off + 8] += _off_kink(v, margin).float()
        assert not (pre().abs() < margin).any(), f'layer {layer}: could not move the pre-activations off the ReLU kink'
    return feat, params, coors, levels, img_inds


def run_head(feat, params, coors, levels, img_inds, g_out, rel, in_stride=8, out_stride=4):
    from boxinstseg_b200.ops.condinst import dynamic_mask_head
    soi = torch.tensor([64, 128, 256, 512, 1024], device=DEV)

    def once():
        f = feat.to(DEV).requires_grad_(True)
        p = params.to(DEV).requires_grad_(True)
        out = dynamic_mask_head(f, p, coors.to(DEV), levels.to(DEV), img_inds.to(DEV), soi, in_stride, out_stride,
                                rel_coors=rel)
        gf, gp = torch.autograd.grad((out * g_out.to(DEV)).sum(), [f, p])
        return out.detach(), gf, gp
    return twice(once)


def head_cmax(C):
    """the head_{fwd,bwd}_kernel instantiation bxs_condinst_head_* launch for C mask-feature channels"""
    return 8 if C <= 8 else (16 if C <= 16 else 32)


def check_head(tag, B, C, h, w, N, rel, seed, want_groups=None):
    groups = head_groups(N, B, h, w)
    vec4 = (B * C * h * w) % 4 == 0
    use_groups = groups if vec4 else 1
    if want_groups is not None:
        assert use_groups == want_groups(groups), (groups, vec4)
    feat, params, coors, levels, img_inds = head_problem(B, C, h, w, N, rel, seed)
    g_out = torch.randn(N, 1, 2 * h, 2 * w, generator=torch.Generator().manual_seed(seed + 1))
    out, gf, gp = run_head(feat, params, coors, levels, img_inds, g_out, rel)
    f64 = feat.double().requires_grad_(True)
    p64 = params.double().requires_grad_(True)
    ref = ob.condinst_mask_head(f64, p64, coors.double(), levels, img_inds, 8, 4, rel_coors=rel)
    rf, rp = torch.autograd.grad((ref * g_out.double()).sum(), [f64, p64])
    check_close(f'{tag} out', out, ref, TOL_HEAD_OUT)
    check_close(f'{tag} g_feat', gf, rf, TOL_HEAD_GFEAT)
    check_close(f'{tag} g_params', gp, rp, TOL_HEAD_GPARAMS)


@pytest.mark.parametrize('rel', [True, False], ids=['rel', 'norel'])
@pytest.mark.parametrize('C', [17, 24, 32])
def test_head_wide_channels(C, rel):
    """head_{fwd,bwd}_kernel<32>: 17..32 mask-feature channels, cin up to 34 with the relative coordinates."""
    check_head(f'head C={C} rel={rel}', 2, C, 13, 40, 9, rel, seed=C * 2 + rel)


@pytest.mark.parametrize('B,C,h,w,N', [(1, 3, 9, 11, 6), (3, 5, 7, 13, 8), (1, 17, 9, 11, 5)])
def test_head_backward_unvectorised(B, C, h, w, N):
    """B*C*h*w not a multiple of 4: the instance groups the SM count asks for are dropped, one group writes d/d feat."""
    assert (B * C * h * w) % 4 != 0 and head_groups(N, B, h, w) > 1
    check_head(f'head B={B} C={C} {h}x{w}', B, C, h, w, N, True, seed=B * 100 + C, want_groups=lambda g: 1)


def test_head_backward_config_a():
    """Config A's whole backward: feat [2,16,100,128], N = 128, 200x256 logits; 52 tiles x 2 images, SM-derived groups."""
    assert head_groups(128, 2, 100, 128) > 1
    check_head('head config A', 2, 16, 100, 128, 128, True, seed=5, want_groups=lambda g: g)


# ================================================================== D. dense projection
def prj_segments(n, h, w):
    """bxs_projection_loss_forward: (rows_per_seg, segs) of prj_cols_kernel."""
    segs = min(-(-h // 8), max(1, -(-(sms() * 8 * 256) // (n * w))))
    rows = -(-h // segs)
    return rows, -(-h // rows)


def planted_scores(n, h, w, rows, seed):
    """Scores in [0, 1) with exact column-maximum ties planted across every computed segment boundary (rows b-1 / b and
    b-3 / b+5), inside the first and last segments, and -0.0 / +0.0 ties in all-negative columns; the first row must win."""
    gen = torch.Generator().manual_seed(seed)
    s = torch.rand(n, 1, h, w, generator=gen)
    bounds = list(range(rows, h, rows))
    pairs = [(b - 1, b) for b in bounds] + [(b - 3, b + 5) for b in bounds if b >= 3 and b + 5 < h]
    pairs += [(0, min(1, h - 1)), (max(h - 2, 0), h - 1), (0, h - 1)]
    col = 0
    for y0, y1 in pairs:
        if y0 == y1:
            continue
        for c in (col % w, (col + 1) % w):                     # a value tie, then a signed-zero tie in the next column
            s[:, 0, :, c] = torch.rand(n, h, generator=gen) * 0.5
        s[:, 0, y0, col % w] = s[:, 0, y1, col % w] = 2.0
        c = (col + 1) % w
        s[:, 0, :, c] = -(torch.rand(n, h, generator=gen) + 0.5)
        s[:, 0, y0, c], s[:, 0, y1, c] = -0.0, 0.0
        col += 3
    assert col < w
    return s


@pytest.mark.parametrize('case', ['segments', 'single'])
def test_dense_projection_segments(case):
    from boxinstseg_b200.models.losses import projection_losses
    if case == 'segments':
        n, h, w = 128, 200, 256                                    # config A's instance maps
        rows, segs = prj_segments(n, h, w)
        assert rows != 8 and segs > 1, (rows, segs)
    else:
        h, w = 40, 256
        n = -(-(sms() * 8 * 256) // w)                             # n * w >= SMs * 8 * 256: one segment
        rows, segs = prj_segments(n, h, w)
        assert segs == 1 and rows == h
    s = planted_scores(n, h, w, rows, seed=n + h)
    gen = torch.Generator().manual_seed(3)
    t = (torch.rand(n, 1, h, w, generator=gen) > 0.6).float()
    gl = torch.rand(n, generator=gen)
    s64 = s.double().requires_grad_(True)
    ref = 2.5 * ob.projection_losses(s64, t.double())
    (gref,) = torch.autograd.grad((ref * gl.double()).sum(), s64)

    def once():
        sg = s.to(DEV).requires_grad_(True)
        out = projection_losses(sg, t.to(DEV), 1e-5, 2.5)
        (gs,) = torch.autograd.grad((out * gl.to(DEV)).sum(), sg)
        return out.detach(), gs
    out, gs = twice(once)
    assert torch.allclose(out.cpu().double(), ref.detach(), rtol=1e-5, atol=1e-6)
    check_close(f'projection {case} n={n} rows_per_seg={rows}', gs, gref, TOL_PRJ_GRAD)
    assert torch.equal(gs.cpu() != 0, gref != 0)                   # the support: first-row arg-max of every column


# ================================================================== which kernel each path runs
# Kernel records are matched by name; anything else in a trace (runtime calls, memcpy / memset records) is ignored.
LIBRARY_KERNEL = re.compile(r'\b(affinity_kernel|lcm_\w+|mf_\w+|head_\w+_kernel|group_by_image|feat_reduce_kernel|'
                            r'params_reduce_kernel|prj_\w+_kernel)\b')


def traced_library_kernels(fn, expected):
    """Names of the library kernels fn launches, from torch.profiler.  fn runs once untraced first, so that module loading
    is not part of the trace.  Every trace is preceded by an empty one that takes any record still pending from earlier
    work, so a late record of another path cannot appear in fn's trace.  The kernel records of a trace arrive
    asynchronously and are occasionally incomplete: a trace that lacks an `expected` kernel is retaken, up to 5 times
    (a kernel that is never launched fails all of them)."""
    from torch.profiler import ProfilerActivity, profile
    activities = [ProfilerActivity.CPU, ProfilerActivity.CUDA]
    fn()
    for _ in range(5):
        torch.cuda.synchronize()
        with profile(activities=activities):
            torch.cuda.synchronize()
        with profile(activities=activities) as prof:
            fn()
            torch.cuda.synchronize()
        everything = {e.name for e in prof.events()}
        names = {n for n in everything if LIBRARY_KERNEL.search(n)}
        if all(any(re.search(p, n) for n in names) for p in expected):
            break
    else:
        print('[kernels] every record of the last trace:', sorted(everything))
    return names


def _tpl(kernel, *args):
    """pattern of a kernel template instantiation, e.g. _tpl('mf_fused_kernel', 0, '__half') -> mf_fused_kernel<0, __half"""
    parts = [rf'(\(int\))?{a}' if isinstance(a, int) else re.escape(a) for a in args]
    return kernel + '<' + r'\s*,\s*'.join(parts) + (r'>' if len(args) == 1 and isinstance(args[0], int) else r'\b')


def _lcm_path(n, h, w):
    from boxinstseg_b200.models.losses.levelset_loss import _LCM
    imgs, phis, box = lcm_inputs(n, 3, h, w, seed=7)
    im, bx = imgs.to(DEV), box.to(DEV)

    def fn():
        pg = phis.to(DEV).requires_grad_(True)
        torch.autograd.grad(_LCM.apply(im, pg, bx, 2, 3), pg)
    fused = lcm_per_instance(n, h, w)
    on = [_tpl('lcm_fused_kernel', 0), _tpl('lcm_fused_kernel', 1)]
    off = [_tpl('lcm_step_global', 0), _tpl('lcm_step_global', 1)]
    return fn, (on, off) if fused else (off, on)


def _mf_path(ks, n, h, w, workspace, logits=None):
    from boxinstseg_b200.models.dense_heads import MeanField
    fm, x, t, obj_img = mf_inputs(n, h, w, seed=3)
    mf = MeanField(fm.to(DEV), kernel_size=ks, alpha0=mf_alpha0(ks), **MF_CFG)
    per_obj = mf_per_object(n, h, w, workspace)
    taps = 3 if ks == 3 else 0
    if logits is None:
        fn = lambda: run_mf_inter(mf, x, t, obj_img, workspace)               # noqa: E731
        on, off = _tpl('mf_fused_kernel', taps, 'float'), _tpl('mf_step_global', taps, 'float')
    else:
        from boxinstseg_b200 import _lib as L
        from boxinstseg_b200.ops.discobox import HALF_DTYPES
        lib = L.lib()
        s, tg, oi = x[:, 0].to(logits).to(DEV), t[:, 0].to(torch.uint8).to(DEV), obj_img.to(DEV)
        ws = torch.empty(lib.bxs_meanfield_workspace_bytes(n, h, w), dtype=torch.uint8, device=DEV) if workspace else None
        out = torch.empty(n, h, w, dtype=torch.uint8, device=DEV)

        def fn():
            L.check(lib.bxs_meanfield_forward_logits(L.ptr(mf.kernel), L.ptr(oi), L.ptr(s), None, L.ptr(tg), HALF_DTYPES[logits],
                                                     mf._neglog.ctypes.data, L.ptr(out), L.ptr(ws), n, h, w, ks, mf.iter,
                                                     L.stream()), 'meanfield_forward_logits')
            # a trace whose only GPU work is this one kernel has been seen to come back without its kernel record once other
            # tests have run in the process; a device copy after it, as every other path here has, keeps it
            return out.clone()
        half = '__half' if logits == torch.float16 else '__nv_bfloat16'
        on, off = _tpl('mf_fused_kernel', taps, half), _tpl('mf_step_global', taps, 'unsigned char')
    return fn, ([on], [off]) if per_obj else ([off], [on])


def _head_path(B, C, h, w, N):
    feat, params, coors, levels, img_inds = head_problem(B, C, h, w, N, True, seed=1)
    g_out = torch.randn(N, 1, 2 * h, 2 * w, generator=torch.Generator().manual_seed(2))
    fn = lambda: run_head(feat, params, coors, levels, img_inds, g_out, True)        # noqa: E731
    cm = head_cmax(C)
    on = [_tpl('head_fwd_kernel', cm), _tpl('head_bwd_kernel', cm)]
    off = [_tpl(k, c) for k in ('head_fwd_kernel', 'head_bwd_kernel') for c in (8, 16, 32) if c != cm]
    grouped = (B * C * h * w) % 4 == 0 and head_groups(N, B, h, w) > 1
    return fn, (on + ['feat_reduce_kernel'], off) if grouped else (on, off + ['feat_reduce_kernel'])


def _prj_path(n, h, w):
    from boxinstseg_b200.models.losses import projection_losses
    s = torch.rand(n, 1, h, w, generator=torch.Generator().manual_seed(4)).to(DEV).requires_grad_(True)
    t = (torch.rand(n, 1, h, w, generator=torch.Generator().manual_seed(5)) > 0.6).float().to(DEV)
    return (lambda: torch.autograd.grad(projection_losses(s, t).sum(), s)), (['prj_cols_kernel'], [])


def _paths():
    many = 2 * sms() + 3
    return {
        'lcm-per-instance-17x23': lambda: _lcm_path(many, 17, 23),
        'lcm-per-instance-160x160': lambda: _lcm_path(many, 160, 160),
        'lcm-grid-few-17x23': lambda: _lcm_path(3, 17, 23),
        'lcm-grid-many-160x161': lambda: _lcm_path(many, 160, 161),
        'mf-k5-per-object-many': lambda: _mf_path(5, many, 40, 50, True),
        'mf-k5-grid-few': lambda: _mf_path(5, 5, 40, 50, True),
        'mf-k5-per-object-no-workspace': lambda: _mf_path(5, 5, 40, 50, False),
        'mf-k3-per-object-many': lambda: _mf_path(3, many, 40, 50, True),
        'mf-k5-per-object-320x320': lambda: _mf_path(5, many, 320, 320, True),
        'mf-k5-grid-many-320x321': lambda: _mf_path(5, many, 320, 321, True),
        'mf-logits-fp16-k5-per-object-many': lambda: _mf_path(5, many, 48, 64, True, torch.float16),
        'mf-logits-bf16-k5-grid-few': lambda: _mf_path(5, 5, 48, 64, True, torch.bfloat16),
        'head-C24-grouped': lambda: _head_path(2, 24, 13, 40, 9),
        'head-C17-unvectorised': lambda: _head_path(1, 17, 9, 11, 5),
        'head-config-a': lambda: _head_path(2, 16, 100, 128, 128),
        'projection-segments': lambda: _prj_path(128, 200, 256),
    }


PATHS = ['lcm-per-instance-17x23', 'lcm-per-instance-160x160', 'lcm-grid-few-17x23', 'lcm-grid-many-160x161',
         'mf-k5-per-object-many', 'mf-k5-grid-few', 'mf-k5-per-object-no-workspace', 'mf-k3-per-object-many',
         'mf-k5-per-object-320x320', 'mf-k5-grid-many-320x321', 'mf-logits-fp16-k5-per-object-many',
         'mf-logits-bf16-k5-grid-few', 'head-C24-grouped', 'head-C17-unvectorised', 'head-config-a', 'projection-segments']


def check_every_path():
    """Once per path: the kernels the restated rule predicts are the ones torch.profiler records, and the other side's
    are absent.  Raises on the first path that disagrees."""
    paths = _paths()
    assert set(PATHS) == set(paths)
    for path in PATHS:
        fn, (expected, absent) = paths[path]()
        names = traced_library_kernels(fn, expected)
        print(f'[kernels] {path}: {sorted(names)}', flush=True)
        for p in expected:
            assert any(re.search(p, n) for n in names), (path, 'missing', p, sorted(names))
        for p in absent:
            assert not any(re.search(p, n) for n in names), (path, 'unexpected', p, sorted(names))


def test_profiler_sees_the_dispatched_kernel():
    """check_every_path in a process of its own.  In a process where the rest of the GPU suite has already run, the
    profiler has come back without the kernel record of the per-object logits mean field in five traces in a row (the
    launch itself recorded, the kernel's results checked bit for bit by test_meanfield_logits_generic_taps); in a fresh
    process every path's records arrive."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, '-c', 'from tests.test_dispatch_paths_gpu import check_every_path; check_every_path()'],
                       cwd=root, capture_output=True, text=True, timeout=900)
    print(r.stdout[-6000:])
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-4000:]
    assert r.stdout.count('[kernels] ') == len(PATHS)
