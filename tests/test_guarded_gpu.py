"""GPU: the suite under the guard-band allocator (tests/guarded_run.py).  First the harness's own tests, on a small test
file written here: fresh memory reads back the poison pattern, payloads are 512-byte aligned, a changed guard byte is
reported with the right allocation size, side and offset, a change made just before an entry point is blamed on that
entry point, and a violation fails its test.  Direct tests of the entry points no other GPU test calls.  Then every GPU
test file, each in a process of its own under guard: it passes and reports no violation; and together they call every
compute entry point of the C ABI."""
import ctypes
import os
import re
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

from tests.guarded_run import compute_entry_points, read_summary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THIS = os.path.basename(__file__)
GPU_FILES = sorted(f for f in os.listdir(os.path.join(ROOT, 'tests'))
                   if f.startswith('test_') and f.endswith('_gpu.py') and f != THIS)
DEV = 'cuda'

pytestmark = pytest.mark.gpu


def guarded(files, tmp_path, timeout):
    """(completed process, summary) of one guarded run of `files`."""
    out = str(tmp_path / 'summary.json')
    r = subprocess.run([sys.executable, '-m', 'tests.guarded_run', '--json', out] + list(files), cwd=ROOT,
                       capture_output=True, text=True, timeout=timeout)
    assert os.path.exists(out), r.stdout[-4000:] + r.stderr[-4000:]
    return r, read_summary(out)


SELF_TEST = textwrap.dedent('''
    import pytest
    import torch
    from boxinstseg_b200 import _lib as L
    from tests import guarded_run as G

    DEV = 'cuda'


    def test_fresh_memory_holds_the_poison_and_is_aligned():
        for dt in (torch.float32, torch.float16, torch.bfloat16, torch.int64, torch.uint8):
            for n in (1, 3, 1000, 1 << 20):
                t = torch.empty(n, dtype=dt, device=DEV)
                assert t.data_ptr() % 512 == 0
                raw = t.view(torch.uint8).cpu().numpy().tobytes()
                assert raw == (b'\\xa5\\xff' * len(raw))[:len(raw)], (dt, n)
                if dt.is_floating_point:
                    assert torch.isnan(t).all()
                if dt == torch.int64:
                    assert (t < -(1 << 50)).all()


    def test_payload_is_not_a_guard():
        t = torch.empty(100, dtype=torch.uint8, device=DEV)
        for off in (0, 99, -4097, 100 + G.STATE.guard.tail_bytes(t)):
            with pytest.raises(ValueError):
                G.STATE.guard.scribble(t, off, 0)


    def test_tail_first_byte():
        t = torch.empty(1000, dtype=torch.uint8, device=DEV)
        G.STATE.guard.scribble(t, 1000, 0)


    def test_tail_last_byte():
        t = torch.empty(1001, dtype=torch.uint8, device=DEV)
        G.STATE.guard.scribble(t, 1001 + G.STATE.guard.tail_bytes(t) - 1, 0x5A)


    def test_front_last_byte():
        t = torch.empty(1002, dtype=torch.uint8, device=DEV)
        G.STATE.guard.scribble(t, -1, 0)


    def test_blamed_on_the_next_entry_point():
        rgb = torch.zeros(5, 3, dtype=torch.uint8, device=DEV)
        lab = torch.empty(5, 3, device=DEV)
        G.STATE.guard.scribble(lab, 60 + 8, 0)
        L.check(L.lib().bxs_rgb_u8_to_lab(L.ptr(rgb), L.ptr(lab), 5, L.stream()), 'rgb_u8_to_lab')
        assert torch.isfinite(lab).all()


    def test_clean():
        x = torch.arange(10, device=DEV, dtype=torch.float32)
        assert (x * 2).sum().item() == 90
''')


def test_harness_reports_what_it_is_shown(tmp_path):
    path = tmp_path / 'test_synthetic_guard.py'
    path.write_text(SELF_TEST.replace('def test_', '@pytest.mark.gpu\ndef test_'))
    r, s = guarded([str(path)], tmp_path, timeout=600)
    log = r.stdout[-4000:] + r.stderr[-4000:]
    ran = {k.split('::')[1] for k in s['passed'] + s['failed']}
    assert ran == set(re.findall(r'def (test_\w+)', SELF_TEST)), log
    failed = {k.split('::')[1] for k in s['failed']}
    assert failed == {'test_tail_first_byte', 'test_tail_last_byte', 'test_front_last_byte',
                      'test_blamed_on_the_next_entry_point'}, log
    assert r.returncode != 0
    got = {v['test'].split('::')[1]: v for v in s['violations']}
    assert len(got) == len(s['violations']) == 4, s['violations']
    tail_bytes = got['test_tail_last_byte']['first'] - 1001
    assert tail_bytes >= (64 << 10) - 1
    want = {'test_tail_first_byte': ('the test code (call)', 1000, 'tail', 1000, '00'),
            'test_tail_last_byte': ('the test code (call)', 1001, 'tail', 1001 + tail_bytes, '5a'),
            'test_front_last_byte': ('the test code (call)', 1002, 'front', -1, '00'),
            'test_blamed_on_the_next_entry_point': ('bxs_rgb_u8_to_lab', 60, 'tail', 68, '00')}
    for t, (entry, size, side, first, byte) in want.items():
        v = got[t]
        assert (v['entry'], v['size'], v['side'], v['first'], v['last']) == (entry, size, side, first, first), v
        assert v['found'].startswith(byte), v
    assert 'bxs_rgb_u8_to_lab' in s['entry_points']
    assert 'guard violation after bxs_rgb_u8_to_lab' in r.stdout


# ------------------------------------------------------------------ entry points no other GPU test calls
def _ptrs(ts, ctype=ctypes.c_void_p):
    return (ctype * len(ts))(*[t.data_ptr() if torch.is_tensor(t) else t for t in ts])


@pytest.mark.parametrize('grids, B, C', [((12, 40, 5), 3, 7), ((36,), 1, 80)])
def test_sigmoid_focal_loss_levels_forward_matches_float64(grids, B, C):
    """The square-grid focal loss (the cells form of the same kernel is what the heads call) against its float64 formula,
    at level sizes that end inside a 64-cell tile, with background and out-of-range labels."""
    from boxinstseg_b200 import _lib as L
    gen = torch.Generator().manual_seed(len(grids) * 100 + C)
    gamma, alpha, weight, avg = 2.0, 0.25, 1.5, 17.0
    xs = [torch.randn(B, C, S, S, generator=gen, dtype=torch.float64) * 3 for S in grids]
    ls = [torch.randint(-1, C + 2, (B, S * S), generator=gen) for S in grids]
    dx = [x.float().to(DEV) for x in xs]
    dl = [l.to(DEV) for l in ls]
    grads = [torch.empty_like(x) for x in dx]
    loss = torch.empty((), device=DEV)
    avg_t = torch.tensor(avg, device=DEV)
    n = len(grids)
    grid = (ctypes.c_int64 * n)(*grids)
    lib = L.lib()
    ws = torch.empty(lib.bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(grid, n, B), dtype=torch.uint8, device=DEV)
    L.check(lib.bxs_sigmoid_focal_loss_levels_forward(_ptrs(dx), _ptrs(dl), grid, _ptrs(grads), L.ptr(avg_t), L.ptr(loss),
                                                      L.ptr(ws), n, B, C, gamma, alpha, weight, L.stream()),
            'sigmoid_focal_loss_levels_forward')
    leaves = [x.clone().requires_grad_(True) for x in xs]
    total = 0
    for x, l in zip(leaves, ls):
        cls = torch.arange(C).view(1, C, 1)
        t = (l.view(B, 1, -1) == cls).double()                        # labels outside [0, C): all-negative cells
        z = x.reshape(B, C, -1)
        p = torch.sigmoid(z)
        pt = (1 - p) * t + p * (1 - t)
        bce = torch.nn.functional.binary_cross_entropy_with_logits(z, t, reduction='none')
        total = total + (bce * (alpha * t + (1 - alpha) * (1 - t)) * pt.pow(gamma)).sum()
    ref = total * weight / (avg + float(np.finfo(np.float32).eps))
    ref.backward()
    assert abs(loss.item() - ref.item()) <= 1e-5 * abs(ref.item()), (loss.item(), ref.item())
    for g, x in zip(grads, leaves):
        assert torch.allclose(g.cpu().double(), x.grad, rtol=1e-4, atol=1e-7), (g.cpu().double() - x.grad).abs().max()


@pytest.mark.parametrize('K', [1, 3])
def test_single_query_corr_solve_and_transfer_equal_the_batched_calls(K):
    """bxs_corr_solve and bxs_corr_transfer are the n = 1 cases of the batched entry points that tests/test_corr_gpu.py
    checks against the reference: same tables and transferred maps, bit for bit."""
    from boxinstseg_b200 import _lib as L
    from oracle.make_golden_corr import SOLVER
    gen = torch.Generator().manual_seed(K)
    h = w = 7
    Hm = Wm = 28
    P = h * w
    Cu = (torch.rand(K, P, P, generator=gen) * 2 - 1).to(DEV)
    m0 = torch.rand(Hm * Wm, generator=gen).to(DEV)
    m1 = torch.rand(K, Hm * Wm, generator=gen).to(DEV)
    args = (SOLVER['dist_kernel'], SOLVER['num_iter'], SOLVER['num_smooth_iter'])
    lib = L.lib()
    T1, Tb = torch.empty_like(Cu), torch.empty_like(Cu)
    L.check(lib.bxs_corr_solve(L.ptr(Cu), L.ptr(T1), K, h, w, *args, L.stream()), 'corr_solve')
    L.check(lib.bxs_corr_solve_batched(L.ptr(Cu), L.ptr(Tb), None, 1, K, h, w, *args, L.stream()), 'corr_solve_batched')
    assert torch.isfinite(T1).all() and torch.equal(T1, Tb)
    ws = torch.empty(lib.bxs_corr_transfer_workspace_bytes(K, Hm, Wm), dtype=torch.uint8, device=DEV)
    out = [torch.empty(Hm * Wm, device=DEV) for _ in range(4)]
    L.check(lib.bxs_corr_transfer(L.ptr(T1), L.ptr(Cu), L.ptr(m0), L.ptr(m1), L.ptr(out[0]), L.ptr(out[1]), L.ptr(ws), K,
                                  h, w, Hm, Wm, L.stream()), 'corr_transfer')
    L.check(lib.bxs_corr_transfer_batched(L.ptr(T1), L.ptr(Cu), L.ptr(m0), L.ptr(m1), None, L.ptr(out[2]), L.ptr(out[3]),
                                          L.ptr(ws), 1, K, h, w, Hm, Wm, L.stream()), 'corr_transfer_batched')
    assert all(torch.isfinite(o).all() for o in out)
    assert torch.equal(out[0], out[2]) and torch.equal(out[1], out[3])


@pytest.fixture(scope='module')
def summaries():
    return {}


# every GPU file, and this file's direct tests of the entry points above (not its guarded runs, not the harness test)
@pytest.mark.parametrize('name', GPU_FILES + [THIS])
def test_file_is_clean_under_guard(name, summaries, tmp_path):
    select = ['--', '-k', 'not under_guard and not harness'] if name == THIS else []
    r, s = guarded([os.path.join('tests', name)] + select, tmp_path, timeout=3000)
    summaries[name] = s
    log = r.stdout[-6000:] + r.stderr[-3000:]
    assert not s['violations'], log
    assert r.returncode == 0 and not s['failed'], log
    assert s['passed'] or s['skipped'], log          # every test of test_detector_glue_gpu.py captures a graph


def test_every_compute_entry_point_ran_under_guard(summaries):
    """The union of the entry points the guarded runs called equals the header's compute entry points, so an entry point
    added without a test that reaches it under guard fails here.  Needs this module's guarded runs of every file."""
    assert set(summaries) == set(GPU_FILES + [THIS]), 'run the whole module: the coverage is the union of every file'
    called = set().union(*(s['entry_points'] for s in summaries.values()))
    missing = sorted(set(compute_entry_points()) - called)
    assert not missing, f'compute entry points no guarded test calls: {missing}'
