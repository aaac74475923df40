"""CPU: the host logic of the guarded GPU run (tests/guarded_run.py): the compute entry points it must cover, which
tests it skips and why, the proxy that checks the guards after each entry point, the JSON summary, and that the
allocator compiles for sm_90a."""
import ast
import ctypes
import os
import re
import shutil
import subprocess
import sys

import pytest

from tests import guarded_run as G

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, 'tests')
GPU_FILES = sorted(f for f in os.listdir(TESTS) if f.startswith('test_') and f.endswith('_gpu.py'))


def test_compute_entry_points_are_the_header_minus_its_queries():
    from boxinstseg_b200 import _lib
    with open(_lib.HEADER_PATH) as f:
        declared = set(re.findall(r'\b(bxs_\w+)\s*\(', re.sub(r'/\*.*?\*/', '', f.read(), flags=re.S)))
    eps = G.compute_entry_points()
    assert eps == sorted(eps) and set(eps) <= declared
    queries = declared - set(eps)
    assert all(n.endswith(('_bytes', '_supported')) or n in ('bxs_version', 'bxs_device_sm_count', 'bxs_last_error')
               for n in queries), queries
    # a query returns a size or a flag and takes no stream; every compute entry point launches on a stream it is given
    assert all(_lib.SIGNATURES[n] and _lib.SIGNATURES[n][-1] is ctypes.c_void_p for n in eps)
    assert {'bxs_boxinst_loss_fused_forward', 'bxs_dynconv1x1_forward', 'bxs_lsap_solve', 'bxs_mask_rle_strings'} <= set(eps)
    assert len(eps) >= 70
    assert G.compute_entry_points({'bxs_a_workspace_bytes': [], 'bxs_a': [], 'bxs_b_supported': []}) == ['bxs_a']


def _unhostable_by_ast():
    """(file, test function) pairs whose body captures a CUDA graph or reads allocator statistics, found from the syntax
    tree rather than the runner's text search."""
    stats = {'memory_allocated', 'max_memory_allocated', 'reset_peak_memory_stats', 'memory_stats', 'memory_reserved'}
    found = set()
    for name in GPU_FILES:
        with open(os.path.join(TESTS, name)) as f:
            tree = ast.parse(f.read())
        for fn in tree.body:
            if not (isinstance(fn, ast.FunctionDef) and fn.name.startswith('test_')):
                continue
            for node in ast.walk(fn):
                attr = node.attr if isinstance(node, ast.Attribute) else node.id if isinstance(node, ast.Name) else None
                if attr == 'CUDAGraph' or attr in stats or (
                        attr == 'graph' and isinstance(node, ast.Attribute) and isinstance(node.value, ast.Attribute) and node.value.attr == 'cuda'):
                    found.add((name, fn.name))
    return found


def test_list_skips_exactly_the_graph_and_allocator_statistics_tests():
    """--list collects every GPU file without touching a device and skips exactly the tests a pluggable allocator cannot
    host; everything else it would run."""
    r = subprocess.run([sys.executable, '-m', 'tests.guarded_run', '--list'] + [os.path.join('tests', f) for f in GPU_FILES],
                       cwd=ROOT, capture_output=True, text=True, timeout=600, env=dict(os.environ, CUDA_VISIBLE_DEVICES=''))
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    skipped, ran = {}, set()
    for line in r.stdout.splitlines():
        m = re.match(r'(run|skip) +tests/(\w+\.py)::(\w+)(\[.*\])?(: (.*))?$', line)
        if m:
            key = (m.group(2), m.group(3))
            if m.group(1) == 'skip':
                skipped[key] = m.group(6)
            else:
                ran.add(key)
    assert set(skipped) == _unhostable_by_ast()
    assert not set(skipped) & ran
    assert {f for f, _ in skipped} >= {'test_boxinst_gpu.py', 'test_lsap_gpu.py', 'test_fcos_loss_gpu.py',
                                       'test_fcos_targets_gpu.py', 'test_dynconv_half_gpu.py', 'test_solo_head_gpu.py'}
    assert skipped[('test_solo_head_gpu.py', 'test_head_config_d_vs_reference_lines_dense_path_never_runs')].startswith(
        "reads the caching allocator's statistics")
    assert skipped[('test_boxinst_gpu.py', 'test_single_pass_scheduler_state_is_reusable')].startswith('captures a CUDA graph')
    assert len(ran) > 200


def test_skip_reason_on_source():
    def graph():
        g = torch.cuda.CUDAGraph()          # noqa: F821
        return g

    def stats():
        return torch.cuda.max_memory_allocated()      # noqa: F821

    def plain():
        return torch.cuda.synchronize()       # noqa: F821
    assert G.skip_reason(graph).startswith('captures a CUDA graph')
    assert G.skip_reason(stats).startswith("reads the caching allocator's statistics")
    assert G.skip_reason(plain) is None and G.skip_reason(None) is None


class _FakeGuard:
    def __init__(self):
        self.pending, self.checks = [], 0

    def check(self):
        self.checks += 1
        new, self.pending = self.pending, []
        return new


class _FakeHandle:
    def __init__(self, guard):
        self.guard = guard

    def bxs_ok(self, scribble=False):
        if scribble:
            self.guard.pending.append(dict(seq=7, size=60, side='tail', first=68, last=71, found='00'))
        return 0

    def bxs_invalid(self):
        return -1

    def bxs_x_workspace_bytes(self, n):
        return 4 * n


def test_proxy_checks_after_every_compute_call_and_blames_it():
    guard = _FakeGuard()
    state = G.State(guard)
    state.test = 'tests/test_x_gpu.py::test_y'
    lib = G.GuardedLib(_FakeHandle(guard), state)
    assert lib.bxs_x_workspace_bytes(3) == 12 and guard.checks == 0       # a size query launches nothing: no check
    assert lib.bxs_ok() == 0 and guard.checks == 1 and not state.violations
    assert lib.bxs_invalid() == -1 and guard.checks == 2
    assert lib.bxs_ok(True) == 0 and guard.checks == 3
    assert state.called == {'bxs_ok'}                     # a call rejected before any launch does not count as covered
    (v,) = state.violations
    assert v['entry'] == 'bxs_ok' and v['test'] == 'tests/test_x_gpu.py::test_y'
    text = G.describe(v)
    for part in ('tests/test_x_gpu.py::test_y', 'bxs_ok', '#7 of 60 bytes', 'tail guard', 'offset 68', '8 bytes past the end'):
        assert part in text, text
    front = dict(v, side='front', first=-3)
    assert '3 bytes before the start' in G.describe(front)


def test_summary_round_trips(tmp_path):
    guard = _FakeGuard()
    state = G.State(guard)
    state.test = 't.py::a'
    guard.pending.append(dict(seq=1, size=4, side='front', first=-1, last=-1, found='00'))
    state.check('bxs_z')
    state.called |= {'bxs_z', 'bxs_a'}
    plugin = G.GuardPlugin(state)
    plugin.skipped = {'t.py::g': 'captures a CUDA graph, which a pluggable allocator cannot host'}
    plugin.outcomes = {'t.py::a': 'failed', 't.py::b': 'passed', 't.py::g': 'skipped'}
    s = plugin.summary(['t.py'], 1)
    path = str(tmp_path / 's.json')
    G.write_summary(path, s)
    back = G.read_summary(path)
    assert back == s
    assert back['failed'] == ['t.py::a'] and back['passed'] == ['t.py::b'] and back['entry_points'] == ['bxs_a', 'bxs_z']
    assert back['violations'] == [dict(seq=1, size=4, side='front', first=-1, last=-1, found='00', test='t.py::a',
                                       entry='bxs_z')]


def test_allocator_compiles_for_sm90a_and_exports_its_interface():
    path = G.allocator_path()
    so = ctypes.CDLL(path)                       # the CUDA runtime is linked statically: loads without a device
    for sym in ('guard_malloc', 'guard_free', 'guard_check', 'guard_report', 'guard_stats', 'guard_scribble_for_test',
                'guard_tail_bytes', 'guard_last_error'):
        assert hasattr(so, sym), sym
    cuobjdump = shutil.which('cuobjdump') or '/usr/local/cuda/bin/cuobjdump'
    if os.path.exists(cuobjdump):
        elf = subprocess.run([cuobjdump, '--list-elf', path], capture_output=True, text=True, check=True).stdout
        assert 'sm_90a' in elf, elf
    assert ctypes.sizeof(G._Violation) == 56

