"""Runs GPU test files under the guard-band allocator of tests/guard_alloc/guard_alloc.cu, in a process of its own:

    python -m tests.guarded_run [--list] [--json SUMMARY] tests/test_x_gpu.py ... [-- extra pytest arguments]

Every CUDA allocation of the process gets a 4 KiB front guard and a tail guard of at least 64 KiB that starts at exactly
the tensor's last byte + 1, and the whole block starts out filled with the pattern 0xFFA5 (a NaN in every float type).
After every call of a compute entry point of the C ABI, and after each phase of each test, the guards of every live
and freed block are checked.  So a kernel that writes past its output or workspace fails the test that called it, with
the entry point, the allocation's size, the guard side and the offset named; an output element a kernel never writes
holds NaN instead of whatever the caching allocator happened to hand back.

The allocator must be installed before the first CUDA allocation, hence the separate process.  Tests that capture CUDA
graphs or read the caching allocator's statistics cannot run on a pluggable allocator; they are found from their source
and skipped with the reason.  --list only collects: it prints what would run and what would be skipped, and touches no
device.  The run writes a JSON summary (tests run and failed, skips with reasons, violations, entry points called)."""
import ctypes
import inspect
import json
import os
import re
import subprocess
import sys
import tempfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
SOURCE = os.path.join(HERE, 'guard_alloc', 'guard_alloc.cu')
NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O2', '-std=c++17', '-Xcompiler', '-fPIC', '-shared']

STATE = None           # the running State, for the harness's own tests

# Entry points that only answer a question about sizes or the device and launch nothing.
QUERIES = {'bxs_version', 'bxs_device_sm_count', 'bxs_last_error'}

SKIPS = [
    (re.compile(r'torch\.cuda\.graph\b|CUDAGraph'), 'captures a CUDA graph, which a pluggable allocator cannot host'),
    (re.compile(r'\b(memory_allocated|max_memory_allocated|reset_peak_memory_stats|memory_stats|memory_reserved)\b'),
     "reads the caching allocator's statistics, which a pluggable allocator does not keep"),
]


def is_query(name):
    return name in QUERIES or name.endswith('_bytes') or name.endswith('_supported')


def compute_entry_points(signatures=None):
    """Sorted names of the C ABI's compute entry points: every ``bxs_*`` function of the header except the size and
    capability queries."""
    if signatures is None:
        from boxinstseg_b200 import _lib
        signatures = _lib.SIGNATURES
    return sorted(n for n in signatures if not is_query(n))


def skip_reason(fn):
    """Why the test function ``fn`` cannot run under the guard allocator, from its source; None when it can."""
    try:
        src = inspect.getsource(fn)
    except (OSError, TypeError):
        return None
    for pattern, reason in SKIPS:
        if pattern.search(src):
            return reason
    return None


def write_summary(path, summary):
    with open(path, 'w') as f:
        json.dump(summary, f, indent=1, sort_keys=True)


def read_summary(path):
    with open(path) as f:
        return json.load(f)


def allocator_path():
    """The guard allocator's shared object, compiled with nvcc on first use and cached in the temporary directory (keyed
    by user and source time), as tests/helpers.py:host_twin does for the host harnesses."""
    out = os.path.join(tempfile.gettempdir(), f'bxs_guard_alloc_{os.getuid()}_{int(os.path.getmtime(SOURCE))}.so')
    if not os.path.exists(out):
        import shutil
        nvcc = shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'
        tmp = f'{out}.{os.getpid()}.tmp'
        subprocess.run([nvcc] + NVCC_FLAGS + [SOURCE, '-o', tmp], check=True)
        os.replace(tmp, out)
    return out


class _Violation(ctypes.Structure):
    _fields_ = [('seq', ctypes.c_int64), ('size', ctypes.c_int64), ('first', ctypes.c_int64), ('last', ctypes.c_int64),
                ('side', ctypes.c_int32), ('nfound', ctypes.c_int32), ('found', ctypes.c_uint8 * 16)]


class Guard:
    """The loaded allocator: installs itself as torch's CUDA allocator and reads its checks back."""

    def __init__(self, path):
        import torch
        self.so = ctypes.CDLL(path)
        self.so.guard_check.restype = ctypes.c_int
        self.so.guard_report.restype = ctypes.c_int64
        self.so.guard_report.argtypes = [ctypes.c_void_p, ctypes.c_int64]
        self.so.guard_stats.argtypes = [ctypes.c_void_p]
        self.so.guard_scribble_for_test.argtypes = [ctypes.c_void_p, ctypes.c_int64, ctypes.c_int]
        self.so.guard_tail_bytes.restype = ctypes.c_int64
        self.so.guard_tail_bytes.argtypes = [ctypes.c_void_p]
        self.so.guard_last_error.restype = ctypes.c_char_p
        alloc = torch.cuda.memory.CUDAPluggableAllocator(path, 'guard_malloc', 'guard_free')
        torch.cuda.memory.change_current_allocator(alloc)
        self.seen = 0

    def check(self):
        """Records of the violations found since the last call (a device synchronise and one check kernel)."""
        if self.so.guard_check() < 0:
            raise RuntimeError('guard check failed: ' + self.so.guard_last_error().decode())
        n = self.so.guard_report(None, 0)
        recs = (_Violation * n)()
        self.so.guard_report(recs, n)
        new = [dict(seq=r.seq, size=r.size, side=('front', 'tail')[r.side], first=r.first, last=r.last,
                    found=bytes(r.found[:r.nfound]).hex()) for r in recs[self.seen:n]]
        self.seen = n
        return new

    def stats(self):
        out = (ctypes.c_int64 * 6)()
        self.so.guard_stats(out)
        return dict(zip(['live_blocks', 'live_bytes', 'quarantined_blocks', 'quarantined_bytes', 'allocations',
                         'pooled_bytes'], out))

    def scribble(self, t, offset, value):
        """Sets the guard byte at ``offset`` bytes from tensor t's first byte (test support for the harness itself)."""
        if self.so.guard_scribble_for_test(ctypes.c_void_p(t.data_ptr()), offset, value) != 0:
            raise ValueError(f'offset {offset} is not a guard byte of this allocation')

    def tail_bytes(self, t):
        return self.so.guard_tail_bytes(ctypes.c_void_p(t.data_ptr()))


def describe(v):
    where = (f'{v["first"] - v["size"]} bytes past the end' if v['side'] == 'tail'
             else f'{-v["first"]} bytes before the start')
    return (f'{v["test"]}: guard violation after {v["entry"]}: allocation #{v["seq"]} of {v["size"]} bytes, {v["side"]} '
            f'guard, first corrupted byte at offset {v["first"]} ({where}), last at {v["last"]}, found {v["found"]}')


class State:
    """What the proxy and the plugin share: the guard, the test running now, the violations and the entry points."""

    def __init__(self, guard):
        self.guard = guard
        self.test = None
        self.violations = []
        self.called = set()

    def check(self, entry):
        new = self.guard.check()
        for v in new:
            v.update(test=self.test, entry=entry)
        self.violations += new
        return new


class GuardedLib:
    """Stands in for the ctypes handle of libboxseg_b200.so: every compute entry point runs, then the guards are checked,
    so that a violation is blamed on the entry point that made it.  Under torch.profiler the check waits for the end of
    the test phase, so that traces hold the library's launches alone."""

    def __init__(self, handle, state):
        self._handle = handle
        self._state = state

    def __getattr__(self, name):
        fn = getattr(self._handle, name)
        if not name.startswith('bxs_') or is_query(name):
            return fn
        state = self._state

        def call(*args):
            rc = fn(*args)
            if rc == 0:
                state.called.add(name)
            import torch
            if not torch._C._autograd._profiler_enabled():
                state.check(name)
            return rc
        call.__name__ = name
        setattr(self, name, call)
        return call


class GuardPlugin:
    """pytest plugin: skips the tests the allocator cannot host, checks the guards after every test phase, turns a
    violation into a failure of the phase it was found in, and keeps the summary."""

    def __init__(self, state=None):
        self.state = state
        self.skipped = {}
        self.outcomes = {}

    def pytest_configure(self, config):
        config.addinivalue_line('markers', 'gpu: needs a CUDA device')

    @pytest.hookimpl(tryfirst=True)
    def pytest_collection_modifyitems(self, items):
        for item in items:
            reason = skip_reason(getattr(item, 'function', None))
            if reason:
                item.add_marker(pytest.mark.skip(reason='under the guard allocator: test ' + reason))
                self.skipped[item.nodeid] = reason

    def pytest_runtest_logstart(self, nodeid, location):
        if self.state is not None:
            self.state.test = nodeid

    @pytest.hookimpl(hookwrapper=True)
    def pytest_runtest_makereport(self, item, call):
        outcome = yield
        rep = outcome.get_result()
        if self.state is None or rep.skipped:
            return
        self.state.check(f'the test code ({call.when})')
        mine = [v for v in self.state.violations if v['test'] == item.nodeid and not v.get('reported')]
        if mine:
            for v in mine:
                v['reported'] = True
            text = '\n'.join(describe(v) for v in mine)
            rep.longrepr = (str(rep.longrepr) + '\n' + text) if rep.failed else text
            rep.outcome = 'failed'

    def pytest_runtest_logreport(self, report):
        if report.failed:
            self.outcomes[report.nodeid] = 'failed'
        elif self.outcomes.get(report.nodeid) != 'failed' and (report.when == 'call' or report.skipped):
            self.outcomes[report.nodeid] = report.outcome

    def summary(self, files, exitstatus):
        s = self.state
        return dict(files=list(files), exitstatus=int(exitstatus),
                    passed=sorted(k for k, o in self.outcomes.items() if o == 'passed'),
                    failed=sorted(k for k, o in self.outcomes.items() if o == 'failed'),
                    skipped=dict(sorted(self.skipped.items())),
                    violations=[{k: v for k, v in x.items() if k != 'reported'} for x in (s.violations if s else [])],
                    entry_points=sorted(s.called) if s else [])


def main(argv):
    import argparse
    if '--' in argv:
        i = argv.index('--')
        argv, extra = argv[:i], argv[i + 1:]
    else:
        extra = []
    ap = argparse.ArgumentParser(prog='python -m tests.guarded_run')
    ap.add_argument('files', nargs='+')
    ap.add_argument('--list', action='store_true', help='collect only: print the tests that would run and be skipped')
    ap.add_argument('--json', default=None, help='where to write the JSON summary')
    args = ap.parse_args(argv)
    base = ['-m', 'gpu', '-p', 'no:cacheprovider', '-q'] + extra + args.files

    if args.list:
        plugin = GuardPlugin()
        selected = []

        class Collected:
            def pytest_collection_finish(self, session):
                selected.extend(item.nodeid for item in session.items)
        rc = pytest.main(['--collect-only'] + base, plugins=[plugin, Collected()])
        for nodeid in selected:
            if nodeid in plugin.skipped:
                print(f'skip {nodeid}: {plugin.skipped[nodeid]}')
            else:
                print(f'run  {nodeid}')
        print(f'{len(selected) - len(plugin.skipped)} to run, {len(plugin.skipped)} to skip')
        return int(rc)

    global STATE
    guard = Guard(allocator_path())                     # before anything allocates on the device
    from boxinstseg_b200 import _lib
    state = STATE = State(guard)
    _lib._lib = GuardedLib(_lib.lib(), state)
    plugin = GuardPlugin(state)
    rc = pytest.main(base, plugins=[plugin])
    summary = plugin.summary(args.files, rc)
    summary['stats'] = guard.stats()
    write_summary(args.json or os.path.join(tempfile.gettempdir(), f'bxs_guarded_run_{os.getpid()}.json'), summary)
    for v in summary['violations']:
        print(describe(v))
    return int(rc) if rc or not summary['violations'] else 1


if __name__ == '__main__':
    from tests import guarded_run       # the importable module holds the state that the tests under guard can reach
    sys.exit(guarded_run.main(sys.argv[1:]))
