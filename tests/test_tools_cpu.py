"""CPU: the measurement scripts under tools/ import without a GPU, and time, count and label their numbers through the one
harness in tools/benchkit.py instead of a copy of their own."""
import ast
import glob
import importlib
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOLS = os.path.join(ROOT, 'tools')
# bench_ops.py and bench_f_rows.py run their work when imported; the duplication check below still covers them
RUN_AT_IMPORT = {'bench_ops', 'bench_f_rows'}
HARNESS = re.compile(r'(card|timed|time_call|timeit|syncs|count_syncs|launches|profile|graph_\w*|host_ms|summary)')


def _scripts(pattern):
    return sorted(glob.glob(os.path.join(TOOLS, pattern)))


def _guarded_benches():
    names = []
    for path in _scripts('bench_*.py'):
        name = os.path.splitext(os.path.basename(path))[0]
        with open(path) as f:
            if name not in RUN_AT_IMPORT and "__name__ == '__main__'" in f.read():
                names.append(name)
    return names


@pytest.mark.parametrize('name', _guarded_benches())
def test_bench_imports_without_running(name, monkeypatch):
    monkeypatch.syspath_prepend(TOOLS)
    monkeypatch.syspath_prepend(ROOT)
    monkeypatch.delitem(sys.modules, name, raising=False)
    importlib.import_module(name)


@pytest.mark.parametrize('path', _scripts('*.py'), ids=os.path.basename)
def test_no_harness_copy_outside_benchkit(path):
    """A function named like a harness helper, at any depth, belongs in benchkit.py alone."""
    if os.path.basename(path) == 'benchkit.py':
        return
    with open(path) as f:
        tree = ast.parse(f.read(), path)
    copies = [f'{n.name} (line {n.lineno})' for n in ast.walk(tree)
              if isinstance(n, (ast.FunctionDef, ast.AsyncFunctionDef)) and HARNESS.fullmatch(n.name)]
    assert not copies, f'{os.path.basename(path)} defines its own {", ".join(copies)}: use tools/benchkit.py'


def test_benchkit_imports_only_torch_and_the_standard_library():
    with open(os.path.join(TOOLS, 'benchkit.py')) as f:
        tree = ast.parse(f.read())
    roots = set()
    for n in ast.walk(tree):
        if isinstance(n, ast.Import):
            roots |= {a.name.split('.')[0] for a in n.names}
        elif isinstance(n, ast.ImportFrom):
            roots.add((n.module or '').split('.')[0] if n.level == 0 else '.')
    assert all(r == 'torch' or r in sys.stdlib_module_names for r in roots), roots
