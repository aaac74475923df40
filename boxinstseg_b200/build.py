"""In-tree build of libboxseg_b200.so (sm_90a, H100) with nvcc; no torch involved.

    python -m boxinstseg_b200.build [--force] [--verbose]

Objects are cached per source under ``boxinstseg_b200/lib/obj`` keyed on the source + header
mtimes, so an incremental rebuild recompiles only what changed.
"""
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
LIBDIR = os.path.join(HERE, 'lib')
LIB = os.path.join(LIBDIR, 'libboxseg_b200.so')
INCLUDE = os.path.join(os.path.dirname(HERE), 'include')

NVCC_FLAGS = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17',
              '-Xcompiler', '-fPIC', '--expt-relaxed-constexpr', '-I', INCLUDE]


def _nvcc():
    return shutil.which('nvcc') or '/usr/local/cuda/bin/nvcc'


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith('.cu'))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(('.cuh', '.h'))]
    hs += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE)]
    return max(os.path.getmtime(h) for h in hs)


def build(force=False, verbose=False):
    os.makedirs(os.path.join(LIBDIR, 'obj'), exist_ok=True)
    hdr = _headers_mtime()
    jobs, objs = [], []
    for src in sources():
        obj = os.path.join(LIBDIR, 'obj', os.path.basename(src)[:-3] + '.o')
        objs.append(obj)
        stale = force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(src), hdr)
        if stale:
            cmd = [_nvcc()] + NVCC_FLAGS + (['-Xptxas', '-v'] if verbose else []) + ['-c', src, '-o', obj]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError('nvcc failed: ' + ' '.join(cmd) + '\n' + r.stdout + r.stderr)
        return r.stderr

    with ThreadPoolExecutor(max_workers=min(8, max(1, len(jobs)))) as ex:
        for log in ex.map(run, jobs):
            if verbose and log:
                print(log)
    if jobs or force or not os.path.exists(LIB):
        run([_nvcc(), '-shared', '-o', LIB] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    return LIB


if __name__ == '__main__':
    print(build(force='--force' in sys.argv, verbose='--verbose' in sys.argv))
