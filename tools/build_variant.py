"""Build an A/B variant of the library with extra -D flags:  python tools/build_variant.py <name> [--src=PATTERN] -DBXS_WQ_R=16 ...
   -> boxinstseg_b200/lib/libboxseg_b200_<name>.so   (run with BXS_LIB_PATH=...).  Only sources whose name contains PATTERN
   (default "onepass") are recompiled with the flags; the others reuse the main build's objects."""
import os, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from boxinstseg_b200 import build as B
name, flags = sys.argv[1], sys.argv[2:]
pattern = 'onepass'
for f in list(flags):
    if f.startswith('--src='):
        pattern = f[6:]
        flags.remove(f)
out = os.path.join(B.LIBDIR, f'libboxseg_b200_{name}.so')
od = os.path.join(B.LIBDIR, 'obj_' + name)
os.makedirs(od, exist_ok=True)
objs = []
for src in B.sources():
    obj = os.path.join(od, os.path.basename(src)[:-3] + '.o')
    base = os.path.join(B.LIBDIR, 'obj', os.path.basename(src)[:-3] + '.o')
    if pattern in os.path.basename(src):
        subprocess.run([B._nvcc()] + B.NVCC_FLAGS + flags + ['-c', src, '-o', obj], check=True)
        objs.append(obj)
    else:
        objs.append(base)          # unchanged sources: reuse the main build's objects
subprocess.run([B._nvcc(), '-shared', '-o', out] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'], check=True)
print(out)
