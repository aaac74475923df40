"""ctypes binding of ``libboxseg_b200.so`` (the C ABI declared in ``include/boxseg_b200.h``).

The product path has NO fallback: if the shared library is missing or a call fails, an
exception is raised.  Build with ``python -m boxinstseg_b200.build`` (or ``__graft_entry__.build()``).
"""
import ctypes
import os
import re

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('BXS_LIB_PATH') or os.path.join(_HERE, 'lib', 'libboxseg_b200.so')   # BXS_LIB_PATH: A/B builds (tools/)
HEADER_PATH = os.path.join(os.path.dirname(_HERE), 'include', 'boxseg_b200.h')

_lib = None

c_p = ctypes.c_void_p
c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_f = ctypes.c_float

# The by-value C types the header uses.  Every pointer binds as c_void_p.  A type outside this table is an error, never a
# guess: on x86-64 a wrong scalar type is not caught by ctypes, the call just receives a wrong value.
_BY_VALUE = {'int64_t': c_i64, 'int': c_int, 'float': c_f, 'bxs_stream_t': c_p}


def _ctype(c_type, where):
    if '*' in c_type:
        return c_p
    if c_type not in _BY_VALUE:
        raise TypeError(f'{where}: no ctypes mapping for the C type {c_type!r}')
    return _BY_VALUE[c_type]


def parse_header(text):
    """(argtypes, restypes): name -> ctypes argument list and name -> ctypes result type of every ``bxs_*`` prototype in
    the C header ``text``.  A ``const char*`` result is a ``c_char_p``; ``(void)`` is no argument."""
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    argtypes, restypes = {}, {}
    for stmt in text.split(';'):
        if not re.search(r'\bbxs_\w+\s*\(', stmt):
            continue
        m = re.fullmatch(r'\s*([\w\s*]+?)\s*\b(bxs_\w+)\s*\(([^()]*)\)\s*', stmt)
        if m is None:
            raise ValueError(f'not a prototype: {" ".join(stmt.split())!r}')
        ret, name, params = m.groups()
        ret = ' '.join(ret.replace('*', ' * ').split())
        restypes[name] = ctypes.c_char_p if ret == 'const char *' else _ctype(ret, name)
        params = [] if params.strip() == 'void' else params.split(',')
        argtypes[name] = [_ctype(' '.join(re.sub(r'\w+\s*$', '', p).split()), name) for p in params]   # drop the name
    return argtypes, restypes


# name -> argtypes and name -> restype of every entry point, from the prototypes the library is compiled against
with open(HEADER_PATH) as _f:
    SIGNATURES, RESTYPES = parse_header(_f.read())

_STATUS = {-1: 'invalid argument', -2: 'kernel launch failed', -3: 'unsupported shape', -4: 'no CUDA device'}


class BoxSegError(RuntimeError):
    pass


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f'{LIB_PATH} is missing: the CUDA extension is the product and there is no fallback. '
                'Build it with `python -m boxinstseg_b200.build`.')
        handle = ctypes.CDLL(LIB_PATH)
        for name, args in SIGNATURES.items():
            fn = getattr(handle, name)          # AttributeError if the .so does not export it
            fn.argtypes = args
            fn.restype = RESTYPES[name]
        _lib = handle
    return _lib


def check(rc, what):
    if rc != 0:
        detail = lib().bxs_last_error().decode() if rc == -2 else ''
        raise BoxSegError(f'{what}: {_STATUS.get(rc, rc)} {detail}'.strip())


def ptr(t):
    return None if t is None else c_p(t.data_ptr())


def stream():
    return c_p(torch.cuda.current_stream().cuda_stream)


def dense_aligned(t, align=16):
    """``t`` as a dense row-major tensor whose base address is a multiple of ``align`` bytes: ``t`` itself when it already
    is one, else one copy into a fresh allocation.  A dense view that starts inside another buffer (``flat[1:1 + n]``,
    ``torch.cat(...)[a:b]`` with an odd row size) is ``is_contiguous()`` but only element-aligned; the kernels that read
    through 8- or 16-byte vectors or a TMA tensor map take their operands through here."""
    t = t.contiguous()
    return t if t.data_ptr() % align == 0 else t.clone(memory_format=torch.contiguous_format)


def require_cuda(*tensors):
    """Same error behaviour as the reference's CHECK_INPUT (pairwise.cu:7-13)."""
    for t in tensors:
        if t is None:
            continue
        if not t.is_cuda:
            raise RuntimeError('boxinstseg_b200: tensor must be a CUDA tensor')
        if not t.is_contiguous():
            raise RuntimeError('boxinstseg_b200: tensor must be contiguous')
