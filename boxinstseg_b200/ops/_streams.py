"""Fork / join of independent latency-bound chains onto a per-device side stream.

The tree-filter path is made of dependent-level walks that keep a handful of SMs busy for a millisecond each (MST rounds, the
BFS order, the aggregation passes).  Chains that do not depend on each other -- the two gradients of ``refine``, the MST + BFS
of the second tree of a head while the first filter runs -- are issued on a side stream so that they overlap.  The fork and the
join are ordinary cross-stream dependencies (``wait_stream``), hence capturable in a CUDA graph; the side stream is created
on the first call made outside a capture, and until it exists everything simply runs in order on the current stream.
"""
import torch

_SIDE = {}     # (device, current stream) -> its partner side stream
_LANES = {}    # device -> list of lane streams


def side_stream(device):
    """The partner of the CURRENT stream (each lane of ``run_concurrently`` gets its own, so forks made inside different lanes
    do not queue up behind each other)."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    st = _SIDE.get(key)
    if st is None and not torch.cuda.is_current_stream_capturing():
        st = _SIDE[key] = torch.cuda.Stream(device)
    return st


def lanes(device, n):
    pool = _LANES.setdefault(device.index, [])
    if len(pool) < n:
        if torch.cuda.is_current_stream_capturing():
            return pool or None
        pool.extend(torch.cuda.Stream(device) for _ in range(n - len(pool)))
    return pool[:n]


def run_concurrently(fns, device, max_lanes=10):
    """[fn() for fn in fns], each on its own lane stream, forked from and joined back into the current stream.  For
    independent chains that each keep only a few SMs busy (the per-level / per-decoder-layer mask losses: their tree filters are
    dependent-level walks of a millisecond on ~20 CTAs).  Autograd runs a node's backward on the stream of its forward, so the
    backward passes of the lanes overlap as well.  Falls back to a plain loop when no lane stream exists yet inside a
    capture."""
    fns = list(fns)
    if len(fns) <= 1:
        return [fn() for fn in fns]
    pool = lanes(device, min(len(fns), max_lanes))
    if not pool:
        return [fn() for fn in fns]
    cur = torch.cuda.current_stream(device)
    for st in pool:
        st.wait_stream(cur)
    outs = []
    for k, fn in enumerate(fns):
        with torch.cuda.stream(pool[k % len(pool)]):
            outs.append(fn())
    for st in pool:
        cur.wait_stream(st)
    for t in _tensors(outs):
        if t.is_cuda:
            t.record_stream(cur)
    return outs


def _tensors(obj):
    if isinstance(obj, torch.Tensor):
        yield obj
    elif isinstance(obj, (tuple, list)):
        for o in obj:
            yield from _tensors(o)


class Forked:
    """``Forked(fn, device)`` runs ``fn()`` on the side stream (after everything issued so far on the current stream);
    ``join()`` makes the current stream wait for it and returns its value."""

    def __init__(self, fn, device):
        self.side = side_stream(device)
        self.device = device
        if self.side is None:
            self.value = fn()
            return
        self.side.wait_stream(torch.cuda.current_stream(device))
        with torch.cuda.stream(self.side):
            self.value = fn()

    def join(self):
        if self.side is not None:
            cur = torch.cuda.current_stream(self.device)
            cur.wait_stream(self.side)
            for t in _tensors(self.value):
                if t.is_cuda:
                    t.record_stream(cur)
        return self.value
