"""f1: linear sum assignment on the GPU -- what MaskHungarianAssigner.assign hands to ``scipy.optimize.linear_sum_assignment``
on the host (mask_hungarian_assigner.py:113-123).  The kernel (csrc/lsap.cu) runs scipy's algorithm with scipy's tie rules in
float64, so ``row_ind`` / ``col_ind`` are the same as scipy's on every input.

``solve_batched`` is the sync-free form: one launch for a list of problems, results and a per-problem status left on the
device.  ``linear_sum_assignment`` is the scipy signature for one matrix; it reads the 4-byte status to raise scipy's errors.
"""
import ctypes

import torch

from .. import _lib as L

_F32, _F64 = 0, 1
OK, INVALID, INFEASIBLE = 0, 1, 2


def raise_for_status(code):
    """scipy's ValueError for a status read back from ``solve_batched``."""
    if code == INVALID:
        raise ValueError('matrix contains invalid numeric entries')
    if code == INFEASIBLE:
        raise ValueError('cost matrix is infeasible')


def solve_batched(costs):
    """costs: list of 2-D CUDA tensors [rows_p, cols_p] on one device (any real or bool dtype; each entry is widened to
    float64 exactly as scipy's conversion does).  Returns (matches, status) without synchronising: ``matches[p]`` int32
    [rows_p] is the column matched to each row or -1, ``status`` int32 [P] holds 0 (ok), 1 (NaN or -inf entry) or 2
    (infeasible) per problem; a failed problem's rows are all -1."""
    costs = list(costs)
    for c in costs:
        if c.dim() != 2:
            raise ValueError(f'expected a matrix (2-D array), got a {c.dim()}-D array')
        if c.is_complex():
            raise ValueError('cost matrices must be real')
    if not costs:
        return [], torch.empty(0, dtype=torch.int32, device='cuda')
    dev = costs[0].device
    if any(c.device != dev for c in costs):
        raise RuntimeError('boxinstseg_b200: all cost matrices must be on one device')
    dt = torch.float32 if all(c.dtype == torch.float32 for c in costs) else torch.float64
    flat = [c.to(dt).reshape(-1) for c in costs]
    flat = flat[0].contiguous() if len(flat) == 1 else torch.cat(flat)
    L.require_cuda(flat)
    n = len(costs)
    rows = [int(c.shape[0]) for c in costs]
    cols = [int(c.shape[1]) for c in costs]
    offs, o = [], 0
    for r, c in zip(rows, cols):
        offs.append(o)
        o += r * c
    arr = ctypes.c_int64 * n
    rows_h, cols_h, offs_h = arr(*rows), arr(*cols), arr(*offs)
    match = torch.empty(sum(rows), dtype=torch.int32, device=dev)
    status = torch.empty(n, dtype=torch.int32, device=dev)
    lib = L.lib()
    ws_bytes = lib.bxs_lsap_workspace_bytes(rows_h, cols_h, n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes > 0 else None
    with torch.cuda.device(dev):
        L.check(lib.bxs_lsap_solve(L.ptr(flat) if flat.numel() else None, offs_h, rows_h, cols_h, n,
                                   _F32 if dt == torch.float32 else _F64, L.ptr(match) if match.numel() else None,
                                   L.ptr(status), L.ptr(ws), L.stream()), 'lsap_solve')
    return list(match.split(rows)), status


def linear_sum_assignment(cost):
    """scipy.optimize.linear_sum_assignment(cost) for one 2-D CUDA tensor: (row_ind, col_ind) int64 CUDA tensors equal to
    scipy's, and scipy's ValueError for a NaN / -inf entry or an infeasible matrix (one 4-byte status read)."""
    (match,), status = solve_batched([cost])
    raise_for_status(int(status[0]))
    k = min(cost.shape)
    row_ind = torch.nonzero_static(match >= 0, size=k).squeeze(1)
    return row_ind, match[row_ind].long()
