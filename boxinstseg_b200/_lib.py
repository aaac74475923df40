"""ctypes binding of ``libboxseg_b200.so`` (the C ABI declared in ``include/boxseg_b200.h``).

The product path has NO fallback: if the shared library is missing or a call fails, an
exception is raised.  Build with ``python -m boxinstseg_b200.build`` (or ``__graft_entry__.build()``).
"""
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('BXS_LIB_PATH') or os.path.join(_HERE, 'lib', 'libboxseg_b200.so')   # BXS_LIB_PATH: A/B builds (tools/)

_lib = None

c_p = ctypes.c_void_p
c_i64 = ctypes.c_int64
c_int = ctypes.c_int
c_f = ctypes.c_float

# name -> argtypes (all return int unless listed in _RESTYPE)
SIGNATURES = {
    'bxs_version': [],
    'bxs_last_error': [],
    'bxs_device_sm_count': [],
    'bxs_pairwise_nlog_forward': [c_p, c_p, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_p],
    'bxs_pairwise_nlog_backward': [c_p, c_p, c_p, c_i64, c_i64, c_i64, c_int, c_int, c_int, c_p],
    'bxs_boxinst_bitmasks': [c_p, c_p, c_i64, c_i64, c_i64, c_p],
    'bxs_boxinst_targets_forward': [c_p] * 13 + [c_i64] * 3 + [c_int] * 3 + [c_f, c_p],
    'bxs_rgb_u8_to_lab': [c_p, c_p, c_i64, c_p],
    'bxs_boxinst_loss_workspace_bytes': [c_i64, c_i64, c_i64],
    'bxs_boxinst_loss_forward': [c_p, c_p, c_p, c_p, c_p, c_p, c_f, c_p, c_p, c_i64, c_i64, c_i64, c_int, c_p],
    'bxs_boxinst_loss_backward': [c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_p, c_i64, c_i64, c_i64, c_int, c_p],
    'bxs_boxinst_loss_fused_supported': [c_i64, c_i64, c_i64, c_int],
    'bxs_boxinst_loss_fused_workspace_bytes': [c_i64, c_i64, c_i64],
    'bxs_boxinst_loss_fused_sched_bytes': [],
    'bxs_boxinst_loss_fused_forward': [c_p] * 6 + [c_f] + [c_p] * 4 + [c_i64] * 3 + [c_int, c_p],
    'bxs_boxinst_loss_fused_backward': [c_p] * 4 + [c_i64] * 3 + [c_p],
    'bxs_boxinst_loss_plan_bytes': [c_i64, c_i64, c_i64, c_int],
    'bxs_boxinst_loss_plan': [c_p] * 5 + [c_i64] * 3 + [c_int, c_p],
    'bxs_boxinst_loss_fused_forward_planned': [c_p] * 4 + [c_f] + [c_p] * 4 + [c_i64] * 3 + [c_int, c_p],
    'bxs_condinst_head_forward': [c_p] * 6 + [c_i64] * 6 + [c_int] * 3 + [c_p],
    'bxs_condinst_head_workspace_bytes': [c_i64] * 5,
    'bxs_condinst_head_backward': [c_p] * 9 + [c_i64] * 6 + [c_int] * 3 + [c_p],
    'bxs_projection_workspace_bytes': [c_i64] * 3,
    'bxs_projection_loss_forward': [c_p] * 4 + [c_i64] * 3 + [c_f, c_f, c_p],
    'bxs_projection_loss_backward': [c_p] * 3 + [c_i64] * 3 + [c_p],
    'bxs_length_reg_forward': [c_p] * 3 + [c_i64] * 4 + [c_p],
    'bxs_length_reg_backward': [c_p] * 3 + [c_i64] * 4 + [c_p],
    'bxs_lcm_workspace_bytes': [c_i64] * 3,
    'bxs_lcm_forward': [c_p] * 5 + [c_i64] * 4 + [c_int, c_int, c_p],
    'bxs_lcm_backward': [c_p] * 5 + [c_i64] * 3 + [c_int, c_int, c_p],
    'bxs_meanfield_kernel': [c_p, c_p] + [c_i64] * 4 + [c_int, c_f, c_f, c_f, c_p],
    'bxs_meanfield_workspace_bytes': [c_i64] * 3,
    'bxs_meanfield_forward_inter': [c_p] * 5 + [c_f] + [c_p] * 4 + [c_i64] * 3 + [c_int, c_int, c_p],
    'bxs_meanfield_forward_logits': [c_p] * 5 + [c_int] + [c_p] * 3 + [c_i64] * 3 + [c_int, c_int, c_p],
    'bxs_discobox_loss_workspace_bytes': [c_i64] * 3,
    'bxs_discobox_loss_forward': [c_p] * 3 + [c_int] + [c_p] * 2 + [c_i64] * 3 + [c_p],
    'bxs_discobox_loss_backward': [c_p] * 3 + [c_int] + [c_p] * 3 + [c_i64] * 3 + [c_p],
    'bxs_mst_workspace_bytes': [c_i64] * 3,
    'bxs_mst_forward': [c_p] * 4 + [c_i64] * 3 + [c_p],
    'bxs_bfs_workspace_bytes': [c_i64] * 2,
    'bxs_bfs_forward_rooted': [c_p] * 7 + [c_i64] * 2 + [c_int, c_i64, c_p],
    'bxs_refine_scratch_bytes': [c_i64] * 3,
    'bxs_refine_forward_grouped': [c_p] * 14 + [c_i64] * 4 + [c_p],
    'bxs_refine_backward_feature_grouped': [c_p] * 11 + [c_i64] * 4 + [c_p],
    'bxs_refine_backward_weight_grouped': [c_p] * 15 + [c_i64] * 4 + [c_p],
    'bxs_dynconv1x1_forward': [c_p] * 3 + [c_i64] * 4 + [c_p],
    'bxs_dynconv1x1_backward_workspace_bytes': [c_i64] * 4,
    'bxs_dynconv1x1_backward': [c_p] * 6 + [c_i64] * 4 + [c_p],
    'bxs_dynconv1x1_cells_forward_workspace_bytes': [c_p] + [c_i64] * 3,
    'bxs_dynconv1x1_cells_forward': [c_p] * 9 + [c_i64] * 4 + [c_p],
    'bxs_dynconv1x1_cells_backward_workspace_bytes': [c_p] * 4 + [c_i64] * 4,
    'bxs_dynconv1x1_cells_backward': [c_p] * 11 + [c_i64] * 4 + [c_p],
    'bxs_dynconv1x1_half_forward': [c_p] * 3 + [c_i64] * 4 + [c_int, c_p],
    'bxs_dynconv1x1_half_backward_workspace_bytes': [c_i64] * 4 + [c_int],
    'bxs_dynconv1x1_half_backward': [c_p] * 6 + [c_i64] * 4 + [c_int, c_p],
    'bxs_upsampled_rowcol_max': [c_p] * 4 + [c_i64] * 5 + [c_int, c_p],
    'bxs_bilinear_resize_forward': [c_p, c_p] + [c_i64] * 5 + [c_int, c_p],
    'bxs_bilinear_resize_backward': [c_p, c_p] + [c_i64] * 5 + [c_int, c_p],
    'bxs_box2mask_attn_mask': [c_p, c_p] + [c_i64] * 7 + [c_int, c_int, c_p],
    'bxs_tree_edge_weight_forward': [c_p] * 4 + [c_i64] * 4 + [c_f, c_p],
    'bxs_tree_edge_weight_backward': [c_p] * 7 + [c_i64] * 4 + [c_f, c_p],
    'bxs_levelset_fused_workspace_bytes': [c_i64],
    'bxs_levelset_fused_forward': [c_p] * 6 + [c_i64] * 4 + [c_f, c_int, c_p],
    'bxs_levelset_fused_backward': [c_p] * 7 + [c_i64] * 4 + [c_f, c_int, c_p],
    'bxs_corr_solve': [c_p, c_p] + [c_i64] * 3 + [c_int] * 3 + [c_p],
    'bxs_corr_solve_batched': [c_p] * 3 + [c_i64] * 4 + [c_int] * 3 + [c_p],
    'bxs_corr_transfer_workspace_bytes': [c_i64] * 3,
    'bxs_corr_transfer': [c_p] * 7 + [c_i64] * 5 + [c_p],
    'bxs_corr_transfer_batched': [c_p] * 8 + [c_i64] * 6 + [c_p],
    'bxs_corr_retrieve': [c_p] * 19 + [c_i64] * 8 + [c_f] * 6 + [c_int] * 2 + [c_p],
    'bxs_corr_paste': [c_p] * 5 + [c_i64] * 5 + [c_p],
    'bxs_corr_bank_append': [c_p] * 12 + [c_i64] * 5 + [c_p],
    'bxs_fcos_targets': [c_p] * 7 + [c_i64] * 2 + [c_p] * 5 + [c_int, c_int, c_i64, c_p],
    'bxs_lsap_workspace_bytes': [c_p, c_p, c_i64],
    'bxs_lsap_solve': [c_p] * 4 + [c_i64, c_int] + [c_p] * 4,
    'bxs_sigmoid_focal_loss_levels_forward_workspace_bytes': [c_p, c_i64, c_i64],
    'bxs_sigmoid_focal_loss_levels_forward': [c_p] * 7 + [c_i64] * 3 + [c_f] * 3 + [c_p],
    'bxs_softmax_cross_entropy_layers_forward_workspace_bytes': [c_i64] * 3,
    'bxs_softmax_cross_entropy_layers_forward': [c_p] * 6 + [c_i64] * 4 + [c_f, c_p],
    'bxs_softmax_cross_entropy_layers_backward': [c_p] * 2 + [c_i64] * 4 + [c_p],
}
_RESTYPE = {'bxs_mst_workspace_bytes': c_i64, 'bxs_bfs_workspace_bytes': c_i64, 'bxs_refine_scratch_bytes': c_i64, 'bxs_lcm_workspace_bytes': c_i64, 'bxs_meanfield_workspace_bytes': c_i64, 'bxs_projection_workspace_bytes': c_i64,'bxs_condinst_head_workspace_bytes': c_i64, 'bxs_last_error': ctypes.c_char_p, 'bxs_boxinst_loss_workspace_bytes': c_i64,
             'bxs_boxinst_loss_fused_workspace_bytes': c_i64, 'bxs_boxinst_loss_fused_sched_bytes': c_i64,
             'bxs_boxinst_loss_plan_bytes': c_i64, 'bxs_levelset_fused_workspace_bytes': c_i64,
             'bxs_dynconv1x1_backward_workspace_bytes': c_i64, 'bxs_corr_transfer_workspace_bytes': c_i64,
             'bxs_dynconv1x1_half_backward_workspace_bytes': c_i64, 'bxs_lsap_workspace_bytes': c_i64,
             'bxs_discobox_loss_workspace_bytes': c_i64, 'bxs_dynconv1x1_cells_forward_workspace_bytes': c_i64,
             'bxs_dynconv1x1_cells_backward_workspace_bytes': c_i64,
             'bxs_sigmoid_focal_loss_levels_forward_workspace_bytes': c_i64,
             'bxs_softmax_cross_entropy_layers_forward_workspace_bytes': c_i64}

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
            fn.restype = _RESTYPE.get(name, c_int)
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
