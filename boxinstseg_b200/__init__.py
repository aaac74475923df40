"""boxinstseg_b200 -- H100 (sm_90a) box-supervised mask-loss hot path of BoxInstSeg.

Layout mirrors the part of the reference it drops into:
  ops/pairwise, ops/tree_filter   <->  mmdet/ops/{pairwise,tree_filter}
  models/builder.py               <->  mmdet/models/builder.py (HEADS / LOSSES registry)
  models/losses, models/dense_heads <-> the loss classes / mask heads on the path
  csrc/ + lib/libboxseg_b200.so   the hand-written CUDA kernels behind a C ABI (include/boxseg_b200.h)
"""
__version__ = '0.1.0'
