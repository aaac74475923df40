// TEST INFRASTRUCTURE: host twin of fcos_loss_kernel's per-point arithmetic (boxinstseg_b200/csrc/fcos_loss.cu).  It
// compiles the very header the kernel is made of (fcos_loss_core.cuh) with g++ (-ffp-contract=off) and evaluates it point
// by point, so that the point locations, the centerness targets, the element losses and their gradients -- ties included
// -- can be checked against the float64 oracle on a box without a GPU.  Never shipped.
#include "../../boxinstseg_b200/csrc/fcos_loss_core.cuh"

extern "C" void host_fcos_points(int64_t n, const int64_t* idx, float stride, float* out) {
  for (int64_t i = 0; i < n; ++i) out[i] = bxs::fcos_point_coord(idx[i], stride);
}

extern "C" void host_fcos_point_loss(int64_t n, const float* xy, const float* pred, const float* target, const float* ctr,
                                     float* ct, float* bbox, float* bce, float* g_pred, float* g_ctr) {
  for (int64_t i = 0; i < n; ++i) {
    const bxs::FcosPointLoss r = bxs::fcos_point_loss(xy[2 * i], xy[2 * i + 1], pred + 4 * i, target + 4 * i, ctr[i]);
    ct[i] = r.ct;
    bbox[i] = r.bbox;
    bce[i] = r.ctr;
    for (int k = 0; k < 4; ++k) g_pred[4 * i + k] = r.g_pred[k];
    g_ctr[i] = r.g_ctr;
  }
}
