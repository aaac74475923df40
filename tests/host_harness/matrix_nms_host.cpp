// TEST INFRASTRUCTURE: host twin of the Matrix NMS and mask-paste arithmetic of csrc/solo_seg.cu.  It compiles the very
// header the kernels are made of (solo_seg_core.cuh, with resize_core.cuh's tap arithmetic) with g++ (-ffp-contract=off)
// and evaluates it element by element, so that the IoU, compensation, decay coefficient and the two-stage bilinear paste
// can be checked against the oracle on a box without a GPU.  Never shipped.
#include <stdint.h>

#include "../../boxinstseg_b200/csrc/solo_seg_core.cuh"

// Decayed scores of n score-sorted candidates (nms_decay_kernel's arithmetic): inter [n,n] float (row-major, i < j used),
// area, label, score [n] -> out [n] = score * min_i ratio(i, j), -inf below a positive filter_thr.
extern "C" void host_matrix_nms(int64_t n, const float* inter, const float* area, const int64_t* label, const float* score,
                                int kernel, float sigma, float filter_thr, float* out) {
  float* comp = new float[n];
  float* iou = new float[n * n];
  for (int64_t j = 0; j < n; ++j) {
    comp[j] = 0.f;
    for (int64_t i = 0; i < n; ++i) {
      const bool need = i < j && label[i] == label[j];
      iou[i * n + j] = need ? bxs::nms_iou(inter[i * n + j], area[i], area[j]) : 0.f;
      if (iou[i * n + j] > comp[j]) comp[j] = iou[i * n + j];
    }
  }
  const float nsig = -1.f * sigma;
  for (int64_t j = 0; j < n; ++j) {
    float m = INFINITY;
    for (int64_t i = 0; i < n; ++i) m = bxs::nan_min(m, bxs::nms_decay_ratio(iou[i * n + j], comp[i], kernel, nsig));
    const float s = score[j] * m;
    out[j] = (filter_thr > 0.f && !(s >= filter_thr)) ? -INFINITY : s;
  }
  delete[] comp;
  delete[] iou;
}

// interpolate(interpolate(p, (4h, 4w))[:H_img, :W_img], (H_ori, W_ori)) of one float32 plane, pixel by pixel
extern "C" void host_paste(const float* p, int h, int w, int H_img, int W_img, int H_ori, int W_ori, float* out) {
  for (int y = 0; y < H_ori; ++y)
    for (int x = 0; x < W_ori; ++x) {
      const bxs::PasteTaps pt = bxs::paste_taps(y, x, H_img, W_img, H_ori, W_ori);
      float v[2][2];
      for (int a = 0; a < 2; ++a) {
        const bxs::RsTap ty = bxs::paste_stage1_tap(pt.y1[a], h);
        for (int c = 0; c < 2; ++c) {
          const bxs::RsTap tx = bxs::paste_stage1_tap(pt.x1[c], w);
          const float* q = p + ty.i0 * w + tx.i0;
          v[a][c] = bxs::rs_lerp2(ty, tx, q[0], q[tx.ip], q[ty.ip * w], q[ty.ip * w + tx.ip]);
        }
      }
      out[y * W_ori + x] = bxs::rs_lerp2(pt.ty2, pt.tx2, v[0][0], v[0][1], v[1][0], v[1][1]);
    }
}
