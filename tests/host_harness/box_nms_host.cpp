// TEST INFRASTRUCTURE: host twin of the box arithmetic of csrc/condinst_infer.cu.  It compiles the very header the kernels
// are made of (box_nms_core.cuh) with g++ (-ffp-contract=off) so that the decode, mmcv's suppression test, the greedy pass
// and the aligned_bilinear paste can be checked against the oracle on a box without a GPU.  Never shipped.
#include <stdint.h>

#include "../../boxinstseg_b200/csrc/box_nms_core.cuh"

// n points (px, py) with distances d [n,4] -> boxes [n,4]; sf: scale_factor [4] or NULL
extern "C" void host_decode(int64_t n, const float* pts, const float* d, float img_h, float img_w, const float* sf, float* out) {
  for (int64_t i = 0; i < n; ++i) bxs::ci_decode_box(pts[2 * i], pts[2 * i + 1], d + 4 * i, img_h, img_w, sf, out + 4 * i);
}

// sup [n,n]: box i suppresses box j (any i, j)
extern "C" void host_suppress(int64_t n, const float* boxes, float thr, uint8_t* sup) {
  for (int64_t i = 0; i < n; ++i)
    for (int64_t j = 0; j < n; ++j) sup[i * n + j] = bxs::ci_suppresses(boxes + 4 * i, boxes + 4 * j, thr);
}

// greedy NMS of n boxes already sorted by descending score -> keep [n] (nms_resolve_kernel's order of decisions)
extern "C" void host_greedy(int64_t n, const float* boxes, float thr, uint8_t* keep) {
  for (int64_t i = 0; i < n; ++i) keep[i] = 1;
  for (int64_t i = 0; i < n; ++i) {
    if (!keep[i]) continue;
    for (int64_t j = i + 1; j < n; ++j)
      if (bxs::ci_suppresses(boxes + 4 * i, boxes + 4 * j, thr)) keep[j] = 0;
  }
}

// aligned_bilinear(p, f)[:H_img, :W_img] of one h x w float32 plane of probabilities, pixel by pixel
extern "C" void host_aligned(const float* p, int h, int w, int f, int H_img, int W_img, float* out) {
  for (int y = 0; y < H_img; ++y)
    for (int x = 0; x < W_img; ++x) {
      const bxs::RsTap ty = bxs::ci_aligned_tap(y, h, f), tx = bxs::ci_aligned_tap(x, w, f);
      auto at = [&](int i, int j) { return p[(i < h - 1 ? i : h - 1) * w + (j < w - 1 ? j : w - 1)]; };
      out[y * W_img + x] = bxs::rs_lerp2(ty, tx, at(ty.i0, tx.i0), at(ty.i0, tx.i0 + tx.ip), at(ty.i0 + ty.ip, tx.i0),
                                         at(ty.i0 + ty.ip, tx.i0 + tx.ip));
    }
}
