// TEST INFRASTRUCTURE: host twin of the MaskFormer instance-mask paste of csrc/solo_seg.cu (bxs_maskformer_paste_masks).
// It compiles the very header the kernel is made of (solo_seg_core.cuh: paste_value and MaskStats, with resize_core.cuh's
// tap arithmetic) with g++ (-ffp-contract=off) and evaluates it pixel by pixel on one float32 logit plane, so that the mask,
// the area, the masked sum and the box can be checked against the oracle on a box without a GPU.  Never shipped.
#include <stdint.h>

#include "../../boxinstseg_b200/csrc/solo_seg_core.cuh"

// interpolate(interpolate(p, (H_pad, W_pad))[:H_img, :W_img], (H_out, W_out)) > 0 of one h x w plane, a stage skipped as
// the kernel skips it, and the statistics of the mask (sigmoid as 1 / (1 + expf(-v)), summed in float64 in pixel order).
extern "C" void host_maskformer_paste(const float* p, int h, int w, int H_pad, int W_pad, int H_img, int W_img, int rescale,
                                      int H_out, int W_out, uint8_t* out, int32_t* area, float* masked_sum, float* box) {
  const bxs::PasteGeom g{h, w, H_pad, W_pad, H_img, W_img, H_out, W_out, h == H_pad && w == W_pad, rescale == 0};
  bxs::MaskStats s = bxs::mask_stats_empty();
  for (int y = 0; y < H_out; ++y)
    for (int x = 0; x < W_out; ++x) {
      const float v = bxs::paste_value<true>(
          g, y, x, [&](int o, int d) { return p[o + d]; }, [](float u) { return u; });
      const bool on = v > 0.f;
      out[y * W_out + x] = on;
      if (on) bxs::mask_stats_add(s, y, x, 1.f / (1.f + expf(-v)));
    }
  *area = s.area;
  *masked_sum = (float)s.sum;
  bxs::mask_stats_box(s, box);
}
