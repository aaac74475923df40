// TEST INFRASTRUCTURE: host twin of the string arithmetic of csrc/mask_rle.cu.  It compiles the very header the kernels
// call (mask_rle_core.cuh) with g++ so that each delta's character count and characters can be checked against the
// oracle on a box without a GPU.  Never shipped.
#include <stdint.h>

#include "../../boxinstseg_b200/csrc/mask_rle_core.cuh"

// n deltas x -> len [n] (rle_char_len) and the characters of each at chars[6 * i ..] (rle_emit); returns 0, or -1 when
// rle_emit and rle_char_len disagree or a delta takes more than kRleMaxChars characters
extern "C" int host_rle_chars(int64_t n, const int64_t* x, int32_t* len, uint8_t* chars) {
  for (int64_t i = 0; i < n; ++i) {
    len[i] = bxs::rle_char_len(x[i]);
    if (len[i] > bxs::kRleMaxChars || bxs::rle_emit(x[i], chars + bxs::kRleMaxChars * i) != len[i]) return -1;
  }
  return 0;
}

// the deltas rleToString writes for the m counts c of one mask -> x [m]
extern "C" void host_rle_deltas(int64_t m, const uint32_t* c, int64_t* x) {
  for (int64_t i = 0; i < m; ++i) x[i] = bxs::rle_delta(c, i);
}
