// COCO RLE string arithmetic of pycocotools' rleToString (maskApi.c): the delta a count is written as, the number of
// characters that delta takes, and the characters themselves.  mask_rle.cu's string kernels call these per count.
//
// The body is BXS_HD so that tests/host_harness/mask_rle_host.cpp can compile the very same lines for the host and check
// them against the oracle without a GPU (test infrastructure; the library itself exports only the CUDA path).
#pragma once
#include <stdint.h>

#include "assign_core.cuh"            // BXS_HD

namespace bxs {

constexpr int kRleMaxChars = 6;      // characters of one delta while |delta| < 2^29, i.e. H * W < 2^29

// rleToString's value for count i (mask-local index) of the counts c: c[i], minus c[i - 2] when i > 2 (not i >= 2).
BXS_HD int64_t rle_delta(const uint32_t* c, int64_t i) {
  int64_t x = (int64_t)c[i];
  if (i > 2) x -= (int64_t)c[i - 2];
  return x;
}

// rleToString's loop on x: 5 bits per character, low bits first; a character continues (0x20) while the bits left are
// not all copies of its own bit 4.  >> on a negative int64_t is arithmetic with gcc and nvcc, as on `long` in maskApi.c.
// Writes the characters to out when it is not NULL; returns how many there are.
BXS_HD int rle_emit(int64_t x, uint8_t* out) {
  int n = 0;
  bool more = true;
  while (more) {
    int c = (int)(x & 0x1f);
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    if (more) c |= 0x20;
    if (out) out[n] = (uint8_t)(c + 48);
    ++n;
  }
  return n;
}

BXS_HD int rle_char_len(int64_t x) { return rle_emit(x, nullptr); }

}  // namespace bxs
