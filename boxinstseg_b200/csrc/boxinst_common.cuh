// Small helpers shared by the BoxInst loss kernels (two-pass kernels in boxinst_loss.cu, the
// single-pass TMA-staged kernel in boxinst_onepass.cu).
#pragma once
#include "common.cuh"

namespace bxs {

constexpr float kFastLimit = 40.f;
constexpr float kDiceEps = 1e-5f;        // condinst_head.py:124

struct Rect { int j0, j1, i0, i1; };

__device__ __forceinline__ Rect load_rect(const int32_t* rects, int g) {
  int4 r = *reinterpret_cast<const int4*>(rects + 4 * (int64_t)g);
  return Rect{r.x, r.y, r.z, r.w};
}
__device__ __forceinline__ bool rect_empty(const Rect& r) { return r.j0 > r.j1 || r.i0 > r.i1; }
__device__ __forceinline__ bool in_rect(const Rect& r, int y, int x) {
  return y >= r.j0 && y <= r.j1 && x >= r.i0 && x <= r.i1;
}

// Order-preserving map float -> uint, so maxima of LOGITS can be combined with integer max /
// atomicMax.  The sigmoid is monotone, hence the arg-max of the scores is the arg-max of the logits
// (first index on exact ties, like torch.max(dim)).  -0 and +0 compare equal in torch.max, so they
// share one key: a negative float maps to -b = ~b + 1, which puts -0 on +0's key and keeps every
// other value in order.  No float maps to 0, the "nothing yet" value of the atomicMax slots.
// Every projection path (single-pass, two-call, dense) merges keys through these three helpers.
__device__ __forceinline__ unsigned fkey(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? 0u - b : (b | 0x80000000u);
}
__device__ __forceinline__ float fkey_inv(unsigned k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : 0u - k);
}
__device__ __forceinline__ unsigned long long pack_key(unsigned key, int index) {
  return ((unsigned long long)key << 32) | (unsigned long long)(0xffffffffu - (unsigned)index);
}
__device__ __forceinline__ unsigned long long pack_max(float v, int index) { return pack_key(fkey(v), index); }

__device__ __forceinline__ float sigmoid_exact(float x) { return 1.f / (1.f + expf(-x)); }

}  // namespace bxs
