// 16-bit mask predictions on the autocast paths of the DiscoBox mask loss (discobox_loss.cu, the logits entry of
// meanfield.cu): widening, rounding and torch's CUDA sigmoid for a float16 / bfloat16 tensor.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "boxinst_common.cuh"         // fkey (the arg-max key), sigmoid_exact

namespace bxs {

template <typename T>
struct Half16Ops;
template <>
struct Half16Ops<__half> {
  static __device__ __forceinline__ __half round(float x) { return __float2half_rn(x); }
  static __device__ __forceinline__ float widen(__half x) { return __half2float(x); }
};
template <>
struct Half16Ops<__nv_bfloat16> {
  static __device__ __forceinline__ __nv_bfloat16 round(float x) { return __float2bfloat16_rn(x); }
  static __device__ __forceinline__ float widen(__nv_bfloat16 x) { return __bfloat162float(x); }
};

// round_T(v) as a float
template <typename T>
__device__ __forceinline__ float round_to(float v) { return Half16Ops<T>::widen(Half16Ops<T>::round(v)); }

// torch.sigmoid of a T tensor on CUDA: 1 / (1 + exp(-x)) in float32 (accurate expf, IEEE divide), rounded to T once.
// Bit-identical to torch's result; returned widened to float (exact).
template <typename T>
__device__ __forceinline__ float sigmoid_rounded(T x) { return round_to<T>(sigmoid_exact(Half16Ops<T>::widen(x))); }

}  // namespace bxs
