// a16: DiscoBox mean-field CRF teacher -- bilateral 3x3 (k x k) kernel from the colour features and
// `iter` rounds of [unfold(-log U) * K -> exp -> * target -> normalise -> re-threshold].
// Replaces MeanField.__init__/forward/simple_forward (mmdet/models/dense_heads/discobox_head.py:585-651),
// which expands every round into a k*k-fold unfold plus ~6 elementwise launches.
//
// Observation that shapes the design: after the first threshold the state of a pixel is ONE BIT
// (U = [1-q, q] with q in {base, 1-base}), so the whole recursion runs on bit maps.  One CTA per
// object keeps the two ping-pong bit maps in shared memory for all rounds; only the kernel K
// (k*k floats per pixel, shared by every object of the image) is streamed from L2.
// The four -log(U) constants are computed by the caller with the reference's own float32
// arithmetic and passed in, so the energies are bit-identical to the reference's.
// Entirely forward / no_grad, exactly like the reference.
// The kernels are templated on where the initial state and the targets come from: float32 maps and targets
// (MeanField.forward) or 16-bit student / teacher logits with uint8 targets (the DiscoBox mask loss under autocast,
// bxs_meanfield_forward_logits, which writes the pseudo-label as uint8 and no `valid`).
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "half_math.cuh"

namespace bxs {
namespace {

constexpr int NT = 1024;

struct MfConst {
  float e_fg[2];   // -log(U_fg) for bit 0 / 1
  float e_bg[2];   // -log(U_bg) for bit 0 / 1
};

// K[j,p] = alpha0 * exp( -sum_c (F_c(p+d_j) - F_c(p))^2 / (2 theta0^2) - |d_j|^2 / (2 theta1^2) ), F = feature + 10,
// zero padded (discobox_head.py:596-610)
__global__ void mf_kernel_kernel(const float* __restrict__ feat, float* __restrict__ K, int C, int h, int w, int ks,
                                 float inv2t0, float inv2t1, float alpha0, int64_t total) {
  const int64_t hw = (int64_t)h * w;
  const int r = ks / 2, kk = ks * ks;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = i % w, y = (i / w) % h;
    const int64_t b = i / hw;
    for (int j = 0; j < kk; ++j) {
      const int dy = j / ks - r, dx = j % ks - r;
      const int qy = y + dy, qx = x + dx;
      const bool in = qy >= 0 && qy < h && qx >= 0 && qx < w;
      float acc = 0.f;
      for (int c = 0; c < C; ++c) {
        const float* f = feat + (b * C + c) * hw;
        const float centre = __fadd_rn(f[(int64_t)y * w + x], 10.f);
        const float nb = in ? __fadd_rn(f[(int64_t)qy * w + qx], 10.f) : 0.f;
        const float d = __fsub_rn(nb, centre);
        acc = __fadd_rn(acc, -__fmul_rn(d, d));
      }
      const float app = __fmul_rn(acc, inv2t0);                      // (-(..)^2).sum(1) / (2 theta0^2)
      const float spa = -__fmul_rn((float)(dy * dy + dx * dx), inv2t1);
      K[(b * kk + j) * hw + (int64_t)y * w + x] = __fmul_rn(alpha0, expf(__fadd_rn(app, spa)));
    }
  }
}

// One pixel of one mean-field round.  KS > 0: compile-time kernel size (taps unrolled, no integer division); KS == 0: `ks`.
// A pixel whose target is exactly 0 (outside the object's box -- most of the map) comes out 0 whatever its neighbours are:
// f_fg = exp(-agg_fg) * 0 + 1e-6 (agg_fg >= 0: the unaries are -log of probabilities and K >= 0, so no inf * 0) and
// f_bg >= 1e-6, hence f_fg / (f_bg + f_fg) <= 0.5, which is not > 0.5.  Skipping it is exact and removes ~85 % of the work.
// (With the inter-image term of corr_loss, f += iiu * gamma before the target product: still exact for iiu >= 0, which holds
// for the reference's iiu -- means of products of non-negative numbers, discobox_head.py:1094-1107.)
template <int KS, typename TG>
__device__ __forceinline__ uint8_t mf_update(const float* __restrict__ Kimg, const uint8_t* bits, const TG tgt,
                                             const MfConst& mc, int h, int w, int ks_rt, int y, int x,
                                             const float* __restrict__ iiu = nullptr, float gamma = 0.f) {
  if (tgt == 0.f) return 0;
  const int ks = KS > 0 ? KS : ks_rt;
  const int64_t hw = (int64_t)h * w, p = (int64_t)y * w + x;
  const int r = ks / 2;
  float agg_bg = 0.f, agg_fg = 0.f;
#pragma unroll
  for (int j = 0; j < ks * ks; ++j) {
    const int qy = y + j / ks - r, qx = x + j % ks - r;
    float ebg = 0.f, efg = 0.f;                                       // unfold zero-pads -log(U)
    if (qy >= 0 && qy < h && qx >= 0 && qx < w) {
      const bool bit = bits[qy * w + qx] != 0;
      ebg = bit ? mc.e_bg[1] : mc.e_bg[0];
      efg = bit ? mc.e_fg[1] : mc.e_fg[0];
    }
    const float kj = __ldg(Kimg + j * hw + p);
    agg_bg = __fadd_rn(agg_bg, __fmul_rn(ebg, kj));                   // (unfold_x * kernel).sum(2), tap order
    agg_fg = __fadd_rn(agg_fg, __fmul_rn(efg, kj));
  }
  float f_bg = expf(-agg_bg), f_fg = expf(-agg_fg);
  if (iiu) {                                                          // f += inter_img_mask * gamma (:643-644); [2,h,w] of the object
    f_bg = __fadd_rn(f_bg, __fmul_rn(__ldg(iiu + p), gamma));
    f_fg = __fadd_rn(f_fg, __fmul_rn(__ldg(iiu + hw + p), gamma));
  }
  f_fg = __fmul_rn(f_fg, (float)tgt);                                 // f[:,1:] *= targets
  f_bg = __fadd_rn(f_bg, 1e-6f);
  f_fg = __fadd_rn(f_fg, 1e-6f);
  const float s = __fadd_rn(f_bg, f_fg);
  return __fdiv_rn(f_fg, s) > 0.5f ? 1 : 0;
}

// The initial bit of pixel i: x * target > 0.5 (:629-630).  Float32: x is the caller's map.
__device__ __forceinline__ uint8_t init_bit(const float* __restrict__ x, const float* __restrict__, int64_t i,
                                            const float* __restrict__ tg, int64_t j) {
  return __fmul_rn(x[i], tg[j]) > 0.5f ? 1 : 0;
}
// 16-bit logits: x = (t + s) / 2 with the reference's autocast arithmetic, s = round_T(sigmoid(student)),
// t = round_T(sigmoid(teacher)) or s without an independent teacher, each T operation rounded to T; the same
// comparison as MeanField.forward on x.float() then follows.
template <typename T>
__device__ __forceinline__ uint8_t init_bit(const T* __restrict__ s_logits, const T* __restrict__ t_logits, int64_t i,
                                            const uint8_t* __restrict__ tg, int64_t j) {
  const float s = sigmoid_rounded(s_logits[i]);
  const float t = t_logits ? sigmoid_rounded(t_logits[i]) : s;
  const float m = round_to<T>(round_to<T>(t + s) * 0.5f);
  return __fmul_rn(m, (float)tg[j]) > 0.5f ? 1 : 0;
}

// one CTA per object; both bit maps in shared memory for all rounds.  R = float: ret / valid as MeanField.forward
// returns them; R = uint8_t: the pseudo-label only (valid unused).  x_t: teacher logits of the 16-bit form, or NULL.
template <int KS, typename X, typename TG, typename R>
__global__ void __launch_bounds__(NT) mf_fused_kernel(const float* __restrict__ K, const int32_t* __restrict__ obj_img,
                                                      const X* __restrict__ x, const TG* __restrict__ targets,
                                                      MfConst mc, R* __restrict__ ret, float* __restrict__ valid,
                                                      int h, int w, int ks, int iters, const float* __restrict__ iiu,
                                                      float gamma, const X* __restrict__ x_t) {
  extern __shared__ uint8_t sm_bits[];
  __shared__ int s_redi[NT / 32];
  const int n = blockIdx.x, hw = h * w;
  uint8_t* a = sm_bits;
  uint8_t* b = sm_bits + ((hw + 15) / 16) * 16;
  const float* Kimg = K + (int64_t)(obj_img ? obj_img[n] : 0) * ks * ks * hw;
  const TG* tg = targets + (int64_t)n * hw;
  const float* io = iiu ? iiu + (int64_t)n * 2 * hw : nullptr;
  for (int i = threadIdx.x; i < hw; i += NT) a[i] = init_bit(x, x_t, (int64_t)n * hw + i, tg, i);
  __syncthreads();
  for (int it = 0; it < iters; ++it) {
    for (int i = threadIdx.x; i < hw; i += NT) b[i] = mf_update<KS, TG>(Kimg, a, tg[i], mc, h, w, ks, i / w, i % w, io, gamma);
    __syncthreads();
    uint8_t* t = a; a = b; b = t;
  }
  if constexpr (std::is_same<R, float>::value) {
    int cnt = 0;
    for (int i = threadIdx.x; i < hw; i += NT) {
      ret[(int64_t)n * hw + i] = (float)a[i];
      cnt += a[i];
    }
    cnt = block_sum<int>(cnt, s_redi);
    if (threadIdx.x == 0)
      valid[n] = ((double)cnt >= (double)hw * 0.05 && (double)cnt <= (double)hw * 0.95) ? 1.f : 0.f;   // :631
  } else {
    for (int i = threadIdx.x; i < hw; i += NT) ret[(int64_t)n * hw + i] = a[i];
  }
}

// global ping-pong fallback for maps larger than shared memory
template <typename X, typename TG>
__global__ void mf_init_global(const X* __restrict__ x, const TG* __restrict__ targets, uint8_t* __restrict__ bits,
                               int64_t total, const X* __restrict__ x_t) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    bits[i] = init_bit(x, x_t, i, targets, i);
}
template <int KS, typename TG>
__global__ void mf_step_global(const float* __restrict__ K, const int32_t* __restrict__ obj_img,
                               const TG* __restrict__ targets, const uint8_t* __restrict__ src,
                               uint8_t* __restrict__ dst, MfConst mc, int h, int w, int ks, int64_t total,
                               const float* __restrict__ iiu, float gamma) {
  const int64_t hw = (int64_t)h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t n = i / hw;
    const int p = i % hw;
    const float* Kimg = K + (int64_t)(obj_img ? obj_img[n] : 0) * ks * ks * hw;
    dst[i] = mf_update<KS, TG>(Kimg, src + n * hw, targets[i], mc, h, w, ks, p / w, p % w, iiu ? iiu + n * 2 * hw : nullptr, gamma);
  }
}
__global__ void __launch_bounds__(256) mf_finish_global(const uint8_t* __restrict__ bits, float* __restrict__ ret,
                                                        float* __restrict__ valid, int hw) {
  __shared__ int s_redi[8];
  const int n = blockIdx.x;
  int cnt = 0;
  for (int i = threadIdx.x; i < hw; i += 256) {
    const int v = bits[(int64_t)n * hw + i];
    ret[(int64_t)n * hw + i] = (float)v;
    cnt += v;
  }
  cnt = block_sum<int>(cnt, s_redi);
  if (threadIdx.x == 0)
    valid[n] = ((double)cnt >= (double)hw * 0.05 && (double)cnt <= (double)hw * 0.95) ? 1.f : 0.f;
}

constexpr size_t kMaxFusedSmem = 200 * 1024;

}  // namespace
}  // namespace bxs

using namespace bxs;

// two_theta0_sq / two_theta1_sq are the reference's Python doubles 2*theta^2 rounded to float32; like
// torch's CUDA true-divide by a scalar the kernel multiplies by their float32 reciprocals.
extern "C" int bxs_meanfield_kernel(const float* feature, float* K, int64_t B, int64_t C, int64_t h, int64_t w,
                                    int kernel_size, float two_theta0_sq, float two_theta1_sq, float alpha0,
                                    bxs_stream_t stream) {
  if (!feature || !K || B <= 0 || C <= 0 || h <= 0 || w <= 0 || kernel_size < 1 || !(kernel_size & 1) ||
      !(two_theta0_sq > 0.f) || !(two_theta1_sq > 0.f))
    return BXS_ERR_INVALID_ARG;
  const int64_t total = B * h * w;
  mf_kernel_kernel<<<grid_for(total, 256), 256, 0, as_stream(stream)>>>(
      feature, K, (int)C, (int)h, (int)w, kernel_size, 1.f / two_theta0_sq, 1.f / two_theta1_sq, alpha0, total);
  return check_launch();
}

extern "C" int64_t bxs_meanfield_workspace_bytes(int64_t n, int64_t h, int64_t w) {
  return n <= 0 ? 0 : 2 * n * h * w + 64;
}

extern "C" int bxs_meanfield_forward_inter(const float* K, const int32_t* obj_img, const float* x, const float* targets,
                                           const float* inter_img_mask, float gamma, const float* neglog4_host, float* ret,
                                           float* valid, void* workspace, int64_t n, int64_t h, int64_t w, int kernel_size,
                                           int num_iter, bxs_stream_t stream) {
  const float* iiu = inter_img_mask;
  if (!K || !x || !targets || !neglog4_host || !ret || !valid || n <= 0 || n >= 65536 || h <= 0 || w <= 0 ||
      kernel_size < 1 || !(kernel_size & 1) || num_iter < 0 || h * w >= (int64_t(1) << 30))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  MfConst mc;
  mc.e_fg[0] = neglog4_host[0]; mc.e_fg[1] = neglog4_host[1];
  mc.e_bg[0] = neglog4_host[2]; mc.e_bg[1] = neglog4_host[3];
  const int64_t hw = h * w;
  const size_t sm = 2 * ((hw + 15) / 16) * 16;
  // One CTA per object keeps both bit maps in shared memory for all rounds, but it is ONE SM per object: a round of a
  // 200x256 map is ~4500 instructions per thread, whatever the number of objects (16 objects run on 16 of 132 SMs).
  // Unless there are enough objects to fill the machine that way, run the rounds as grid-wide
  // kernels over all objects' pixels (bit maps ping-pong through L2; the launches are graph-captured by the callers).
  const bool per_object = sm <= kMaxFusedSmem && (n >= 2 * (int64_t)sm_count() || !workspace);
  if (per_object) {
    auto fused = kernel_size == 3 ? mf_fused_kernel<3, float, float, float> : mf_fused_kernel<0, float, float, float>;
    if (opt_in_smem(fused, kMaxFusedSmem) != BXS_OK) return BXS_ERR_LAUNCH;
    fused<<<(unsigned)n, NT, sm, st>>>(K, obj_img, x, targets, mc, ret, valid, (int)h, (int)w, kernel_size, num_iter, iiu, gamma,
                                       nullptr);
  } else {
    if (!workspace) return BXS_ERR_INVALID_ARG;
    uint8_t* a = (uint8_t*)workspace;
    uint8_t* b = a + n * hw;
    const int64_t total = n * hw;
    mf_init_global<float, float><<<grid_for(total, 256), 256, 0, st>>>(x, targets, a, total, nullptr);
    for (int it = 0; it < num_iter; ++it) {
      if (kernel_size == 3)
        mf_step_global<3, float><<<grid_for(total, 256), 256, 0, st>>>(K, obj_img, targets, a, b, mc, (int)h, (int)w, kernel_size, total, iiu, gamma);
      else
        mf_step_global<0, float><<<grid_for(total, 256), 256, 0, st>>>(K, obj_img, targets, a, b, mc, (int)h, (int)w, kernel_size, total, iiu, gamma);
      std::swap(a, b);
    }
    mf_finish_global<<<(unsigned)n, 256, 0, st>>>(a, ret, valid, (int)hw);
  }
  return check_launch();
}

namespace bxs {
namespace {

template <typename T>
int meanfield_logits(const float* K, const int32_t* obj_img, const T* s, const T* t, const uint8_t* targets,
                     const MfConst& mc, uint8_t* out, void* workspace, int64_t n, int64_t h, int64_t w, int ks, int iters,
                     cudaStream_t st) {
  const int64_t hw = h * w;
  const size_t sm = 2 * ((hw + 15) / 16) * 16;
  // the same choice of schedule as bxs_meanfield_forward_inter
  const bool per_object = sm <= kMaxFusedSmem && (n >= 2 * (int64_t)sm_count() || !workspace);
  if (per_object) {
    auto fused = ks == 3 ? mf_fused_kernel<3, T, uint8_t, uint8_t> : mf_fused_kernel<0, T, uint8_t, uint8_t>;
    if (opt_in_smem(fused, kMaxFusedSmem) != BXS_OK) return BXS_ERR_LAUNCH;
    fused<<<(unsigned)n, NT, sm, st>>>(K, obj_img, s, targets, mc, out, nullptr, (int)h, (int)w, ks, iters, nullptr, 0.f, t);
  } else {
    // ping-pong between the workspace and `out`, starting on the side that makes the last round land in `out`
    uint8_t* a = iters % 2 == 0 ? out : (uint8_t*)workspace;
    uint8_t* b = iters % 2 == 0 ? (uint8_t*)workspace : out;
    const int64_t total = n * hw;
    mf_init_global<T, uint8_t><<<grid_for(total, 256), 256, 0, st>>>(s, targets, a, total, t);
    for (int it = 0; it < iters; ++it) {
      if (ks == 3)
        mf_step_global<3, uint8_t><<<grid_for(total, 256), 256, 0, st>>>(K, obj_img, targets, a, b, mc, (int)h, (int)w, ks, total, nullptr, 0.f);
      else
        mf_step_global<0, uint8_t><<<grid_for(total, 256), 256, 0, st>>>(K, obj_img, targets, a, b, mc, (int)h, (int)w, ks, total, nullptr, 0.f);
      std::swap(a, b);
    }
  }
  return check_launch();
}

}  // namespace
}  // namespace bxs

extern "C" int bxs_meanfield_forward_logits(const float* K, const int32_t* obj_img, const void* s_logits,
                                            const void* t_logits, const uint8_t* targets, int dtype,
                                            const float* neglog4_host, uint8_t* pseudo, void* workspace, int64_t n,
                                            int64_t h, int64_t w, int kernel_size, int num_iter, bxs_stream_t stream) {
  if (n < 0 || h <= 0 || w <= 0 || kernel_size < 1 || !(kernel_size & 1) || num_iter < 0 ||
      (dtype != BXS_F16 && dtype != BXS_BF16))
    return BXS_ERR_INVALID_ARG;
  if (n > 0 && (!K || !s_logits || !targets || !neglog4_host || !pseudo)) return BXS_ERR_INVALID_ARG;
  if (h * w >= (int64_t(1) << 30)) return BXS_ERR_UNSUPPORTED;
  if (!workspace && 2 * ((h * w + 15) / 16) * 16 > (int64_t)kMaxFusedSmem) return BXS_ERR_INVALID_ARG;
  if (n == 0) return BXS_OK;
  MfConst mc;
  mc.e_fg[0] = neglog4_host[0]; mc.e_fg[1] = neglog4_host[1];
  mc.e_bg[0] = neglog4_host[2]; mc.e_bg[1] = neglog4_host[3];
  cudaStream_t st = as_stream(stream);
  if (dtype == BXS_F16)
    return meanfield_logits(K, obj_img, static_cast<const __half*>(s_logits), static_cast<const __half*>(t_logits), targets,
                            mc, pseudo, workspace, n, h, w, kernel_size, num_iter, st);
  return meanfield_logits(K, obj_img, static_cast<const __nv_bfloat16*>(s_logits),
                          static_cast<const __nv_bfloat16*>(t_logits), targets, mc, pseudo, workspace, n, h, w, kernel_size,
                          num_iter, st);
}
