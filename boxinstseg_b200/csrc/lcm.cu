// a11: Local Consistency Module of Box2Mask -- 8 dilated-neighbour affinity (softmax of the
// std-normalised colour distance) and `num_iter` propagation steps phi <- sum_k aff_k phi_k with
// replicate padding; loss = sum |phi_T - phi_0| box / max(sum box, 1).  Forward + backward wrt phi_0.
// Replaces LCM / LocalConsistencyModule (mmdet/models/losses/levelset_loss.py:64-126), which builds
// a fresh nn.Module per call and runs ~35 small launches (pad, one-hot conv, elementwise) whose
// autograd tape is replayed backwards through all iterations.
//
// Design: the maps are small (96x96 in every config of the reference), so ONE CTA per instance
// keeps phi ping-ponged in shared memory across all iterations (forward) and applies the
// transposed operator the same way (backward, gather form -> deterministic, no float atomics).
// Maps that do not fit shared memory use the same step function over global ping-pong buffers,
// one launch per iteration.
#include <algorithm>

#include "common.cuh"

namespace bxs {
namespace {

constexpr int NT = 1024;
constexpr float kAlpha = 0.3f;     // levelset_loss.py:84
constexpr float kStdEps = 1e-8f;   // :115

// neighbour k of the 3x3 stencil without centre: taps (0,0),(0,1),(0,2),(1,0),(1,2),(2,0),(2,1),(2,2)
__device__ __forceinline__ void tap(int k, int& dy, int& dx) {
  const int kk = k < 4 ? k : k + 1;
  dy = kk / 3 - 1;
  dx = kk % 3 - 1;
}
__device__ __forceinline__ int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

__global__ void affinity_kernel(const float* __restrict__ imgs, float* __restrict__ aff, int C, int h, int w, int d,
                                int64_t total) {
  const int64_t hw = (int64_t)h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = i % w, y = (i / w) % h;
    const int64_t n = i / hw;
    float logit[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) logit[k] = 0.f;
    for (int c = 0; c < C; ++c) {
      const float* im = imgs + (n * C + c) * hw;
      const float centre = im[(int64_t)y * w + x];
      float v[8], mean = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        int dy, dx;
        tap(k, dy, dx);
        v[k] = im[(int64_t)clampi(y + dy * d, 0, h - 1) * w + clampi(x + dx * d, 0, w - 1)];
        mean += v[k];
      }
      mean *= 0.125f;
      float var = 0.f;
#pragma unroll
      for (int k = 0; k < 8; ++k) var = fmaf(v[k] - mean, v[k] - mean, var);
      const float sd = sqrtf(var / 7.f);                           // torch.std: unbiased over the 8 neighbours
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float z = fabsf(v[k] - centre) / (sd + kStdEps) / kAlpha;
        logit[k] -= z * z;
      }
    }
    float mx = -INFINITY;
#pragma unroll
    for (int k = 0; k < 8; ++k) { logit[k] /= (float)C; mx = fmaxf(mx, logit[k]); }
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 8; ++k) { logit[k] = expf(logit[k] - mx); sum += logit[k]; }
#pragma unroll
    for (int k = 0; k < 8; ++k) aff[(n * 8 + k) * hw + (int64_t)y * w + x] = logit[k] / sum;
  }
}

// forward step at pixel (y,x): sum_k aff_k(p) * src[clamp(p + delta_k)]
__device__ __forceinline__ float step_fwd(const float* __restrict__ aff_n, const float* src, int h, int w, int d, int y,
                                          int x) {
  const int64_t hw = (int64_t)h * w, p = (int64_t)y * w + x;
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int dy, dx;
    tap(k, dy, dx);
    acc = fmaf(__ldg(aff_n + k * hw + p), src[clampi(y + dy * d, 0, h - 1) * w + clampi(x + dx * d, 0, w - 1)], acc);
  }
  return acc;
}

// transposed step at pixel q: sum over k and over all p with clamp(p + delta_k) == q of aff_k(p) * src[p]
__device__ __forceinline__ float step_bwd(const float* __restrict__ aff_n, const float* src, int h, int w, int d, int y,
                                          int x) {
  const int64_t hw = (int64_t)h * w;
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    int dy, dx;
    tap(k, dy, dx);
    dy *= d; dx *= d;
    // 1-D preimage of q under p -> clamp(p + delta): a single point in the interior, a short run at a border
    int y_lo = y - dy, y_hi = y - dy, x_lo = x - dx, x_hi = x - dx;
    if (y == 0 && dy < 0) y_lo = 0;               // p + dy <= 0  <=>  p <= -dy
    if (y == h - 1 && dy > 0) y_hi = h - 1;       // p + dy >= h-1
    if (x == 0 && dx < 0) x_lo = 0;
    if (x == w - 1 && dx > 0) x_hi = w - 1;
    y_lo = max(y_lo, 0); y_hi = min(y_hi, h - 1); x_lo = max(x_lo, 0); x_hi = min(x_hi, w - 1);
    for (int py = y_lo; py <= y_hi; ++py)
      for (int px = x_lo; px <= x_hi; ++px) {
        const int64_t p = (int64_t)py * w + px;
        acc = fmaf(__ldg(aff_n + k * hw + p), src[p], acc);
      }
  }
  return acc;
}

// one CTA per instance, all iterations in shared memory.  MODE 0: forward (writes phi_T and the
// per-instance loss numerator / box sum); MODE 1: backward (g_phi0 = (A^T)^iters r - r).
template <int MODE>
__global__ void __launch_bounds__(NT) lcm_fused_kernel(const float* __restrict__ aff, const float* __restrict__ phi0,
                                                       const float* __restrict__ box, float* __restrict__ phiT,
                                                       float* __restrict__ inst_sums, const float* __restrict__ scale_ptr,
                                                       float* __restrict__ g_phi0, int h, int w, int d, int iters) {
  extern __shared__ float smem[];
  __shared__ float s_red[NT / 32];
  const int n = blockIdx.x, hw = h * w;
  float* a = smem;
  float* b = smem + hw;
  const float* aff_n = aff + (int64_t)n * 8 * hw;
  const float scale = MODE == 1 ? scale_ptr[0] : 0.f;
  for (int i = threadIdx.x; i < hw; i += NT) {
    if (MODE == 0) {
      a[i] = phi0[(int64_t)n * hw + i];
    } else {
      const float dlt = phiT[(int64_t)n * hw + i] - phi0[(int64_t)n * hw + i];
      a[i] = ((dlt > 0.f) - (dlt < 0.f)) * box[(int64_t)n * hw + i] * scale;      // d|x| = sign(x), sign(0) = 0
    }
  }
  __syncthreads();
  for (int it = 0; it < iters; ++it) {
    for (int i = threadIdx.x; i < hw; i += NT) {
      const int y = i / w, x = i - y * w;
      b[i] = MODE == 0 ? step_fwd(aff_n, a, h, w, d, y, x) : step_bwd(aff_n, a, h, w, d, y, x);
    }
    __syncthreads();
    float* t = a; a = b; b = t;
  }
  if (MODE == 0) {
    float num = 0.f, den = 0.f;
    for (int i = threadIdx.x; i < hw; i += NT) {
      const float bx = box[(int64_t)n * hw + i];
      phiT[(int64_t)n * hw + i] = a[i];
      num = fmaf(fabsf(a[i] - phi0[(int64_t)n * hw + i]), bx, num);
      den += bx;
    }
    num = block_sum<float>(num, s_red);
    den = block_sum<float>(den, s_red);
    if (threadIdx.x == 0) { inst_sums[2 * n] = num; inst_sums[2 * n + 1] = den; }
  } else {
    for (int i = threadIdx.x; i < hw; i += NT) {
      const float dlt = phiT[(int64_t)n * hw + i] - phi0[(int64_t)n * hw + i];
      const float r = ((dlt > 0.f) - (dlt < 0.f)) * box[(int64_t)n * hw + i] * scale;
      g_phi0[(int64_t)n * hw + i] = a[i] - r;
    }
  }
}

// global-memory variants for maps that do not fit shared memory (one launch per iteration)
template <int MODE>
__global__ void lcm_step_global(const float* __restrict__ aff, const float* __restrict__ src, float* __restrict__ dst,
                                int h, int w, int d, int64_t total) {
  const int64_t hw = (int64_t)h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = i % w, y = (i / w) % h;
    const int64_t n = i / hw;
    dst[i] = MODE == 0 ? step_fwd(aff + n * 8 * hw, src + n * hw, h, w, d, y, x)
                       : step_bwd(aff + n * 8 * hw, src + n * hw, h, w, d, y, x);
  }
}

__global__ void __launch_bounds__(256) lcm_sums_global(const float* __restrict__ phiT, const float* __restrict__ phi0,
                                                       const float* __restrict__ box, float* __restrict__ inst_sums,
                                                       int hw) {
  __shared__ float s_red[8];
  const int n = blockIdx.x;
  float num = 0.f, den = 0.f;
  for (int i = threadIdx.x; i < hw; i += 256) {
    const float bx = box[(int64_t)n * hw + i];
    num = fmaf(fabsf(phiT[(int64_t)n * hw + i] - phi0[(int64_t)n * hw + i]), bx, num);
    den += bx;
  }
  num = block_sum<float>(num, s_red);
  den = block_sum<float>(den, s_red);
  if (threadIdx.x == 0) { inst_sums[2 * n] = num; inst_sums[2 * n + 1] = den; }
}

__global__ void lcm_residual_global(const float* __restrict__ phiT, const float* __restrict__ phi0,
                                    const float* __restrict__ box, const float* __restrict__ scale_ptr,
                                    float* __restrict__ r, int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const float dlt = phiT[i] - phi0[i];
    r[i] = ((dlt > 0.f) - (dlt < 0.f)) * box[i] * scale_ptr[0];
  }
}

__global__ void lcm_sub_global(const float* __restrict__ a, const float* __restrict__ r, float* __restrict__ out,
                               int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = a[i] - r[i];
}

// loss = sum_n num_n / max(sum_n den_n, 1); also 1/max(.,1) for the backward
__global__ void lcm_total_kernel(const float* __restrict__ inst_sums, int n, float* __restrict__ out) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  float num = 0.f, den = 0.f;
  for (int i = 0; i < n; ++i) { num += inst_sums[2 * i]; den += inst_sums[2 * i + 1]; }
  const float z = fmaxf(den, 1.f);
  out[0] = num / z;
  out[1] = 1.f / z;
}

__global__ void lcm_scale_kernel(const float* __restrict__ out, const float* __restrict__ g_loss, float* __restrict__ scale) {
  if (threadIdx.x == 0 && blockIdx.x == 0) scale[0] = g_loss[0] * out[1];
}

inline int grid_for(int64_t total, int block) {
  const int64_t g = ceil_div(total, block), cap = (int64_t)sm_count() * 8;
  return (int)std::max<int64_t>(1, std::min(g, cap));
}

constexpr size_t kMaxFusedSmem = 200 * 1024;

}  // namespace
}  // namespace bxs

using namespace bxs;

// workspace layout (floats): aff [n*8*hw] | phiT [n*hw] | tmpA [n*hw] | tmpB [n*hw] | inst_sums [2n] | out2 [2] | scale [1]
extern "C" int64_t bxs_lcm_workspace_bytes(int64_t n, int64_t h, int64_t w) {
  if (n <= 0 || h <= 0 || w <= 0) return 0;
  return (int64_t)sizeof(float) * (n * 11 * h * w + 2 * n + 8);
}

extern "C" int bxs_lcm_forward(const float* imgs, const float* phis, const float* box, float* loss_out, void* workspace,
                               int64_t n, int64_t C, int64_t h, int64_t w, int dilation, int num_iter,
                               bxs_stream_t stream) {
  if (!imgs || !phis || !box || !loss_out || !workspace || n <= 0 || n >= 65536 || C <= 0 || h <= 0 || w <= 0 ||
      dilation < 1 || num_iter < 0 || h * w >= (int64_t(1) << 30))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  const int64_t hw = h * w, total = n * hw;
  float* aff = (float*)workspace;
  float* phiT = aff + n * 8 * hw;
  float* tmpA = phiT + total;
  float* tmpB = tmpA + total;
  float* inst = tmpB + total;
  float* out2 = inst + 2 * n;
  affinity_kernel<<<grid_for(total, 256), 256, 0, st>>>(imgs, aff, (int)C, (int)h, (int)w, dilation, total);
  const size_t sm = 2 * hw * sizeof(float);
  // One CTA per instance keeps phi in shared memory for all iterations, but it is ONE SM per instance: 8 instances of a
  // 96x96 map run on 8 of 132 SMs, issue-bound.
  // Unless the instances fill the machine that way, run the iterations as grid-wide kernels (phi ping-pongs through L2; same arithmetic
  // per pixel, same results; the launches are graph-captured by the callers).
  if (sm <= kMaxFusedSmem && n >= 2 * (int64_t)sm_count()) {
    cudaFuncSetAttribute(lcm_fused_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxFusedSmem);
    lcm_fused_kernel<0><<<(unsigned)n, NT, sm, st>>>(aff, phis, box, phiT, inst, nullptr, nullptr, (int)h, (int)w,
                                                     dilation, num_iter);
  } else {
    const float* src = phis;
    for (int it = 0; it < num_iter; ++it) {
      float* dst = (it == num_iter - 1) ? phiT : ((it & 1) ? tmpB : tmpA);
      lcm_step_global<0><<<grid_for(total, 256), 256, 0, st>>>(aff, src, dst, (int)h, (int)w, dilation, total);
      src = dst;
    }
    if (num_iter == 0) cudaMemcpyAsync(phiT, phis, total * sizeof(float), cudaMemcpyDeviceToDevice, st);
    lcm_sums_global<<<(unsigned)n, 256, 0, st>>>(phiT, phis, box, inst, (int)hw);
  }
  lcm_total_kernel<<<1, 32, 0, st>>>(inst, (int)n, out2);
  cudaMemcpyAsync(loss_out, out2, sizeof(float), cudaMemcpyDeviceToDevice, st);
  return check_launch();
}

extern "C" int bxs_lcm_backward(const float* phis, const float* box, const void* workspace, const float* g_loss,
                                float* g_phis, int64_t n, int64_t h, int64_t w, int dilation, int num_iter,
                                bxs_stream_t stream) {
  if (!phis || !box || !workspace || !g_loss || !g_phis || n <= 0 || n >= 65536 || h <= 0 || w <= 0 || dilation < 1 ||
      num_iter < 0)
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  const int64_t hw = h * w, total = n * hw;
  float* aff = (float*)const_cast<void*>(workspace);
  float* phiT = aff + n * 8 * hw;
  float* tmpA = phiT + total;
  float* tmpB = tmpA + total;
  float* inst = tmpB + total;
  float* out2 = inst + 2 * n;
  float* scale = out2 + 2;
  lcm_scale_kernel<<<1, 32, 0, st>>>(out2, g_loss, scale);
  const size_t sm = 2 * hw * sizeof(float);
  if (sm <= kMaxFusedSmem && n >= 2 * (int64_t)sm_count()) {
    cudaFuncSetAttribute(lcm_fused_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kMaxFusedSmem);
    lcm_fused_kernel<1><<<(unsigned)n, NT, sm, st>>>(aff, phis, box, phiT, nullptr, scale, g_phis, (int)h, (int)w,
                                                     dilation, num_iter);
  } else {
    // r -> tmpA ; iterate the transposed operator between g_phis / tmpB ; out = result - r
    lcm_residual_global<<<grid_for(total, 256), 256, 0, st>>>(phiT, phis, box, scale, tmpA, total);
    const float* src = tmpA;
    float* bufs[2] = {g_phis, tmpB};
    for (int it = 0; it < num_iter; ++it) {
      float* dst = bufs[it & 1];
      lcm_step_global<1><<<grid_for(total, 256), 256, 0, st>>>(aff, src, dst, (int)h, (int)w, dilation, total);
      src = dst;
    }
    lcm_sub_global<<<grid_for(total, 256), 256, 0, st>>>(src, tmpA, g_phis, total);
  }
  return check_launch();
}
