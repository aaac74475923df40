// f4: DiscoBox's semantic-correspondence path as kernels (mmdet/models/dense_heads/discobox_head.py):
//   bxs_corr_solve     SemanticCorrSolver.solve :393-410 -- one CTA per retrieved object, the [P,P] vote table and its
//                      ping-pong copy in shared memory for all num_iter x num_smooth rounds (ONE launch instead of ~250).
//   bxs_corr_transfer  corr_loss :1086-1096 + superres_T :851-865 -- one thread per (object, query mask pixel); the six
//                      [K,784,784] intermediates of the reference (T_superres, fg/bg masks, their products: 12 MB each)
//                      are never built; the mean over the objects is a second, fixed-order pass (deterministic).
// The per-element arithmetic lives in corr_core.cuh (compiled for the host as well by tests/host_harness/corr_host.cpp).
#include "common.cuh"
#include "corr_core.cuh"

namespace bxs {
namespace {

constexpr int NT_SOLVE = 1024;
constexpr int NT_XFER = 128;
constexpr int64_t kMaxSmem = 200 * 1024;

__global__ void __launch_bounds__(NT_SOLVE) corr_solve_kernel(const float* __restrict__ Cu, float* __restrict__ T, int h, int w,
                                                              int dist_kernel, int num_iter, int num_smooth) {
  extern __shared__ float sm[];
  const int P = h * w, PP = P * P;
  const int64_t k = blockIdx.x;
  corr_solve(Cu + k * PP, T + k * PP, sm, sm + PP, sm + 2 * PP, h, w, dist_kernel, num_iter, num_smooth);
}

__global__ void __launch_bounds__(NT_XFER) corr_transfer_kernel(const float* __restrict__ T, const float* __restrict__ Cu,
                                                                const float* __restrict__ m0, const float* __restrict__ m1,
                                                                float* __restrict__ partial, int h, int w, int Hm, int Wm) {
  extern __shared__ float sm[];
  const int P = h * w, PP = P * P, M = Hm * Wm;
  const int64_t k = blockIdx.y;
  float* t2 = sm;                 // [PP]
  float* rs = t2 + PP;            // [P]
  float* mx = rs + P;             // [P]
  float* s_m1 = mx + P;           // [M]
  float* R = s_m1 + M;            // [NT_XFER * P]
  CorrTap* tapV = reinterpret_cast<CorrTap*>(R + NT_XFER * P);   // [Hm]
  CorrTap* tapU = tapV + Hm;                                      // [Wm]
  corr_phase(Hm, [&](int i) { tapV[i] = corr_tap(i, h, Hm); });
  corr_phase(Wm, [&](int i) { tapU[i] = corr_tap(i, w, Wm); });
  corr_weighted(T + k * PP, Cu + k * PP, t2, rs, mx, P, [](float v) { return expf(v); });
  corr_phase(M, [&](int i) { s_m1[i] = m1[k * M + i]; });
  const int pq = blockIdx.x * NT_XFER + threadIdx.x;
  if (pq < M) {
    float fg, bg;
    corr_transfer_pixel(t2, m0[pq], s_m1, R + threadIdx.x * P, tapV, tapU, h, w, Hm, Wm, pq, &fg, &bg);
    partial[(k * 2 + 0) * M + pq] = fg;
    partial[(k * 2 + 1) * M + pq] = bg;
  }
}

// .mean(0) over the objects, in object order
__global__ void __launch_bounds__(NT_XFER) corr_mean_kernel(const float* __restrict__ partial, float* __restrict__ fg,
                                                            float* __restrict__ bg, int K, int M) {
  const int pq = blockIdx.x * NT_XFER + threadIdx.x;
  if (pq >= M) return;
  float a = 0.f, b = 0.f;
  for (int k = 0; k < K; ++k) {
    a = __fadd_rn(a, partial[(k * 2 + 0) * (int64_t)M + pq]);
    b = __fadd_rn(b, partial[(k * 2 + 1) * (int64_t)M + pq]);
  }
  fg[pq] = __fdiv_rn(a, (float)K);
  bg[pq] = __fdiv_rn(b, (float)K);
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_corr_solve(const float* Cu, float* T, int64_t K, int64_t h, int64_t w, int dist_kernel, int num_iter,
                              int num_smooth, bxs_stream_t stream) {
  if (!Cu || !T || K <= 0 || h <= 0 || w <= 0 || dist_kernel <= 0 || (dist_kernel & 1) == 0 || num_iter < 0 || num_smooth < 0)
    return BXS_ERR_INVALID_ARG;        // an even window would change the size of the reference's max_pool2d output (:394)
  const int64_t P = h * w;
  const int64_t smem = (2 * P * P + (1 + kCorrLanes) * P) * 4;
  if (smem > kMaxSmem || K > 65535) return BXS_ERR_UNSUPPORTED;
  if (smem > 48 * 1024 && opt_in_smem(corr_solve_kernel, smem) != BXS_OK) return BXS_ERR_LAUNCH;
  corr_solve_kernel<<<(unsigned)K, NT_SOLVE, smem, as_stream(stream)>>>(Cu, T, (int)h, (int)w, dist_kernel, num_iter, num_smooth);
  return check_launch();
}

extern "C" int64_t bxs_corr_transfer_workspace_bytes(int64_t K, int64_t Hm, int64_t Wm) {
  if (K <= 0 || Hm <= 0 || Wm <= 0) return 0;
  return K * 2 * Hm * Wm * 4;
}

extern "C" int bxs_corr_transfer(const float* T, const float* Cu, const float* m0, const float* m1, float* fg_ci, float* bg_ci,
                                 void* workspace, int64_t K, int64_t h, int64_t w, int64_t Hm, int64_t Wm,
                                 bxs_stream_t stream) {
  if (!T || !Cu || !m0 || !m1 || !fg_ci || !bg_ci || !workspace || K <= 0 || h <= 0 || w <= 0 || Hm <= 0 || Wm <= 0)
    return BXS_ERR_INVALID_ARG;
  const int64_t P = h * w, M = Hm * Wm;
  const int64_t smem = (P * P + 2 * P + M + (int64_t)NT_XFER * P) * 4 + (Hm + Wm) * (int64_t)sizeof(CorrTap);
  if (smem > kMaxSmem || K > 65535 || M > (int64_t(1) << 24)) return BXS_ERR_UNSUPPORTED;
  if (smem > 48 * 1024 && opt_in_smem(corr_transfer_kernel, smem) != BXS_OK) return BXS_ERR_LAUNCH;
  float* partial = static_cast<float*>(workspace);
  const unsigned gx = (unsigned)ceil_div(M, NT_XFER);
  corr_transfer_kernel<<<dim3(gx, (unsigned)K), NT_XFER, smem, as_stream(stream)>>>(T, Cu, m0, m1, partial, (int)h, (int)w,
                                                                                    (int)Hm, (int)Wm);
  int rc = check_launch();
  if (rc != BXS_OK) return rc;
  corr_mean_kernel<<<gx, NT_XFER, 0, as_stream(stream)>>>(partial, fg_ci, bg_ci, (int)K, (int)M);
  return check_launch();
}
