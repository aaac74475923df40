// f4: DiscoBox's semantic-correspondence path as kernels (mmdet/models/dense_heads/discobox_head.py):
//   bxs_corr_solve     SemanticCorrSolver.solve :393-410 -- one CTA per retrieved object, the [P,P] vote table and its
//                      ping-pong copy in shared memory for all num_iter x num_smooth rounds (ONE launch instead of ~250).
//   bxs_corr_transfer  corr_loss :1086-1096 + superres_T :851-865 -- one thread per (object, query mask pixel); the six
//                      [K,784,784] intermediates of the reference (T_superres, fg/bg masks, their products: 12 MB each)
//                      are never built; the mean over the objects is a second, fixed-order pass (deterministic).
//   bxs_corr_retrieve  get_similar_obj :174-221 for all query objects of a level, the order dependence of the per-object
//                      loop (:1056-1125) resolved on the device: one CTA per query (corr_core.cuh: corr_retrieve_query).
//   bxs_corr_paste     :1098-1107 -- the two transferred maps of every query resized to its box and written into iiu.
//   bxs_corr_bank_append  :1113-1124 -- the ordered ring append of the level's eligible objects (last writer wins) and the
//                      ptr / exists / first-query state, on the device.
// bxs_corr_solve_batched / bxs_corr_transfer_batched run over all the level's tables in one launch each, with a per-query
// count; bxs_corr_solve / bxs_corr_transfer are their single-query cases.
// The per-element arithmetic lives in corr_core.cuh (compiled for the host as well by tests/host_harness/corr_host.cpp and,
// for the retrieval, corr_retrieve_host.cpp).
#include "common.cuh"
#include "corr_core.cuh"
#include "resize_core.cuh"

namespace bxs {
namespace {

constexpr int NT_SOLVE = 1024;
constexpr int NT_XFER = 128;
constexpr int NT_RETR = 512;
constexpr int NT_PASTE = 256;
constexpr int NT_APPEND = 256;
constexpr int64_t kMaxSmem = 200 * 1024;

// table k of query k / kmax; with counts, the tables at or past the query's count are zero-filled and cost no solve
__global__ void __launch_bounds__(NT_SOLVE) corr_solve_kernel(const float* __restrict__ Cu, float* __restrict__ T,
                                                              const int32_t* __restrict__ counts, int kmax, int h, int w,
                                                              int dist_kernel, int num_iter, int num_smooth) {
  extern __shared__ float sm[];
  const int P = h * w, PP = P * P;
  const int64_t k = blockIdx.x;
  if (counts && (int)(k % kmax) >= counts[k / kmax]) {
    for (int i = threadIdx.x; i < PP; i += NT_SOLVE) T[k * PP + i] = 0.f;
    return;
  }
  corr_solve(Cu + k * PP, T + k * PP, sm, sm + PP, sm + 2 * PP, h, w, dist_kernel, num_iter, num_smooth);
}

// CTA (pixel block, table j, query q): table q * kmax + j against query mask q; tables past the query's count do nothing
__global__ void __launch_bounds__(NT_XFER) corr_transfer_kernel(const float* __restrict__ T, const float* __restrict__ Cu,
                                                                const float* __restrict__ m0, const float* __restrict__ m1,
                                                                const int32_t* __restrict__ counts, float* __restrict__ partial,
                                                                int kmax, int h, int w, int Hm, int Wm) {
  extern __shared__ float sm[];
  const int P = h * w, PP = P * P, M = Hm * Wm;
  const int q = blockIdx.z;
  if (counts && (int)blockIdx.y >= counts[q]) return;
  const int64_t k = (int64_t)q * kmax + blockIdx.y;
  m0 += (int64_t)q * M;
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

// .mean(0) over the objects of query blockIdx.y, in object order (zero for a query without tables)
__global__ void __launch_bounds__(NT_XFER) corr_mean_kernel(const float* __restrict__ partial, const int32_t* __restrict__ counts,
                                                            float* __restrict__ fg, float* __restrict__ bg, int kmax, int M) {
  const int pq = blockIdx.x * NT_XFER + threadIdx.x;
  if (pq >= M) return;
  const int q = blockIdx.y;
  const int K = counts ? counts[q] : kmax;
  const float* part = partial + (int64_t)q * kmax * 2 * M;
  float a = 0.f, b = 0.f;
  for (int k = 0; k < K; ++k) {
    a = __fadd_rn(a, part[(k * 2 + 0) * (int64_t)M + pq]);
    b = __fadd_rn(b, part[(k * 2 + 1) * (int64_t)M + pq]);
  }
  fg[(int64_t)q * M + pq] = K > 0 ? __fdiv_rn(a, (float)K) : 0.f;
  bg[(int64_t)q * M + pq] = K > 0 ? __fdiv_rn(b, (float)K) : 0.f;
}

__global__ void __launch_bounds__(NT_RETR) corr_retrieve_kernel(CorrBank bank, CorrLevel lvl, CorrRetrieveCfg cfg,
                                                                const int32_t* __restrict__ first, CorrRetrieveOut out) {
  extern __shared__ float sm[];
  corr_retrieve_query(bank, lvl, cfg, *first, blockIdx.x, sm, out);
}

// iiu[2q] / iiu[2q+1] over the box of query q = the bilinear resize of bg / fg to the box (F.interpolate, align_corners
// False); the rest of iiu is left as it is.  grid (pixel blocks, 2, n)
__global__ void __launch_bounds__(NT_PASTE) corr_paste_kernel(const float* __restrict__ fg, const float* __restrict__ bg,
                                                              const float* __restrict__ box, const int32_t* __restrict__ counts,
                                                              float* __restrict__ iiu, int Hm, int Wm, int H, int W) {
  const int q = blockIdx.z, ch = blockIdx.y;
  if (counts[q] <= 0) return;
  const int x1 = (int)box[4 * q + 0], y1 = (int)box[4 * q + 1], x2 = (int)box[4 * q + 2], y2 = (int)box[4 * q + 3];
  const int bh = y2 - y1, bw = x2 - x1;
  if (bh <= 0 || bw <= 0) return;
  const int e = blockIdx.x * NT_PASTE + threadIdx.x;
  if (e >= bh * bw) return;
  const int oy = e / bw, ox = e - oy * bw, Y = y1 + oy, X = x1 + ox;
  if (Y < 0 || Y >= H || X < 0 || X >= W) return;
  const float* in = (ch == 0 ? bg : fg) + (int64_t)q * Hm * Wm;
  iiu[((int64_t)(2 * q + ch) * H + Y) * W + X] = rs_pixel(in, Hm, Wm, rs_scale(Hm, bh, false), rs_scale(Wm, bw, false), oy, ox, false);
}

// CTA per object of the level: copy its teacher RoI feature / mask / box to its slot unless a later object of the level
// writes the same slot; the last appending object of a class sets the class's ptr and exists; CTA 0 clears the head's
// first-query flag once the level had a live object.
__global__ void __launch_bounds__(NT_APPEND) corr_append_kernel(float* __restrict__ feat, float* __restrict__ mask,
                                                                float* __restrict__ bbox, int32_t* __restrict__ ptr,
                                                                int32_t* __restrict__ exists, int32_t* __restrict__ first,
                                                                CorrLevel lvl, const int32_t* __restrict__ slot, int num_class,
                                                                int L, int CP, int M) {
  __shared__ int s_copy;
  const int i = blockIdx.x;
  if (threadIdx.x == 0) {
    int copy = 0;
    const int si = slot[i];
    if (si >= 0) {
      const int c = lvl.label[i];
      bool overwritten = false, last = true;
      for (int j = i + 1; j < lvl.n; ++j) {
        if (slot[j] < 0 || lvl.label[j] != c) continue;
        last = false;
        if (slot[j] == si) overwritten = true;
      }
      copy = !overwritten;
      if (last) {
        ptr[c] = (si + 1) % L;
        exists[c] = 1;
      }
    }
    if (i == 0) {
      bool any = false;
      for (int j = 0; j < lvl.n; ++j) any = any || corr_live(lvl, num_class, j);
      if (any) *first = 0;
    }
    s_copy = copy;
  }
  __syncthreads();
  if (!s_copy) return;
  const int64_t row = (int64_t)lvl.label[i] * L + slot[i];
  for (int e = threadIdx.x; e < CP; e += NT_APPEND) feat[row * CP + e] = lvl.t_feat[(int64_t)i * CP + e];
  for (int e = threadIdx.x; e < M; e += NT_APPEND) mask[row * M + e] = lvl.t_mask[(int64_t)i * M + e];
  if (threadIdx.x < 4) bbox[row * 4 + threadIdx.x] = lvl.box[4 * i + threadIdx.x];
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_corr_solve_batched(const float* Cu, float* T, const int32_t* counts, int64_t n, int64_t kmax, int64_t h,
                                      int64_t w, int dist_kernel, int num_iter, int num_smooth, bxs_stream_t stream) {
  if (!Cu || !T || n <= 0 || kmax <= 0 || h <= 0 || w <= 0 || dist_kernel <= 0 || (dist_kernel & 1) == 0 || num_iter < 0 ||
      num_smooth < 0)
    return BXS_ERR_INVALID_ARG;        // an even window would change the size of the reference's max_pool2d output (:394)
  const int64_t P = h * w, K = n * kmax;
  const int64_t smem = (2 * P * P + (1 + kCorrLanes) * P) * 4;
  if (smem > kMaxSmem || n > INT32_MAX / kmax) return BXS_ERR_UNSUPPORTED;
  if (smem > 48 * 1024 && opt_in_smem(corr_solve_kernel, smem) != BXS_OK) return BXS_ERR_LAUNCH;
  corr_solve_kernel<<<(unsigned)K, NT_SOLVE, smem, as_stream(stream)>>>(Cu, T, counts, (int)kmax, (int)h, (int)w, dist_kernel,
                                                                        num_iter, num_smooth);
  return check_launch();
}

extern "C" int bxs_corr_solve(const float* Cu, float* T, int64_t K, int64_t h, int64_t w, int dist_kernel, int num_iter,
                              int num_smooth, bxs_stream_t stream) {
  if (K > 65535) return BXS_ERR_UNSUPPORTED;
  return bxs_corr_solve_batched(Cu, T, nullptr, 1, K, h, w, dist_kernel, num_iter, num_smooth, stream);
}

extern "C" int64_t bxs_corr_transfer_workspace_bytes(int64_t K, int64_t Hm, int64_t Wm) {
  if (K <= 0 || Hm <= 0 || Wm <= 0) return 0;
  return K * 2 * Hm * Wm * 4;
}

extern "C" int bxs_corr_transfer_batched(const float* T, const float* Cu, const float* m0, const float* m1, const int32_t* counts,
                                         float* fg_ci, float* bg_ci, void* workspace, int64_t n, int64_t kmax, int64_t h,
                                         int64_t w, int64_t Hm, int64_t Wm, bxs_stream_t stream) {
  if (!T || !Cu || !m0 || !m1 || !fg_ci || !bg_ci || !workspace || n <= 0 || kmax <= 0 || h <= 0 || w <= 0 || Hm <= 0 || Wm <= 0)
    return BXS_ERR_INVALID_ARG;
  const int64_t P = h * w, M = Hm * Wm;
  const int64_t smem = (P * P + 2 * P + M + (int64_t)NT_XFER * P) * 4 + (Hm + Wm) * (int64_t)sizeof(CorrTap);
  if (smem > kMaxSmem || kmax > 65535 || n > 65535 || M > (int64_t(1) << 24)) return BXS_ERR_UNSUPPORTED;
  if (smem > 48 * 1024 && opt_in_smem(corr_transfer_kernel, smem) != BXS_OK) return BXS_ERR_LAUNCH;
  float* partial = static_cast<float*>(workspace);
  const unsigned gx = (unsigned)ceil_div(M, NT_XFER);
  corr_transfer_kernel<<<dim3(gx, (unsigned)kmax, (unsigned)n), NT_XFER, smem, as_stream(stream)>>>(
      T, Cu, m0, m1, counts, partial, (int)kmax, (int)h, (int)w, (int)Hm, (int)Wm);
  int rc = check_launch();
  if (rc != BXS_OK) return rc;
  corr_mean_kernel<<<dim3(gx, (unsigned)n), NT_XFER, 0, as_stream(stream)>>>(partial, counts, fg_ci, bg_ci, (int)kmax, (int)M);
  return check_launch();
}

extern "C" int bxs_corr_transfer(const float* T, const float* Cu, const float* m0, const float* m1, float* fg_ci, float* bg_ci,
                                 void* workspace, int64_t K, int64_t h, int64_t w, int64_t Hm, int64_t Wm,
                                 bxs_stream_t stream) {
  return bxs_corr_transfer_batched(T, Cu, m0, m1, nullptr, fg_ci, bg_ci, workspace, 1, K, h, w, Hm, Wm, stream);
}

extern "C" int bxs_corr_retrieve(const float* bank_feat, const float* bank_mask, const float* bank_box, const int32_t* bank_ptr,
                                 const int32_t* bank_exists, const int32_t* first, const float* q_feat, const float* q_feat_first,
                                 const float* q_mask, const float* t_feat, const float* t_mask, const float* box,
                                 const int32_t* label, const int32_t* valid, int32_t* src, int32_t* count, int32_t* kcount,
                                 int32_t* slot, int32_t* exists, int64_t n, int64_t num_class, int64_t L, int64_t C, int64_t h,
                                 int64_t w, int64_t Hm, int64_t Wm, float fg_thr, float bg_thr, float app_thr, float ratio_lo,
                                 float ratio_hi, float min_size, int max_objs, int min_objs, bxs_stream_t stream) {
  if (n == 0) return BXS_OK;
  if (!bank_feat || !bank_mask || !bank_box || !bank_ptr || !bank_exists || !first || !q_feat || !q_feat_first || !q_mask ||
      !t_feat || !t_mask || !box || !label || !valid || !src || !count || !kcount || !slot || !exists || n < 0 ||
      num_class <= 0 || L <= 0 || C <= 0 || h <= 0 || w <= 0 || Hm <= 0 || Wm <= 0 || max_objs < 0)
    return BXS_ERR_INVALID_ARG;
  const int64_t smem = corr_retrieve_scratch((int)std::min<int64_t>(L, 1 << 20), (int)std::min<int64_t>(h * w, 1 << 20));
  if (smem > kMaxSmem || n > INT32_MAX || num_class * L > INT32_MAX || C * h * w > INT32_MAX || Hm * Wm > INT32_MAX)
    return BXS_ERR_UNSUPPORTED;
  if (smem > 48 * 1024 && opt_in_smem(corr_retrieve_kernel, smem) != BXS_OK) return BXS_ERR_LAUNCH;
  const CorrBank bank{bank_feat, bank_mask, bank_box, bank_ptr, bank_exists, (int)num_class, (int)L};
  const CorrLevel lvl{q_feat, q_feat_first, q_mask, t_feat, t_mask, box, label, valid, (int)n};
  const CorrRetrieveCfg cfg{(int)C, (int)h, (int)w, (int)Hm, (int)Wm, fg_thr, bg_thr, app_thr, ratio_lo, ratio_hi, min_size,
                            max_objs, min_objs};
  const CorrRetrieveOut out{src, count, kcount, slot, exists};
  corr_retrieve_kernel<<<(unsigned)n, NT_RETR, smem, as_stream(stream)>>>(bank, lvl, cfg, first, out);
  return check_launch();
}

extern "C" int bxs_corr_paste(const float* fg, const float* bg, const float* box, const int32_t* counts, float* iiu, int64_t n,
                              int64_t Hm, int64_t Wm, int64_t H, int64_t W, bxs_stream_t stream) {
  if (n == 0) return BXS_OK;
  if (!fg || !bg || !box || !counts || !iiu || n < 0 || Hm <= 0 || Wm <= 0 || H <= 0 || W <= 0) return BXS_ERR_INVALID_ARG;
  if (n > 65535 || H * W > INT32_MAX || Hm * Wm > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  const unsigned gx = (unsigned)ceil_div(H * W, NT_PASTE);     // a box lies inside the H x W map
  corr_paste_kernel<<<dim3(gx, 2, (unsigned)n), NT_PASTE, 0, as_stream(stream)>>>(fg, bg, box, counts, iiu, (int)Hm, (int)Wm,
                                                                                  (int)H, (int)W);
  return check_launch();
}

extern "C" int bxs_corr_bank_append(float* bank_feat, float* bank_mask, float* bank_box, int32_t* bank_ptr, int32_t* bank_exists,
                                    int32_t* first, const float* t_feat, const float* t_mask, const float* box,
                                    const int32_t* label, const int32_t* valid, const int32_t* slot, int64_t n,
                                    int64_t num_class, int64_t L, int64_t CP, int64_t M, bxs_stream_t stream) {
  if (n == 0) return BXS_OK;
  if (!bank_feat || !bank_mask || !bank_box || !bank_ptr || !bank_exists || !first || !t_feat || !t_mask || !box || !label ||
      !valid || !slot || n < 0 || num_class <= 0 || L <= 0 || CP <= 0 || M <= 0)
    return BXS_ERR_INVALID_ARG;
  if (n > INT32_MAX || num_class * L > INT32_MAX || CP > INT32_MAX || M > INT32_MAX) return BXS_ERR_UNSUPPORTED;
  const CorrLevel lvl{nullptr, nullptr, nullptr, t_feat, t_mask, box, label, valid, (int)n};
  corr_append_kernel<<<(unsigned)n, NT_APPEND, 0, as_stream(stream)>>>(bank_feat, bank_mask, bank_box, bank_ptr, bank_exists,
                                                                       first, lvl, slot, (int)num_class, (int)L, (int)CP, (int)M);
  return check_launch();
}
