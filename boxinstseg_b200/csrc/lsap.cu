// f1: a batch of independent linear sum assignments (MaskHungarianAssigner.assign step 3, mask_hungarian_assigner.py:113-123)
// in one launch per kLsapChunk problems, one warp per problem, the same row_ind / col_ind as scipy's
// linear_sum_assignment (see lsap_core.cuh).  The problem table travels by value in the kernel parameters: no host-to-device
// copy and no host read, so the call can be captured in a CUDA graph.  Every problem's state (duals and shortest-path
// costs in fp64, path / assignment / remaining-column lists, reached flags) lives in shared memory when the chunk's largest
// problem fits (kLsapSmemMax for the CTA's kLsapWarps problems: Box2Mask's 100 x 150 takes 5.6 KB), else in the caller's
// workspace.  Each Dijkstra step is a chain of dependent loads of that state, so its latency sets the speed.
#include "common.cuh"
#include "lsap_core.cuh"

namespace bxs {
namespace {

constexpr int kLsapChunk = 64;
constexpr int kLsapWarps = 4;          // problems per CTA
constexpr int64_t kLsapSmemMax = 160 << 10;

struct LsapTable {
  int64_t cost_off[kLsapChunk];    // elements from the cost base
  int64_t ws_off[kLsapChunk];      // bytes from the workspace base
  int64_t match_off[kLsapChunk];   // rows before this problem
  int32_t rows[kLsapChunk], cols[kLsapChunk];
};

template <class T>
__global__ void __launch_bounds__(kLsapWarps * kWarp) lsap_kernel(const T* __restrict__ cost, const LsapTable tab, int n,
                                                                  char* __restrict__ workspace, int64_t smem_per_warp,
                                                                  int32_t* __restrict__ match, int32_t* __restrict__ status) {
  extern __shared__ __align__(16) char lsap_smem[];
  const int wi = (int)(threadIdx.x / kWarp), p = blockIdx.x * kLsapWarps + wi;
  if (p >= n) return;
  const LsapWarp team{(int)(threadIdx.x % kWarp)};
  char* state = smem_per_warp ? lsap_smem + wi * smem_per_warp : workspace + tab.ws_off[p];
  const int st = lsap_solve(cost + tab.cost_off[p], tab.rows[p], tab.cols[p], state, match + tab.match_off[p], team);
  if (team.lane == 0) status[p] = st;
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_lsap_workspace_bytes(const int64_t* rows_host, const int64_t* cols_host, int64_t num_problems) {
  if (!rows_host || !cols_host || num_problems < 0) return 0;
  int64_t total = 0;
  for (int64_t p = 0; p < num_problems; ++p) total += lsap_work_bytes(rows_host[p], cols_host[p]);
  return total;
}

extern "C" int bxs_lsap_solve(const void* cost, const int64_t* offset_host, const int64_t* rows_host,
                              const int64_t* cols_host, int64_t num_problems, int dtype, int32_t* match, int32_t* status,
                              void* workspace, bxs_stream_t stream) {
  if (num_problems < 0 || (dtype != BXS_LSAP_F32 && dtype != BXS_LSAP_F64)) return BXS_ERR_INVALID_ARG;
  if (num_problems == 0) return BXS_OK;
  if (!offset_host || !rows_host || !cols_host || !status) return BXS_ERR_INVALID_ARG;
  int64_t total_rows = 0, ws_bytes = 0, elems = 0;
  for (int64_t p = 0; p < num_problems; ++p) {
    if (rows_host[p] < 0 || cols_host[p] < 0 || offset_host[p] < 0) return BXS_ERR_INVALID_ARG;
    if (rows_host[p] > INT32_MAX || cols_host[p] > INT32_MAX) return BXS_ERR_UNSUPPORTED;
    total_rows += rows_host[p];
    ws_bytes += lsap_work_bytes(rows_host[p], cols_host[p]);
    elems += rows_host[p] * cols_host[p];
  }
  if ((total_rows > 0 && !match) || (ws_bytes > 0 && !workspace) || (elems > 0 && !cost)) return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  LsapTable tab;
  int64_t ws = 0, mo = 0;
  for (int64_t p0 = 0; p0 < num_problems; p0 += kLsapChunk) {
    const int n = (int)std::min<int64_t>(num_problems - p0, kLsapChunk);
    int64_t largest = 0;
    for (int k = 0; k < kLsapChunk; ++k) {
      const bool in = k < n;
      const int64_t r = in ? rows_host[p0 + k] : 0, c = in ? cols_host[p0 + k] : 0;
      tab.cost_off[k] = in ? offset_host[p0 + k] : 0;
      tab.ws_off[k] = ws;
      tab.match_off[k] = mo;
      tab.rows[k] = (int32_t)r;
      tab.cols[k] = (int32_t)c;
      ws += lsap_work_bytes(r, c);
      largest = std::max(largest, lsap_work_bytes(r, c));
      mo += r;
    }
    const unsigned grid = (unsigned)ceil_div(n, kLsapWarps);
    char* wsp = static_cast<char*>(workspace);
    const int64_t per_warp = kLsapWarps * largest <= kLsapSmemMax ? largest : 0;
    const size_t smem = (size_t)(kLsapWarps * per_warp);
    int rc;
    if (dtype == BXS_LSAP_F32) {
      rc = opt_in_smem(lsap_kernel<float>, smem);
      if (rc == BXS_OK)
        lsap_kernel<float><<<grid, kLsapWarps * kWarp, smem, st>>>(static_cast<const float*>(cost), tab, n, wsp, per_warp,
                                                                   match, status + p0);
    } else {
      rc = opt_in_smem(lsap_kernel<double>, smem);
      if (rc == BXS_OK)
        lsap_kernel<double><<<grid, kLsapWarps * kWarp, smem, st>>>(static_cast<const double*>(cost), tab, n, wsp, per_warp,
                                                                    match, status + p0);
    }
    if (rc == BXS_OK) rc = check_launch();
    if (rc != BXS_OK) return rc;
  }
  return BXS_OK;
}
