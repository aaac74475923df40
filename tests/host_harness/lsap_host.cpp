// TEST INFRASTRUCTURE: host twin of lsap_kernel (boxinstseg_b200/csrc/lsap.cu).  It compiles the very header the kernel is
// made of (lsap_core.cuh: lsap_solve with a one-lane team instead of a warp, the same column-choice order and workspace
// layout) with g++ -ffp-contract=off, so that the CPU suite can check the matching against scipy bit for bit on a box
// without a GPU.  Never shipped: the product library exports only the CUDA path.
#include <vector>

#include "../../boxinstseg_b200/csrc/lsap_core.cuh"

// cost: row-major rows x cols, float32 (dtype 0) or float64 (dtype 1); match [rows]; returns the status
extern "C" int host_lsap_solve(const void* cost, int dtype, int rows, int cols, int32_t* match) {
  std::vector<double> ws((bxs::lsap_work_bytes(rows, cols) + 7) / 8 + 1);
  const bxs::LsapSerial team;
  if (dtype == 0) return bxs::lsap_solve(static_cast<const float*>(cost), rows, cols, ws.data(), match, team);
  return bxs::lsap_solve(static_cast<const double*>(cost), rows, cols, ws.data(), match, team);
}
