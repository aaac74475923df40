// f1: the linear sum assignment of MaskHungarianAssigner.assign step 3 (mmdet/core/bbox/assigners/
// mask_hungarian_assigner.py:113-123), which the reference hands to scipy.optimize.linear_sum_assignment on the host.
//
// The algorithm is the shortest augmenting path for rectangular matrices (D. F. Crouse, "On implementing 2D rectangular
// assignment algorithms", IEEE TAES 52(4), 2016) with the conventions of scipy's implementation, so that row_ind / col_ind
// are the same as scipy's on every input, ties included:
//   * a tall matrix (cols < rows) is solved transposed (read in place through the strides, never copied);
//   * every entry is widened to double; a NaN or -inf entry is an invalid matrix (status 1), a row that cannot be
//     augmented is an infeasible one (status 2);
//   * the list of columns not yet reached starts as cols-1 ... 0, and a reached column is removed by moving the last
//     entry into its slot;
//   * reduced cost ((minVal + c[i][j]) - u[i]) - v[j], dual updates u[cur] += minVal, u[i] += minVal - spc[col4row[i]],
//     v[j] -= minVal - spc[j]: additions and subtractions only, so no FMA contraction can change a result;
//   * the column a Dijkstra step reaches is the minimum shortest-path cost; among the columns at that minimum, the LAST
//     unassigned one in list order, else the FIRST one.  scipy finds it with one left-to-right scan; written as the key
//     order `lsap_better` it is a total order, so any reduction tree (a warp's shuffles, the host's plain loop) picks the
//     same column.
//
// `lsap_solve` is written for a `Team`: on the device a warp (columns strided over the lanes, the choice as a shuffle
// reduction, sequential steps on lane 0), on the host a single lane.  tests/host_harness/lsap_host.cpp runs this very
// source on the CPU against scipy; the kernel is csrc/lsap.cu.
#pragma once
#include <stdint.h>

#include "assign_core.cuh"      // BXS_HD

namespace bxs {

#if defined(__CUDA_ARCH__)
#define BXS_DADD(a, b) __dadd_rn((a), (b))
#define BXS_DSUB(a, b) __dsub_rn((a), (b))
#else
#define BXS_DADD(a, b) ((a) + (b))
#define BXS_DSUB(a, b) ((a) - (b))
#endif
#if defined(__CUDACC__)
#define BXS_NO_UNROLL _Pragma("unroll 1")   // the strided loops run 1-5 times per lane at Box2Mask's sizes
#else
#define BXS_NO_UNROLL
#endif

enum { kLsapOk = 0, kLsapInvalid = 1, kLsapInfeasible = 2 };

// candidate column of one Dijkstra step: shortest-path cost, position in the remaining list, unassigned flag; pos < 0 = none
struct LsapKey {
  double cost;
  int pos;
  int free;
};

// true when a is chosen over b (see the header comment); positions are distinct, so this is a strict total order
BXS_HD bool lsap_better(const LsapKey& a, const LsapKey& b) {
  if (b.pos < 0) return a.pos >= 0;
  if (a.pos < 0) return false;
  if (a.cost != b.cost) return a.cost < b.cost;
  if (a.free != b.free) return a.free > b.free;
  return a.free ? a.pos > b.pos : a.pos < b.pos;
}

// the per-problem state in the caller's workspace: solving orientation nr <= nc
struct LsapWork {
  double* u;        // [nr]
  double* v;        // [nc]
  double* spc;      // [nc] shortest-path costs
  int32_t* path;    // [nc]
  int32_t* row4col; // [nc]
  int32_t* col4row; // [nr]
  int32_t* remaining;   // [nc]
  uint8_t* sr;      // [nr] rows reached in the current augmentation
  uint8_t* sc;      // [nc] columns reached
};

BXS_HD int64_t lsap_align(int64_t n) { return (n + 15) & ~(int64_t)15; }

// bytes of one problem's state (either orientation); 0 for an empty problem
BXS_HD int64_t lsap_work_bytes(int64_t rows, int64_t cols) {
  if (rows <= 0 || cols <= 0) return 0;
  const int64_t nr = rows < cols ? rows : cols, nc = rows < cols ? cols : rows;
  return lsap_align(8 * nr) + 2 * lsap_align(8 * nc) + 3 * lsap_align(4 * nc) + lsap_align(4 * nr) + lsap_align(nr) +
         lsap_align(nc);
}

BXS_HD LsapWork lsap_carve(void* base, int64_t nr, int64_t nc) {
  char* p = static_cast<char*>(base);
  LsapWork w;
  w.u = reinterpret_cast<double*>(p);          p += lsap_align(8 * nr);
  w.v = reinterpret_cast<double*>(p);          p += lsap_align(8 * nc);
  w.spc = reinterpret_cast<double*>(p);        p += lsap_align(8 * nc);
  w.path = reinterpret_cast<int32_t*>(p);      p += lsap_align(4 * nc);
  w.row4col = reinterpret_cast<int32_t*>(p);   p += lsap_align(4 * nc);
  w.remaining = reinterpret_cast<int32_t*>(p); p += lsap_align(4 * nc);
  w.col4row = reinterpret_cast<int32_t*>(p);   p += lsap_align(4 * nr);
  w.sr = reinterpret_cast<uint8_t*>(p);        p += lsap_align(nr);
  w.sc = reinterpret_cast<uint8_t*>(p);
  return w;
}

// One lane doing everything (the host twin).
struct LsapSerial {
  static constexpr int lane = 0, size = 1;
  void sync() const {}
  bool any(bool b) const { return b; }
  LsapKey reduce(const LsapKey& k) const { return k; }
};

#if defined(__CUDACC__)
// One warp per problem.
struct LsapWarp {
  int lane;
  static constexpr int size = 32;
  __device__ void sync() const { __syncwarp(); }
  __device__ bool any(bool b) const { return __any_sync(0xffffffffu, b); }
  __device__ LsapKey reduce(LsapKey k) const {
    for (int o = 16; o > 0; o >>= 1) {
      LsapKey t;
      t.cost = __shfl_xor_sync(0xffffffffu, k.cost, o);
      t.pos = __shfl_xor_sync(0xffffffffu, k.pos, o);
      t.free = __shfl_xor_sync(0xffffffffu, k.free, o);
      if (lsap_better(t, k)) k = t;
    }
    return k;
  }
};
#endif

// Solves one rows x cols problem of the cost matrix `cost` (row-major, widened from T to double) and writes match[r] =
// the column of row r, or -1, for every row of the caller's orientation.  Returns the status (kLsap*), the same on
// every lane; a failed problem leaves every row at -1.
template <class T, class Team>
BXS_HD int lsap_solve(const T* cost, int rows, int cols, void* workspace, int32_t* match, const Team& team) {
  for (int r = team.lane; r < rows; r += team.size) match[r] = -1;
  if (rows == 0 || cols == 0) return kLsapOk;
  const bool tr = cols < rows;
  const int nr = tr ? cols : rows, nc = tr ? rows : cols;
  const int64_t si = tr ? 1 : cols, sj = tr ? cols : 1;      // element (i, j) of the solving orientation
  const double kInf = __builtin_inf();
  bool bad = false;
  BXS_NO_UNROLL
  for (int64_t e = team.lane; e < (int64_t)rows * cols; e += team.size) {
    const double c = (double)cost[e];
    bad |= c != c || c == -kInf;
  }
  if (team.any(bad)) return kLsapInvalid;
  const LsapWork w = lsap_carve(workspace, nr, nc);
  for (int i = team.lane; i < nr; i += team.size) { w.u[i] = 0.0; w.col4row[i] = -1; }
  for (int j = team.lane; j < nc; j += team.size) { w.v[j] = 0.0; w.row4col[j] = -1; w.path[j] = -1; }
  team.sync();
  for (int cur = 0; cur < nr; ++cur) {
    for (int i = team.lane; i < nr; i += team.size) w.sr[i] = 0;
    BXS_NO_UNROLL
    for (int j = team.lane; j < nc; j += team.size) {
      w.remaining[j] = nc - 1 - j;
      w.sc[j] = 0;
      w.spc[j] = kInf;
    }
    team.sync();
    double minVal = 0.0;
    int i = cur, sink = -1, num_remaining = nc;
    while (sink < 0) {
      if (team.lane == 0) w.sr[i] = 1;
      const double ui = w.u[i];
      const T* ci = cost + (int64_t)i * si;
      LsapKey best;
      best.cost = kInf; best.pos = -1; best.free = 0;
      BXS_NO_UNROLL
      for (int it = team.lane; it < num_remaining; it += team.size) {
        const int j = w.remaining[it];
        const double r = BXS_DSUB(BXS_DSUB(BXS_DADD(minVal, (double)ci[j * sj]), ui), w.v[j]);
        double s = w.spc[j];
        if (r < s) {
          w.path[j] = i;
          w.spc[j] = r;
          s = r;
        }
        LsapKey k;
        k.cost = s; k.pos = it; k.free = w.row4col[j] < 0;
        if (lsap_better(k, best)) best = k;
      }
      best = team.reduce(best);
      minVal = best.cost;
      if (!(minVal < kInf)) return kLsapInfeasible;            // scipy: minVal == INFINITY
      const int j = w.remaining[best.pos];
      if (w.row4col[j] < 0) sink = j;
      else i = w.row4col[j];
      team.sync();                                           // every lane has read remaining[] and spc[]
      if (team.lane == 0) {
        w.sc[j] = 1;
        w.remaining[best.pos] = w.remaining[num_remaining - 1];
      }
      --num_remaining;
      team.sync();
    }
    for (int r = team.lane; r < nr; r += team.size)
      if (w.sr[r]) w.u[r] = r == cur ? BXS_DADD(w.u[r], minVal) : BXS_DADD(w.u[r], BXS_DSUB(minVal, w.spc[w.col4row[r]]));
    for (int j = team.lane; j < nc; j += team.size)
      if (w.sc[j]) w.v[j] = BXS_DSUB(w.v[j], BXS_DSUB(minVal, w.spc[j]));
    team.sync();
    if (team.lane == 0) {                                     // augment along the path
      int j = sink;
      for (;;) {
        const int r = w.path[j];
        w.row4col[j] = r;
        const int prev = w.col4row[r];
        w.col4row[r] = j;
        j = prev;
        if (r == cur) break;
      }
    }
    team.sync();
  }
  for (int i = team.lane; i < nr; i += team.size) {
    if (tr) match[w.col4row[i]] = i;
    else match[i] = w.col4row[i];
  }
  return kLsapOk;
}

}  // namespace bxs
