// a12-a15: learnable tree filter -- minimum spanning tree, breadth-first ordering, two-pass tree
// aggregation (forward + both backwards).  Drop-in for mmdet/ops/tree_filter (tree_filter_cuda):
//   mst_forward  (src/mst/mst.cu:86-117 + boruvka.cpp)  : in the reference this runs ON THE CPU (sync copy,
//                one std::thread per tree); here Boruvka runs on the GPU with 64-bit (weight,index) keys and
//                integer atomicMin, so the result is the unique MST of the strict total order -- the same
//                edge SET as the reference's; edges are returned sorted by edge id (deterministic).
//   bfs_forward  (src/bfs/bfs.cu:100-135)               : deterministic adjacency (sorted neighbours, no
//                atomics-dependent order), one CTA per tree, block scans assign positions level by level;
//                also emits the level boundaries the aggregation kernels use.
//   refine_*     (src/refine/refine.cu:201-370)         : the reference walks a tree with a 64-thread
//                wavefront polling shared flags (>= V/64 barriers, each behind a global-memory round trip).
//                Here the order is level-contiguous, one CTA owns a (tree, channel), the running values
//                live in SHARED memory (V floats) and each level is one barrier.
#include <cooperative_groups.h>

#include <algorithm>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace bxs {
namespace {

constexpr int NT = 256;     // levels hold ~30 nodes on average: a small CTA keeps the per-level barrier and the idle-warp issue cost low
constexpr unsigned long long kInf = ~0ull;

__device__ __forceinline__ unsigned fkey(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// ---------------------------------------------------------------------------------------
// MST (Boruvka)
// ---------------------------------------------------------------------------------------
struct MstWs {
  unsigned long long* best;   // [B*V]
  int* P;                     // [B*V] component label (always a root id)
  int* Q;                     // [B*V] hook parents
  uint8_t* in_tree;           // [B*E]
  int* round_flags;           // [B*64] "this round hooked something"
  size_t total_bytes;
};
inline MstWs carve_mst(void* base, int64_t B, int64_t E, int64_t V) {
  MstWs w{};
  Carver c(base);
  w.best = (unsigned long long*)c.take(8 * B * V);
  w.P = (int*)c.take(4 * B * V);
  w.Q = (int*)c.take(4 * B * V);
  w.in_tree = (uint8_t*)c.take(B * E);
  w.round_flags = (int*)c.take(4 * B * 64);
  w.total_bytes = c.off;
  return w;
}

__global__ void mst_init_kernel(MstWs ws, int64_t BV, int64_t BE, int V) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < BV; i += (int64_t)gridDim.x * blockDim.x) {
    ws.P[i] = (int)(i % V);
    ws.best[i] = kInf;
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < BE; i += (int64_t)gridDim.x * blockDim.x)
    ws.in_tree[i] = 0;
}

// every edge offers itself to the two components it connects
__global__ void mst_min_edge_kernel(const int32_t* __restrict__ edge_index, const float* __restrict__ edge_weight,
                                    MstWs ws, int E, int V) {
  const int b = blockIdx.y;
  const int32_t* ei = edge_index + (int64_t)b * E * 2;
  const float* ew = edge_weight + (int64_t)b * E;
  const int* P = ws.P + (int64_t)b * V;
  unsigned long long* best = ws.best + (int64_t)b * V;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < E; e += gridDim.x * blockDim.x) {
    const int cu = P[ei[2 * e]], cv = P[ei[2 * e + 1]];
    if (cu == cv) continue;
    const unsigned long long key = ((unsigned long long)fkey(ew[e]) << 32) | (unsigned)e;
    atomicMin(best + cu, key);
    atomicMin(best + cv, key);
  }
}

// roots with an outgoing edge hook onto the component at its other end (2-cycles broken by id)
__global__ void mst_hook_kernel(const int32_t* __restrict__ edge_index, MstWs ws, int E, int V) {
  const int b = blockIdx.y;
  const int32_t* ei = edge_index + (int64_t)b * E * 2;
  const int* P = ws.P + (int64_t)b * V;
  int* Q = ws.Q + (int64_t)b * V;
  const unsigned long long* best = ws.best + (int64_t)b * V;
  uint8_t* in_tree = ws.in_tree + (int64_t)b * E;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
    int q = P[v];
    if (q == v && best[v] != kInf) {
      const int e = (int)(best[v] & 0xffffffffull);
      const int cu = P[ei[2 * e]], cv = P[ei[2 * e + 1]];
      const int other = cu == v ? cv : cu;
      const bool mutual = best[other] == best[v];
      if (!(mutual && v < other)) {
        q = other;
        in_tree[e] = 1;
      }
    }
    Q[v] = q;
  }
}

__global__ void mst_compress_kernel(MstWs ws, int V) {
  const int b = blockIdx.y;
  int* P = ws.P + (int64_t)b * V;
  const int* Q = ws.Q + (int64_t)b * V;
  unsigned long long* best = ws.best + (int64_t)b * V;
  for (int v = blockIdx.x * blockDim.x + threadIdx.x; v < V; v += gridDim.x * blockDim.x) {
    int r = P[v];
    while (Q[r] != r) r = Q[r];
    P[v] = r;
    best[v] = kInf;
  }
}

// ---------------------------------------------------------------------------------------
// The whole Boruvka iteration in ONE launch: a thread-block cluster of 8 CTAs per tree runs the three phases of a round
// (min edge per component, hook, compress) back to back with cluster barriers in between and stops as soon as a round
// hooks nothing (one component left).  The per-round kernels above needed 3 launches x ceil(log2 V) rounds (48
// launches at 200x256, most of them doing nothing: components shrink ~3-4x per round) and were launch-bound:
// ~0.67 ms whether for 16 trees or for 2.  Same keys, same integer atomicMin, same edge set.
// ---------------------------------------------------------------------------------------
constexpr int MST_CL = 8;
constexpr int MST_NT = 1024;

__global__ void __cluster_dims__(MST_CL, 1, 1) __launch_bounds__(MST_NT)
mst_cluster_kernel(const int32_t* __restrict__ edge_index, const float* __restrict__ edge_weight, MstWs ws, int E, int V,
                   int max_rounds, int* __restrict__ round_flags) {
  cg::cluster_group cluster = cg::this_cluster();
  const int b = blockIdx.x / MST_CL;
  const int t0 = (int)cluster.block_rank() * MST_NT + threadIdx.x, stride = MST_CL * MST_NT;
  const int32_t* ei = edge_index + (int64_t)b * E * 2;
  const float* ew = edge_weight + (int64_t)b * E;
  int* P = ws.P + (int64_t)b * V;
  int* Q = ws.Q + (int64_t)b * V;
  unsigned long long* best = ws.best + (int64_t)b * V;
  uint8_t* in_tree = ws.in_tree + (int64_t)b * E;
  int* flags = round_flags + (int64_t)b * max_rounds;
  for (int v = t0; v < V; v += stride) { P[v] = v; best[v] = kInf; }
  for (int e = t0; e < E; e += stride) in_tree[e] = 0;
  for (int r = t0; r < max_rounds; r += stride) flags[r] = 0;
  cluster.sync();
  for (int round = 0; round < max_rounds; ++round) {
    // every edge offers itself to the two components it connects
    for (int e = t0; e < E; e += stride) {
      const int2 uv = *reinterpret_cast<const int2*>(ei + 2 * e);
      const int cu = P[uv.x], cv = P[uv.y];
      if (cu == cv) continue;
      const unsigned long long key = ((unsigned long long)fkey(ew[e]) << 32) | (unsigned)e;
      atomicMin(best + cu, key);
      atomicMin(best + cv, key);
    }
    cluster.sync();
    // roots with an outgoing edge hook onto the component at its other end (2-cycles broken by id)
    bool hooked = false;
    for (int v = t0; v < V; v += stride) {
      int q = P[v];
      if (q == v) {
        const unsigned long long bv = best[v];
        if (bv != kInf) {
          const int e = (int)(bv & 0xffffffffull);
          const int cu = P[ei[2 * e]], cv = P[ei[2 * e + 1]];
          const int other = cu == v ? cv : cu;
          if (!(best[other] == bv && v < other)) {
            q = other;
            in_tree[e] = 1;
          }
          hooked = true;                      // an outgoing edge exists: more than one component
        }
      }
      Q[v] = q;
    }
    if (hooked) flags[round] = 1;
    cluster.sync();
    if (flags[round] == 0) break;             // uniform over the cluster: nothing left to merge
    for (int v = t0; v < V; v += stride) {
      int r = P[v];
      while (Q[r] != r) r = Q[r];
      P[v] = r;
      best[v] = kInf;
    }
    cluster.sync();
  }
}

// tree edges in ascending edge id; one CTA per tree
// The tree's edges in ascending edge id (the edge SET is the reference's; its order is Boruvka discovery order, boruvka.cpp).
// Two small grids instead of one CTA per image walking 100 edges per thread (134 us at 200x256, 6 % of config D):
// chunk counts, then an ordered compaction of each 4096-edge chunk behind the sum of the counts before it.
constexpr int MC_T = 256, MC_PER = 16, MC_CHUNK = MC_T * MC_PER;

__device__ __forceinline__ unsigned mc_mask(const uint8_t* __restrict__ in_tree, int lo, int E) {
  unsigned mask = 0u;
#pragma unroll
  for (int k = 0; k < MC_PER; ++k)
    if (lo + k < E && in_tree[lo + k]) mask |= 1u << k;
  return mask;
}

__global__ void __launch_bounds__(MC_T) mst_count_kernel(MstWs ws, int* __restrict__ counts, int E) {
  __shared__ int s_w[MC_T / 32];
  const int c = blockIdx.x, b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int cnt = __popc(mc_mask(ws.in_tree + (int64_t)b * E, c * MC_CHUNK + threadIdx.x * MC_PER, E));
  cnt = __reduce_add_sync(kFull, cnt);
  if (lane == 0) s_w[warp] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    int t = 0;
#pragma unroll
    for (int i = 0; i < MC_T / 32; ++i) t += s_w[i];
    counts[b * gridDim.x + c] = t;
  }
}

__global__ void __launch_bounds__(MC_T) mst_compact_kernel(const int32_t* __restrict__ edge_index, MstWs ws,
                                                           const int* __restrict__ counts, int32_t* __restrict__ edge_out,
                                                           int E, int V) {
  __shared__ int s_w[MC_T / 32];
  __shared__ int s_before;
  const int c = blockIdx.x, b = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int2* ei = reinterpret_cast<const int2*>(edge_index + (int64_t)b * E * 2);
  int2* out = reinterpret_cast<int2*>(edge_out + (int64_t)b * (V - 1) * 2);
  const int lo = c * MC_CHUNK + threadIdx.x * MC_PER;
  const unsigned mask = mc_mask(ws.in_tree + (int64_t)b * E, lo, E);
  const int cnt = __popc(mask);
  int incl = cnt;                                           // inclusive warp scan
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int o = __shfl_up_sync(kFull, incl, d);
    if (lane >= d) incl += o;
  }
  if (lane == 31) s_w[warp] = incl;
  if (warp == 0) {                                          // tree edges of this image in the chunks before this one
    int t = 0;
    for (int i = lane; i < c; i += 32) t += counts[b * gridDim.x + i];
    t = __reduce_add_sync(kFull, t);
    if (lane == 0) s_before = t;
  }
  __syncthreads();
  int pos = s_before + incl - cnt;
  for (int i = 0; i < warp; ++i) pos += s_w[i];
#pragma unroll
  for (int k = 0; k < MC_PER; ++k)
    if ((mask >> k) & 1u) {
      if (pos < V - 1) out[pos] = ei[lo + k];
      ++pos;
    }
}

// ---------------------------------------------------------------------------------------
// BFS ordering
// ---------------------------------------------------------------------------------------
struct BfsWs {
  int* deg;        // [B*V]
  int* adj;        // [B*V*4]
  int* counts;     // [B*V] scratch of the level scan
  int* flags;      // [B]   1: ordered by the grid fast path
  size_t total_bytes;
};
inline BfsWs carve_bfs(void* base, int64_t B, int64_t V) {
  BfsWs w{};
  Carver c(base);
  w.deg = (int*)c.take(4 * B * V);
  w.adj = (int*)c.take(16 * B * V);
  w.counts = (int*)c.take(4 * B * V);
  w.flags = (int*)c.take(4 * B);
  w.total_bytes = c.off;
  return w;
}

__global__ void bfs_adj_kernel(const int32_t* __restrict__ tree, BfsWs ws, int V, int* __restrict__ err,
                               const int* __restrict__ flags) {
  const int b = blockIdx.y;
  if (flags && flags[b]) return;
  const int32_t* te = tree + (int64_t)b * (V - 1) * 2;
  int* deg = ws.deg + (int64_t)b * V;
  int* adj = ws.adj + (int64_t)b * V * 4;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < V - 1; i += gridDim.x * blockDim.x) {
    const int u = te[2 * i], v = te[2 * i + 1];
    const int su = atomicAdd(deg + u, 1), sv = atomicAdd(deg + v, 1);
    if (su < 4) adj[u * 4 + su] = v; else *err = 1;
    if (sv < 4) adj[v * 4 + sv] = u; else *err = 1;
  }
}

// ascending neighbour ids, unused slots = INT_MAX, so one 16-byte load per vertex describes its adjacency
__global__ void bfs_sort_adj_kernel(BfsWs ws, int64_t BV, int V, const int* __restrict__ flags) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < BV; i += (int64_t)gridDim.x * blockDim.x) {
    if (flags && flags[i / V]) continue;              // ordered by the grid fast path
    int* a = ws.adj + i * 4;
    const int d = min(ws.deg[i], 4);
    int v[4];
    for (int x = 0; x < 4; ++x) v[x] = x < d ? a[x] : 0x7fffffff;
    for (int x = 1; x < 4; ++x)
      for (int y = x; y > 0 && v[y] < v[y - 1]; --y) { const int t = v[y]; v[y] = v[y - 1]; v[y - 1] = t; }
    *reinterpret_cast<int4*>(a) = make_int4(v[0], v[1], v[2], v[3]);
  }
}

// exclusive scan of `val` over the CTA (NT threads); returns the prefix, total in *total (all threads)
__device__ __forceinline__ int block_excl_scan(int val, int* s_warp, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = val;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(kFull, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = lane < NT / 32 ? s_warp[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(kFull, winc, o);
      if (lane >= o) winc += t;
    }
    s_warp[lane] = winc - w;                       // exclusive warp offsets
    if (lane == 31) s_warp[32] = winc;             // grand total
  }
  __syncthreads();
  *total = s_warp[32];
  return s_warp[wid] + inc - val;
}

// one CTA per tree.  Level l occupies positions [level_start[l], level_start[l+1]); children of a
// vertex are contiguous and ordered by ascending vertex id; parents are non-decreasing in position.
// The frontier's (vertex, parent vertex) pairs are handed from level to level through shared memory, so a level
// costs ONE dependent global load (the 16-byte adjacency record) plus a block scan.
__global__ void __launch_bounds__(NT) bfs_block_kernel(BfsWs ws, int V, int32_t* __restrict__ sorted_index,
                                                       int32_t* __restrict__ sorted_parent,
                                                       int32_t* __restrict__ sorted_child,
                                                       int32_t* __restrict__ level_start,
                                                       int32_t* __restrict__ num_levels, const int* __restrict__ flags,
                                                       int root) {
  __shared__ int s_warp[33];
  __shared__ int s_v[2][NT], s_pv[2][NT];
  const int b = blockIdx.x;
  if (flags && flags[b]) return;                     // bfs_grid_kernel already ordered this tree
  const int4* adj = reinterpret_cast<const int4*>(ws.adj + (int64_t)b * V * 4);
  int* pvert = ws.counts + (int64_t)b * V;           // parent VERTEX of each position (frontiers wider than NT)
  int32_t* idx = sorted_index + (int64_t)b * V;
  int32_t* par = sorted_parent + (int64_t)b * V;
  int32_t* chd = sorted_child + (int64_t)b * V * 4;
  int32_t* lvl = level_start + (int64_t)b * (V + 1);
  for (int i = threadIdx.x; i < V; i += NT) reinterpret_cast<int4*>(chd)[i] = make_int4(0, 0, 0, 0);
  if (threadIdx.x == 0) { idx[0] = root; par[0] = 0; lvl[0] = 0; pvert[0] = -1; s_v[0][0] = root; s_pv[0][0] = -1; }
  __syncthreads();
  int ls = 0, le = 1, level = 0, cur = 0;
  while (ls < le) {
    int next = le;                                  // first free position
    for (int base = ls; base < le; base += NT) {    // frontier in chunks of NT positions
      const int p = base + threadIdx.x;
      int v = -1, pv = -1, cnt = 0;
      int4 a = make_int4(0x7fffffff, 0x7fffffff, 0x7fffffff, 0x7fffffff);
      if (p < le) {
        if (p - ls < NT) { v = s_v[cur][p - ls]; pv = s_pv[cur][p - ls]; }
        else { v = idx[p]; pv = pvert[p]; }
        a = __ldg(adj + v);
        cnt = (a.x < V && a.x != pv) + (a.y < V && a.y != pv) + (a.z < V && a.z != pv) + (a.w < V && a.w != pv);
      }
      int total;
      const int off = block_excl_scan(cnt, s_warp, &total);
      if (p < le) {
        int q = next + off, k2 = 0;
        const int nb[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const int u = nb[k];
          if (u >= V || u == pv) continue;
          idx[q] = u;
          par[q] = p;
          pvert[q] = v;
          if (q - le < NT) { s_v[cur ^ 1][q - le] = u; s_pv[cur ^ 1][q - le] = v; }
          chd[p * 4 + k2++] = q;
          ++q;
        }
      }
      next += total;
      __syncthreads();
    }
    ls = le;
    le = next;
    cur ^= 1;
    ++level;
    if (threadIdx.x == 0) lvl[level] = ls;
    __syncthreads();
  }
  if (threadIdx.x == 0) num_levels[b] = level;      // lvl[level] == number of reached vertices
}

// ---------------------------------------------------------------------------------------
// BFS, fast path for trees of a 4-connected GRID graph (every tree the heads build: tree_filter.py:15-25 lists the
// vertical edges (v, v + W) and the horizontal edges (v, v + 1)).  The adjacency of such a tree is 4 bits per vertex
// (up, left, right, down), i.e. V bytes: it lives in SHARED memory, so a level costs a shared-memory read + a warp
// scan instead of a dependent L2 round trip per level (bfs_block_kernel: ~0.9 us per level, 1667 levels at 200x256).
// One warp per tree: no CTA barrier.  Children are emitted in ascending vertex order (up, left, right, down minus the
// parent), exactly the order bfs_block_kernel produces, so both paths give the same result.
// `flags[b]`: 0 = not a grid tree (or too large for shared memory): bfs_block_kernel must run; 1 = done here.
// ---------------------------------------------------------------------------------------
#ifdef BXS_TREE_TRACE
// per-level clock stamps of the first CTA's up pass: [0..2] consumer thread 0 (level top, after its store was issued,
// at the barrier), [3..5] producer thread RW (level top, copies issued, group wait done)
__device__ long long g_tree_trace[6][4096];
#define TREE_TT(k, i) do { if (DIR < 0 && blockIdx.x == 0 && blockIdx.y == 0 && (i) < 4096) g_tree_trace[k][i] = clock64(); } while (0)
#define BFS_TT(k, i) do { if (blockIdx.x == 0 && lane == 0 && (i) < 4096) g_tree_trace[k][i] = clock64(); } while (0)
#else
#define TREE_TT(k, i) do { } while (0)
#define BFS_TT(k, i) do { } while (0)
#endif
constexpr int BFS_FRONT = 1024;         // frontier entries kept in shared memory (a wider frontier declines to the generic path)
constexpr int BFS_STRIDE = BFS_FRONT + 32;
constexpr int BFS_BUFS = 4;             // frontier buffers in rotation: level L is written during L-1, expanded during L, and
                                        // turned into global output by a helper warp during L+1..L+2

__global__ void __launch_bounds__(NT) bfs_grid_kernel(const int32_t* __restrict__ tree, int V, int32_t* __restrict__ sorted_index,
                                                      int32_t* __restrict__ sorted_parent, int32_t* __restrict__ sorted_child,
                                                      int32_t* __restrict__ level_start, int32_t* __restrict__ num_levels,
                                                      int* __restrict__ flags, int root) {
  extern __shared__ unsigned bfs_smem[];
  __shared__ int s_wd[NT / 32];
  __shared__ int s_ok;
  unsigned* s_adj = bfs_smem;                                   // V bytes, packed 4 per word
  // frontier records, [BFS_BUFS][BFS_STRIDE]: vertex id | (direction bit of its PARENT, seen from the vertex) << 28; the 32
  // entries behind BFS_FRONT are a per-lane dump zone for the unconditional stores of absent children
  int* s_v = reinterpret_cast<int*>(bfs_smem + (V + 3) / 4);
  int* s_q = s_v + BFS_BUFS * BFS_STRIDE;                       // [BFS_BUFS][BFS_STRIDE] first child position | child bits << 28
  __shared__ int s_lev[BFS_BUFS][2];                            // [level & 3] = {level start, level end}; start < 0: stop
  const int b = blockIdx.x, lane = threadIdx.x & 31, tid = threadIdx.x;
  const int2* te = reinterpret_cast<const int2*>(tree + (int64_t)b * (V - 1) * 2);
  // ---- prologue, whole CTA: row pitch of the grid (the single non-unit difference of an edge's end points), then the
  //      adjacency bits.  (One warp alone spends ~1 ms here on 51 200 dependent-latency loads.) ----
  int Wd = 0;
  bool ok = true;
  for (int i = tid; i < V - 1; i += NT) {
    const int2 e = __ldg(te + i);
    const int d = abs(e.y - e.x);
    if (d == 0) ok = false;
    else if (d != 1) Wd = max(Wd, d);
  }
  Wd = __reduce_max_sync(kFull, Wd);
  if (lane == 0) s_wd[tid >> 5] = Wd;
  if (tid == 0) s_ok = 1;
  for (int i = tid; i < (V + 3) / 4; i += NT) s_adj[i] = 0u;
  __syncthreads();
#pragma unroll
  for (int i = 0; i < NT / 32; ++i) Wd = max(Wd, s_wd[i]);
  if (Wd == 0) Wd = V;                                          // a single row: no vertical edge
  for (int i = tid; i < V - 1; i += NT) {
    const int2 e = __ldg(te + i);
    const int u = min(e.x, e.y), v = max(e.x, e.y), d = v - u;
    if (u < 0 || v >= V || (d != 1 && d != Wd) || (d == 1 && Wd < V && (v % Wd) == 0)) { ok = false; continue; }
    // bit 0 = up (v - Wd), 1 = left (v - 1), 2 = right (v + 1), 3 = down (v + Wd)
    atomicOr(&s_adj[u >> 2], (d == 1 ? 4u : 8u) << ((u & 3) * 8));
    atomicOr(&s_adj[v >> 2], (d == 1 ? 2u : 1u) << ((v & 3) * 8));
  }
  if (!ok) s_ok = 0;
  __syncthreads();
  // ---- level loop.  A level is the instruction stream of ONE warp (a frontier is ~30 vertices), so that stream is kept
  //      to the dependent part -- frontier -> adjacency bits -> ballot scan -> next frontier, all in shared memory -- and
  //      everything that only PRODUCES OUTPUT (sorted_index / sorted_parent / sorted_child / level_start stores: two thirds of
  //      the instructions of round 2a's single-warp loop) is done one level later by two helper warps taking alternate
  //      levels, from the frontier buffer and a per-vertex (first child position | child bits) record.  Warp 0 and the
  //      helper of a level meet at a 64-thread named barrier; no CTA-wide barrier from here on. ----
  if (tid >= 96) return;
  const int warp = tid >> 5;
  if (!s_ok) { if (tid == 0) flags[b] = 0; return; }
  int32_t* idx = sorted_index + (int64_t)b * V;
  int32_t* par = sorted_parent + (int64_t)b * V;
  int4* chd = reinterpret_cast<int4*>(sorted_child + (int64_t)b * V * 4);
  int32_t* lvl = level_start + (int64_t)b * (V + 1);
  // named barriers 1 and 2 (immediate ids), 64 participating threads each: warp 0 + the helper of that level parity
  auto pair_sync = [](int parity) {
    if (parity) asm volatile("bar.sync 2, 64;" ::: "memory");
    else asm volatile("bar.sync 1, 64;" ::: "memory");
  };
  if (warp == 0) {
    if (lane == 0) { idx[0] = root; par[0] = 0; s_v[0] = root; }          // the root has no parent bit
    __syncwarp();
    const unsigned lt_mask = (1u << lane) - 1u;
    int ls = 0, le = 1, level = 0;
    bool fail = false;
    while (ls < le && !fail) {
      const int cur = level & (BFS_BUFS - 1), nxt = (level + 1) & (BFS_BUFS - 1);
      const int* cv = s_v + cur * BFS_STRIDE;
      int* cq = s_q + cur * BFS_STRIDE;
      int* nv = s_v + nxt * BFS_STRIDE;
      int next = le;
      BFS_TT(0, level);
      for (int base = ls; base < le; base += 32) {
        // Straight-line code: an idle lane expands entry 0 with its bits masked off, absent children are stored into the
        // lane's dump slot.  (The branchy form of this block -- `if (on)`, a compare chain for the parent, four conditional
        // child stores -- cost ~900 of the ~1200 cycles of a level: clock-stamp trace, tools/trace_bfs.py.)
        const bool on = base + lane < le;
        const int i = on ? base - ls + lane : 0;
        const int rec = cv[i];
        const int v = rec & 0x0fffffff;
        unsigned bits = (s_adj[v >> 2] >> ((v & 3) * 8)) & 15u & ~((unsigned)rec >> 28);
        bits = on ? bits : 0u;
        const int cnt = __popc(bits);
        if (cnt >= 0) BFS_TT(1, level);
        // exclusive prefix of the child counts (0..3 per lane; only the root can have 4): ballots instead of a shuffle scan
        const unsigned b0 = __ballot_sync(kFull, cnt & 1), b1 = __ballot_sync(kFull, cnt & 2);
        int excl = __popc(b0 & lt_mask) + 2 * __popc(b1 & lt_mask), total = __popc(b0) + 2 * __popc(b1);
        if (level == 0) total = __shfl_sync(kFull, cnt, 0);             // the root: lane 0 alone, excl == 0
        if (next + total - le > BFS_FRONT) { fail = true; break; }      // warp-uniform
        if (total >= 0) BFS_TT(2, level);
        const int q0 = next + excl;                   // this vertex's children occupy positions [q0, q0 + cnt)
        const int r0 = q0 - le, r1 = r0 + (bits & 1u), r2 = r1 + ((bits >> 1) & 1u), r3 = r2 + ((bits >> 2) & 1u);
        const int dump = BFS_FRONT + lane;
        cq[on ? i : dump] = q0 | (int)(bits << 28);
        // children in ascending vertex order (up, left, right, down); the parent of a child reached through direction k is in
        // direction 3 - k seen from the child
        nv[(bits & 1u) ? r0 : dump] = (int)((unsigned)(v - Wd) & 0x0fffffffu | (8u << 28));
        nv[(bits & 2u) ? r1 : dump] = (int)((unsigned)(v - 1) & 0x0fffffffu | (4u << 28));
        nv[(bits & 4u) ? r2 : dump] = (int)((unsigned)(v + 1) & 0x0fffffffu | (2u << 28));
        nv[(bits & 8u) ? r3 : dump] = (int)((unsigned)(v + Wd) & 0x0fffffffu | (1u << 28));
        next += total;
      }
      BFS_TT(3, level);
      if (lane == 0) { s_lev[cur][0] = fail ? -1 : ls; s_lev[cur][1] = le; }
      pair_sync(level & 1);
      BFS_TT(4, level);                          // hand level `level` to its helper (which finished level - 2 long ago)
      if (fail) break;
      ls = le;
      le = next;
      ++level;
    }
    // stop markers for both helpers (the failing level already carries one for its own helper)
    const int stops = fail ? 1 : 2;
    for (int k = 0; k < stops; ++k) {
      const int lv2 = level + (fail ? 1 : 0) + k;
      if (lane == 0) s_lev[lv2 & (BFS_BUFS - 1)][0] = -1;
      pair_sync(lv2 & 1);
    }
    if (lane == 0) {
      if (!fail) lvl[level] = ls;                    // == V for a spanning tree
      num_levels[b] = level;
      flags[b] = (!fail && ls == V) ? 1 : 0;         // every vertex reached <=> a spanning tree; else the generic path runs
    }
  } else {
    // helper of the levels of parity (warp - 1): global output of a level, while warp 0 is one or two levels further on
    const int parity = warp - 1;
    for (int level = parity;; level += 2) {
      pair_sync(parity);
      const int cur = level & (BFS_BUFS - 1);
      const int ls = s_lev[cur][0], le = s_lev[cur][1];
      if (ls < 0) break;
      if (lane == 0) lvl[level] = ls;
      const int* cv = s_v + cur * BFS_STRIDE;
      const int* cq = s_q + cur * BFS_STRIDE;
      for (int i = lane; i < le - ls; i += 32) {
        const int v = cv[i] & 0x0fffffff, qb = cq[i], p = ls + i;
        const int q0 = qb & 0x0fffffff;
        const unsigned bits = (unsigned)qb >> 28;
        int q = q0;
        if (bits & 1u) { idx[q] = v - Wd; par[q] = p; ++q; }
        if (bits & 2u) { idx[q] = v - 1; par[q] = p; ++q; }
        if (bits & 4u) { idx[q] = v + 1; par[q] = p; ++q; }
        if (bits & 8u) { idx[q] = v + Wd; par[q] = p; ++q; }
        const int cnt = q - q0;
        chd[p] = make_int4(cnt > 0 ? q0 : 0, cnt > 1 ? q0 + 1 : 0, cnt > 2 ? q0 + 2 : 0, cnt > 3 ? q0 + 3 : 0);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------
// tree aggregation
// ---------------------------------------------------------------------------------------
// The recursion has one dependent step per tree level (~1700 levels for a 200x256 image MST, ~30 nodes each), so the
// cost of a level IS the kernel time, and a level is the INSTRUCTION STREAM of the one warp that owns its nodes: an
// in-order warp at ~4-7 cycles per dependent instruction.  History of the level loop:
//   round 1   : dependent global loads inside the level                             ~1600 cycles / level
//   round 2a  : register prefetch rings (node data PF levels ahead, bounds 2 PF)     ~500 cycles / level: ~90 warp
//               instructions, two thirds of them the address arithmetic of the prefetch, four LDS -> FFMA -> BRA steps
//   round 2b  : this version.  PRODUCER warps (4-7) run the prefetch: per level they read the level's bounds from a
//               shared-memory window, issue cp.async copies of the node records into a PF-deep shared-memory ring and
//               retire the group of two levels ahead (cp.async groups complete in order).  CONSUMER warps (0-3; warp 0
//               alone for a level of <= 32 nodes) only read the ring -- one level ahead, into registers, in the shadow of
//               the current level's loads -- and do: five shared-memory loads, one FMA chain, one store, the barrier.
// One __syncthreads per level publishes the consumers' values and the producers' ring slots at once.
constexpr int PF = 6;                    // levels in flight in the copy ring
constexpr int RNT = 256;                 // threads of a refine CTA (parallel pre-passes; 4 consumer + 4 producer warps)
constexpr int RW = 128;                  // ring width = consumer threads; wider levels: the other threads load directly
constexpr int LWIN = 1024;               // level-bound window (entries), power of two
constexpr int LCHUNK = 256;              // window refill granularity (two entries per producer thread)
static_assert(RNT == 2 * RW && LCHUNK == 2 * RW && (LWIN & (LWIN - 1)) == 0 && LWIN >= 4 * LCHUNK, "refine CTA shape");

struct RingSmem {
  float4 q[PF][RW];                      // up: child weights; sweep: (ind, outd[parent], grad so far)
  int ia[PF][RW];                        // up: child range; down / sweep: parent position
  float fa[PF][RW];                      // down / sweep: edge weight
  int lvl[LWIN];
};
struct Rec { float4 q; int ia; float fa; };



__device__ __forceinline__ void cpa4(void* dst, const void* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cpa16(void* dst, const void* src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct TreeView {
  const int32_t* idx;     // [V] position -> vertex
  const int32_t* par;     // [V] position of the parent
  const int32_t* lvl;     // [L+1]
  const float* w;         // [V] edge weight to the parent, position order (w[0] treated as 0)
  const int32_t* cinfo;   // [V] first child position | (child count << 28)
  const float4* cw;       // [V] weights of the (<= 4) children, in child order
  int V, L;
};

// children are contiguous in position order (bfs_block_kernel); pack the range and the child weights per node
__global__ void tree_pack_kernel(const float* __restrict__ w, const int32_t* __restrict__ chd, int32_t* __restrict__ cinfo,
                                 float4* __restrict__ cw, int V, int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t b = i / V;
    const int32_t* c = chd + i * 4;
    const float* wb = w + b * V;
    int first = 0, n = 0;
    float cv[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int q = c[k];
      if (q > 0 && n == k) { if (k == 0) first = q; cv[k] = wb[q]; ++n; }
    }
    cinfo[i] = first | (n << 28);
    cw[i] = make_float4(cv[0], cv[1], cv[2], cv[3]);
  }
}

// PADDED (shared-memory buffer with 4 zeroed floats behind position V-1): the four child slots are read and
// accumulated unconditionally -- a missing child has weight 0 (tree_pack_kernel) and its slot holds some finite node
// value, so it adds an exact zero.  The conditional form serialises up to four shared-memory round trips and four
// branches on the critical path of EVERY level (SASS: LDS -> FFMA -> BRA, four times); this one is four independent
// loads and one FMA chain.  (A NaN/Inf input makes every output NaN in either form: the down pass spreads the root's
// aggregate to all nodes.)
template <bool PADDED>
__device__ __forceinline__ float up_node(float own, int ci, const float4& cw, const float* buf) {
  const int first = ci & 0x0fffffff, n = ci >> 28;
  float acc = own;
  if (PADDED) {
    const float b0 = buf[first], b1 = buf[first + 1], b2 = buf[first + 2], b3 = buf[first + 3];
    acc = fmaf(b0, cw.x, acc);
    acc = fmaf(b1, cw.y, acc);
    acc = fmaf(b2, cw.z, acc);
    acc = fmaf(b3, cw.w, acc);
  } else {
    if (n > 0) acc = fmaf(buf[first], cw.x, acc);
    if (n > 1) acc = fmaf(buf[first + 1], cw.y, acc);
    if (n > 2) acc = fmaf(buf[first + 2], cw.z, acc);
    if (n > 3) acc = fmaf(buf[first + 3], cw.w, acc);
  }
  return acc;
}

// Walk the levels in dependency order (DIR = -1: deepest level .. root, DIR = +1: level 1 .. deepest).
//   issue(p, slot, i)        producer thread: cp.async copies of the record of position p into ring[slot][i]
//   compute(p, on, rec)      consumer thread i < RW: position p = level start + i (`on`: p is inside the level), `rec` =
//                            its record (UNDEFINED when !on: idle threads must not use it for addresses)
//   direct(p)                any thread: the same work for position p with plain global loads (levels wider than RW)
template <int DIR, typename Issue, typename Compute, typename Direct>
__device__ __forceinline__ void level_walk(const TreeView& t, RingSmem& R, Issue issue, Compute compute, Direct direct) {
  const int tid = threadIdx.x;
  const bool producer = tid >= RW;
  const int slot_i = producer ? tid - RW : tid;
  const int first = DIR > 0 ? 1 : t.L - 1, last = DIR > 0 ? t.L - 1 : 0;
  __syncthreads();                                          // the previous walk is done with the ring and the window
  if (DIR > 0 ? first > last : first < last) return;
  if (DIR > 0) {
    for (int e = tid; e < LWIN - LCHUNK; e += RNT)
      if (e <= t.L) cpa4(&R.lvl[e & (LWIN - 1)], t.lvl + e);
  } else {
    const int hi = ((t.L - 1) | (LCHUNK - 1)) + 1;
    for (int k = tid; k < LWIN - LCHUNK; k += RNT) {
      const int e = hi - k;
      if (e >= 0 && e <= t.L) cpa4(&R.lvl[e & (LWIN - 1)], t.lvl + e);
    }
  }
  cp_commit();
  cp_wait<0>();
  __syncthreads();
  auto lv = [&](int l) { return R.lvl[l & (LWIN - 1)]; };
  auto inside = [&](int l) { return DIR > 0 ? l <= last : l >= last; };
  // copies of level l (bounds s0, e0) into ring slot `slot`; one group per level, empty or not: the count is what matters
  auto issue_level = [&](int l, int slot, int s0, int e0) {
    if (inside(l) && s0 + (slot_i & ~31) < e0) {            // warp-uniform: most levels need only the first producer warp
      const int p = s0 + slot_i;
      if (p < e0) issue(p, slot, slot_i);
    }
    cp_commit();
  };
  auto load_rec = [&](int slot) {
    Rec r;
    r.q = R.q[slot][slot_i]; r.ia = R.ia[slot][slot_i]; r.fa = R.fa[slot][slot_i];
    return r;
  };
  // producer registers: bounds of the level whose copies sit in slot j (its wide-level remainder is done from them PF
  // levels later), bounds of the next level to issue (read one level ahead, in the shadow of the barrier), and the level
  // at which the window is refilled next
  int bs[PF], be[PF], nis = 0, nie = 0;
  int refill_at = DIR > 0 ? LCHUNK : (((t.L - 1) | (LCHUNK - 1)) + 1) - LCHUNK - 1;
  if (producer) {
#pragma unroll
    for (int j = 0; j < PF; ++j) {
      const int l = first + DIR * j;
      bs[j] = be[j] = 0;
      if (inside(l)) { bs[j] = lv(l); be[j] = lv(l + 1); }
      issue_level(l, j, bs[j], be[j]);
    }
    if (inside(first + DIR * PF)) { nis = lv(first + DIR * PF); nie = lv(first + DIR * PF + 1); }
    cp_wait<PF - 2>();                                      // the first two levels have landed
  }
  __syncthreads();
  Rec rec;
  rec.q = make_float4(0.f, 0.f, 0.f, 0.f); rec.ia = 0; rec.fa = 0.f;
  int s = 0, e = 0;
  if (!producer) {
    s = lv(first); e = lv(first + 1);
    rec = load_rec(0);
  }
  for (int l0 = first; DIR > 0 ? l0 <= last : l0 >= last; l0 += DIR * PF) {
    // window refill (producers, two entries each), once per chunk of LCHUNK levels, up to PF levels early; the copies ride
    // in the next level's group and are read 250+ levels later
    if (producer && (DIR > 0 ? l0 + PF > refill_at : l0 - PF < refill_at)) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int en = DIR > 0 ? refill_at + LWIN - 2 * LCHUNK + slot_i + h * RW : refill_at - (2 * LCHUNK - 1) - slot_i - h * RW;
        if (en >= 0 && en <= t.L) cpa4(&R.lvl[en & (LWIN - 1)], t.lvl + en);
      }
      refill_at += DIR * LCHUNK;
    }
#pragma unroll
    for (int j = 0; j < PF; ++j) {
      const int l = l0 + DIR * j;
      if (DIR > 0 ? l > last : l < last) break;
      if (!producer) {
        if (tid == 0) TREE_TT(0, DIR * (l - first));
        const int p = s + tid;
        compute(p, p < e, rec);
        if (tid == 0) TREE_TT(1, DIR * (l - first));
        asm volatile("" ::: "memory");                      // keep the next level's loads BEHIND this level's store
        // next level's bounds and record (complete since the previous barrier): their latency hides in the barrier.
        // Loaded unconditionally (no dependent round trip); compute() ignores the record of an idle thread.
        Rec nrec = rec;
        int ns = 0, ne = 0;
        if (inside(l + DIR)) { ns = lv(l + DIR); ne = lv(l + DIR + 1); nrec = load_rec((j + 1) % PF); }
#pragma unroll 1
        for (int p2 = p + RNT; p2 < e; p2 += RNT) direct(p2);
        rec = nrec; s = ns; e = ne;
        if (tid == 0) TREE_TT(2, DIR * (l - first));
      } else {
        if (tid == RW) TREE_TT(3, DIR * (l - first));
#pragma unroll 1
        for (int p2 = bs[j] + tid; p2 < be[j]; p2 += RNT) direct(p2);      // positions RW.. of a wide level
        issue_level(l + DIR * PF, j, nis, nie);             // slot j: its record was read by the consumers a level ago
        bs[j] = nis; be[j] = nie;
        if (tid == RW) TREE_TT(4, DIR * (l - first));
        cp_wait<PF - 2>();                                  // level l + 2 has landed: visible to the consumers after the barrier
        if (tid == RW) TREE_TT(5, DIR * (l - first));
        const int ln = l + DIR * (PF + 1);                  // the level the next iteration issues
        nis = nie = 0;
        if (inside(ln)) { nis = lv(ln); nie = lv(ln + 1); }
      }
      __syncthreads();
    }
  }
  if (producer) cp_wait<0>();
}

// buf[p] holds the node's own input on entry; on exit U[p] = in(p) + sum_children w[c] U[c].  Deepest level first.
template <bool PADDED>
__device__ __forceinline__ void up_pass(const TreeView& t, RingSmem& R, float* buf, float* __restrict__ save_up) {
  level_walk<-1>(
      t, R,
      [&](int p, int slot, int i) {
        cpa4(&R.ia[slot][i], t.cinfo + p);
        cpa16(&R.q[slot][i], t.cw + p);
      },
      [&](int p, bool on, const Rec& r) {
        if (PADDED) {
          const int first = on ? (r.ia & 0x0fffffff) : 0;
          const float own = buf[on ? p : 0], b0 = buf[first], b1 = buf[first + 1], b2 = buf[first + 2], b3 = buf[first + 3];
          if (on) buf[p] = fmaf(b3, r.q.w, fmaf(b2, r.q.z, fmaf(b1, r.q.y, fmaf(b0, r.q.x, own))));
        } else {
          if (on) buf[p] = up_node<false>(buf[p], r.ia, r.q, buf);
        }
      },
      [&](int p) { buf[p] = up_node<PADDED>(buf[p], __ldg(t.cinfo + p), __ldg(t.cw + p), buf); });
  // U of every position is in `buf`: one coalesced sweep instead of a global store on every level's critical path
  if (save_up)
    for (int p = threadIdx.x; p < t.V; p += RNT) save_up[p] = buf[p];
}

// in place: A[0] = U[0]; A[p] = (1 - w^2) U[p] + w A[par]; writes the vertex-ordered result
__device__ __forceinline__ void down_pass(const TreeView& t, RingSmem& R, float* buf, float* __restrict__ out_vertex) {
  level_walk<1>(
      t, R,
      [&](int p, int slot, int i) {
        cpa4(&R.ia[slot][i], t.par + p);
        cpa4(&R.fa[slot][i], t.w + p);
      },
      [&](int p, bool on, const Rec& r) {
        const float a_par = buf[on ? r.ia : 0], u_own = buf[on ? p : 0];
        if (on) buf[p] = fmaf(a_par, r.fa, u_own * (1.f - r.fa * r.fa));
      },
      [&](int p) {
        const float ew = __ldg(t.w + p);
        buf[p] = fmaf(buf[__ldg(t.par + p)], ew, buf[p] * (1.f - ew * ew));
      });
  __syncthreads();
  // A of every position is in `buf`: scatter to vertex order in one parallel sweep (not level by level)
  if (out_vertex)
#pragma unroll 8
    for (int p = threadIdx.x; p < t.V; p += RNT) out_vertex[__ldg(t.idx + p)] = buf[p];
}

__device__ __forceinline__ TreeView make_view(const float* w, const int32_t* idx, const int32_t* par, const int32_t* cinfo,
                                              const float4* cw, const int32_t* lvl, const int32_t* nlv, int b, int V) {
  TreeView t;
  t.idx = idx + (int64_t)b * V; t.par = par + (int64_t)b * V; t.cinfo = cinfo + (int64_t)b * V;
  t.cw = cw + (int64_t)b * V; t.lvl = lvl + (int64_t)b * (V + 1); t.w = w + (int64_t)b * V; t.V = V; t.L = nlv[b];
  return t;
}

// MODE 0: forward (feature CTAs, then one normaliser CTA with input 1 per tree)
// MODE 1: backward wrt feature: input = g / Z
template <int MODE, bool SMEM>
__global__ void __launch_bounds__(RNT) refine_updown_kernel(const float* __restrict__ feature, const float* __restrict__ w,
                                                           const int32_t* __restrict__ idx, const int32_t* __restrict__ par,
                                                           const int32_t* __restrict__ cinfo, const float4* __restrict__ cw,
                                                           const int32_t* __restrict__ lvl, const int32_t* __restrict__ nlv,
                                                           const float* __restrict__ wsum, float* __restrict__ aggr,
                                                           float* __restrict__ aggr_up, float* __restrict__ wsum_out,
                                                           float* __restrict__ wsum_up, float* __restrict__ scratch, int C,
                                                           int V, const int32_t* __restrict__ tree_of, int norm_from) {
  // tree_of (may be null): the tree / edge weights / normaliser of batch entry b are those of group tree_of[b] -- the
  // instances of one image share one tree (box_solov2_head.py:300-305,353; box2mask_head.py:271-276), so the order,
  // the packed child weights and the normaliser Z exist once per image instead of once per instance.
  // norm_from = the instance count.  Forward: CTAs with blockIdx.x >= norm_from compute the normaliser of TREE
  // blockIdx.x - norm_from (one per tree, blockIdx.y == 0 only) in the same launch as the feature CTAs -- the two are
  // independent until the division, and as two launches on one stream they cost two level walks back to back.
  // The backward launches exactly norm_from CTAs per channel.
  extern __shared__ float s_buf[];
  __shared__ RingSmem R;
  const bool split_norm = (int)blockIdx.x >= norm_from;
  if (split_norm && blockIdx.y != 0) return;
  const int b = split_norm ? (int)blockIdx.x - norm_from : (int)blockIdx.x, c = split_norm ? C : (int)blockIdx.y;
  const int tb = (tree_of && !split_norm) ? __ldg(tree_of + b) : b;
  const TreeView t = make_view(w, idx, par, cinfo, cw, lvl, nlv, tb, V);
  float* buf = SMEM ? s_buf : scratch + ((int64_t)b * (C + 1) + c) * V;
  const bool norm = MODE == 0 && c == C;
  const float* x = norm ? nullptr : feature + ((int64_t)b * C + c) * V;
  const float* z = MODE == 1 ? wsum + (int64_t)tb * V : nullptr;
  float* save_up = MODE == 0 ? (norm ? wsum_up + (int64_t)b * V : aggr_up + ((int64_t)b * C + c) * V) : nullptr;
  float* out_v = MODE == 0 ? (norm ? wsum_out + (int64_t)b * V : aggr + ((int64_t)b * C + c) * V)
                           : aggr + ((int64_t)b * C + c) * V;     // MODE 1: aggr == grad_feature
  // (dependent index -> value loads with 256 threads per CTA: unrolled so that 8 round trips are in flight per thread)
#pragma unroll 8
  for (int p = threadIdx.x; p < V; p += RNT) {               // parallel gather of the inputs into position order
    const int v = __ldg(t.idx + p);
    buf[p] = norm ? 1.f : (MODE == 1 ? x[v] / z[v] : x[v]);
  }
  if (SMEM && threadIdx.x < 4) buf[V + threadIdx.x] = 0.f;      // the pad up_node<true> may read
  __syncthreads();
  up_pass<SMEM>(t, R, buf, save_up);
  down_pass(t, R, buf, out_v);
}

__global__ void refine_div_kernel(const float* __restrict__ aggr, const float* __restrict__ wsum, float* __restrict__ out,
                                  int C, int V, int64_t total, const int32_t* __restrict__ tree_of) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = i % V;
    const int64_t b = i / ((int64_t)C * V);
    const int64_t tb = tree_of ? __ldg(tree_of + b) : b;
    out[i] = aggr[i] / wsum[tb * V + v];
  }
}

// backward wrt the edge weights (refine.cu:302-370): per channel
//   gn = g / Z, fg = gn * out;  gnU = up(gn), fgU = up(fg)
//   grad[p] += sweep(aggr_up_c, gnU, aggr_c)[p] - sweep(wsum_up, fgU, wsum)[p]
// sweep: G[0] = gup[0]; for p > 0: grad = gup (outd[v_par] - w ind) + ind (G[par] - w gup); G = gup (1 - w^2) + G[par] w
// `outd_par` [2][V] is the position-ordered gather outd[idx[par[p]]] for the two data sets (parallel pre-pass).

template <bool SMEM>
__global__ void __launch_bounds__(RNT) refine_bwd_weight_kernel(
    const float* __restrict__ w, const int32_t* __restrict__ idx, const int32_t* __restrict__ par,
    const int32_t* __restrict__ cinfo, const float4* __restrict__ cw, const int32_t* __restrict__ lvl,
    const int32_t* __restrict__ nlv, const float* __restrict__ out, const float* __restrict__ aggr,
    const float* __restrict__ aggr_up, const float* __restrict__ wsum, const float* __restrict__ wsum_up,
    const float* __restrict__ g_out, float* __restrict__ grad_w, float* __restrict__ scratch, float* __restrict__ outd_par,
    int C, int V, const int32_t* __restrict__ tree_of) {
  // The two terms of d/d w (refine.cu:302-370) are independent passes over the tree: blockIdx.y selects the term, the two
  // CTAs of an instance run concurrently on different SMs and write separate buffers (grad_w and its twin B*V further),
  // summed by refine_add_kernel -- the dependent-level chain of this backward is 2 passes long instead of 4.
  extern __shared__ float s_buf[];
  __shared__ RingSmem R;
  const int b = blockIdx.x, nb = gridDim.x, phase = blockIdx.y;
  const int tb = tree_of ? __ldg(tree_of + b) : b;          // tree / weights / normaliser of the instance's image
  const TreeView t = make_view(w, idx, par, cinfo, cw, lvl, nlv, tb, V);
  float* buf = SMEM ? s_buf : scratch + ((int64_t)phase * nb + b) * V;
  float* gw = grad_w + ((int64_t)phase * nb + b) * V;
  float* op = outd_par + ((int64_t)phase * nb + b) * V;
  const float* z = wsum + (int64_t)tb * V;
  const float* zu = wsum_up + (int64_t)tb * V;
  for (int p = threadIdx.x; p < V; p += RNT) gw[p] = 0.f;
  for (int c = 0; c < C; ++c) {
    const float* g = g_out + ((int64_t)b * C + c) * V;
    const float* o = out + ((int64_t)b * C + c) * V;
    const float* ag = aggr + ((int64_t)b * C + c) * V;
    const float* au = aggr_up + ((int64_t)b * C + c) * V;
    {
      // phase 0: gup = up(g/Z), data = (aggr_up, aggr), sign +   phase 1: gup = up(g/Z * out), data = (wsum_up, wsum), sign -
      const float* ind = phase ? zu : au;
      const float* outd = phase ? z : ag;
      const float sign = phase ? -1.f : 1.f;
      __syncthreads();
#pragma unroll 4
      for (int p = threadIdx.x; p < V; p += RNT) {           // parallel pre-pass: inputs and parent data, position order
        const int v = __ldg(t.idx + p);
        const float gn = g[v] / z[v];
        buf[p] = phase ? gn * o[v] : gn;
        op[p] = p == 0 ? 0.f : outd[__ldg(t.idx + __ldg(t.par + p))];
      }
      if (SMEM && threadIdx.x < 4) buf[V + threadIdx.x] = 0.f;   // the pad up_node<true> may read
      __syncthreads();
      up_pass<SMEM>(t, R, buf, nullptr);
      // top-down: buf[p] holds gup[p] until visited, then G[p].  gw[p] is updated once per (channel, phase) and the
      // channels are separated by barriers: its old value travels with the prefetched record instead of being a dependent
      // global load inside the level.
      level_walk<1>(
          t, R,
          [&](int p, int slot, int i) {
            cpa4(&R.ia[slot][i], t.par + p);
            cpa4(&R.fa[slot][i], t.w + p);
            cpa4(&R.q[slot][i].x, ind + p);
            cpa4(&R.q[slot][i].y, op + p);
            cpa4(&R.q[slot][i].z, gw + p);
          },
          [&](int p, bool on, const Rec& r) {
            const float gup = buf[on ? p : 0], Gp = buf[on ? r.ia : 0];
            if (on) {
              const float ew = r.fa, in_p = r.q.x;
              buf[p] = fmaf(Gp, ew, gup * (1.f - ew * ew));
              gw[p] = r.q.z + sign * (gup * (r.q.y - ew * in_p) + in_p * (Gp - ew * gup));
            }
          },
          [&](int p) {
            const float ew = __ldg(t.w + p), in_p = ind[p], gup = buf[p], Gp = buf[__ldg(t.par + p)];
            gw[p] += sign * (gup * (op[p] - ew * in_p) + in_p * (Gp - ew * gup));
            buf[p] = fmaf(Gp, ew, gup * (1.f - ew * ew));
          });
    }
  }
}

__global__ void refine_add_kernel(float* __restrict__ a, const float* __restrict__ b2, int64_t total) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) a[i] += b2[i];
}

constexpr size_t kMaxTreeSmem = 220 * 1024;
// refine kernels: the position-ordered values (dynamic) next to the copy ring + level window (static)
constexpr size_t kMaxRefineSmem = 227 * 1024 - sizeof(RingSmem) - 64;

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_mst_workspace_bytes(int64_t B, int64_t E, int64_t V) {
  return (B <= 0 || E <= 0 || V <= 0) ? 0 : (int64_t)carve_mst(nullptr, B, E, V).total_bytes;
}

extern "C" int bxs_mst_forward(const int32_t* edge_index, const float* edge_weight, int32_t* edge_out, void* workspace,
                               int64_t B, int64_t E, int64_t V, bxs_stream_t stream) {
  if (!edge_index || !edge_weight || !edge_out || !workspace || B <= 0 || B >= 65536 || E <= 0 || V <= 1 ||
      E >= (int64_t(1) << 31) || V >= (int64_t(1) << 31))
    return BXS_ERR_INVALID_ARG;
  // both edge lists are read and written one int2 per edge
  if ((reinterpret_cast<uintptr_t>(edge_index) & 7) || (reinterpret_cast<uintptr_t>(edge_out) & 7))
    return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  MstWs ws = carve_mst(workspace, B, E, V);
  int rounds = 0;
  while ((int64_t(1) << rounds) < V) ++rounds;             // components at least halve per round
  if (rounds <= 64 && B * MST_CL < 65536 * 8) {
    mst_cluster_kernel<<<(unsigned)(B * MST_CL), MST_NT, 0, st>>>(edge_index, edge_weight, ws, (int)E, (int)V, rounds,
                                                                  ws.round_flags);
  } else {
    mst_init_kernel<<<grid_for(B * std::max(E, V), 256), 256, 0, st>>>(ws, B * V, B * E, (int)V);
    const dim3 ge((unsigned)std::min<int64_t>(ceil_div(E, 256), 1024), (unsigned)B);
    const dim3 gv((unsigned)std::min<int64_t>(ceil_div(V, 256), 1024), (unsigned)B);
    for (int r = 0; r < rounds; ++r) {
      mst_min_edge_kernel<<<ge, 256, 0, st>>>(edge_index, edge_weight, ws, (int)E, (int)V);
      mst_hook_kernel<<<gv, 256, 0, st>>>(edge_index, ws, (int)E, (int)V);
      mst_compress_kernel<<<gv, 256, 0, st>>>(ws, (int)V);
    }
  }
  {
    const int nchunks = (int)ceil_div(E, MC_CHUNK);
    int* counts = reinterpret_cast<int*>(ws.best);          // the Boruvka keys are dead by now: B * nchunks <= B * V ints
    mst_count_kernel<<<dim3((unsigned)nchunks, (unsigned)B), MC_T, 0, st>>>(ws, counts, (int)E);
    mst_compact_kernel<<<dim3((unsigned)nchunks, (unsigned)B), MC_T, 0, st>>>(edge_index, ws, counts, edge_out, (int)E, (int)V);
  }
  return check_launch();
}

extern "C" int64_t bxs_bfs_workspace_bytes(int64_t B, int64_t V) {
  return (B <= 0 || V <= 0) ? 0 : (int64_t)carve_bfs(nullptr, B, V).total_bytes + 256;
}

// level_start [B, V+1] and num_levels [B] are required outputs: the level table bxs_refine_* runs on.
// The reference roots every tree at vertex 0 (bfs.cu:100-135); here the caller picks the root: the tree filter's result
// does not depend on it, but the number of dependent levels of every pass does (a 200x256 image MST is ~1900 levels deep
// from the corner, about half of that from the centre).
extern "C" int bxs_bfs_forward_rooted(const int32_t* tree_edges, int32_t* sorted_index, int32_t* sorted_parent,
                                      int32_t* sorted_child, int32_t* level_start, int32_t* num_levels, void* workspace,
                                      int64_t B, int64_t V, int max_adj, int64_t root, bxs_stream_t stream) {
  if (!tree_edges || !sorted_index || !sorted_parent || !sorted_child || !level_start || !num_levels || !workspace ||
      B <= 0 || B >= 65536 || V <= 1 || root < 0 || root >= V)
    return BXS_ERR_INVALID_ARG;
  if (max_adj != 4) return BXS_ERR_UNSUPPORTED;             // the reference only ever passes 4 (tree_filter.py:137)
  // the edges are read one int2 each, the child table is written one int4 per node
  if ((reinterpret_cast<uintptr_t>(tree_edges) & 7) || (reinterpret_cast<uintptr_t>(sorted_child) & 15))
    return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  BfsWs ws = carve_bfs(workspace, B, V);
  int* err = (int*)((char*)workspace + ws.total_bytes);
  int* flags = ws.flags;
  cudaMemsetAsync(ws.deg, 0, sizeof(int) * B * V, st);
  cudaMemsetAsync(err, 0, sizeof(int), st);
  // fast path: 4-connected grid trees with the adjacency bits in shared memory (one warp per tree)
  const size_t grid_smem = ((size_t)(V + 3) / 4) * 4 + (size_t)BFS_BUFS * 2 * BFS_STRIDE * sizeof(int);
  const bool try_grid = grid_smem <= kMaxTreeSmem;
  if (try_grid) {
    if (opt_in_smem(bfs_grid_kernel, kMaxTreeSmem) != BXS_OK) return BXS_ERR_LAUNCH;
    bfs_grid_kernel<<<(unsigned)B, NT, grid_smem, st>>>(tree_edges, (int)V, sorted_index, sorted_parent, sorted_child,
                                                        level_start, num_levels, flags, (int)root);
  } else {
    cudaMemsetAsync(flags, 0, sizeof(int) * B, st);
  }
  // generic path for whatever the fast path declined (its CTAs return at once otherwise)
  bfs_adj_kernel<<<dim3((unsigned)std::min<int64_t>(ceil_div(V, 256), 1024), (unsigned)B), 256, 0, st>>>(tree_edges, ws,
                                                                                                         (int)V, err, flags);
  bfs_sort_adj_kernel<<<grid_for(B * V, 256), 256, 0, st>>>(ws, B * V, (int)V, flags);
  bfs_block_kernel<<<(unsigned)B, NT, 0, st>>>(ws, (int)V, sorted_index, sorted_parent, sorted_child, level_start,
                                               num_levels, flags, (int)root);
  return check_launch();
}

// scratch layout: cinfo int[B*V] | cw float4[B*V] | outd_par float[B*V] | global buffers float[B*(C+1)*V] (maps too large for smem)
namespace bxs {
namespace {
struct RefineScratch {
  int32_t* cinfo;
  float4* cw;
  float* outd_par;
  float* gw2;
  float* bufs;
  size_t total_bytes;
};
inline RefineScratch carve_refine(void* base, int64_t B, int64_t C, int64_t V) {
  RefineScratch r{};
  Carver c(base);
  r.cw = (float4*)c.take(16 * B * V);
  r.cinfo = (int32_t*)c.take(4 * B * V);
  r.outd_par = (float*)c.take(2 * 4 * B * V);             // per d/d w term
  r.gw2 = (float*)c.take(2 * 4 * B * V);                  // the two d/d w terms before they are summed
  r.bufs = (float*)c.take(4 * B * (C + 2) * V);
  r.total_bytes = c.off;
  return r;
}
inline void pack_tree(const float* w, const int32_t* chd, const RefineScratch& rs, int64_t B, int64_t V, cudaStream_t st) {
  tree_pack_kernel<<<grid_for(B * V, 256), 256, 0, st>>>(w, chd, rs.cinfo, rs.cw, (int)V, B * V);
}
}  // namespace
}  // namespace bxs

extern "C" int64_t bxs_refine_scratch_bytes(int64_t B, int64_t C, int64_t V) {
  return (B <= 0 || C <= 0 || V <= 0) ? 0 : (int64_t)carve_refine(nullptr, B, C, V).total_bytes;
}

// ---------------------------------------------------------------------------------------
// n instances share G trees (tree_of [n] -> group; NULL: instance i uses tree i, n == G).  Order, packed child weights,
// edge weights and the normaliser exist once per group; per-instance work is one CTA per (instance, channel).
// ---------------------------------------------------------------------------------------
extern "C" int bxs_refine_forward_grouped(const float* feature, const float* edge_weight, const int32_t* sorted_index,
                                          const int32_t* sorted_parent, const int32_t* sorted_child,
                                          const int32_t* level_start, const int32_t* num_levels, const int32_t* tree_of,
                                          float* feature_out, float* aggr, float* aggr_up, float* wsum, float* wsum_up,
                                          void* scratch, int64_t n, int64_t G, int64_t C, int64_t V, bxs_stream_t stream) {
  if (!feature || !edge_weight || !sorted_index || !sorted_parent || !sorted_child || !level_start || !num_levels ||
      !feature_out || !aggr || !aggr_up || !wsum || !wsum_up || !scratch || n <= 0 || n >= 65536 || G <= 0 ||
      G >= 65536 || C <= 0 || C >= 65535 || V <= 0 || V >= (int64_t(1) << 28) || (!tree_of && n != G))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  RefineScratch rs = carve_refine(scratch, std::max(n, G), C, V);
  pack_tree(edge_weight, sorted_child, rs, G, V, st);
  const size_t sm = (V + 4) * sizeof(float);
  if (sm <= kMaxRefineSmem) {
    if (opt_in_smem(refine_updown_kernel<0, true>, kMaxRefineSmem) != BXS_OK) return BXS_ERR_LAUNCH;
    refine_updown_kernel<0, true><<<dim3((unsigned)(n + G), (unsigned)C), RNT, sm, st>>>(
        feature, edge_weight, sorted_index, sorted_parent, rs.cinfo, rs.cw, level_start, num_levels, nullptr, aggr, aggr_up,
        wsum, wsum_up, nullptr, (int)C, (int)V, tree_of, (int)n);
  } else {
    refine_updown_kernel<0, false><<<dim3((unsigned)(n + G), (unsigned)C), RNT, 0, st>>>(
        feature, edge_weight, sorted_index, sorted_parent, rs.cinfo, rs.cw, level_start, num_levels, nullptr, aggr, aggr_up,
        wsum, wsum_up, rs.bufs, (int)C, (int)V, tree_of, (int)n);
  }
  refine_div_kernel<<<grid_for(n * C * V, 256), 256, 0, st>>>(aggr, wsum, feature_out, (int)C, (int)V, n * C * V, tree_of);
  return check_launch();
}

extern "C" int bxs_refine_backward_feature_grouped(const float* edge_weight, const int32_t* sorted_index,
                                                   const int32_t* sorted_parent, const int32_t* sorted_child,
                                                   const int32_t* level_start, const int32_t* num_levels,
                                                   const int32_t* tree_of, const float* wsum, const float* grad_out,
                                                   float* grad_feature, void* scratch, int64_t n, int64_t G, int64_t C,
                                                   int64_t V, bxs_stream_t stream) {
  if (!edge_weight || !sorted_index || !sorted_parent || !sorted_child || !level_start || !num_levels || !wsum ||
      !grad_out || !grad_feature || !scratch || n <= 0 || n >= 65536 || G <= 0 || G >= 65536 || C <= 0 || C >= 65535 ||
      V <= 0 || V >= (int64_t(1) << 28) || (!tree_of && n != G))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  RefineScratch rs = carve_refine(scratch, std::max(n, G), C, V);
  pack_tree(edge_weight, sorted_child, rs, G, V, st);
  const size_t sm = (V + 4) * sizeof(float);
  const dim3 grid((unsigned)n, (unsigned)C);
  if (sm <= kMaxRefineSmem) {
    if (opt_in_smem(refine_updown_kernel<1, true>, kMaxRefineSmem) != BXS_OK) return BXS_ERR_LAUNCH;
    refine_updown_kernel<1, true><<<grid, RNT, sm, st>>>(grad_out, edge_weight, sorted_index, sorted_parent, rs.cinfo, rs.cw,
                                                        level_start, num_levels, wsum, grad_feature, nullptr, nullptr,
                                                        nullptr, nullptr, (int)C, (int)V, tree_of, (int)n);
  } else {
    refine_updown_kernel<1, false><<<grid, RNT, 0, st>>>(grad_out, edge_weight, sorted_index, sorted_parent, rs.cinfo, rs.cw,
                                                        level_start, num_levels, wsum, grad_feature, nullptr, nullptr,
                                                        nullptr, rs.bufs, (int)C, (int)V, tree_of, (int)n);
  }
  return check_launch();
}

// grad_weight [n,V]: per INSTANCE (the caller sums the rows of a group: d/d w of a shared tree)
extern "C" int bxs_refine_backward_weight_grouped(const float* edge_weight, const int32_t* sorted_index,
                                                  const int32_t* sorted_parent, const int32_t* sorted_child,
                                                  const int32_t* level_start, const int32_t* num_levels,
                                                  const int32_t* tree_of, const float* feature_out, const float* aggr,
                                                  const float* aggr_up, const float* wsum, const float* wsum_up,
                                                  const float* grad_out, float* grad_weight, void* scratch, int64_t n,
                                                  int64_t G, int64_t C, int64_t V, bxs_stream_t stream) {
  if (!edge_weight || !sorted_index || !sorted_parent || !sorted_child || !level_start || !num_levels || !feature_out ||
      !aggr || !aggr_up || !wsum || !wsum_up || !grad_out || !grad_weight || !scratch || n <= 0 || n >= 65536 || G <= 0 ||
      G >= 65536 || C <= 0 || V <= 0 || V >= (int64_t(1) << 28) || (!tree_of && n != G))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  RefineScratch rs = carve_refine(scratch, std::max(n, G), C, V);
  pack_tree(edge_weight, sorted_child, rs, G, V, st);
  const size_t sm = (V + 4) * sizeof(float);
  if (sm <= kMaxRefineSmem) {
    if (opt_in_smem(refine_bwd_weight_kernel<true>, kMaxRefineSmem) != BXS_OK) return BXS_ERR_LAUNCH;
    refine_bwd_weight_kernel<true><<<dim3((unsigned)n, 2), RNT, sm, st>>>(edge_weight, sorted_index, sorted_parent, rs.cinfo,
                                                                         rs.cw, level_start, num_levels, feature_out, aggr,
                                                                         aggr_up, wsum, wsum_up, grad_out, rs.gw2, nullptr,
                                                                         rs.outd_par, (int)C, (int)V, tree_of);
  } else {
    refine_bwd_weight_kernel<false><<<dim3((unsigned)n, 2), RNT, 0, st>>>(edge_weight, sorted_index, sorted_parent, rs.cinfo,
                                                                          rs.cw, level_start, num_levels, feature_out, aggr,
                                                                          aggr_up, wsum, wsum_up, grad_out, rs.gw2, rs.bufs,
                                                                          rs.outd_par, (int)C, (int)V, tree_of);
  }
  cudaMemcpyAsync(grad_weight, rs.gw2, sizeof(float) * n * V, cudaMemcpyDeviceToDevice, st);
  refine_add_kernel<<<grid_for(n * V, 256), 256, 0, st>>>(grad_weight, rs.gw2 + n * V, n * V);
  return check_launch();
}

#ifdef BXS_TREE_TRACE
extern "C" int bxs_debug_tree_trace(long long* out_host) {
  return cudaMemcpyFromSymbol(out_host, bxs::g_tree_trace, sizeof(long long) * 6 * 4096) == cudaSuccess ? 0 : -2;
}
#endif
