// a6 + a7 + a8: the fused BoxInst mask loss (projection term + colour-pairwise term) and its
// backward.  Replaces the arithmetic of CondInstMaskHead.loss, condinst_head.py:1288-1343
// (sigmoid -> compute_project_term :134-143 -> pairwise_nlog -> threshold weights -> reduction).
//
// Design (DESIGN.md "BoxInst loss"):
//   * the [N,8,H,W] pairwise tensor, the [N,8,H,W] gathered similarity and the [N,1,H,W] gathered
//     bitmask of the reference are never materialised.  The similarity enters as ONE BYTE per
//     pixel per image (bit c = sim[c] >= thresh) and the box bitmask as 4 integers per GT.
//   * forward kernel 1 streams the logits once (HBM-bound): row / column maxima of the scores
//     with first-index tie-breaking, combined across CTAs with order-independent 64-bit
//     atomicMax on (score bits, ~index) -> deterministic.
//   * forward kernel 2 evaluates pair terms ONLY where a weight can be non-zero (inside the GT
//     box +- dilation), walking a device-built work list of 16x64 tiles so every CTA has work.
//     Each unordered pair is evaluated once (pl is symmetric) with an integer multiplier 0/1/2.
//   * the finalize kernel turns the profiles into dice losses and into per-row/per-column
//     gradient coefficients; the last CTA (ticket counter) writes the scalars.
//   * backward is one tile kernel writing every g_logits element exactly once: zeros + arg-max
//     scatter outside the box, gather-form pairwise gradient inside.  No atomics on floats.
#include <algorithm>

#include "boxinst_common.cuh"

namespace bxs {
namespace {

constexpr int TH = 16, TW = 64, NT = 256;

struct Workspace {
  // zeroed at the start of every forward (fast path: up to zero_bytes_fast)
  unsigned long long* col_packed;  // [N*W]  (key(max logit) << 32) | ~y
  unsigned long long* weight_sum;  // [1]    sum of weights (integer)
  unsigned int* ticket;            // [1]    instances finalized
  unsigned int* inst_ticket;       // [N]    strips finished per instance (fast path)
  size_t zero_bytes_fast;
  unsigned long long* row_packed;  // [N*H]  (key(max logit) << 32) | ~x  (atomics only on the generic path)
  size_t zero_bytes;
  // plain
  float* coef_row;     // [N*H] d loss_prj / d logit at the row arg-max
  float* coef_col;     // [N*W]
  int* row_arg;        // [N*H]
  int* col_arg;        // [N*W]
  int* tile_prefix;    // [N+1]            generic path work list
  float* pair_partial; // [N*max(tiles,H)] per tile (generic) / per row (fast) numerators
  int* den_partial;    // [N*H]            per row weight counts (fast)
  float* inst_prj;     // [N]
  float* inst_num;     // [N]
  float* scale_pair;   // [1] warmup / max(weight_sum, 1)
  int* inst_rec;       // [N*16] per-instance record of the fast path (rectangle, image, span, chain split)
  size_t total_bytes;
};

inline size_t align_up(size_t v, size_t a = 256) { return (v + a - 1) / a * a; }

inline Workspace carve(void* base, int64_t N, int64_t H, int64_t W) {
  Workspace w{};
  char* p = (char*)base;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* r = p + off; off = align_up(off + bytes); return r; };
  w.col_packed = (unsigned long long*)take(sizeof(unsigned long long) * N * W);
  w.weight_sum = (unsigned long long*)take(sizeof(unsigned long long));
  w.ticket = (unsigned int*)take(sizeof(unsigned int));
  w.inst_ticket = (unsigned int*)take(sizeof(unsigned int) * N);
  w.zero_bytes_fast = off;
  w.row_packed = (unsigned long long*)take(sizeof(unsigned long long) * N * H);
  w.zero_bytes = off;
  w.coef_row = (float*)take(sizeof(float) * N * H);
  w.coef_col = (float*)take(sizeof(float) * N * W);
  w.row_arg = (int*)take(sizeof(int) * N * H);
  w.col_arg = (int*)take(sizeof(int) * N * W);
  w.tile_prefix = (int*)take(sizeof(int) * (N + 1));
  const int64_t tiles_full = ceil_div(H, TH) * ceil_div(W, TW);
  const int64_t per_inst = std::max<int64_t>(tiles_full, 128);         // generic: tiles; fast: one per pair-role warp
  w.pair_partial = (float*)take(sizeof(float) * N * per_inst);
  w.den_partial = (int*)take(sizeof(int) * N * per_inst);
  w.inst_prj = (float*)take(sizeof(float) * N);
  w.inst_num = (float*)take(sizeof(float) * N);
  w.scale_pair = (float*)take(sizeof(float));
  w.inst_rec = (int*)take(sizeof(int) * 16 * N);
  w.total_bytes = off;
  return w;
}


// tiles (map aligned) that contain a pixel p for which pair (p, p+forward offset) can carry weight:
// rows [j0-d, j1], cols [i0-d, i1+d], clipped to the map.
__device__ __forceinline__ bool fwd_tile_range(const Rect& r, int d, int H, int W, int& ty0, int& ty1,
                                               int& tx0, int& tx1) {
  if (rect_empty(r)) return false;
  int y0 = max(r.j0 - d, 0), y1 = min(r.j1, H - 1), x0 = max(r.i0 - d, 0), x1 = min(r.i1 + d, W - 1);
  if (y0 > y1 || x0 > x1) return false;
  ty0 = y0 / TH; ty1 = y1 / TH; tx0 = x0 / TW; tx1 = x1 / TW;
  return true;
}

// ---------------------------------------------------------------------------------------
// work list: exclusive prefix of per-instance tile counts (one CTA)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) prep_worklist(const int32_t* __restrict__ rects,
                                                    const int32_t* __restrict__ inst_gt, int N, int H, int W,
                                                    int d, int* __restrict__ tile_prefix) {
  __shared__ int s_sum[NT];
  const int per = (N + NT - 1) / NT;
  const int lo = threadIdx.x * per, hi = min(lo + per, N);
  int local = 0;
  for (int n = lo; n < hi; ++n) {
    int a, b, c, e;
    if (fwd_tile_range(load_rect(rects, inst_gt[n]), d, H, W, a, b, c, e)) local += (b - a + 1) * (e - c + 1);
  }
  s_sum[threadIdx.x] = local;
  __syncthreads();
  if (threadIdx.x == 0) {     // NT partial sums: a serial scan is cheaper than it looks (256 adds)
    int run = 0;
    for (int i = 0; i < NT; ++i) { int v = s_sum[i]; s_sum[i] = run; run += v; }
    tile_prefix[N] = run;
  }
  __syncthreads();
  int run = s_sum[threadIdx.x];
  for (int n = lo; n < hi; ++n) {
    tile_prefix[n] = run;
    int a, b, c, e;
    if (fwd_tile_range(load_rect(rects, inst_gt[n]), d, H, W, a, b, c, e)) run += (b - a + 1) * (e - c + 1);
  }
}

// ---------------------------------------------------------------------------------------
// forward 1: projection maxima.  grid (strips, N, panels); one warp per row.
// ---------------------------------------------------------------------------------------

template <int NCHUNK, int V>
__global__ void __launch_bounds__(NT) prj_max_kernel(const float* __restrict__ logits, int H, int W,
                                                     int rows_per_block,
                                                     unsigned long long* __restrict__ row_packed,
                                                     unsigned long long* __restrict__ col_packed) {
  constexpr int PANEL = NCHUNK * 32 * V;
  constexpr int NWARP = NT / 32;
  __shared__ unsigned long long s_col[NWARP][PANEL];
  const int n = blockIdx.y, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(r0 + rows_per_block, H);
  const int panel0 = blockIdx.z * PANEL;
  const float* img = logits + (int64_t)n * H * W;

  float cbest[NCHUNK * V];
  int cy[NCHUNK * V];
#pragma unroll
  for (int i = 0; i < NCHUNK * V; ++i) { cbest[i] = -INFINITY; cy[i] = -1; }

  for (int y = r0 + warp; y < r1; y += NWARP) {
    const float* row = img + (int64_t)y * W;
    float v[NCHUNK * V];
#pragma unroll
    for (int ch = 0; ch < NCHUNK; ++ch) {           // issue all loads of the row first
      const int col = panel0 + (ch * 32 + lane) * V;
      if constexpr (V == 4) {
        float4 q = col < W ? __ldg(reinterpret_cast<const float4*>(row + col)) : make_float4(0, 0, 0, 0);
        v[ch * 4 + 0] = q.x; v[ch * 4 + 1] = q.y; v[ch * 4 + 2] = q.z; v[ch * 4 + 3] = q.w;
      } else {
        v[ch] = col < W ? __ldg(row + col) : 0.f;
      }
    }
    float rbest = -INFINITY;
    int rx = -1;
#pragma unroll
    for (int ch = 0; ch < NCHUNK; ++ch) {
#pragma unroll
      for (int e = 0; e < V; ++e) {
        const int col = panel0 + (ch * 32 + lane) * V + e;
        if (col < W) {
          const float s = v[ch * V + e];
          if (s > rbest || rx < 0) { rbest = s; rx = col; }             // ascending cols: first wins
          if (s > cbest[ch * V + e] || cy[ch * V + e] < 0) { cbest[ch * V + e] = s; cy[ch * V + e] = y; }
        }
      }
    }
    unsigned long long rp = rx >= 0 ? pack_max(rbest, rx) : 0ull;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      unsigned long long other = __shfl_xor_sync(kFull, rp, o);
      rp = other > rp ? other : rp;
    }
    if (lane == 0 && rp) atomicMax(row_packed + (int64_t)n * H + y, rp);
  }
#pragma unroll
  for (int ch = 0; ch < NCHUNK; ++ch)
#pragma unroll
    for (int e = 0; e < V; ++e)
      s_col[warp][(ch * 32 + lane) * V + e] = cy[ch * V + e] >= 0 ? pack_max(cbest[ch * V + e], cy[ch * V + e]) : 0ull;
  __syncthreads();
  for (int c = threadIdx.x; c < PANEL; c += NT) {
    unsigned long long best = 0ull;
#pragma unroll
    for (int w = 0; w < NWARP; ++w) best = s_col[w][c] > best ? s_col[w][c] : best;
    if (best && panel0 + c < W) atomicMax(col_packed + (int64_t)n * W + panel0 + c, best);
  }
}

// ---------------------------------------------------------------------------------------
// shared-memory tile of (x, s, n, edge byte) with an asymmetric halo
// ---------------------------------------------------------------------------------------
struct PairTile {
  float *x, *s, *n;
  uint8_t* e;
  int pitch;
};

__device__ __forceinline__ PairTile load_pair_tile(const float* __restrict__ img, const uint8_t* __restrict__ bits,
                                                   int H, int W, int y_lo, int x_lo, int ph, int pw,
                                                   float* smem) {
  PairTile t{smem, smem + ph * pw, smem + 2 * ph * pw, reinterpret_cast<uint8_t*>(smem + 3 * ph * pw), pw};
  for (int i = threadIdx.x; i < ph * pw; i += NT) {
    int ly = i / pw, lx = i - ly * pw;
    int gy = y_lo + ly, gx = x_lo + lx;
    float v = 0.f, s = 0.f, n = 0.f;
    uint8_t e = 0;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      v = __ldg(img + (int64_t)gy * W + gx);
      e = __ldg(bits + (int64_t)gy * W + gx);
      sigmoid_pair(v, s, n);
    }
    t.x[i] = v; t.s[i] = s; t.n[i] = n; t.e[i] = e;
  }
  __syncthreads();
  return t;
}

// ---------------------------------------------------------------------------------------
// forward 2: pairwise numerators over the work list
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) pair_fwd_kernel(const float* __restrict__ logits,
                                                      const uint8_t* __restrict__ edge_bits,
                                                      const int32_t* __restrict__ rects,
                                                      const int32_t* __restrict__ inst_gt,
                                                      const int32_t* __restrict__ gt_img, int N, int H, int W,
                                                      int d, const int* __restrict__ tile_prefix,
                                                      float* __restrict__ pair_partial,
                                                      unsigned long long* __restrict__ weight_sum) {
  extern __shared__ float smem[];
  __shared__ float s_red[NT / 32];
  __shared__ int s_redi[NT / 32];
  const int total = tile_prefix[N];
  const int ph = TH + d, pw = TW + 2 * d;
  for (int item = blockIdx.x; item < total; item += gridDim.x) {
    int lo = 0, hi = N;                       // largest n with tile_prefix[n] <= item
    while (hi - lo > 1) {
      int mid = (lo + hi) >> 1;
      if (tile_prefix[mid] <= item) lo = mid; else hi = mid;
    }
    const int n = lo;
    const int g = inst_gt[n];
    const Rect r = load_rect(rects, g);
    int ty0, ty1, tx0, tx1;
    fwd_tile_range(r, d, H, W, ty0, ty1, tx0, tx1);
    const int local = item - tile_prefix[n];
    const int ntx = tx1 - tx0 + 1;
    const int y0 = (ty0 + local / ntx) * TH, x0 = (tx0 + local % ntx) * TW;
    const float* img = logits + (int64_t)n * H * W;
    const uint8_t* bits = edge_bits + (int64_t)gt_img[g] * H * W;
    __syncthreads();                          // previous item's readers are done with smem
    PairTile t = load_pair_tile(img, bits, H, W, y0, x0 - d, ph, pw, smem);

    float acc = 0.f;
    int wsum = 0;
    const int tx = threadIdx.x % TW;
    const int gx = x0 + tx;
    for (int ty = threadIdx.x / TW; ty < TH; ty += NT / TW) {
      const int gy = y0 + ty;
      if (gy >= H || gx >= W) continue;
      const int ci = ty * t.pitch + tx + d;
      const bool pin = in_rect(r, gy, gx);
      const unsigned ep = t.e[ci];
      if (pin) wsum += __popc(ep);
      const float xa = t.x[ci], sa = t.s[ci], na = t.n[ci];
      // forward half of the neighbourhood: c = 4..7 <-> (0,+d), (+d,-d), (+d,0), (+d,+d)
#pragma unroll
      for (int c = 4; c < 8; ++c) {
        const int dy = c == 4 ? 0 : d;
        const int dx = c == 4 ? d : (c - 6) * d;
        const int qy = gy + dy, qx = gx + dx;
        if (qy >= H || qx < 0 || qx >= W) continue;
        const int qi = ci + (c == 4 ? 0 : d * t.pitch) + dx;
        const unsigned eq = t.e[qi];
        const int m = (pin ? (ep >> c) & 1u : 0u) + (in_rect(r, qy, qx) ? (eq >> (7 - c)) & 1u : 0u);
        if (m) {
          const float xb = t.x[qi];
          float pl;
          if (fmaxf(fabsf(xa), fabsf(xb)) <= kFastLimit)
            pl = -__logf(sa * t.s[qi] + na * t.n[qi]);
          else
            pl = pair_nlog_logspace<float>(xa, xb, true);
          acc = fmaf((float)m, pl, acc);
        }
      }
    }
    const float tot = block_sum<float>(acc, s_red);
    const int wtot = block_sum<int>(wsum, s_redi);
    if (threadIdx.x == 0) {
      pair_partial[item] = tot;
      if (wtot) atomicAdd(weight_sum, (unsigned long long)wtot);
    }
  }
}

// ---------------------------------------------------------------------------------------
// finalize: dice terms, gradient coefficients, scalars.  Executed by ONE CTA per instance (a
// dedicated kernel on the generic path; the last CTA of the instance on the fast path); the CTA
// that finalizes the last instance (global ticket) writes the scalars.
// ---------------------------------------------------------------------------------------
struct FinalizeShared {
  float red[NT / 32];
  int redi[NT / 32];
  float bc[2];
  bool last;
};


__device__ void finalize_instance(const int n, const Rect r, const int N, const int H, const int W, const Workspace& ws,
                                  const float* __restrict__ partial, const int npartial,
                                  const int* __restrict__ den_partial, const int nden,
                                  const float* __restrict__ iter_ptr, const float warmup_iters,
                                  float* __restrict__ losses_out, FinalizeShared& sh) {
  const bool empty = rect_empty(r);
  const float inv_n = 1.f / (float)N;
  float inst_loss = 0.f;
  // axis 0: row profile (max over x) of length H;  axis 1: column profile of length W
  for (int axis = 0; axis < 2; ++axis) {
    const int L = axis == 0 ? H : W;
    const int lo = axis == 0 ? r.j0 : r.i0, hi = axis == 0 ? r.j1 : r.i1;
    const unsigned long long* packed = (axis == 0 ? ws.row_packed + (int64_t)n * H : ws.col_packed + (int64_t)n * W);
    float* coef = axis == 0 ? ws.coef_row + (int64_t)n * H : ws.coef_col + (int64_t)n * W;
    int* arg = axis == 0 ? ws.row_arg + (int64_t)n * H : ws.col_arg + (int64_t)n * W;
    float inter = 0.f, x2 = 0.f;
    for (int i = threadIdx.x; i < L; i += NT) {
      const float s = sigmoid_exact(fkey_inv((unsigned)(__ldcg(packed + i) >> 32)));
      const bool t = !empty && i >= lo && i <= hi;
      inter += t ? s : 0.f;
      x2 = fmaf(s, s, x2);
    }
    inter = block_sum<float>(inter, sh.red);
    x2 = block_sum<float>(x2, sh.red);
    if (threadIdx.x == 0) {
      const float t2 = empty ? 0.f : (float)(max(min(hi, L - 1) - max(lo, 0) + 1, 0));
      const float u = x2 + t2 + kDiceEps;
      sh.bc[0] = inter; sh.bc[1] = u;
      inst_loss += 1.f - 2.f * inter / u;
    }
    __syncthreads();
    const float I = sh.bc[0], U = sh.bc[1];
    for (int i = threadIdx.x; i < L; i += NT) {
      const unsigned long long p = __ldcg(packed + i);
      const float s = sigmoid_exact(fkey_inv((unsigned)(p >> 32)));
      const float t = (!empty && i >= lo && i <= hi) ? 1.f : 0.f;
      // d dice / d s = -2 t / U + 4 I s / U^2 ; through the sigmoid: * s (1 - s); mean over N
      coef[i] = inv_n * (-2.f * t / U + 4.f * I * s / (U * U)) * s * (1.f - s);
      arg[i] = (int)(0xffffffffu - (unsigned)(p & 0xffffffffull));
    }
    __syncthreads();
  }
  // pairwise numerator / weight count of this instance: fixed-order sums of its partials
  float num = 0.f;
  for (int i = threadIdx.x; i < npartial; i += NT) num += __ldcg(partial + i);
  num = block_sum<float>(num, sh.red);
  int den = 0;
  for (int i = threadIdx.x; i < nden; i += NT) den += __ldcg(den_partial + i);
  den = block_sum<int>(den, sh.redi);
  if (threadIdx.x == 0) {
    ws.inst_prj[n] = inst_loss;
    ws.inst_num[n] = num;
    if (den) atomicAdd(ws.weight_sum, (unsigned long long)den);
    __threadfence();
    sh.last = atomicAdd(ws.ticket, 1u) == (unsigned)(N - 1);
  }
  __syncthreads();
  if (!sh.last) return;
  __threadfence();
  float prj = 0.f, pn = 0.f;
  for (int i = threadIdx.x; i < N; i += NT) { prj += __ldcg(ws.inst_prj + i); pn += __ldcg(ws.inst_num + i); }
  prj = block_sum<float>(prj, sh.red);
  pn = block_sum<float>(pn, sh.red);
  if (threadIdx.x == 0) {
    const float wsum = (float)__ldcg(ws.weight_sum);
    const float warm = fminf(iter_ptr[0] / warmup_iters, 1.f);
    const float scale = warm / fmaxf(wsum, 1.f);
    losses_out[0] = prj * inv_n;
    losses_out[1] = pn * scale;
    losses_out[2] = pn;
    losses_out[3] = wsum;
    ws.scale_pair[0] = scale;
  }
}

__global__ void __launch_bounds__(NT) finalize_kernel(const int32_t* __restrict__ rects,
                                                      const int32_t* __restrict__ inst_gt, int N, int H, int W,
                                                      Workspace ws, const float* __restrict__ iter_ptr,
                                                      float warmup_iters, float* __restrict__ losses_out) {
  __shared__ FinalizeShared sh;
  const int n = blockIdx.x;
  const int p0 = ws.tile_prefix[n], p1 = ws.tile_prefix[n + 1];
  finalize_instance(n, load_rect(rects, inst_gt[n]), N, H, W, ws, ws.pair_partial + p0, p1 - p0, nullptr, 0,
                    iter_ptr, warmup_iters, losses_out, sh);
}

// =========================================================================================
// FAST PATH (W % 4 == 0, 16-byte aligned, W <= 512, dilation <= 4): no shared-memory tiles, no
// work list.  One warp owns a full row; a lane owns NCHUNK groups of 4 consecutive pixels.
// =========================================================================================
constexpr int RPW = 2;                      // rows per warp, all in flight before any use
constexpr int PASSES = 2;                   // streaming CTAs repeat: the cross-warp column reduction is paid once per CTA
constexpr int ROWS_PER_CTA = PASSES * RPW * (NT / 32);

// ---- pair terms, lane-per-pixel: a warp walks the box columns [c_lo, c_hi] of one row in segments of
// 32 lanes of which the inner 32-2D "own" a pixel; horizontal neighbours come from warp shuffles, the
// row below is a second (L1-resident) load.  Out-of-image / out-of-box neighbours need no test at all:
// their effective weight bits are zero by construction.
__device__ __forceinline__ float pair_value(bool extreme, float xa, float sa, float na, float xb, float sb, float nb) {
  if (!extreme) return -__logf(sa * sb + na * nb);
  return pair_nlog_logspace<float>(xa, xb, true);
}
__device__ __forceinline__ float pair_grad_a(bool extreme, float xa, float sa, float na, float xb, float sb, float nb) {
  if (!extreme) return -(sb - nb) * __frcp_rn(sa * sb + na * nb) * (sa * na);
  return pair_nlog_grad_a_logspace<float>(xa, xb, true, pair_nlog_logspace<float>(xa, xb, true));
}

struct RowSeg {            // one lane's pixel of a row segment
  float x, s, n;
  unsigned eff;            // edge bits masked by "pixel lies in the box"
  unsigned raw;            // unmasked edge bits
};

// raw (x, bits) of one lane's pixel: issued one row ahead of its use so that the load latency hides behind
// the pair arithmetic of the previous row
struct RawSeg { float x; unsigned raw; };
__device__ __forceinline__ RawSeg load_raw(const float* __restrict__ img, const uint8_t* __restrict__ bits, int H, int W,
                                           int y, int x, bool x_ok) {
  RawSeg v;
  const bool in = x_ok && y >= 0 && y < H;
  const int64_t o = (int64_t)y * W + x;
  v.x = in ? __ldg(img + o) : 0.f;
  v.raw = in ? (unsigned)__ldg(bits + o) : 0u;
  return v;
}
__device__ __forceinline__ RowSeg finish_seg(const RawSeg& w, int y, bool x_box, const Rect& r) {
  RowSeg v;
  v.x = w.x;
  v.raw = w.raw;
  v.eff = (x_box && y >= r.j0 && y <= r.j1) ? w.raw : 0u;
  sigmoid_pair(v.x, v.s, v.n);
  return v;
}

// The pair role walks CHAINS: rows y0, y0 + D, y0 + 2D, ... of one 32-lane column segment.  The row "below"
// (y + D) of one step is the row "at" of the next, so every row of the chain is loaded and sigmoid-ed once,
// and each unordered pair {p, q} is evaluated once (neighbours c = 4..7: right, below-left, below, below-right)
// with multiplicity m = [edge bit of p towards q, p in box] + [edge bit of q towards p, q in box].
template <int D>
struct Neigh { float x, s, n; unsigned e; };

template <int D, int C>
__device__ __forceinline__ Neigh<D> neighbour(const RowSeg& cur, const RowSeg& nxt, bool extreme, int lane, bool& valid) {
  Neigh<D> q;
  if (C == 4) {
    q.s = __shfl_down_sync(kFull, cur.s, D); q.n = __shfl_down_sync(kFull, cur.n, D); q.e = __shfl_down_sync(kFull, cur.eff, D);
    q.x = extreme ? __shfl_down_sync(kFull, cur.x, D) : 0.f;
    valid = lane + D < 32;
  } else if (C == 5) {
    q.s = __shfl_up_sync(kFull, nxt.s, D); q.n = __shfl_up_sync(kFull, nxt.n, D); q.e = __shfl_up_sync(kFull, nxt.eff, D);
    q.x = extreme ? __shfl_up_sync(kFull, nxt.x, D) : 0.f;
    valid = lane >= D;
  } else if (C == 6) {
    q.s = nxt.s; q.n = nxt.n; q.e = nxt.eff; q.x = nxt.x;
    valid = true;
  } else {
    q.s = __shfl_down_sync(kFull, nxt.s, D); q.n = __shfl_down_sync(kFull, nxt.n, D); q.e = __shfl_down_sync(kFull, nxt.eff, D);
    q.x = extreme ? __shfl_down_sync(kFull, nxt.x, D) : 0.f;
    valid = lane + D < 32;
  }
  return q;
}

// forward: sum of m * pair_value over the chain's owner pixels; wsum = weight count of the owner pixels
template <int D>
__device__ __forceinline__ void pair_chain_fwd(const float* __restrict__ img, const uint8_t* __restrict__ bits, int H, int W,
                                               int y0, int nrows, int xs, int c_hi, const Rect& r, int lane, float& acc,
                                               int& wsum) {
  const int x = xs + lane;
  const bool x_ok = x >= 0 && x < W, x_box = x >= r.i0 && x <= r.i1;
  const bool owner = lane >= D && lane < 32 - D && x <= c_hi;
  RowSeg a = finish_seg(load_raw(img, bits, H, W, y0, x, x_ok), y0, x_box, r);
  RawSeg ahead = load_raw(img, bits, H, W, y0 + D, x, x_ok);
  for (int k = 0; k < nrows; ++k) {
    const int y = y0 + k * D;
    const RowSeg b = finish_seg(ahead, y + D, x_box, r);
    if (k + 1 < nrows) ahead = load_raw(img, bits, H, W, y + 2 * D, x, x_ok);
    const bool extreme = __any_sync(kFull, fmaxf(fabsf(a.x), fabsf(b.x)) > kFastLimit);
    if (owner) wsum += __popc(a.eff);
    float row = 0.f;
#define BXS_FWD_PAIR(C)                                                                         \
    {                                                                                           \
      bool valid;                                                                               \
      const Neigh<D> q = neighbour<D, C>(a, b, extreme, lane, valid);                           \
      const unsigned m = ((a.eff >> C) & 1u) + ((q.e >> (7 - C)) & 1u);                         \
      const float pv = pair_value(extreme, a.x, a.s, a.n, q.x, q.s, q.n);                       \
      row = fmaf((float)m, pv, row);                                                            \
    }
    BXS_FWD_PAIR(4) BXS_FWD_PAIR(5) BXS_FWD_PAIR(6) BXS_FWD_PAIR(7)
#undef BXS_FWD_PAIR
    if (owner) acc += row;
    a = b;
  }
}

// backward: gradient rows of the chain.  Each unordered pair yields the gradient of both of its pixels: the
// one of the left/upper pixel stays in the lane, the one of the right/lower pixel travels by one shuffle
// (same row) or through `carry` (row below -> next step).  The step before the chain (row y0 - D) only feeds
// the carry.  Also adds the projection arg-max terms and stores the row.
template <int D>
__device__ __forceinline__ void pair_chain_bwd(const float* __restrict__ img, const uint8_t* __restrict__ bits, int H, int W,
                                               int y0, int nrows, int xs, int c_hi, const Rect& r, int lane, float g_pair,
                                               const int* __restrict__ row_arg, const float* __restrict__ coef_row,
                                               const int* __restrict__ acol, const float* __restrict__ ccol, float g_prj,
                                               float* __restrict__ ginst) {
  const int x = xs + lane;
  const bool x_ok = x >= 0 && x < W, x_box = x >= r.i0 && x <= r.i1;
  const bool owner = lane >= D && lane < 32 - D && x <= c_hi;
  const int acx = owner ? acol[x] : -1;
  const float ccx = owner ? ccol[x] * g_prj : 0.f;
  RowSeg cur = finish_seg(load_raw(img, bits, H, W, y0 - D, x, x_ok), y0 - D, x_box, r);
  RawSeg ahead = load_raw(img, bits, H, W, y0, x, x_ok);
  float carry = 0.f;
  for (int k = -1; k < nrows; ++k) {
    const int y = y0 + k * D;
    const RowSeg nxt = finish_seg(ahead, y + D, x_box, r);
    if (k + 1 < nrows) ahead = load_raw(img, bits, H, W, y + 2 * D, x, x_ok);
    const bool extreme = __any_sync(kFull, fmaxf(fabsf(cur.x), fabsf(nxt.x)) > kFastLimit);
    float acc = carry;
    carry = 0.f;
    const float sn_a = cur.s * cur.n, df_a = cur.s - cur.n;
#define BXS_BWD_PAIR(C, GA, GQ)                                                                 \
    float GA, GQ;                                                                               \
    {                                                                                           \
      bool valid;                                                                               \
      const Neigh<D> q = neighbour<D, C>(cur, nxt, extreme, lane, valid);                       \
      const unsigned m = valid ? ((cur.eff >> C) & 1u) + ((q.e >> (7 - C)) & 1u) : 0u;          \
      if (!extreme) {                                                                           \
        const float t = (float)m * rcp_approx(fmaf(cur.s, q.s, cur.n * q.n));                   \
        GA = -(q.s - q.n) * t * sn_a;                                                           \
        GQ = -df_a * t * (q.s * q.n);                                                           \
      } else {                                                                                  \
        GA = (float)m * pair_grad_a(true, cur.x, cur.s, cur.n, q.x, q.s, q.n);                  \
        GQ = (float)m * pair_grad_a(true, q.x, q.s, q.n, cur.x, cur.s, cur.n);                  \
      }                                                                                         \
    }
    if (k >= 0) {                                              // warp-uniform
      BXS_BWD_PAIR(4, ga4, gq4)
      const float from_left = __shfl_up_sync(kFull, gq4, D);  // pair (x - D, x): this lane is the right pixel
      acc += ga4 + (lane >= D ? from_left : 0.f);
    }
    BXS_BWD_PAIR(5, ga5, gq5)
    BXS_BWD_PAIR(6, ga6, gq6)
    BXS_BWD_PAIR(7, ga7, gq7)
#undef BXS_BWD_PAIR
    {
      const float to_left = __shfl_down_sync(kFull, gq5, D);  // lower-left pixel of lane + D is this lane's column
      const float to_right = __shfl_up_sync(kFull, gq7, D);
      carry = gq6 + (lane + D < 32 ? to_left : 0.f) + (lane >= D ? to_right : 0.f);
    }
    if (k >= 0) {
      acc += ga5 + ga6 + ga7;
      if (owner) {
        float v = 0.f;
        if (x == row_arg[y]) v += coef_row[y] * g_prj;
        if (acx == y) v += ccx;
        ginst[(int64_t)y * W + x] = fmaf(acc, g_pair, v);
      }
    }
    cur = nxt;
  }
}

// Both fast-path kernels use a HETEROGENEOUS grid, blockIdx.x = instance, blockIdx.y = role:
//   y <  PAIR_BLOCKS : pair role      -- the (row, 28-pixel segment) items of the box span, round-robin over
//                                        PAIR_BLOCKS * 8 warps (scheduled first: they are the long, latency-bound CTAs)
//   y >= PAIR_BLOCKS : streaming role -- 16 rows of the map (2 per warp), full width
// The two roles touch disjoint outputs and overlap on the SMs (one is load/store bound, the other ALU/latency bound).
constexpr int PAIR_BLOCKS = 16;
constexpr int PAIR_PARTS = PAIR_BLOCKS * 8;   // numerator / weight-count partials per instance (one per pair-role warp)

struct Span { int y_lo, y_hi, c_lo, c_hi, nseg; };
template <int D>
__device__ __forceinline__ Span pair_span(const Rect& r, int H, int W, bool backward) {
  Span s;
  if (rect_empty(r)) { s.y_lo = 0; s.y_hi = -1; s.c_lo = 0; s.c_hi = -1; s.nseg = 0; return s; }
  s.y_lo = max(r.j0 - D, 0);
  s.y_hi = backward ? min(r.j1 + D, H - 1) : min(r.j1, H - 1);
  s.c_lo = max(r.i0 - D, 0);
  s.c_hi = min(r.i1 + D, W - 1);
  s.nseg = (s.c_hi - s.c_lo + 1 + (32 - 2 * D) - 1) / (32 - 2 * D);
  return s;
}

__device__ __forceinline__ int div_small(int a, int b) {
  return __float2int_rz((__int2float_rn(a) + 0.5f) * rcp_approx(__int2float_rn(b)));
}

// Per-instance record written by prep_fast_kernel (one 64-byte line): everything a CTA of either role needs to
// know about its instance, so that its prologue is ONE load instead of the inst_gt -> rects -> gt_img chain plus
// a dozen integer divisions per warp.
struct InstRec {
  Rect r;                          // box rectangle on the loss grid
  int img, nseg, c_lo, c_hi;       // image index; column span [c_lo, c_hi] in nseg segments of 32 - 2D owner lanes
  int y_lo, y_hi_f, y_hi_b, len_f; // row span (forward ends at j1, backward at j1 + D); chain piece lengths
  int pc_f, len_b, pc_b, pad;      // pieces per parity class
};
__device__ __forceinline__ InstRec load_rec(const int* __restrict__ recs, int n) {
  const int4* q = reinterpret_cast<const int4*>(recs + 16 * (int64_t)n);
  const int4 a = __ldg(q), b = __ldg(q + 1), c = __ldg(q + 2), d = __ldg(q + 3);
  InstRec v;
  v.r = Rect{a.x, a.y, a.z, a.w};
  v.img = b.x; v.nseg = b.y; v.c_lo = b.z; v.c_hi = b.w;
  v.y_lo = c.x; v.y_hi_f = c.y; v.y_hi_b = c.z; v.len_f = c.w;
  v.pc_f = d.x; v.len_b = d.y; v.pc_b = d.z; v.pad = 0;
  return v;
}
__device__ __forceinline__ Span span_of(const InstRec& v, bool backward) {
  return Span{v.y_lo, backward ? v.y_hi_b : v.y_hi_f, v.c_lo, v.c_hi, v.nseg};
}

// Chain split of one span: class p = row parity mod D, pieces of `len` chain rows, nseg column segments; at most
// one chain per pair-role warp: len is the smallest piece length (>= 4) for which D * pc * nseg <= PAIR_PARTS.
template <int D>
__device__ __forceinline__ void chain_split(int rows, int nseg, int& len, int& pc) {
  len = 4; pc = 0;
  if (nseg <= 0 || rows <= 0) return;
  const int RC = (rows + D - 1) / D;                     // chain rows of the longest class
  const int pc_max = PAIR_PARTS / (D * nseg);            // >= 1: D * nseg <= 88
  len = max((RC + pc_max - 1) / pc_max, 4);
  pc = (RC + len - 1) / len;
}

// zeroes the accumulators of a forward pass and writes the instance records (replaces the memset node)
template <int D>
__global__ void __launch_bounds__(128) prep_fast_kernel(const int32_t* __restrict__ rects, const int32_t* __restrict__ inst_gt,
                                                        const int32_t* __restrict__ gt_img, int H, int W, Workspace ws) {
  const int n = blockIdx.x;
  for (int c = threadIdx.x; c < W; c += 128) ws.col_packed[(int64_t)n * W + c] = 0ull;
  if (threadIdx.x < PAIR_PARTS) {
    ws.pair_partial[(int64_t)n * PAIR_PARTS + threadIdx.x] = 0.f;
    ws.den_partial[(int64_t)n * PAIR_PARTS + threadIdx.x] = 0;
  }
  if (threadIdx.x != 0) return;
  if (n == 0) { *ws.weight_sum = 0ull; *ws.ticket = 0u; }
  const int g = inst_gt[n];
  const Rect r = load_rect(rects, g);
  const Span f = pair_span<D>(r, H, W, false), b = pair_span<D>(r, H, W, true);
  int len_f, pc_f, len_b, pc_b;
  chain_split<D>(f.y_hi - f.y_lo + 1, f.nseg, len_f, pc_f);
  chain_split<D>(b.y_hi - b.y_lo + 1, b.nseg, len_b, pc_b);
  int4* q = reinterpret_cast<int4*>(ws.inst_rec + 16 * (int64_t)n);
  q[0] = make_int4(r.j0, r.j1, r.i0, r.i1);
  q[1] = make_int4(gt_img[g], f.nseg, f.c_lo, f.c_hi);
  q[2] = make_int4(f.y_lo, f.y_hi, b.y_hi, len_f);
  q[3] = make_int4(pc_f, len_b, pc_b, 0);
}

// chain of pair-role warp gw in [0, PAIR_PARTS).  The two divisions run on MUFU.RCP: for operands < 2^20,
// floor((a + 0.5) / b) in fp32 is exact (error q * 2^-22 < 0.5 / b).
struct Chain { int seg, y0, nrows; };
template <int D>
__device__ __forceinline__ Chain chain_of(const Span& sp, int len, int pc, int gw) {
  Chain c;
  c.seg = 0; c.y0 = 0; c.nrows = 0;
  if (pc <= 0) return c;
  const int u = div_small(gw, sp.nseg);
  const int p = div_small(u, pc), piece = u - p * pc;
  if (p >= D) return c;
  const int R = sp.y_hi - sp.y_lo + 1;
  const int Rp = (R - p + D - 1) / D;                    // chain rows of class p
  const int k0 = piece * len;
  if (k0 >= Rp) return c;
  c.seg = gw - u * sp.nseg;
  c.y0 = sp.y_lo + p + D * k0;
  c.nrows = min(len, Rp - k0);
  return c;
}

template <int NCHUNK, int D>
__global__ void __launch_bounds__(NT, 4) fwd_fused_kernel(const float* __restrict__ logits,
                                                       const uint8_t* __restrict__ edge_bits,
                                                       const int32_t* __restrict__ rects,
                                                       const int32_t* __restrict__ inst_gt,
                                                       const int32_t* __restrict__ gt_img, int H, int W, Workspace ws) {
  constexpr int PANEL = NCHUNK * 128, NWARP = NT / 32;
  __shared__ float s_val[NWARP][PANEL];
  __shared__ int s_row[NWARP][PANEL];
  const int n = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int role = blockIdx.y;
  const float* img = logits + (int64_t)n * H * W;

  if (role >= PAIR_BLOCKS) {
    // ================= streaming role: row / column maxima =================
    const int ybase = (role - PAIR_BLOCKS) * ROWS_PER_CTA + warp;     // this warp's rows: ybase + k * NWARP
    float cv[NCHUNK * 4];                                   // running column maxima of this lane's columns
    int cy[NCHUNK * 4];
#pragma unroll
    for (int i = 0; i < NCHUNK * 4; ++i) { cv[i] = -INFINITY; cy[i] = H; }
#pragma unroll
    for (int ps = 0; ps < PASSES; ++ps) {
      const int yp = ybase + ps * RPW * NWARP;
      float v[RPW][NCHUNK * 4];
#pragma unroll
      for (int k = 0; k < RPW; ++k) {                       // all loads first (memory-level parallelism)
        const int y = yp + k * NWARP;
#pragma unroll
        for (int ch = 0; ch < NCHUNK; ++ch) {
          const int col0 = (ch * 32 + lane) * 4;
          float4 q = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
          if (col0 < W && y < H) q = __ldg(reinterpret_cast<const float4*>(img + (int64_t)y * W + col0));
          v[k][ch * 4] = q.x; v[k][ch * 4 + 1] = q.y; v[k][ch * 4 + 2] = q.z; v[k][ch * 4 + 3] = q.w;
        }
      }
#pragma unroll
      for (int k = 0; k < RPW; ++k) {                       // row maxima: integer redux on the order-preserving key
        const int y = yp + k * NWARP;
        if (y < H) {                                        // warp-uniform
          float m = v[k][0];
#pragma unroll
          for (int i = 1; i < NCHUNK * 4; ++i) m = fmaxf(m, v[k][i]);
          const unsigned kmax = __reduce_max_sync(kFull, fkey(m));
          const float mv = fkey_inv(kmax);
          int cand = 0x7fffffff;
#pragma unroll
          for (int i = NCHUNK * 4 - 1; i >= 0; --i)
            if (v[k][i] == mv) cand = ((i >> 2) * 32 + lane) * 4 + (i & 3);
          const int amin = __reduce_min_sync(kFull, cand);
          if (lane == 0) ws.row_packed[(int64_t)n * H + y] = pack_key(kmax, amin == 0x7fffffff ? 0 : amin);
        }
      }
#pragma unroll
      for (int i = 0; i < NCHUNK * 4; ++i) {                // column maxima (strict '>': the earlier row wins ties;
#pragma unroll
        for (int k = 0; k < RPW; ++k)                       //  rows >= H hold -inf and never win)
          if (v[k][i] > cv[i]) { cv[i] = v[k][i]; cy[i] = yp + k * NWARP; }
      }
    }
#pragma unroll
    for (int i = 0; i < NCHUNK * 4; ++i) {
      const int col = ((i >> 2) * 32 + lane) * 4 + (i & 3);
      s_val[warp][col] = cv[i];
      s_row[warp][col] = cy[i];
    }
    __syncthreads();
    for (int c = threadIdx.x; c < PANEL; c += NT) {
      float best = s_val[0][c];
      int brow = s_row[0][c];
#pragma unroll
      for (int w = 1; w < NWARP; ++w) {
        const float val = s_val[w][c];
        const int row = s_row[w][c];
        if (val > best || (val == best && row < brow)) { best = val; brow = row; }
      }
      if (c < W && brow < H) atomicMax(ws.col_packed + (int64_t)n * W + c, pack_key(fkey(best), brow));
    }
  } else {
    // ================= pair role: (row, segment) items of the box span =================
    const InstRec rec = load_rec(ws.inst_rec, n);
    if (role * NWARP >= D * rec.pc_f * rec.nseg) return;    // no chain for any warp of this CTA (partials pre-zeroed)
    const Rect r = rec.r;
    const uint8_t* bits = edge_bits + (int64_t)rec.img * H * W;
    const Span sp = span_of(rec, false);
    // one chain (rows of one parity class, one column segment) per warp; per-lane accumulation, one shuffle
    // tree and one store at the end: PAIR_PARTS partials per instance, summed in fixed order by the finalize
    const int gw = role * NWARP + warp;
    const Chain ch = chain_of<D>(sp, rec.len_f, rec.pc_f, gw);
    float acc = 0.f;
    int wsum = 0;
    if (ch.nrows > 0)
      pair_chain_fwd<D>(img, bits, H, W, ch.y0, ch.nrows, sp.c_lo - D + ch.seg * (32 - 2 * D), sp.c_hi, r, lane, acc, wsum);
    acc = warp_sum(acc);
    wsum = warp_sum(wsum);
    if (lane == 0) {
      ws.pair_partial[(int64_t)n * PAIR_PARTS + gw] = acc;
      ws.den_partial[(int64_t)n * PAIR_PARTS + gw] = wsum;
    }
  }
}

// Finalize (separate launch: no fences / tickets in the streaming kernel).  Each instance gets a group of four
// warps whose reductions are independent and use warp shuffles only:
//   warp 0: row profile -> dice + row coefficients     warp 1: column profile -> dice + column coefficients
//   warp 2: pairwise numerator (fixed order)           warp 3: weight count
// A CTA holds FIN_GROUPS instances so that only N / FIN_GROUPS CTAs touch the two same-address atomics
// (weight sum, ticket) -- 128 serialised L2 atomics cost more than the arithmetic.
constexpr int FIN_GROUPS = 4;

template <int D>
__global__ void __launch_bounds__(FIN_GROUPS * 128) finalize_fast_kernel(const int32_t* __restrict__ rects,
                                                                         const int32_t* __restrict__ inst_gt, int N, int H,
                                                                         int W, Workspace ws,
                                                                         const float* __restrict__ iter_ptr,
                                                                         float warmup_iters, float* __restrict__ losses_out) {
  __shared__ float s_part[FIN_GROUPS][4];
  __shared__ int s_den[FIN_GROUPS];
  __shared__ bool s_last;
  const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3, group = threadIdx.x >> 7;
  const int n = blockIdx.x * FIN_GROUPS + group;
  const float inv_n = 1.f / (float)N;
  if (n < N) {
    const Rect r = load_rec(ws.inst_rec, n).r;
    const bool empty = rect_empty(r);
    if (warp < 2) {
      const int axis = warp;
      const int L = axis == 0 ? H : W;
      const int lo = axis == 0 ? r.j0 : r.i0, hi = axis == 0 ? r.j1 : r.i1;
      const unsigned long long* packed = (axis == 0 ? ws.row_packed + (int64_t)n * H : ws.col_packed + (int64_t)n * W);
      float* coef = axis == 0 ? ws.coef_row + (int64_t)n * H : ws.coef_col + (int64_t)n * W;
      int* arg = axis == 0 ? ws.row_arg + (int64_t)n * H : ws.col_arg + (int64_t)n * W;
      // the whole profile (L <= 512) sits in registers: all loads issue back to back, one latency round trip
      constexpr int PER_LANE = 16;
      unsigned long long pk[PER_LANE];
#pragma unroll
      for (int k = 0; k < PER_LANE; ++k) pk[k] = (k * 32 + lane < L) ? packed[k * 32 + lane] : 0ull;
      float sv[PER_LANE];
      float inter = 0.f, x2 = 0.f;
#pragma unroll
      for (int k = 0; k < PER_LANE; ++k) {
        const int i = k * 32 + lane;
        sv[k] = i < L ? sigmoid_exact(fkey_inv((unsigned)(pk[k] >> 32))) : 0.f;
        inter += (!empty && i >= lo && i <= hi) ? sv[k] : 0.f;
        x2 = fmaf(sv[k], sv[k], x2);
      }
      inter = warp_sum(inter);
      x2 = warp_sum(x2);
      const float t2 = empty ? 0.f : (float)(max(min(hi, L - 1) - max(lo, 0) + 1, 0));
      const float U = x2 + t2 + kDiceEps, I = inter;
#pragma unroll
      for (int k = 0; k < PER_LANE; ++k) {
        const int i = k * 32 + lane;
        if (i < L) {
          const float t = (!empty && i >= lo && i <= hi) ? 1.f : 0.f;
          coef[i] = inv_n * (-2.f * t / U + 4.f * I * sv[k] / (U * U)) * sv[k] * (1.f - sv[k]);
          arg[i] = (int)(0xffffffffu - (unsigned)(pk[k] & 0xffffffffull));
        }
      }
      if (lane == 0) s_part[group][axis] = 1.f - 2.f * I / U;
    } else {
      if (warp == 2) {
        float num = 0.f;
#pragma unroll
        for (int i = 0; i < PAIR_PARTS / 32; ++i) num += ws.pair_partial[(int64_t)n * PAIR_PARTS + i * 32 + lane];
        num = warp_sum(num);
        if (lane == 0) s_part[group][2] = num;
      } else {
        int den = 0;
#pragma unroll
        for (int i = 0; i < PAIR_PARTS / 32; ++i) den += ws.den_partial[(int64_t)n * PAIR_PARTS + i * 32 + lane];
        den = warp_sum(den);
        if (lane == 0) s_den[group] = den;
      }
    }
  } else if (lane == 0) {
    if (warp == 3) s_den[group] = 0;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int den = 0;
    for (int gq = 0; gq < FIN_GROUPS; ++gq) {
      const int m = blockIdx.x * FIN_GROUPS + gq;
      if (m < N) { ws.inst_prj[m] = s_part[gq][0] + s_part[gq][1]; ws.inst_num[m] = s_part[gq][2]; den += s_den[gq]; }
    }
    if (den) atomicAdd(ws.weight_sum, (unsigned long long)den);
    __threadfence();
    s_last = atomicAdd(ws.ticket, 1u) == gridDim.x - 1;
  }
  __syncthreads();
  if (!s_last || threadIdx.x >= 32) return;
  __threadfence();
  float prj = 0.f, pn = 0.f;
  for (int i = lane; i < N; i += 32) { prj += __ldcg(ws.inst_prj + i); pn += __ldcg(ws.inst_num + i); }
  prj = warp_sum(prj);
  pn = warp_sum(pn);
  if (lane == 0) {
    const float wsum = (float)__ldcg(ws.weight_sum);
    const float warm = fminf(iter_ptr[0] / warmup_iters, 1.f);
    const float scale = warm / fmaxf(wsum, 1.f);
    losses_out[0] = prj * inv_n;
    losses_out[1] = pn * scale;
    losses_out[2] = pn;
    losses_out[3] = wsum;
    ws.scale_pair[0] = scale;
  }
}

template <int NCHUNK, int D>
__global__ void __launch_bounds__(NT, 4) bwd_rows_kernel(const float* __restrict__ logits,
                                                      const uint8_t* __restrict__ edge_bits,
                                                      const int32_t* __restrict__ rects,
                                                      const int32_t* __restrict__ inst_gt,
                                                      const int32_t* __restrict__ gt_img, int H, int W, Workspace ws,
                                                      const float* __restrict__ g_losses,
                                                      float* __restrict__ g_logits) {
  constexpr int NWARP = NT / 32;
  const int n = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int role = blockIdx.y;
  const InstRec rec = load_rec(ws.inst_rec, n);
  if (role < PAIR_BLOCKS && role * NWARP >= D * rec.pc_b * rec.nseg) return;   // pair CTA without a chain
  const Rect r = rec.r;
  const float g_prj = g_losses[0];
  const float* ccol = ws.coef_col + (int64_t)n * W;
  const int* acol = ws.col_arg + (int64_t)n * W;
  const Span sp = span_of(rec, true);                     // pixels that can receive a pairwise gradient

  if (role >= PAIR_BLOCKS) {
    // ================= streaming role: zeros + projection arg-max terms outside the box span =================
    const int y0 = (role - PAIR_BLOCKS) * ROWS_PER_CTA + warp;
    int4 ac[NCHUNK];                                        // loop invariant: column arg-max rows of this lane's chunks
#pragma unroll
    for (int ch = 0; ch < NCHUNK; ++ch) {
      const int col0 = (ch * 32 + lane) * 4;
      ac[ch] = col0 < W ? __ldg(reinterpret_cast<const int4*>(acol + col0)) : make_int4(-1, -1, -1, -1);
    }
#pragma unroll
    for (int k = 0; k < PASSES * RPW; ++k) {
      const int y = y0 + k * NWARP;
      if (y >= H) continue;
      const int ra = ws.row_arg[(int64_t)n * H + y];
      const bool row_in = y >= sp.y_lo && y <= sp.y_hi;     // warp-uniform
      const int c_lo = row_in ? sp.c_lo : W, c_hi = row_in ? sp.c_hi : -1;
      float* grow = g_logits + (int64_t)n * H * W + (int64_t)y * W;
#pragma unroll
      for (int ch = 0; ch < NCHUNK; ++ch) {
        const int col0 = (ch * 32 + lane) * 4;
        if (col0 >= W) continue;
        if (col0 >= c_lo && col0 + 3 <= c_hi) continue;     // fully inside the span: the pair role writes it
        const bool hit = (ac[ch].x == y) | (ac[ch].y == y) | (ac[ch].z == y) | (ac[ch].w == y) |
                         ((unsigned)(ra - col0) < 4u);
        const bool outside = col0 + 3 < c_lo || col0 > c_hi;
        if (!hit && outside) {                              // the common case: a plain zero store
          *reinterpret_cast<float4*>(grow + col0) = make_float4(0.f, 0.f, 0.f, 0.f);
          continue;
        }
        float out[4] = {0.f, 0.f, 0.f, 0.f};
        if ((unsigned)(ra - col0) < 4u) {
          const float rc = ws.coef_row[(int64_t)n * H + y] * g_prj;
#pragma unroll
          for (int e = 0; e < 4; ++e) if (ra - col0 == e) out[e] += rc;
        }
        if (ac[ch].x == y) out[0] += ccol[col0] * g_prj;
        if (ac[ch].y == y) out[1] += ccol[col0 + 1] * g_prj;
        if (ac[ch].z == y) out[2] += ccol[col0 + 2] * g_prj;
        if (ac[ch].w == y) out[3] += ccol[col0 + 3] * g_prj;
        if (outside) {
          *reinterpret_cast<float4*>(grow + col0) = make_float4(out[0], out[1], out[2], out[3]);
        } else {                                            // straddles the span boundary
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (col0 + e < c_lo || col0 + e > c_hi) grow[col0 + e] = out[e];
        }
      }
    }
  } else {
    // ================= pair role: gather-form gradient of the span pixels =================
    const float g_pair = g_losses[1] * ws.scale_pair[0];
    const float* img = logits + (int64_t)n * H * W;
    const uint8_t* bits = edge_bits + (int64_t)rec.img * H * W;
    const Chain ch = chain_of<D>(sp, rec.len_b, rec.pc_b, role * NWARP + warp);
    if (ch.nrows > 0)
      pair_chain_bwd<D>(img, bits, H, W, ch.y0, ch.nrows, sp.c_lo - D + ch.seg * (32 - 2 * D), sp.c_hi, r, lane, g_pair,
                        ws.row_arg + (int64_t)n * H, ws.coef_row + (int64_t)n * H, acol, ccol, g_prj,
                        g_logits + (int64_t)n * H * W);
  }
}

// ---------------------------------------------------------------------------------------
// generic-path backward: one tile kernel, every g_logits element written exactly once
// ---------------------------------------------------------------------------------------
template <bool VEC>
__global__ void __launch_bounds__(NT) loss_bwd_kernel(const float* __restrict__ logits,
                                                      const uint8_t* __restrict__ edge_bits,
                                                      const int32_t* __restrict__ rects,
                                                      const int32_t* __restrict__ inst_gt,
                                                      const int32_t* __restrict__ gt_img, int H, int W, int d,
                                                      Workspace ws, const float* __restrict__ g_losses,
                                                      float* __restrict__ g_logits) {
  extern __shared__ float smem[];
  const int n = blockIdx.z, y0 = blockIdx.y * TH, x0 = blockIdx.x * TW;
  const int g = inst_gt[n];
  const Rect r = load_rect(rects, g);
  const float g_prj = g_losses[0];
  const float g_pair = g_losses[1] * ws.scale_pair[0];
  // pixels that can receive a pairwise gradient: the box grown by d
  const bool box_tile = !rect_empty(r) && y0 <= r.j1 + d && y0 + TH - 1 >= r.j0 - d && x0 <= r.i1 + d &&
                        x0 + TW - 1 >= r.i0 - d;
  PairTile t{};
  if (box_tile) {
    const float* img = logits + (int64_t)n * H * W;
    const uint8_t* bits = edge_bits + (int64_t)gt_img[g] * H * W;
    t = load_pair_tile(img, bits, H, W, y0 - d, x0 - d, TH + 2 * d, TW + 2 * d, smem);
  }
  const int ty = threadIdx.x / (TW / 4), tx = (threadIdx.x % (TW / 4)) * 4;
  const int gy = y0 + ty, gx = x0 + tx;
  if (gy >= H || gx >= W) return;
  const float* crow = ws.coef_row + (int64_t)n * H;
  const int* arow = ws.row_arg + (int64_t)n * H;
  const float* ccol = ws.coef_col + (int64_t)n * W;
  const int* acol = ws.col_arg + (int64_t)n * W;
  const int ra = arow[gy];
  const float rc = crow[gy] * g_prj;
  float out[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int x = gx + k;
    float v = 0.f;
    if (x < W) {
      if (x == ra) v += rc;
      if (acol[x] == gy) v += ccol[x] * g_prj;
      if (box_tile) {
        const int ci = (ty + d) * t.pitch + (tx + k + d);
        const bool pin = in_rect(r, gy, x);
        const unsigned ep = t.e[ci];
        const float xa = t.x[ci], sa = t.s[ci], na = t.n[ci];
        float acc = 0.f;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const int cc = c < 4 ? c : c + 1;              // skip the centre of the 3x3 stencil
          const int dy = (cc / 3 - 1) * d, dx = (cc % 3 - 1) * d;
          const int qy = gy + dy, qx = x + dx;
          if (qy < 0 || qy >= H || qx < 0 || qx >= W) continue;
          const int qi = ci + dy * t.pitch + dx;
          const unsigned eq = t.e[qi];
          const int m = (pin ? (ep >> c) & 1u : 0u) + (in_rect(r, qy, qx) ? (eq >> (7 - c)) & 1u : 0u);
          if (m) {
            const float xb = t.x[qi];
            float dd;
            if (fmaxf(fabsf(xa), fabsf(xb)) <= kFastLimit) {
              const float sb = t.s[qi], nb = t.n[qi];
              dd = -(sb - nb) * __frcp_rn(sa * sb + na * nb);
              dd *= sa * na;
            } else {
              dd = pair_nlog_grad_a_logspace<float>(xa, xb, true, pair_nlog_logspace<float>(xa, xb, true));
            }
            acc = fmaf((float)m, dd, acc);
          }
        }
        v = fmaf(acc, g_pair, v);
      }
    }
    out[k] = v;
  }
  float* dst = g_logits + (int64_t)n * H * W + (int64_t)gy * W + gx;
  if (VEC) {
    *reinterpret_cast<float4*>(dst) = make_float4(out[0], out[1], out[2], out[3]);
  } else {
#pragma unroll
    for (int k = 0; k < 4; ++k)
      if (gx + k < W) dst[k] = out[k];
  }
}

inline bool args_ok(int64_t N, int64_t H, int64_t W, int d) {
  return N > 0 && N < 65536 && H > 0 && W > 0 && H * W < (int64_t(1) << 31) && d >= 1 && d <= 16;
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_boxinst_loss_workspace_bytes(int64_t N, int64_t H, int64_t W) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  return (int64_t)carve(nullptr, N, H, W).total_bytes;
}

namespace bxs {
namespace {
inline bool fast_ok(const void* logits, const void* edge_bits, const void* out, int64_t H, int64_t W, int d) {
  return (W % 4 == 0) && W <= 512 && H <= 512 && d >= 1 && d <= 4 && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0) &&
         ((reinterpret_cast<uintptr_t>(edge_bits) & 3) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
}

template <int NCHUNK>
void launch_fwd_fast(int d, dim3 grid, cudaStream_t st, const float* logits, const uint8_t* edge_bits,
                     const int32_t* rects, const int32_t* inst_gt, const int32_t* gt_img, int N, int H, int W,
                     Workspace ws, const float* iter_ptr, float warmup_iters, float* losses_out) {
#define BXS_CASE(DD)                                                                                             \
  case DD:                                                                                                       \
    prep_fast_kernel<DD><<<N, 128, 0, st>>>(rects, inst_gt, gt_img, H, W, ws);                                   \
    fwd_fused_kernel<NCHUNK, DD><<<grid, NT, 0, st>>>(logits, edge_bits, rects, inst_gt, gt_img, H, W, ws);      \
    finalize_fast_kernel<DD><<<(N + FIN_GROUPS - 1) / FIN_GROUPS, FIN_GROUPS * 128, 0, st>>>(                    \
        rects, inst_gt, N, H, W, ws, iter_ptr, warmup_iters, losses_out);                                        \
    break;
  switch (d) { BXS_CASE(1) BXS_CASE(2) BXS_CASE(3) BXS_CASE(4) }
#undef BXS_CASE
}

template <int NCHUNK>
void launch_bwd_fast(int d, dim3 grid, cudaStream_t st, const float* logits, const uint8_t* edge_bits,
                     const int32_t* rects, const int32_t* inst_gt, const int32_t* gt_img, int H, int W, Workspace ws,
                     const float* g_losses, float* g_logits) {
#define BXS_CASE(DD)                                                                                              \
  case DD:                                                                                                        \
    bwd_rows_kernel<NCHUNK, DD><<<grid, NT, 0, st>>>(logits, edge_bits, rects, inst_gt, gt_img, H, W, ws, g_losses, \
                                                     g_logits);                                                   \
    break;
  switch (d) { BXS_CASE(1) BXS_CASE(2) BXS_CASE(3) BXS_CASE(4) }
#undef BXS_CASE
}
}  // namespace
}  // namespace bxs

extern "C" int bxs_boxinst_loss_forward(const float* logits, const uint8_t* edge_bits, const int32_t* rects,
                                        const int32_t* inst_gt, const int32_t* gt_img, const float* iter_ptr,
                                        float warmup_iters, void* workspace, float* losses_out, int64_t N,
                                        int64_t H, int64_t W, int dilation, bxs_stream_t stream) {
  if (!logits || !edge_bits || !rects || !inst_gt || !gt_img || !iter_ptr || !workspace || !losses_out ||
      !args_ok(N, H, W, dilation) || !(warmup_iters > 0.f))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  Workspace ws = carve(workspace, N, H, W);
  const int d = dilation;
  if (fast_ok(logits, edge_bits, logits, H, W, d)) {
    // one fused streaming kernel: maxima + in-box pair terms + per-instance finalize
    dim3 grid((unsigned)N, (unsigned)ceil_div(H, ROWS_PER_CTA) + PAIR_BLOCKS);
    if (W <= 128) launch_fwd_fast<1>(d, grid, st, logits, edge_bits, rects, inst_gt, gt_img, (int)N, (int)H, (int)W, ws, iter_ptr, warmup_iters, losses_out);
    else if (W <= 256) launch_fwd_fast<2>(d, grid, st, logits, edge_bits, rects, inst_gt, gt_img, (int)N, (int)H, (int)W, ws, iter_ptr, warmup_iters, losses_out);
    else launch_fwd_fast<4>(d, grid, st, logits, edge_bits, rects, inst_gt, gt_img, (int)N, (int)H, (int)W, ws, iter_ptr, warmup_iters, losses_out);
    return check_launch();
  }
  // ---- generic path (any W / alignment / dilation): tile kernels over a device-built work list ----
  cudaMemsetAsync(workspace, 0, ws.zero_bytes, st);
  prep_worklist<<<1, NT, 0, st>>>(rects, inst_gt, (int)N, (int)H, (int)W, d, ws.tile_prefix);
  const int sms = sm_count();
  int strips = (int)ceil_div((int64_t)sms * 4, N);
  strips = (int)std::max<int64_t>(1, std::min<int64_t>(strips, ceil_div(H, 8)));
  const int rows = (int)ceil_div(H, strips);
  strips = (int)ceil_div(H, rows);
  const bool vec = (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(logits) & 15) == 0);
  if (vec && W <= 128) {
    prj_max_kernel<1, 4><<<dim3(strips, (unsigned)N, 1), NT, 0, st>>>(logits, (int)H, (int)W, rows, ws.row_packed, ws.col_packed);
  } else if (vec && W <= 256) {
    prj_max_kernel<2, 4><<<dim3(strips, (unsigned)N, 1), NT, 0, st>>>(logits, (int)H, (int)W, rows, ws.row_packed, ws.col_packed);
  } else if (vec) {
    prj_max_kernel<4, 4><<<dim3(strips, (unsigned)N, (unsigned)ceil_div(W, 512)), NT, 0, st>>>(logits, (int)H, (int)W, rows, ws.row_packed, ws.col_packed);
  } else {
    prj_max_kernel<8, 1><<<dim3(strips, (unsigned)N, (unsigned)ceil_div(W, 256)), NT, 0, st>>>(logits, (int)H, (int)W, rows, ws.row_packed, ws.col_packed);
  }
  int rc = check_launch();
  if (rc) return rc;
  const size_t sm2 = (size_t)(TH + d) * (TW + 2 * d) * (3 * sizeof(float) + 1) + 16;
  pair_fwd_kernel<<<sms * 4, NT, sm2, st>>>(logits, edge_bits, rects, inst_gt, gt_img, (int)N, (int)H, (int)W, d,
                                            ws.tile_prefix, ws.pair_partial, ws.weight_sum);
  rc = check_launch();
  if (rc) return rc;
  finalize_kernel<<<(unsigned)N, NT, 0, st>>>(rects, inst_gt, (int)N, (int)H, (int)W, ws, iter_ptr, warmup_iters,
                                              losses_out);
  return check_launch();
}

extern "C" int bxs_boxinst_loss_backward(const float* logits, const uint8_t* edge_bits, const int32_t* rects,
                                         const int32_t* inst_gt, const int32_t* gt_img, const void* workspace,
                                         const float* g_losses, float* g_logits, int64_t N, int64_t H,
                                         int64_t W, int dilation, bxs_stream_t stream) {
  if (!logits || !edge_bits || !rects || !inst_gt || !gt_img || !workspace || !g_losses || !g_logits ||
      !args_ok(N, H, W, dilation))
    return BXS_ERR_INVALID_ARG;
  cudaStream_t st = as_stream(stream);
  Workspace ws = carve(const_cast<void*>(workspace), N, H, W);
  const int d = dilation;
  if (fast_ok(logits, edge_bits, g_logits, H, W, d)) {
    dim3 grid((unsigned)N, (unsigned)ceil_div(H, ROWS_PER_CTA) + PAIR_BLOCKS);
    if (W <= 128) launch_bwd_fast<1>(d, grid, st, logits, edge_bits, rects, inst_gt, gt_img, (int)H, (int)W, ws, g_losses, g_logits);
    else if (W <= 256) launch_bwd_fast<2>(d, grid, st, logits, edge_bits, rects, inst_gt, gt_img, (int)H, (int)W, ws, g_losses, g_logits);
    else launch_bwd_fast<4>(d, grid, st, logits, edge_bits, rects, inst_gt, gt_img, (int)H, (int)W, ws, g_losses, g_logits);
    return check_launch();
  }
  const size_t sm = (size_t)(TH + 2 * d) * (TW + 2 * d) * (3 * sizeof(float) + 1) + 16;
  dim3 grid((unsigned)ceil_div(W, TW), (unsigned)ceil_div(H, TH), (unsigned)N);
  const bool vec = (W % 4 == 0) && ((reinterpret_cast<uintptr_t>(g_logits) & 15) == 0);
  if (vec)
    loss_bwd_kernel<true><<<grid, NT, sm, st>>>(logits, edge_bits, rects, inst_gt, gt_img, (int)H, (int)W, d, ws,
                                                g_losses, g_logits);
  else
    loss_bwd_kernel<false><<<grid, NT, sm, st>>>(logits, edge_bits, rects, inst_gt, gt_img, (int)H, (int)W, d, ws,
                                                 g_losses, g_logits);
  return check_launch();
}
