// a6 + a7 + a8, single pass: the fused BoxInst mask loss AND its gradient from ONE read of the logits.
// Same arithmetic as boxinst_loss.cu (CondInstMaskHead.loss, condinst_head.py:1288-1343), different
// schedule: the pairwise normaliser (sum of weights) does not depend on the logits and the projection
// term back-propagates only to H + W arg-max positions per instance, so the dense part of the gradient
// can be produced while the logits stream through the SM the first time.
//
//   onepass_main_kernel   persistent CTAs, dynamic tile scheduler (one atomic per work item).  A work
//       item is a strip of 16 rows of one instance: ONE cp.async.bulk (TMA, 1-D) brings the strip
//       (+ the dilation halo when the strip meets the box) into shared memory, double buffered on
//       mbarriers, so the next strip is in flight while this one is processed.  From shared memory:
//       row maxima (integer redux), column maxima, zero stores of the gradient outside the box
//       span, and -- inside the span -- the pair terms and the RAW (unscaled) pairwise gradient,
//       gathered from a (sigmoid, 1 - sigmoid, edge bits) tile.  HBM traffic: logits read once,
//       gradient written once.
//   onepass_finalize_kernel   one CTA per instance: dice terms and their gradient coefficients; scales
//       the (small) box span of the gradient by warmup / weights (the weight total is an integer
//       atomic sum of the main kernel) and adds the projection terms at the H + W arg-max positions
//       for upstream gradients (1, 1); the last CTA writes the losses.
//   onepass_backward_kernel   returns at once when the upstream gradients are (1, 1) (the result is in
//       place); otherwise converts the gradient in place, exactly (the pairwise part at the arg-max
//       positions is kept in the workspace).
//
// Everything is summed in a fixed order: results do not depend on which CTA processed which strip.
#include <algorithm>
#include <cstdlib>

#include "boxinst_common.cuh"

namespace bxs {
namespace {

constexpr int OP_NT = 256;          // threads per CTA of the main kernel
constexpr int OP_NW = OP_NT / 32;
constexpr int OP_R = 16;            // rows per strip
constexpr int OP_FIN_NT = 512;      // threads per CTA of the finalize / backward kernels
constexpr int OP_MAX_N = 2048;      // instance records live in shared memory (12 B each)

struct OpWorkspace {
  unsigned long long* row_packed;  // [N*H]    (key(max logit) << 32) | ~x
  unsigned long long* col_part;    // [N*S*W]  per strip (key(max logit) << 32) | ~y
  float* num_part;                 // [N*MAXG] per chain group pairwise numerator
  float* coef_row;                 // [N*H]    d loss_prj / d logit at the row arg-max
  float* coef_col;                 // [N*W]
  int* arg_row;                    // [N*H]
  int* arg_col;                    // [N*W]
  int* span;                       // [N*4]    y_lo, y_hi, c_lo, c_hi of the gradient span (y_lo > y_hi: none)
  float* inst_prj;                 // [N]
  float* inst_num;                 // [N]
  float* sv_row;                   // [N*H]    scaled pairwise gradient at the row arg-max position
  float* sv_col;                   // [N*W]
  size_t total_bytes;
};

#ifndef BXS_OP_LEN
#define BXS_OP_LEN 12
#endif
constexpr int OP_LEN = BXS_OP_LEN;  // rows per pair-chain piece (build-time tunable for A/B runs)

inline int64_t op_max_groups(int64_t H, int64_t W) {      // upper bound of ceil(chains / 8) for any box and dilation 1..4
  int64_t best = 1;
  for (int d = 1; d <= 4; ++d) {
    const int64_t nseg = ceil_div(W, 32 - 2 * d) + 1, pc = ceil_div(ceil_div(H, d), OP_LEN) + 1;
    best = std::max<int64_t>(best, ceil_div(d * pc * nseg, OP_NW));
  }
  return best;
}

inline OpWorkspace op_carve(void* base, int64_t N, int64_t H, int64_t W) {
  OpWorkspace w{};
  Carver c(base);
  const int64_t S = ceil_div(H, OP_R);
  w.row_packed = (unsigned long long*)c.take(8 * N * H);
  w.col_part = (unsigned long long*)c.take(8 * N * S * W);
  const int64_t G = op_max_groups(H, W);
  w.num_part = (float*)c.take(4 * N * G);
  w.coef_row = (float*)c.take(4 * N * H);
  w.coef_col = (float*)c.take(4 * N * W);
  w.arg_row = (int*)c.take(4 * N * H);
  w.arg_col = (int*)c.take(4 * N * W);
  w.span = (int*)c.take(16 * N);
  w.inst_prj = (float*)c.take(4 * N);
  w.inst_num = (float*)c.take(4 * N);
  w.sv_row = (float*)c.take(4 * N * H);
  w.sv_col = (float*)c.take(4 * N * W);
  w.total_bytes = c.off;
  return w;
}

// ---------------------------------------------------------------------------------------
// instance records
// ---------------------------------------------------------------------------------------
struct SRec { short j0, j1, i0, i1; int img; };     // box rectangle clipped to the map; canonical empty = (1,0,1,0)

__device__ __forceinline__ SRec make_srec(const int32_t* __restrict__ rects, const int32_t* __restrict__ inst_gt,
                                          const int32_t* __restrict__ gt_img, int n, int H, int W) {
  const int g = __ldg(inst_gt + n);
  const int4 r = __ldg(reinterpret_cast<const int4*>(rects + 4 * (int64_t)g));
  int j0 = max(r.x, 0), j1 = min(r.y, H - 1), i0 = max(r.z, 0), i1 = min(r.w, W - 1);
  if (r.x > r.y || r.z > r.w || j0 > j1 || i0 > i1) { j0 = 1; j1 = 0; i0 = 1; i1 = 0; }
  SRec v;
  v.j0 = (short)j0; v.j1 = (short)j1; v.i0 = (short)i0; v.i1 = (short)i1;
  v.img = __ldg(gt_img + g);
  return v;
}

// pixels that can receive a pairwise gradient: the box grown by D, columns rounded out to float4 groups
struct OpSpan { int y_lo, y_hi, c_lo, c_hi; };
template <int D>
__device__ __forceinline__ OpSpan op_span(const SRec& r, int H, int W) {
  OpSpan s;
  if (r.j0 > r.j1) { s.y_lo = 1; s.y_hi = 0; s.c_lo = 4; s.c_hi = 3; return s; }
  s.y_lo = max(r.j0 - D, 0);
  s.y_hi = min(r.j1 + D, H - 1);
  s.c_lo = max(r.i0 - D, 0) & ~3;
  s.c_hi = min(r.i1 + D, W - 1) | 3;      // < W because W % 4 == 0
  return s;
}

__device__ __forceinline__ int op_div(int a, int b) {      // exact for 0 <= a < 2^20, 0 < b < 2^10
  return __float2int_rz((__int2float_rn(a) + 0.5f) * rcp_approx(__int2float_rn(b)));
}
__device__ __forceinline__ float op_lg2(float v) {         // MUFU.LG2 (v is a normal number here)
  float o;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(o) : "f"(v));
  return o;
}
__device__ __forceinline__ float op_ex2(float v) {
  float o;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(o) : "f"(v));
  return o;
}
// (sigmoid(x), sigmoid(-x)), both to a few ulp relative (no 1 - s cancellation); exact enough for |x| <= kFastLimit
__device__ __forceinline__ void op_sigmoid_pair(float x, float& s, float& n) {
  const float e = op_ex2(-1.4426950408889634f * fabsf(x));
  const float big = rcp_approx(1.f + e);
  const float small = e * big;
  s = x >= 0.f ? big : small;
  n = x >= 0.f ? small : big;
}

// ---------------------------------------------------------------------------------------
// pair chains
// ---------------------------------------------------------------------------------------
// A chain is one warp walking rows y0, y0 + D, y0 + 2D, ... of one 32-lane column segment whose inner 32 - 2D
// lanes own a pixel.  The row below (y + D) of one step is the row at of the next, so every row is loaded and
// sigmoid-ed once, and each unordered pair {p, q} is evaluated once (q = right, below-left, below, below-right
// of p) with multiplicity m = [edge bit of p towards q, p in box] + [edge bit of q towards p, q in box].  The
// gradient of the left / upper pixel stays in the lane, the one of the other pixel travels by a shuffle (same
// row) or through `carry` (row below -> next step).  The step before the chain (row y0 - D) only feeds the carry.
struct PSeg { float x, s, n; unsigned e; };        // one lane's pixel: logit, sigmoid pair, box-masked edge bits
struct PRaw { float x; unsigned e; };

struct ChainGeom {                 // chain layout of one instance (pure function of its record)
  int y_lo, rows, c_lo, c_hi, nseg, pc, nch;
};
template <int D>
__device__ __forceinline__ ChainGeom chain_geom(const SRec& r, int H, int W) {
  ChainGeom g;
  const OpSpan sp = op_span<D>(r, H, W);
  g.y_lo = sp.y_lo; g.rows = sp.y_hi - sp.y_lo + 1; g.c_lo = sp.c_lo; g.c_hi = sp.c_hi;
  if (g.rows <= 0) { g.rows = 0; g.nseg = 0; g.pc = 0; g.nch = 0; return g; }
  g.nseg = (sp.c_hi - sp.c_lo + 1 + (32 - 2 * D) - 1) / (32 - 2 * D);
  g.pc = ((g.rows + D - 1) / D + OP_LEN - 1) / OP_LEN;        // pieces of the longest parity class
  g.nch = D * g.pc * g.nseg;
  return g;
}

template <int D>
__device__ __forceinline__ void op_chain(const float* __restrict__ img, const uint8_t* __restrict__ bits, int H, int W,
                                         int y0, int nrows, int xs, int c_hi, const SRec& r, int lane,
                                         float* __restrict__ ginst, float gscale, float& acc_lg, float& acc_slow,
                                         int& acc_w) {
  const int x = xs + lane;
  const bool x_ok = x >= 0 && x < W, x_box = x >= r.i0 && x <= r.i1;
  const bool owner = lane >= D && lane < 32 - D && x <= c_hi;
  const bool up_ok = lane >= D, dn_ok = lane + D < 32;       // the lane a shuffle by D reads from exists
  auto load = [&](int y) {
    PRaw v;
    const bool in = x_ok && y >= 0 && y < H;
    v.x = in ? __ldg(img + y * W + x) : 0.f;
    v.e = (in && x_box && y >= r.j0 && y <= r.j1) ? (unsigned)__ldg(bits + y * W + x) : 0u;
    return v;
  };
  auto finish = [&](const PRaw& w) {
    PSeg v;
    v.x = w.x; v.e = w.e;
    op_sigmoid_pair(w.x, v.s, v.n);
    return v;
  };
  {  // every row this chain will read, requested from HBM into L2 NOW (one prefetch per lane: row = lane & 15, 64-byte half
     // = lane >> 4): the step-ahead loads below then hit L2 even while the stream items keep HBM saturated
    const int pr = y0 + ((lane & 15) - 1) * D, px = xs + (lane >> 4) * 16;
    if ((lane & 15) < nrows + 2 && pr >= 0 && pr < H) {
      const int pxc = min(max(px, 0), W - 1);
      asm volatile("prefetch.global.L2 [%0];" ::"l"(img + (size_t)pr * W + pxc));
      if (lane < 16 && pr >= r.j0 && pr <= r.j1) asm volatile("prefetch.global.L2 [%0];" ::"l"(bits + (size_t)pr * W + pxc));
    }
  }
  PSeg cur = finish(load(y0 - D));
  PRaw ahead = load(y0);
  float carry = 0.f;
  for (int k = -1; k < nrows; ++k) {
    const int y = y0 + k * D;
    const PSeg nxt = finish(ahead);
    if (k + 1 < nrows) ahead = load(y + 2 * D);
    const bool extreme = __any_sync(kFull, fmaxf(fabsf(cur.x), fabsf(nxt.x)) > kFastLimit);
    const bool count = owner && k >= 0;
    // neighbours: 4 = (y, x + D), 5 = (y + D, x - D), 6 = (y + D, x), 7 = (y + D, x + D)
    const float s4 = __shfl_down_sync(kFull, cur.s, D), n4 = __shfl_down_sync(kFull, cur.n, D);
    const unsigned e4 = __shfl_down_sync(kFull, cur.e, D);
    const float s5 = __shfl_up_sync(kFull, nxt.s, D), n5 = __shfl_up_sync(kFull, nxt.n, D);
    const unsigned e5 = __shfl_up_sync(kFull, nxt.e, D);
    const float s7 = __shfl_down_sync(kFull, nxt.s, D), n7 = __shfl_down_sync(kFull, nxt.n, D);
    const unsigned e7 = __shfl_down_sync(kFull, nxt.e, D);
    const unsigned m4 = (dn_ok && k >= 0) ? ((cur.e >> 4) & 1u) + ((e4 >> 3) & 1u) : 0u;
    const unsigned m5 = up_ok ? ((cur.e >> 5) & 1u) + ((e5 >> 2) & 1u) : 0u;
    const unsigned m6 = ((cur.e >> 6) & 1u) + ((nxt.e >> 1) & 1u);
    const unsigned m7 = dn_ok ? ((cur.e >> 7) & 1u) + (e7 & 1u) : 0u;
    float ga, gq4, gq5, gq6, gq7;     // d/d this pixel (complete), d/d the neighbour (complete)
    if (!extreme) {
      const float dfa = cur.n - cur.s, sna = cur.s * cur.n;
      float lg = 0.f, gs = 0.f;
#define BXS_OP_PAIR(M, QS, QN, GQ)                                        \
      {                                                                    \
        const float den = fmaf(cur.s, QS, cur.n * QN);                     \
        const float mf = (float)(M);                                       \
        const float t = mf * rcp_approx(den);                              \
        lg = fmaf(mf, op_lg2(den), lg);                                    \
        gs = fmaf(QN - QS, t, gs);                                         \
        GQ = dfa * t * (QS * QN);                                          \
      }
      BXS_OP_PAIR(m4, s4, n4, gq4)
      BXS_OP_PAIR(m5, s5, n5, gq5)
      BXS_OP_PAIR(m6, nxt.s, nxt.n, gq6)
      BXS_OP_PAIR(m7, s7, n7, gq7)
#undef BXS_OP_PAIR
      ga = gs * sna;
      if (count) acc_lg += lg;
    } else {                           // a logit beyond +-40 in these two rows: log-space formulas
      const float x4 = __shfl_down_sync(kFull, cur.x, D), x5 = __shfl_up_sync(kFull, nxt.x, D);
      const float x7 = __shfl_down_sync(kFull, nxt.x, D);
      float val = 0.f;
      ga = 0.f;
#define BXS_OP_SLOW(M, QX, GQ)                                                                  \
      {                                                                                          \
        GQ = 0.f;                                                                                \
        if (M) {                                                                                 \
          const float pl = pair_nlog_logspace<float>(cur.x, QX, true);                           \
          val = fmaf((float)(M), pl, val);                                                       \
          ga = fmaf((float)(M), pair_nlog_grad_a_logspace<float>(cur.x, QX, true, pl), ga);      \
          GQ = (float)(M) * pair_nlog_grad_a_logspace<float>(QX, cur.x, true, pl);               \
        }                                                                                        \
      }
      BXS_OP_SLOW(m4, x4, gq4)
      BXS_OP_SLOW(m5, x5, gq5)
      BXS_OP_SLOW(m6, nxt.x, gq6)
      BXS_OP_SLOW(m7, x7, gq7)
#undef BXS_OP_SLOW
      if (count) acc_slow += val;
    }
    const float from_left = __shfl_up_sync(kFull, gq4, D);        // pair (x - D, x): this lane is the right pixel
    const float to_left = __shfl_down_sync(kFull, gq5, D);        // lane + D's lower-left pixel is this lane's column
    const float to_right = __shfl_up_sync(kFull, gq7, D);
    if (count) {
      acc_w += __popc(cur.e);
      ginst[y * W + x] = ((ga + carry) + from_left) * gscale;     // owners have lane >= D: from_left is a real lane's value
    }
    carry = gq6 + (dn_ok ? to_left : 0.f) + (up_ok ? to_right : 0.f);
    cur = nxt;
  }
}

#ifdef BXS_OP_TRACE
// diagnostic build only (tools/trace_onepass.py): per-CTA event log {globaltimer, tag}; 64 slots per CTA
__device__ unsigned long long* g_op_trace = nullptr;
__device__ __forceinline__ void op_trace(int& slot, unsigned long long tag) {
  if (g_op_trace && slot < 64) {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    g_op_trace[(blockIdx.x * 64 + slot) * 2] = t;
    g_op_trace[(blockIdx.x * 64 + slot) * 2 + 1] = tag;
    ++slot;
  }
}
#define OP_TRACE(tag) if (tid == 0) op_trace(trace_slot, (unsigned long long)(tag))
#else
#define OP_TRACE(tag)
#endif

struct OpSched { unsigned next, done, ticket, pad; unsigned long long wtot, pad2; };   // wtot: total weight count of the step

constexpr int OP_STAGES = 2;       // strips staged per CTA: one copy in flight while one strip is processed

// Everything a thread needs to know about a work item, written by thread 0 when it issues the item.
struct ItemInfo {
  int kind;              // 0: stream item (n, strip s)   1: pair item (n, chain group s)   -1: the queue is empty
  int n, s;
  int ya, yb;            // stream: span rows inside the strip (ya > yb: none)
  int c_lo, c_hi;        // span columns (float4-aligned)
  int pad;
};

// One work queue (one atomic per item), two kinds of items:
//   pair items    8 chains (one per warp) of one instance: pair terms, weight counts and the raw pairwise gradient of the
//                 box span, straight from global memory (L2).  No shared memory, no barrier inside.  Long: queued first.
//   stream items  one strip of 16 rows of one instance: ONE bulk copy into a shared-memory stage; row / column maxima and
//                 the zero part of the gradient.  Short: they end the queue, so the dynamic scheduler has a short tail.
// The copy of the next stream item is in flight while the current item is processed.
// FULLW: W == NCHUNK * 128 (every lane of a row warp owns NCHUNK full float4 groups; W folds to a constant)
template <int NCHUNK, int D, bool FULLW>
__global__ void __launch_bounds__(OP_NT, NCHUNK <= 2 ? 4 : 2)
onepass_main_kernel(const float* __restrict__ logits, const uint8_t* __restrict__ edge_bits,
                    const int32_t* __restrict__ rects, const int32_t* __restrict__ inst_gt,
                    const int32_t* __restrict__ gt_img, int N, int H, int W_rt, int S, int MAXG, OpWorkspace ws,
                    OpSched* __restrict__ sched, float* __restrict__ g_logits) {
  const int W = FULLW ? NCHUNK * 128 : W_rt;
  extern __shared__ __align__(128) unsigned char op_smem[];
  const int stage_floats = OP_R * W;
  float* xbuf = reinterpret_cast<float*>(op_smem);                               // [OP_STAGES][OP_R][W]
  SRec* s_rec = reinterpret_cast<SRec*>(xbuf + OP_STAGES * stage_floats);        // [N]
  int* s_gpre = reinterpret_cast<int*>(s_rec + N);                               // [N + 1] prefix of chain-group counts
  __shared__ __align__(8) uint64_t s_bar[OP_STAGES];
  __shared__ __align__(16) ItemInfo s_info[OP_STAGES];
  __shared__ float s_redf[OP_NW];
  __shared__ int s_redi[OP_NW];
  __shared__ int s_scan[OP_NW];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#ifdef BXS_OP_TRACE
  int trace_slot = 0;
#endif
  OP_TRACE(1);
  // programmatic dependent launch: the finalize grid may be scheduled as soon as SM resources free up (it still waits
  // for this grid's completion before reading its results)
  asm volatile("griddepcontrol.launch_dependents;");

  // queue position v -> stage: the item's description for all threads and, for a stream item, ONE bulk copy
  auto issue = [&](int v, int stage) {
    ItemInfo info;
    const int gtot = s_gpre[N];
    info.ya = 1; info.yb = 0; info.c_lo = 4; info.c_hi = 3; info.pad = 0;
    if (v < gtot) {
      int lo = 0, hi = N;                          // largest n with s_gpre[n] <= v
      while (hi - lo > 1) {
        const int mid = (lo + hi) >> 1;
        if (s_gpre[mid] <= v) lo = mid; else hi = mid;
      }
      info.kind = 1; info.n = lo; info.s = v - s_gpre[lo];
      s_info[stage] = info;
      return;
    }
    const int u = v - gtot;
    info.kind = 0;
    info.n = op_div(u, S); info.s = u - info.n * S;
    const int y0 = info.s * OP_R;
    const int rows = min(OP_R, H - y0);
    const OpSpan sp = op_span<D>(s_rec[info.n], H, W);
    if (sp.y_lo <= sp.y_hi) { info.ya = max(y0, sp.y_lo); info.yb = min(y0 + rows - 1, sp.y_hi); }
    info.c_lo = sp.c_lo; info.c_hi = sp.c_hi;
    s_info[stage] = info;
    const uint32_t bytes = (uint32_t)rows * (uint32_t)W * 4u;
    mbar_expect_tx(&s_bar[stage], bytes);
    bulk_g2s(xbuf + (size_t)stage * stage_floats, logits + ((int64_t)info.n * H + y0) * W, bytes, &s_bar[stage]);
  };

  unsigned fetched = 0;          // thread 0: next queue position (fetched one iteration ahead of its use)
  if (tid == 0) {
#pragma unroll
    for (int i = 0; i < OP_STAGES; ++i) mbar_init(&s_bar[i], 1);
    fence_mbarrier_init();
    fence_proxy_async_smem();
    fetched = gridDim.x + atomicAdd(&sched->next, 1u);
  }
  for (int n = tid; n < N; n += OP_NT) s_rec[n] = make_srec(rects, inst_gt, gt_img, n, H, W);
  __syncthreads();
  {                              // exclusive prefix of the chain-group counts (block scan, 256 instances per round)
    int run = 0;
    for (int base = 0; base < N; base += OP_NT) {
      const int n = base + tid;
      const int cnt = n < N ? (chain_geom<D>(s_rec[n], H, W).nch + OP_NW - 1) / OP_NW : 0;
      int inc = cnt;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(kFull, inc, o); if (lane >= o) inc += t; }
      if (lane == 31) s_scan[warp] = inc;
      __syncthreads();
      int wbase = 0, tot = 0;
#pragma unroll
      for (int i = 0; i < OP_NW; ++i) { const int t = s_scan[i]; if (i < warp) wbase += t; tot += t; }
      if (n < N) s_gpre[n] = run + wbase + inc - cnt;
      run += tot;
      if (base + OP_NT < N) __syncthreads();
    }
    if (tid == 0) s_gpre[N] = run;
  }
  __syncthreads();
  const int total = s_gpre[N] + N * S;
  if (tid == 0) issue(blockIdx.x, 0);             // gridDim.x <= N * S <= total (host)
  __syncthreads();

  unsigned phases = 0;           // mbarrier parity per stage (bit s): only stream items complete a phase
  int stage = 0;
  OP_TRACE(2);
  for (;;) {
    const ItemInfo it = s_info[stage];
    if (it.kind < 0) break;
    OP_TRACE(16 + it.kind + ((unsigned long long)it.n << 8));
    if (tid == 0) {              // prefetch the next item into the other stage (its readers finished before the last barrier)
      if (fetched < (unsigned)total) {
        issue((int)fetched, stage ^ 1);
        fetched = gridDim.x + atomicAdd(&sched->next, 1u);
      } else {
        s_info[stage ^ 1].kind = -1;
      }
    }
    const int n = it.n;
    float* ginst = g_logits + (int64_t)n * H * W;
    if (it.kind == 0) {
      // =============================== stream item: strip it.s of instance n ===============================
      const int y0 = it.s * OP_R;
      const int rows = min(OP_R, H - y0);
      const int ya = it.ya, yb = it.yb;
      mbar_wait(&s_bar[stage], (phases >> stage) & 1u);
      phases ^= 1u << stage;
      const float* xb = xbuf + (size_t)stage * stage_floats;       // strip row r at xb[r * W + col]
      // ---- row maxima (one warp per row, the warp's rows unrolled together) + zero stores outside the span ----
#pragma unroll
      for (int rr = 0; rr < OP_R / OP_NW; ++rr) {
        const int r = warp + rr * OP_NW;
        if (r < rows) {
          const int y = y0 + r;
          const float* row = xb + r * W;
          float v[NCHUNK][4];
          float cm[NCHUNK];
#pragma unroll
          for (int ch = 0; ch < NCHUNK; ++ch) {
            const int col0 = (ch * 32 + lane) * 4;
            float4 q;
            if (FULLW || col0 < W) q = *reinterpret_cast<const float4*>(row + col0);
            else q = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
            v[ch][0] = q.x; v[ch][1] = q.y; v[ch][2] = q.z; v[ch][3] = q.w;
            cm[ch] = fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w));
          }
          float m = cm[0];
#pragma unroll
          for (int ch = 1; ch < NCHUNK; ++ch) m = fmaxf(m, cm[ch]);
          const unsigned kmax = __reduce_max_sync(kFull, fkey(m));
          const float mv = fkey_inv(kmax);
          // first chunk (lowest columns) that holds the maximum, first lane within it, first element within the lane
          unsigned bal = __ballot_sync(kFull, cm[0] == mv);
          int chunk = 0;
#pragma unroll
          for (int ch = 1; ch < NCHUNK; ++ch) {
            const unsigned b = __ballot_sync(kFull, cm[ch] == mv);
            if (bal == 0u) { bal = b; chunk = ch; }
          }
          if (lane == (bal ? __ffs(bal) - 1 : 0)) {                  // bal == 0 only for an all-NaN row: any in-range index
            float w0 = v[0][0], w1 = v[0][1], w2 = v[0][2];
#pragma unroll
            for (int ch = 1; ch < NCHUNK; ++ch)
              if (chunk == ch) { w0 = v[ch][0]; w1 = v[ch][1]; w2 = v[ch][2]; }
            const int e = w0 == mv ? 0 : (w1 == mv ? 1 : (w2 == mv ? 2 : 3));
            ws.row_packed[n * H + y] = pack_key(kmax, min((chunk * 32 + lane) * 4 + e, W - 1));
          }
          float* grow = ginst + y * W + lane * 4;
          const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
          if (y >= ya && y <= yb) {                                  // warp-uniform: a span row (the chains write the span)
#pragma unroll
            for (int ch = 0; ch < NCHUNK; ++ch) {
              const int col0 = (ch * 32 + lane) * 4;
              if ((FULLW || col0 < W) && (col0 < it.c_lo || col0 > it.c_hi)) *reinterpret_cast<float4*>(grow + ch * 128) = z;
            }
          } else {
#pragma unroll
            for (int ch = 0; ch < NCHUNK; ++ch)
              if (FULLW || (ch * 32 + lane) * 4 < W) *reinterpret_cast<float4*>(grow + ch * 128) = z;
          }
        }
      }
      // ---- column maxima of the strip (one thread per column; first row wins ties) ----
      for (int col = tid; col < W; col += OP_NT) {
        const float* p = xb + col;
        float best = p[0];
        int brow = 0;
        if (rows == OP_R) {
#pragma unroll
          for (int r = 1; r < OP_R; ++r) {
            const float val = p[r * W];
            if (val > best) { best = val; brow = r; }
          }
        } else {
          for (int r = 1; r < rows; ++r) {
            const float val = p[r * W];
            if (val > best) { best = val; brow = r; }
          }
        }
        ws.col_part[(n * S + it.s) * W + col] = pack_key(fkey(best), y0 + brow);
      }
    } else {
      // =============================== pair item: chains 8 s .. 8 s + 7 of instance n ===============================
      const SRec rec = s_rec[n];
      const ChainGeom cg = chain_geom<D>(rec, H, W);
      const int gw = it.s * OP_NW + warp;
      float acc_lg = 0.f, acc_slow = 0.f;
      int acc_w = 0;
      if (gw < cg.nch) {                           // warp-uniform
        const int u = op_div(gw, cg.nseg), seg = gw - u * cg.nseg;
        const int p = op_div(u, cg.pc), piece = u - p * cg.pc;       // parity class, piece within the class
        const int rows_p = (cg.rows - p + D - 1) / D;                // rows of class p
        const int k0 = piece * OP_LEN;
        if (k0 < rows_p)
          op_chain<D>(logits + (int64_t)n * H * W, edge_bits + (int64_t)rec.img * H * W, H, W, cg.y_lo + p + D * k0,
                      min(OP_LEN, rows_p - k0), cg.c_lo - D + seg * (32 - 2 * D), cg.c_hi, rec, lane, ginst, 1.f, acc_lg,
                      acc_slow, acc_w);
      }
      const float v = warp_sum(fmaf(acc_lg, -0.69314718055994531f, acc_slow));
      const int w = warp_sum(acc_w);
      if (lane == 0) { s_redf[warp] = v; s_redi[warp] = w; }
    }
    __syncthreads();             // stage `stage` is free; the next s_info entries are visible; pair partials are in place
    if (it.kind == 1 && tid == 0) {                // fixed-order sum over the 8 chains of the group
      float v = 0.f;
      int w = 0;
#pragma unroll
      for (int i = 0; i < OP_NW; ++i) { v += s_redf[i]; w += s_redi[i]; }
      ws.num_part[n * MAXG + it.s] = v;
      if (w) atomicAdd(&sched->wtot, (unsigned long long)w);      // integer: order-independent, deterministic
    }
    stage ^= 1;
  }
  OP_TRACE(3);
  // ---- scheduler reset by the last CTA (every fetch of a CTA precedes its `done` increment) ----
  if (tid == 0) {
    __threadfence();
    if (atomicAdd(&sched->done, 1u) == gridDim.x - 1) {
      sched->next = 0u;
      sched->done = 0u;
      __threadfence();
    }
  }
}

// ---------------------------------------------------------------------------------------
// finalize: one CTA per instance.  Profiles -> dice terms and gradient coefficients; global weight sum -> scale;
// the last CTA (ticket) reduces the per-instance terms in a fixed order and writes the losses.  Does not touch
// the gradient.  All global loads of a phase are issued before the first use.
// ---------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(OP_FIN_NT)
onepass_finalize_kernel(const int32_t* __restrict__ rects, const int32_t* __restrict__ inst_gt,
                        const int32_t* __restrict__ gt_img, int N, int H, int W, int S, int MAXG, OpWorkspace ws,
                        OpSched* __restrict__ sched, const float* __restrict__ iter_ptr, float warmup_iters,
                        float* __restrict__ losses_out, float* __restrict__ g_logits) {
  constexpr int NWF = OP_FIN_NT / 32;
  __shared__ float s_f[4][NWF];
  __shared__ float s_coef[1024];      // rows [0, H), columns [512, 512 + W)
  __shared__ int s_arg[1024];
  __shared__ bool s_last;
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  // the record depends only on the targets: read it before waiting for the main grid (programmatic dependent launch)
  asm volatile("griddepcontrol.launch_dependents;");
  const SRec rec = make_srec(rects, inst_gt, gt_img, n, H, W);
  const OpSpan sp = op_span<D>(rec, H, W);
  const bool empty = rec.j0 > rec.j1;
  asm volatile("griddepcontrol.wait;" ::: "memory");
  float* ginst = g_logits + (unsigned)(n * H * W);
  // independent loads first: the step's weight total, this thread's row key and its column keys of every strip
  const unsigned long long wtot = *reinterpret_cast<volatile unsigned long long*>(&sched->wtot);
  const float warm = fminf(iter_ptr[0] / warmup_iters, 1.f);
  const int row_i = tid, col_i = tid;                   // H, W <= 512 = OP_FIN_NT
  unsigned long long rp = 0ull, cp = 0ull;
  if (row_i < H) rp = ws.row_packed[n * H + row_i];
  if (col_i < W) {
    const unsigned long long* src = ws.col_part + (int64_t)n * S * W + col_i;
#pragma unroll 4
    for (int s = 0; s < S; ++s) {
      const unsigned long long p = src[s * W];
      cp = p > cp ? p : cp;
    }
  }
  // chain-group numerators of this instance (warp 0; fixed order: lane-strided, then a shuffle tree at the end)
  float num = 0.f;
  if (wid == 0) {
    const int ng = (chain_geom<D>(rec, H, W).nch + OP_NW - 1) / OP_NW;
    for (int g = lane; g < ng; g += 32) num += ws.num_part[n * MAXG + g];
  }
  // ---- the box span of the gradient: raw pairwise gradient -> * warmup / weights (float4 read-modify-write) ----
  const float scale = warm / fmaxf((float)wtot, 1.f);
  const int sw4 = (sp.c_hi - sp.c_lo + 1) >> 2, srows = sp.y_hi - sp.y_lo + 1;
  if (srows > 0) {
    for (int i = tid; i < srows * sw4; i += OP_FIN_NT) {
      const int ry = op_div(i, sw4), c4 = i - ry * sw4;
      float4* p = reinterpret_cast<float4*>(ginst + (sp.y_lo + ry) * W + sp.c_lo + 4 * c4);
      float4 q = *p;
      q.x *= scale; q.y *= scale; q.z *= scale; q.w *= scale;
      *p = q;
    }
  }
  // ---- dice terms and their gradient coefficients ----
  const float sr = row_i < H ? sigmoid_exact(fkey_inv((unsigned)(rp >> 32))) : 0.f;
  const float sc = col_i < W ? sigmoid_exact(fkey_inv((unsigned)(cp >> 32))) : 0.f;
  const bool tr = !empty && row_i >= rec.j0 && row_i <= rec.j1, tc = !empty && col_i >= rec.i0 && col_i <= rec.i1;
  const float r0 = warp_sum(tr ? sr : 0.f), r1 = warp_sum(sr * sr), r2 = warp_sum(tc ? sc : 0.f), r3 = warp_sum(sc * sc);
  if (lane == 0) { s_f[0][wid] = r0; s_f[1][wid] = r1; s_f[2][wid] = r2; s_f[3][wid] = r3; }
  const int ar = (int)(0xffffffffu - (unsigned)(rp & 0xffffffffull)), ac = (int)(0xffffffffu - (unsigned)(cp & 0xffffffffull));
  if (row_i < H) s_arg[row_i] = ar;
  if (col_i < W) s_arg[512 + col_i] = ac;
  __syncthreads();               // also: every span store of this CTA is visible to its threads
  float Ir = 0.f, Xr = 0.f, Ic = 0.f, Xc = 0.f;
#pragma unroll
  for (int i = 0; i < NWF; ++i) { Ir += s_f[0][i]; Xr += s_f[1][i]; Ic += s_f[2][i]; Xc += s_f[3][i]; }
  const float inv_n = 1.f / (float)N;
  const float Ur = Xr + (empty ? 0.f : (float)(rec.j1 - rec.j0 + 1)) + kDiceEps;
  const float Uc = Xc + (empty ? 0.f : (float)(rec.i1 - rec.i0 + 1)) + kDiceEps;
  // d dice / d s = -2 t / U + 4 I s / U^2 ; through the sigmoid: * s (1 - s); mean over N
  const float crow = inv_n * (-2.f * (tr ? 1.f : 0.f) / Ur + 4.f * Ir * sr / (Ur * Ur)) * sr * (1.f - sr);
  const float ccol = inv_n * (-2.f * (tc ? 1.f : 0.f) / Uc + 4.f * Ic * sc / (Uc * Uc)) * sc * (1.f - sc);
  // scaled pairwise gradient at the arg-max positions (kept for upstream gradients != 1)
  float svr = 0.f, svc = 0.f;
  if (row_i < H) { svr = ginst[row_i * W + ar]; s_coef[row_i] = crow; }
  if (col_i < W) { svc = ginst[ac * W + col_i]; s_coef[512 + col_i] = ccol; }
  __syncthreads();               // all reads of the arg-max positions precede the writes below
  // ---- projection terms for upstream gradients (1, 1); a position that is both a row and a column arg-max is
  //      written once, by its column ----
  if (row_i < H) {
    if (s_arg[512 + ar] != row_i) ginst[row_i * W + ar] = svr + crow;
    ws.coef_row[n * H + row_i] = crow; ws.arg_row[n * H + row_i] = ar; ws.sv_row[n * H + row_i] = svr;
  }
  if (col_i < W) {
    ginst[ac * W + col_i] = s_arg[ac] == col_i ? (svc + s_coef[ac]) + ccol : svc + ccol;
    ws.coef_col[n * W + col_i] = ccol; ws.arg_col[n * W + col_i] = ac; ws.sv_col[n * W + col_i] = svc;
  }
  if (wid == 0) {
    num = warp_sum(num);
    if (lane == 0) {
      ws.inst_prj[n] = (1.f - 2.f * Ir / Ur) + (1.f - 2.f * Ic / Uc);
      ws.inst_num[n] = num;
      reinterpret_cast<int4*>(ws.span)[n] = make_int4(sp.y_lo, sp.y_hi, sp.c_lo, sp.c_hi);
      __threadfence();
      s_last = atomicAdd(&sched->ticket, 1u) == (unsigned)(N - 1);
    }
  }
  __syncthreads();
  if (!s_last || tid >= 32) return;
  __threadfence();
  float prj = 0.f, pn = 0.f;
  for (int i = lane; i < N; i += 32) { prj += __ldcg(ws.inst_prj + i); pn += __ldcg(ws.inst_num + i); }
  prj = warp_sum(prj);
  pn = warp_sum(pn);
  if (lane == 0) {
    losses_out[0] = prj * inv_n;
    losses_out[1] = pn * scale;
    losses_out[2] = pn;
    losses_out[3] = (float)wtot;
    sched->ticket = 0u;          // every CTA of this grid has read wtot before taking its ticket
    sched->wtot = 0ull;
  }
}

// ---------------------------------------------------------------------------------------
// backward: the gradient for upstream gradients (1, 1) is already in place (finalize); anything else converts it in
// place, exactly: span *= g_pair, arg-max positions = g_pair * saved pairwise part + g_prj * coefficients.
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(OP_FIN_NT)
onepass_backward_kernel(int H, int W, OpWorkspace ws, const float* __restrict__ g_prj_p,
                        const float* __restrict__ g_pair_p, float* __restrict__ g_logits) {
  __shared__ int s_ar[512], s_ac[512];
  __shared__ float s_cr[512];
  asm volatile("griddepcontrol.wait;" ::: "memory");     // everything below may read the previous kernel's results
  const float gp = g_prj_p[0], gq = g_pair_p[0];
  if (gp == 1.f && gq == 1.f) return;
  const int n = blockIdx.x, tid = threadIdx.x;
  float* ginst = g_logits + (unsigned)(n * H * W);
  const int4 sp = reinterpret_cast<const int4*>(ws.span)[n];
  int ar = 0, ac = 0;
  float cr = 0.f, cc = 0.f, svr = 0.f, svc = 0.f;
  if (tid < H) { ar = ws.arg_row[n * H + tid]; cr = ws.coef_row[n * H + tid] * gp; svr = ws.sv_row[n * H + tid] * gq; s_ar[tid] = ar; s_cr[tid] = cr; }
  if (tid < W) { ac = ws.arg_col[n * W + tid]; cc = ws.coef_col[n * W + tid] * gp; svc = ws.sv_col[n * W + tid] * gq; s_ac[tid] = ac; }
  const int sw4 = (sp.w - sp.z + 1) >> 2, srows = sp.y - sp.x + 1;
  if (srows > 0) {
    for (int i = tid; i < srows * sw4; i += OP_FIN_NT) {
      const int ry = op_div(i, sw4), c4 = i - ry * sw4;
      float4* p = reinterpret_cast<float4*>(ginst + (sp.x + ry) * W + sp.z + 4 * c4);
      float4 q = *p;
      q.x *= gq; q.y *= gq; q.z *= gq; q.w *= gq;
      *p = q;
    }
  }
  __syncthreads();
  if (tid < H && s_ac[ar] != tid) ginst[tid * W + ar] = svr + cr;
  if (tid < W) ginst[ac * W + tid] = s_ar[ac] == tid ? (svc + s_cr[ac]) + cc : svc + cc;
}

// ---------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------
// launch with programmatic stream serialization: the kernel may start while its predecessor in the stream drains
// (it calls griddepcontrol.wait before touching the predecessor's results)
template <typename... KArgs, typename... Args>
inline cudaError_t op_launch_pdl(void (*kern)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, static_cast<KArgs>(args)...);
}

inline bool op_supported(int64_t N, int64_t H, int64_t W, int d) {
  return N > 0 && N <= OP_MAX_N && H > 0 && H <= 512 && W > 0 && W <= 512 && (W % 4 == 0) && d >= 1 && d <= 4;
}

inline size_t op_smem_bytes(int64_t N, int64_t W) {
  return (size_t)OP_STAGES * OP_R * W * 4 + (size_t)N * sizeof(SRec) + (size_t)(N + 1) * 4;
}

template <int NCHUNK, int D, bool FULLW>
int op_launch_main(cudaStream_t st, const float* logits, const uint8_t* edge_bits, const int32_t* rects,
                   const int32_t* inst_gt, const int32_t* gt_img, int N, int H, int W, OpWorkspace ws, OpSched* sched,
                   float* g_logits) {
  const size_t smem = op_smem_bytes(N, W);
  auto kern = onepass_main_kernel<NCHUNK, D, FULLW>;
  if (opt_in_smem(kern, smem) != BXS_OK) return BXS_ERR_UNSUPPORTED;
  const int occ = max_active_ctas(kern, OP_NT, smem);
  if (occ < 1) return BXS_ERR_UNSUPPORTED;
  const int S = (int)ceil_div(H, OP_R);
  const int64_t total = (int64_t)N * S;           // stream items alone; pair items come on top
  const int grid = (int)std::min<int64_t>(total, (int64_t)sm_count() * occ);
  kern<<<grid, OP_NT, smem, st>>>(logits, edge_bits, rects, inst_gt, gt_img, N, H, W, S, (int)op_max_groups(H, W), ws, sched,
                                  g_logits);
  return check_launch();
}

#include "boxinst_warpq.cuh"

// which schedule bxs_boxinst_loss_fused_forward runs: the warp-granular queue (default) or, with
// BXS_ONEPASS_CTA=1 in the environment, the CTA-granular kernels above (kept for A/B measurements on one box)
inline bool op_use_cta_schedule() {
  static const bool v = [] { const char* e = getenv("BXS_ONEPASS_CTA"); return e && e[0] == '1'; }();
  return v;
}

}  // namespace
}  // namespace bxs

using namespace bxs;

#ifdef BXS_OP_TRACE
extern "C" int bxs_debug_set_trace(void* buf) {
  return cudaMemcpyToSymbol(g_op_trace, &buf, sizeof(buf)) == cudaSuccess ? 0 : -2;
}
#endif

extern "C" int bxs_boxinst_loss_fused_supported(int64_t N, int64_t H, int64_t W, int dilation) {
  return op_supported(N, H, W, dilation) ? 1 : 0;
}

// workspace = the forward->backward tables (op_carve) followed by room for a plan (used when the caller passes none)
extern "C" int64_t bxs_boxinst_loss_fused_workspace_bytes(int64_t N, int64_t H, int64_t W) {
  if (N <= 0 || H <= 0 || W <= 0) return 0;
  size_t plan = 0;
  for (int d = 1; d <= 4; ++d) plan = std::max(plan, wq_plan_bytes(N, H, W, d));
  return (int64_t)(align_up(op_carve(nullptr, N, H, W).total_bytes) + plan);
}

extern "C" int64_t bxs_boxinst_loss_fused_sched_bytes(void) {
  return (int64_t)std::max(sizeof(OpSched), sizeof(WqSched));
}

extern "C" int64_t bxs_boxinst_loss_plan_bytes(int64_t N, int64_t H, int64_t W, int dilation) {
  if (N <= 0 || H <= 0 || W <= 0 || dilation < 1 || dilation > 4) return 0;
  return (int64_t)wq_plan_bytes(N, H, W, dilation);
}

extern "C" int bxs_boxinst_loss_plan(const uint8_t* edge_bits, const int32_t* rects, const int32_t* inst_gt,
                                     const int32_t* gt_img, void* plan, int64_t N, int64_t H, int64_t W, int dilation,
                                     bxs_stream_t stream) {
  if (!edge_bits || !rects || !inst_gt || !gt_img || !plan || N <= 0 || H <= 0 || W <= 0) return BXS_ERR_INVALID_ARG;
  if (!op_supported(N, H, W, dilation)) return BXS_ERR_UNSUPPORTED;
  return wq_build_plan(as_stream(stream), edge_bits, rects, inst_gt, gt_img, reinterpret_cast<unsigned char*>(plan), (int)N,
                       (int)H, (int)W, dilation);
}

extern "C" int bxs_boxinst_loss_fused_forward_planned(const float* logits, const uint8_t* edge_bits, void* plan,
                                                      const float* iter_ptr, float warmup_iters, void* workspace,
                                                      void* sched_state, float* losses_out, float* g_logits, int64_t N,
                                                      int64_t H, int64_t W, int dilation, bxs_stream_t stream) {
  if (!logits || !edge_bits || !plan || !iter_ptr || !workspace || !sched_state || !losses_out || !g_logits || N <= 0 ||
      H <= 0 || W <= 0 || !(warmup_iters > 0.f))
    return BXS_ERR_INVALID_ARG;
  if (!op_supported(N, H, W, dilation) || (reinterpret_cast<uintptr_t>(logits) & 15) ||
      (reinterpret_cast<uintptr_t>(g_logits) & 15) || (reinterpret_cast<uintptr_t>(plan) & 15))
    return BXS_ERR_UNSUPPORTED;
  return wq_forward(as_stream(stream), logits, edge_bits, reinterpret_cast<unsigned char*>(plan), iter_ptr, warmup_iters,
                    op_carve(workspace, N, H, W), reinterpret_cast<WqSched*>(sched_state), losses_out, g_logits, (int)N, (int)H,
                    (int)W, dilation);
}

extern "C" int bxs_boxinst_loss_fused_forward(const float* logits, const uint8_t* edge_bits, const int32_t* rects,
                                              const int32_t* inst_gt, const int32_t* gt_img, const float* iter_ptr,
                                              float warmup_iters, void* workspace, void* sched_state,
                                              float* losses_out, float* g_logits, int64_t N, int64_t H, int64_t W,
                                              int dilation, bxs_stream_t stream) {
  if (!logits || !edge_bits || !rects || !inst_gt || !gt_img || !iter_ptr || !workspace || !sched_state ||
      !losses_out || !g_logits || N <= 0 || H <= 0 || W <= 0 || !(warmup_iters > 0.f))
    return BXS_ERR_INVALID_ARG;
  if (!op_supported(N, H, W, dilation) || (reinterpret_cast<uintptr_t>(logits) & 15) ||
      (reinterpret_cast<uintptr_t>(g_logits) & 15))
    return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  OpWorkspace ws = op_carve(workspace, N, H, W);
  if (!op_use_cta_schedule()) {            // plan in the tail of the workspace, then the warp-granular kernel
    unsigned char* plan = reinterpret_cast<unsigned char*>(workspace) + align_up(ws.total_bytes);
    const int prc = wq_build_plan(st, edge_bits, rects, inst_gt, gt_img, plan, (int)N, (int)H, (int)W, dilation);
    if (prc != BXS_OK) return prc;
    return wq_forward(st, logits, edge_bits, plan, iter_ptr, warmup_iters, ws, reinterpret_cast<WqSched*>(sched_state),
                      losses_out, g_logits, (int)N, (int)H, (int)W, dilation);
  }
  OpSched* sched = reinterpret_cast<OpSched*>(sched_state);
  const int S = (int)ceil_div(H, OP_R);
  int rc = BXS_ERR_UNSUPPORTED;
#define BXS_OP_CASE(NC, DD)                                                                                          \
  rc = (W == NC * 128) ? op_launch_main<NC, DD, true>(st, logits, edge_bits, rects, inst_gt, gt_img, (int)N, (int)H,  \
                                                      (int)W, ws, sched, g_logits)                                  \
                       : op_launch_main<NC, DD, false>(st, logits, edge_bits, rects, inst_gt, gt_img, (int)N, (int)H, \
                                                       (int)W, ws, sched, g_logits);                                \
  if (rc == BXS_OK) {                                                                                               \
    op_launch_pdl(onepass_finalize_kernel<DD>, dim3((unsigned)N), dim3(OP_FIN_NT), 0, st, rects, inst_gt, gt_img, (int)N, \
                  (int)H, (int)W, S, (int)op_max_groups(H, W), ws, sched, iter_ptr, warmup_iters, losses_out, g_logits); \
    rc = check_launch();                                                                                            \
  }
#define BXS_OP_D(NC)                                                  \
  switch (dilation) {                                                 \
    case 1: { BXS_OP_CASE(NC, 1) } break;                             \
    case 2: { BXS_OP_CASE(NC, 2) } break;                             \
    case 3: { BXS_OP_CASE(NC, 3) } break;                             \
    default: { BXS_OP_CASE(NC, 4) } break;                            \
  }
  if (W <= 128) { BXS_OP_D(1) }
  else if (W <= 256) { BXS_OP_D(2) }
  else { BXS_OP_D(4) }
#undef BXS_OP_D
#undef BXS_OP_CASE
  return rc;
}

extern "C" int bxs_boxinst_loss_fused_backward(const void* workspace, const float* g_prj, const float* g_pair,
                                               float* g_logits, int64_t N, int64_t H, int64_t W,
                                               bxs_stream_t stream) {
  if (!workspace || !g_prj || !g_pair || !g_logits || N <= 0 || H <= 0 || W <= 0) return BXS_ERR_INVALID_ARG;
  OpWorkspace ws = op_carve(const_cast<void*>(workspace), N, H, W);
  op_launch_pdl(onepass_backward_kernel, dim3((unsigned)N), dim3(OP_FIN_NT), 0, as_stream(stream), (int)H, (int)W, ws, g_prj,
                g_pair, g_logits);
  return check_launch();
}
