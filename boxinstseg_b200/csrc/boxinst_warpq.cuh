// a6 + a7 + a8, single pass, second schedule: ONE persistent kernel whose unit of work is a WARP item, plus a small
// finalize kernel.  (Included by boxinst_onepass.cu inside namespace bxs::{anonymous}; shares SRec / op_span /
// chain_geom / op_chain and the PTX wrappers with the CTA-granular schedule there.)
//
// Why: the CTA-granular kernel (onepass_main_kernel) spent 31 % of its duration with SMs idle (per-CTA prologue of
// 128 record loads + a block scan, a tail of CTA-wide pair items), its top stall was the CTA barrier around the strip
// buffers, and its finalize kernel re-scaled the whole box span.  Here
//   * the work list is a PLAN built once per target set (wq_count_kernel + wq_build_kernel): instance records, every
//     pair item as a 32-byte descriptor (long chains first) and the logit-independent weight total -- the main kernel
//     has no prologue beyond one header load;
//   * every item is processed by ONE warp, there is no CTA barrier anywhere:
//       - stream item = 24 rows x W of one instance, owned STATICALLY by one of the WQ_STREAMERS streamer warps of a
//         CTA (a queue atomic costs microseconds under load; the streamers are the long pole).  The logits flow
//         through the warp's own 4-stage shared-memory ring, one cp.async.bulk (TMA engine) per 4-row group
//         completing on the warp's own mbarrier, 3 groups in flight ACROSS item boundaries.  Row maxima by integer
//         redux + ballot; per-item column maxima with the 4-row group that holds them; float4 zero stores of the
//         gradient outside the box span;
//       - pair item = one chain (op_chain) = 8 rows of a 32-lane column segment; the weight total is known from the
//         plan, so the chain stores the FINAL scaled pairwise gradient (no second pass over the span).  The other
//         warps (and the streamers once the stream queue is empty) pull them from the pair queue;
//   * the loss sums are 64-bit fixed-point atomics (order-independent => deterministic);
//   * wq_finalize_kernel (one CTA per instance) resolves the exact arg-max positions, the dice terms and their
//     gradient coefficients and adds them at the H + W arg-max positions.  It is released by a flag the main kernel's
//     last warp publishes, not by the main grid's retirement.
// Every gradient element is written by exactly one warp and every sum is either fixed-order or integer: results do not
// depend on which warp processed which item.

constexpr int WQ_NT = 256;          // threads per CTA
constexpr int WQ_NW = WQ_NT / 32;
constexpr int WQ_SUB = 4;           // rows per ring stage (one bulk copy)
#ifndef BXS_WQ_R
#define BXS_WQ_R 24
#endif
#ifndef BXS_WQ_STREAMERS
#define BXS_WQ_STREAMERS 2
#endif
constexpr int WQ_R = BXS_WQ_R;      // rows per stream item (tunable at build time for A/B runs: tools/ab_variants.sh)
constexpr int WQ_RING = 4;          // ring stages of a streamer warp
constexpr int WQ_STREAMERS = BXS_WQ_STREAMERS;     // warps per CTA that take stream items first (the others take pair items)
constexpr double WQ_NUM_FX = 16777216.0;            // 2^24: fixed-point scale of the pairwise numerator
constexpr double WQ_PRJ_FX = 4294967296.0;          // 2^32: fixed-point scale of the projection terms (N <= 2048 terms <= 2 fit 48 bits)
static_assert(WQ_R % WQ_SUB == 0 && WQ_R / WQ_SUB <= 16, "stream items start on a 4-row group; <= 16 groups per item (4-bit fields)");

struct WqHeader {                   // first 64 bytes of the plan
  int total, n_pair, n_stream, S;
  int N, H, W, D;
  unsigned long long wtot;          // sum over instances of the edge bits set inside their boxes
  int pad[6];
};
static_assert(sizeof(WqHeader) == 64, "plan header is 64 bytes");

// 32-byte pair item.  a = {n, y0 | nrows << 16, xs | c_hi << 16, 0}   b = {j0 | j1 << 16, i0 | i1 << 16, image, 0}
struct __align__(16) WqItem { int4 a, b; };

struct WqSched {                    // device state: zero before the first call, left zero by every call
  unsigned next_s, next_p, done, ticket;      // stream / pair queue positions, main-kernel warps arrived, (unused)
  unsigned long long num_fx, prj_fx;          // fixed-point loss sums
};

inline int wq_strips(int64_t H) { return (int)ceil_div(H, WQ_R); }
inline int64_t wq_max_chains(int64_t H, int64_t W, int d) {
  const int64_t nseg = ceil_div(W + 4, 32 - 2 * d) + 1, pc = ceil_div(ceil_div(H, d), OP_LEN) + 1;
  return d * pc * nseg;
}
// plan layout: header (64 B) | inst_w [N] uint32 | recs [N] int4 (j0, j1, i0, i1) | pair items
__host__ __device__ inline size_t wq_plan_rec_offset(int64_t N) { return (64 + 4 * (size_t)N + 63) / 64 * 64; }
__host__ __device__ inline size_t wq_plan_items_offset(int64_t N, int64_t /*W*/) {
  return (wq_plan_rec_offset(N) + 16 * (size_t)N + 63) / 64 * 64;
}
inline size_t wq_plan_bytes(int64_t N, int64_t H, int64_t W, int d) {
  return wq_plan_items_offset(N, W) + (size_t)N * (size_t)wq_max_chains(H, W, d) * sizeof(WqItem);
}

__device__ __forceinline__ int wq_pack16(int lo, int hi) { return (lo & 0xffff) | (hi << 16); }
__device__ __forceinline__ int wq_lo16(int v) { return (int)(short)(v & 0xffff); }
__device__ __forceinline__ int wq_hi16(int v) { return v >> 16; }

// ---------------------------------------------------------------------------------------
// plan, step 1: per-instance weight count = edge bits set inside the box (one CTA per instance)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
wq_count_kernel(const uint8_t* __restrict__ edge_bits, const int32_t* __restrict__ rects,
                const int32_t* __restrict__ inst_gt, const int32_t* __restrict__ gt_img, int H, int W,
                unsigned* __restrict__ inst_w) {
  __shared__ int s_red[4];
  const int n = blockIdx.x, tid = threadIdx.x;
  const SRec r = make_srec(rects, inst_gt, gt_img, n, H, W);
  int cnt = 0;
  if (r.j0 <= r.j1) {
    const uint8_t* bits = edge_bits + (int64_t)r.img * H * W;
    const int bw = r.i1 - r.i0 + 1, tot = (r.j1 - r.j0 + 1) * bw;
    for (int i = tid; i < tot; i += 128) {
      const int ry = i / bw, rx = i - ry * bw;
      cnt += __popc((unsigned)__ldg(bits + (r.j0 + ry) * W + r.i0 + rx));
    }
  }
  cnt = warp_sum(cnt);
  if ((tid & 31) == 0) s_red[tid >> 5] = cnt;
  __syncthreads();
  if (tid == 0) inst_w[n] = (unsigned)(s_red[0] + s_red[1] + s_red[2] + s_red[3]);
}

// chains of one instance by length: `full` = pieces of OP_LEN rows, `part` = the shorter last piece of a parity class
template <int D>
__device__ __forceinline__ void wq_chain_counts(const ChainGeom& cg, int& full, int& part) {
  full = 0; part = 0;
  if (cg.rows <= 0) return;
#pragma unroll
  for (int p = 0; p < D; ++p) {
    const int rows_p = (cg.rows - p + D - 1) / D;
    if (rows_p <= 0) continue;
    full += (rows_p / OP_LEN) * cg.nseg;
    part += (rows_p % OP_LEN) ? cg.nseg : 0;
  }
}

// ---------------------------------------------------------------------------------------
// plan, step 2: the pair queue (one CTA).  Instances are ranked by chain count (large boxes first); the queue holds
// all full-length chains in rank order, then the shorter ones: longest-processing-time-first, so the dynamic queue
// ends with its cheapest items.  Stream items need no descriptors: item q = rows [8 s, 8 s + 8) of instance q / S.
// ---------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(1024)
wq_build_kernel(const int32_t* __restrict__ rects, const int32_t* __restrict__ inst_gt,
                const int32_t* __restrict__ gt_img, int N, int H, int W, unsigned char* __restrict__ plan) {
  __shared__ int s_full[OP_MAX_N], s_part[OP_MAX_N];
  __shared__ int s_order[OP_MAX_N];
  __shared__ int s_pre_f[OP_MAX_N + 1], s_pre_p[OP_MAX_N + 1];
  __shared__ int s_scan[2][32];
  __shared__ unsigned long long s_w[32];
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const unsigned* inst_w = reinterpret_cast<const unsigned*>(plan + 64);
  int4* recs = reinterpret_cast<int4*>(plan + wq_plan_rec_offset(N));
  const int S = (H + WQ_R - 1) / WQ_R;
  unsigned long long wsum = 0ull;
  for (int n = tid; n < N; n += 1024) {
    const SRec r = make_srec(rects, inst_gt, gt_img, n, H, W);
    recs[n] = make_int4(r.j0, r.j1, r.i0, r.i1);
    int f, p;
    wq_chain_counts<D>(chain_geom<D>(r, H, W), f, p);
    s_full[n] = f; s_part[n] = p;
    wsum += inst_w[n];
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) wsum += __shfl_xor_sync(kFull, wsum, o);
  if (lane == 0) s_w[wid] = wsum;
  __syncthreads();
  // rank (descending chain count, ties by instance id) -> order
  for (int n = tid; n < N; n += 1024) {
    const int c = s_full[n] + s_part[n];
    int rank = 0;
    for (int m = 0; m < N; ++m) {
      const int cm = s_full[m] + s_part[m];
      rank += (cm > c || (cm == c && m < n)) ? 1 : 0;
    }
    s_order[rank] = n;
  }
  __syncthreads();
  // exclusive prefixes of the full / partial chain counts in rank order (two elements per thread)
  {
    const int i0 = 2 * tid, i1 = 2 * tid + 1;
    const int f0 = i0 < N ? s_full[s_order[i0]] : 0, f1 = i1 < N ? s_full[s_order[i1]] : 0;
    const int p0 = i0 < N ? s_part[s_order[i0]] : 0, p1 = i1 < N ? s_part[s_order[i1]] : 0;
    int incf = f0 + f1, incp = p0 + p1;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int tf = __shfl_up_sync(kFull, incf, o), tp = __shfl_up_sync(kFull, incp, o);
      if (lane >= o) { incf += tf; incp += tp; }
    }
    if (lane == 31) { s_scan[0][wid] = incf; s_scan[1][wid] = incp; }
    __syncthreads();
    int bf = 0, bp = 0;
    for (int i = 0; i < wid; ++i) { bf += s_scan[0][i]; bp += s_scan[1][i]; }
    const int ef = bf + incf - (f0 + f1), ep = bp + incp - (p0 + p1);
    if (i0 < N) { s_pre_f[i0] = ef; s_pre_p[i0] = ep; }
    if (i1 < N) { s_pre_f[i1] = ef + f0; s_pre_p[i1] = ep + p0; }
    if (tid == 1023) { s_pre_f[N] = bf + incf; s_pre_p[N] = bp + incp; }   // N <= 2048 = 2 * 1024
  }
  __syncthreads();
  const int Pf = s_pre_f[N], Pp = s_pre_p[N], P = Pf + Pp, T = N * S;
  if (tid == 0) {
    WqHeader h{};
    h.total = P + T; h.n_pair = P; h.n_stream = T; h.S = S; h.N = N; h.H = H; h.W = W; h.D = D;
    unsigned long long w = 0ull;
    for (int i = 0; i < 32; ++i) w += s_w[i];
    h.wtot = w;
    *reinterpret_cast<WqHeader*>(plan) = h;
  }
  WqItem* items = reinterpret_cast<WqItem*>(plan + wq_plan_items_offset(N, W));
  for (int q = tid; q < P; q += 1024) {
    const bool is_full = q < Pf;
    const int* pre = is_full ? s_pre_f : s_pre_p;
    const int idx = is_full ? q : q - Pf;
    int lo = 0, hi = N;                     // largest r with pre[r] <= idx
    while (hi - lo > 1) {
      const int mid = (lo + hi) >> 1;
      if (pre[mid] <= idx) lo = mid; else hi = mid;
    }
    const int n = s_order[lo];
    int c = idx - pre[lo];
    const SRec r = make_srec(rects, inst_gt, gt_img, n, H, W);
    const ChainGeom cg = chain_geom<D>(r, H, W);
    int p = 0, piece = 0, seg = 0, nrows = 0;
#pragma unroll
    for (int pp = 0; pp < D; ++pp) {
      const int rows_p = (cg.rows - pp + D - 1) / D;
      if (rows_p <= 0 || c < 0) continue;
      const int cnt = is_full ? (rows_p / OP_LEN) * cg.nseg : ((rows_p % OP_LEN) ? cg.nseg : 0);
      if (c < cnt) {
        p = pp;
        piece = is_full ? c / cg.nseg : rows_p / OP_LEN;
        seg = is_full ? c - piece * cg.nseg : c;
        nrows = is_full ? OP_LEN : rows_p % OP_LEN;
        c = -1;                               // found
      } else {
        c -= cnt;
      }
    }
    WqItem it;
    it.a = make_int4(n, wq_pack16(cg.y_lo + p + D * piece * OP_LEN, nrows),
                     wq_pack16(cg.c_lo - D + seg * (32 - 2 * D), cg.c_hi), 0);
    it.b = make_int4(wq_pack16(r.j0, r.j1), wq_pack16(r.i0, r.i1), r.img, 0);
    items[q] = it;
  }
}

#ifdef BXS_OP_TRACE
// diagnostic build only (tools/trace_wq.py): per-WARP event log {globaltimer, tag}; 16 slots per warp
#define WQ_TRACE(tag)                                                                          \
  if (lane == 0 && g_op_trace && trace_slot < 16) {                                             \
    unsigned long long t_;                                                                     \
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));                                     \
    const size_t w_ = (size_t)blockIdx.x * WQ_NW + warp;                                       \
    g_op_trace[(w_ * 16 + trace_slot) * 2] = t_;                                               \
    g_op_trace[(w_ * 16 + trace_slot) * 2 + 1] = (unsigned long long)(tag);                    \
    ++trace_slot;                                                                              \
  }
#else
#define WQ_TRACE(tag)
#endif

// ---------------------------------------------------------------------------------------
// main kernel.  Items are independent (no completion protocol).
//   row results    row_packed[n*H + y] = key(max logit of the row) << 32 | ~(first float4 group holding it)
//   column results col_part[(n*S + s)*W + x] = key(max logit of column x within stream item s) << 32 | ~(first 4-row
//                                               group of the item holding it)
// (the exact element / row inside the group is resolved by the finalize kernel, one thread per row / column: the
//  first one that equals the maximum, like torch.max(dim))
// ---------------------------------------------------------------------------------------
template <int NCHUNK, int D, bool FULLW>
__global__ void __launch_bounds__(WQ_NT, NCHUNK <= 2 ? 4 : 1)
wq_main_kernel(const float* __restrict__ logits, const uint8_t* __restrict__ edge_bits,
               unsigned char* __restrict__ plan, int N, int H, int W_rt, int NS,
               unsigned long long* __restrict__ row_packed, unsigned long long* __restrict__ col_part,
               WqSched* __restrict__ sched, const float* __restrict__ iter_ptr, float warmup_iters,
               float* __restrict__ g_logits) {
  const int W = FULLW ? NCHUNK * 128 : W_rt;
  extern __shared__ __align__(128) unsigned char wq_smem[];
  __shared__ __align__(8) uint64_t s_bar[WQ_STREAMERS][WQ_RING];
  __shared__ unsigned s_exit;            // warps of this CTA that have finished
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int stage_floats = WQ_SUB * W;
#ifdef BXS_OP_TRACE
  int trace_slot = 0;
#endif
  WQ_TRACE(1);
  asm volatile("griddepcontrol.launch_dependents;");
  if (warp < WQ_STREAMERS && lane == 0) {
#pragma unroll
    for (int i = 0; i < WQ_RING; ++i) op_mbar_init(&s_bar[warp][i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  if (threadIdx.x == 0) s_exit = 0u;
  __syncthreads();                                         // the only CTA-wide barrier of this kernel
  asm volatile("griddepcontrol.wait;" ::: "memory");     // the plan, the scheduler state and the workspace may belong to the predecessor
  const WqHeader* hdr = reinterpret_cast<const WqHeader*>(plan);
  const int S = (H + WQ_R - 1) / WQ_R, T = N * S;

  if (warp < WQ_STREAMERS) {
    // ======================================= streamer =======================================
    float* ring = reinterpret_cast<float*>(wq_smem) + (size_t)warp * WQ_RING * stage_floats;
    uint64_t* bar = s_bar[warp];
    const int4* __restrict__ recs = reinterpret_cast<const int4*>(plan + wq_plan_rec_offset(N));
    // Stream items are STATIC: streamer slot i < NS owns items i, i + NS, ... (NS is chosen by the host so that every
    // streamer owns the same number of items).  A queue atomic costs microseconds under load and a stream item is the
    // long pole of the kernel, so nothing on this path waits for one.  q0 is being processed, q1 is next (its groups
    // may already be in flight).
    const int slot = (int)(blockIdx.x * WQ_STREAMERS + warp);
    int q0 = slot < NS && slot < T ? slot : -1;
    int q1 = q0 >= 0 && q0 + NS < T ? q0 + NS : -1;
    int4 rec0 = make_int4(1, 0, 1, 0), rec1 = rec0;
    if (q0 >= 0) rec0 = __ldg(recs + q0 / S);
    if (q1 >= 0) rec1 = __ldg(recs + q1 / S);
    int gi = 0, gp = 0;              // 4-row groups issued / processed so far (ring stage = g & 3, parity = (g >> 2) & 1)
    int iq = 0, ik = 0;              // issue cursor: item (0 = q0, 1 = q1), group within it
    auto issue_one = [&]() {
      const int q = iq == 0 ? q0 : (iq == 1 ? q1 : -1);
      if (q < 0) return;
      const int n = q / S, row0 = (q - n * S) * WQ_R, nrows = min(WQ_R, H - row0);
      if (lane == 0) {
        const uint32_t bytes = (uint32_t)min(WQ_SUB, nrows - ik * WQ_SUB) * (uint32_t)W * 4u;
        uint64_t* bb = &bar[gi & (WQ_RING - 1)];
        op_mbar_expect_tx(bb, bytes);
        op_bulk_g2s(ring + (gi & (WQ_RING - 1)) * stage_floats, logits + ((size_t)n * H + row0) * W + (size_t)ik * stage_floats,
                    bytes, bb);
      }
      ++gi;
      if (++ik == (nrows + WQ_SUB - 1) / WQ_SUB) { ik = 0; ++iq; }
    };
#pragma unroll
    for (int i = 0; i < WQ_RING - 1; ++i) issue_one();
    while (q0 >= 0) {
      const int n = q0 / S, s_idx = q0 - n * S;
      const int row0 = s_idx * WQ_R, nrows = min(WQ_R, H - row0);
      SRec rec;
      rec.j0 = (short)rec0.x; rec.j1 = (short)rec0.y; rec.i0 = (short)rec0.z; rec.i1 = (short)rec0.w; rec.img = 0;
      const OpSpan sp = op_span<D>(rec, H, W);
      const int ya = max(row0, sp.y_lo), yb = min(row0 + nrows - 1, sp.y_hi);    // ya > yb: no span row in this item
      const int c_lo = sp.c_lo, c_hi = sp.c_hi;
      WQ_TRACE(2 + ((unsigned long long)n << 8));
      const int nsub = (nrows + WQ_SUB - 1) / WQ_SUB;
      float cbest[NCHUNK][4];            // column maxima of this item ...
      unsigned cpk[(NCHUNK + 1) / 2];    // ... and the 4-row group (0..5 within the item) that holds each: 4-bit fields
#pragma unroll
      for (int ch = 0; ch < NCHUNK; ++ch)
#pragma unroll
        for (int e = 0; e < 4; ++e) cbest[ch][e] = -INFINITY;
#pragma unroll
      for (int i = 0; i < (NCHUNK + 1) / 2; ++i) cpk[i] = 0u;
      unsigned long long* rdst = row_packed + (size_t)n * H + row0;
      float* grow = g_logits + ((size_t)n * H + row0) * W + lane * 4;
      const int sub0 = row0 / WQ_SUB;
      int y = row0;
      for (int k = 0; k < nsub; ++k) {
        const int st = gp & (WQ_RING - 1);
        op_mbar_wait(&bar[st], (unsigned)(gp >> 2) & 1u);
        const float* xb = ring + st * stage_floats + lane * 4;
        const int rows_here = min(WQ_SUB, nrows - k * WQ_SUB);
        float gm[NCHUNK][4];                 // column maxima of this 4-row group
#pragma unroll
        for (int ch = 0; ch < NCHUNK; ++ch)
#pragma unroll
          for (int e = 0; e < 4; ++e) gm[ch][e] = -INFINITY;
#pragma unroll
        for (int r = 0; r < WQ_SUB; ++r) {
          if (r < rows_here) {                                         // warp-uniform
            float cm[NCHUNK];
#pragma unroll
            for (int ch = 0; ch < NCHUNK; ++ch) {
              float4 q;
              if (FULLW || (ch * 32 + lane) * 4 < W) q = *reinterpret_cast<const float4*>(xb + r * W + ch * 128);
              else q = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
              cm[ch] = fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w));
              gm[ch][0] = fmaxf(gm[ch][0], q.x); gm[ch][1] = fmaxf(gm[ch][1], q.y);
              gm[ch][2] = fmaxf(gm[ch][2], q.z); gm[ch][3] = fmaxf(gm[ch][3], q.w);
            }
            float m = cm[0];
#pragma unroll
            for (int ch = 1; ch < NCHUNK; ++ch) m = fmaxf(m, cm[ch]);
            const unsigned kmax = __reduce_max_sync(kFull, fkey(m));
            const float mv = fkey_inv(kmax);
            // first float4 group (lowest columns) that holds the row maximum: chunk-major, then lane
            unsigned bal = __ballot_sync(kFull, cm[0] == mv);
            int grp = 0;
#pragma unroll
            for (int ch = 1; ch < NCHUNK; ++ch) {
              const unsigned b = __ballot_sync(kFull, cm[ch] == mv);
              if (bal == 0u) { bal = b; grp = ch * 32; }
            }
            grp += bal ? __ffs(bal) - 1 : 0;                          // bal == 0 only for an all-NaN row: any in-range group
            if (lane == 0) rdst[y - row0] = pack_key(kmax, grp);
            // zero part of the gradient: everything outside the span (the chains write the span)
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            if (y >= ya && y <= yb) {                                  // warp-uniform: a span row
#pragma unroll
              for (int ch = 0; ch < NCHUNK; ++ch) {
                const int col0 = (ch * 32 + lane) * 4;
                if ((FULLW || col0 < W) && (col0 < c_lo || col0 > c_hi)) *reinterpret_cast<float4*>(grow + ch * 128) = z;
              }
            } else {
#pragma unroll
              for (int ch = 0; ch < NCHUNK; ++ch)
                if (FULLW || (ch * 32 + lane) * 4 < W) *reinterpret_cast<float4*>(grow + ch * 128) = z;
            }
            grow += W;
            ++y;
          }
        }
        // column maxima: the first 4-row group wins ties
#pragma unroll
        for (int ch = 0; ch < NCHUNK; ++ch)
#pragma unroll
          for (int e = 0; e < 4; ++e)
            if (gm[ch][e] > cbest[ch][e]) {
              cbest[ch][e] = gm[ch][e];
              constexpr unsigned kDummy = 0u; (void)kDummy;
              const int f = ch * 4 + e;
              asm("bfi.b32 %0, %1, %0, %2, 4;" : "+r"(cpk[f >> 3]) : "r"(k), "r"((f & 7) * 4));
            }
        __syncwarp();                        // every lane has read stage st
        ++gp;
        issue_one();                         // refill the ring: the stage read one group ago is free
      }
      unsigned long long* cdst = col_part + ((size_t)n * S + s_idx) * W;
#pragma unroll
      for (int ch = 0; ch < NCHUNK; ++ch) {
        const int col0 = (ch * 32 + lane) * 4;
        if (FULLW || col0 < W) {
          ulonglong2 p0, p1;
          const unsigned f4 = cpk[ch >> 1] >> ((ch & 1) * 16);       // this chunk's four 4-bit group fields
          p0.x = pack_key(fkey(cbest[ch][0]), sub0 + (int)(f4 & 15u)); p0.y = pack_key(fkey(cbest[ch][1]), sub0 + (int)((f4 >> 4) & 15u));
          p1.x = pack_key(fkey(cbest[ch][2]), sub0 + (int)((f4 >> 8) & 15u)); p1.y = pack_key(fkey(cbest[ch][3]), sub0 + (int)((f4 >> 12) & 15u));
          *reinterpret_cast<ulonglong2*>(cdst + col0) = p0;
          *reinterpret_cast<ulonglong2*>(cdst + col0 + 2) = p1;
        }
      }
      WQ_TRACE(4);
      // advance to this streamer's next item
      q0 = q1; rec0 = rec1; --iq;
      q1 = q0 >= 0 && q0 + NS < T ? q0 + NS : -1;
      if (q0 >= 0) {
        if (q1 >= 0) rec1 = __ldg(recs + q1 / S);
        if (iq < 0) iq = 0;
        while (gi - gp < WQ_RING - 1) {      // top the ring up (the item after next just became known)
          const int before = gi;
          issue_one();
          if (gi == before) break;
        }
      }
    }
  }

  // ======================================= pair queue =======================================
  const WqItem* __restrict__ items = reinterpret_cast<const WqItem*>(plan + wq_plan_items_offset(N, W));
  const unsigned long long wtot = __ldg(&hdr->wtot);
  const float scale = fminf(__ldg(iter_ptr) / warmup_iters, 1.f) / fmaxf((float)wtot, 1.f);
  const int n_pair = __ldg(&hdr->n_pair);
  const unsigned n_idle_slots = gridDim.x * WQ_STREAMERS > (unsigned)NS ? gridDim.x * WQ_STREAMERS - (unsigned)NS : 0u;
  const unsigned n_pair_static = gridDim.x * (WQ_NW - WQ_STREAMERS) + n_idle_slots;
  // the first pair item of a warp that did not stream is static; later ones (and a finished streamer's first) come from
  // the queue counter, fetched two items ahead of their use
  unsigned raw_l0 = 0xffffffffu;
  const int sslot = (int)(blockIdx.x * WQ_STREAMERS + warp);
  if (warp >= WQ_STREAMERS) raw_l0 = blockIdx.x * (WQ_NW - WQ_STREAMERS) + (warp - WQ_STREAMERS);
  else if (sslot >= NS) raw_l0 = gridDim.x * (WQ_NW - WQ_STREAMERS) + (unsigned)(sslot - NS);
  else if (lane == 0) raw_l0 = n_pair_static + atomicAdd(&sched->next_p, 1u);
  unsigned raw = __shfl_sync(kFull, raw_l0, 0);
  int q_cur = raw < (unsigned)n_pair ? (int)raw : -1;
  int4 ia = make_int4(0, 0, 0, 0), ib = ia;
  if (q_cur >= 0) { ia = __ldg(&items[q_cur].a); ib = __ldg(&items[q_cur].b); }
  if (lane == 0 && q_cur >= 0) raw_l0 = n_pair_static + atomicAdd(&sched->next_p, 1u);
  while (q_cur >= 0) {
    raw = __shfl_sync(kFull, raw_l0, 0);
    const int q_nxt = raw < (unsigned)n_pair ? (int)raw : -1;
    int4 na = make_int4(0, 0, 0, 0), nb = na;
    if (q_nxt >= 0) { na = __ldg(&items[q_nxt].a); nb = __ldg(&items[q_nxt].b); }
    if (lane == 0 && q_nxt >= 0) raw_l0 = n_pair_static + atomicAdd(&sched->next_p, 1u);
    const int n = ia.x;
    WQ_TRACE(3 + ((unsigned long long)n << 8));
    const int y0 = wq_lo16(ia.y), nrows = wq_hi16(ia.y);
    const int xs = wq_lo16(ia.z), c_hi = wq_hi16(ia.z);
    SRec rec;
    rec.j0 = (short)wq_lo16(ib.x); rec.j1 = (short)wq_hi16(ib.x);
    rec.i0 = (short)wq_lo16(ib.y); rec.i1 = (short)wq_hi16(ib.y);
    rec.img = ib.z;
    if (nrows > 0) {
      float acc_lg = 0.f, acc_slow = 0.f;
      int acc_w = 0;
      op_chain<D>(logits + (size_t)n * H * W, edge_bits + (size_t)rec.img * H * W, H, W, y0, nrows, xs, c_hi, rec, lane,
                  g_logits + (size_t)n * H * W, scale, acc_lg, acc_slow, acc_w);
      const float val = warp_sum(fmaf(acc_lg, -0.69314718055994531f, acc_slow));
      if (lane == 0 && val != 0.f)           // fixed-point sum: order-independent, hence deterministic
        atomicAdd(&sched->num_fx, (unsigned long long)__double2ll_rn((double)val * WQ_NUM_FX));
    }
    WQ_TRACE(4);
    q_cur = q_nxt; ia = na; ib = nb;
  }
  WQ_TRACE(7);
  // ---- arrival: this warp's results are fenced, then counted (nobody waits for the count here: the finalize CTAs
  //      poll it, and the last of them resets the queue counters) ----
  __syncwarp();
  if (lane == 0) {
#ifdef BXS_WQ_SC_FENCE
    __threadfence();                      // fence.sc.gpu + relaxed atomic (round 2a)
    atomicAdd(&sched->done, 1u);
#elif defined(BXS_WQ_WARP_ARRIVAL)
    // one RELEASE reduction per warp instead of a sequentially-consistent fence followed by a relaxed atomic
    asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(&sched->done) : "memory");
#else
    // Arrival per CTA: the warps count themselves in shared memory (acq_rel at CTA scope), the LAST one adds the whole CTA
    // to the global counter with one RELEASE reduction at GPU scope -- 592 reductions on one L2 address at the end of the
    // kernel instead of 4736 (they serialise there, right on the critical path of the finalize kernel's poll), and no
    // sequentially-consistent fence.  The other warps' stores reach the finalize CTAs by cumulativity: store -> release
    // (cta) -> acquire (cta) by the last warp -> release (gpu) -> acquire (gpu) by the poll.
    unsigned old;
    asm volatile("atom.acq_rel.cta.shared::cta.add.u32 %0, [%1], 1;" : "=r"(old) : "r"((unsigned)__cvta_generic_to_shared(&s_exit)) : "memory");
    if (old == WQ_NW - 1)
      asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(&sched->done), "r"((unsigned)WQ_NW) : "memory");
#endif
  }
}

// ---------------------------------------------------------------------------------------
// finalize: one CTA per instance, one thread per row and per column.  Resolves the arg-max positions, dice terms,
// gradient coefficients, adds the projection terms at the H + W arg-max positions for upstream gradients (1, 1)
// (a position that is both a row and a column arg-max is written once, by its column); the loss sums are 64-bit
// fixed-point atomics (order-independent); the last CTA (ticket) writes the four scalars.
// ---------------------------------------------------------------------------------------
template <int D>
__global__ void __launch_bounds__(OP_FIN_NT)
wq_finalize_kernel(const float* __restrict__ logits, unsigned char* __restrict__ plan, int N, int H, int W,
                   OpWorkspace ws, WqSched* __restrict__ sched, const float* __restrict__ iter_ptr, float warmup_iters,
                   float* __restrict__ losses_out, float* __restrict__ g_logits, int first_pass, unsigned main_warps) {
  constexpr int NWF = OP_FIN_NT / 32;
  __shared__ float s_f[4][NWF];
  __shared__ float s_coef[512];       // row coefficients
  __shared__ int s_arow[512], s_acol[512];
  const int n = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  asm volatile("griddepcontrol.launch_dependents;");
#ifdef BXS_OP_TRACE
  constexpr size_t kFinTrace = (size_t)148 * 4 * 8 * 16;          // after the main kernel's per-warp slots
  if (tid == 0 && g_op_trace) {
    unsigned long long t_;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));
    g_op_trace[(kFinTrace + blockIdx.x * 8 + 0) * 2] = t_;
  }
#endif
  // Launched with programmatic stream serialization and NOT waiting for the main grid to retire (griddepcontrol.wait
  // costs ~2.5 us after the last warp's exit: grid completion + flush): the CTAs become resident as main CTAs leave
  // and poll the main kernel's arrival counter (every warp fences its results, then counts itself in).  The main
  // kernel never waits for this one, so there is nothing to deadlock on.
  //
  // While it waits, a CTA runs the whole body ONCE AS A REHEARSAL (pass 0: every load in range by construction, every
  // global store / atomic switched off): this kernel runs once per SM per step, right after a 60 KB kernel, so its
  // instructions are never in the instruction caches when the flag arrives -- the trace (tools/trace_wq.py) showed
  // 2.9 us from release to the first loaded value on cold code, i.e. instruction fetch, not data.
  const WqHeader* hdr = reinterpret_cast<const WqHeader*>(plan);
  const float* xin = logits + (size_t)n * H * W;
  float* ginst = g_logits + (size_t)n * H * W;
  const int row_i = tid, col_i = tid;                   // H, W <= 512 = OP_FIN_NT
  const int S = (H + WQ_R - 1) / WQ_R;
  for (int pass = first_pass; pass < 2; ++pass) {
    const bool real = pass >= 1;
    if (real) {
      if (tid == 0) {
        unsigned arrived = 0u;                    // every main-kernel warp fences its results, then counts itself in
        for (;;) {
          asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(arrived) : "l"(&sched->done) : "memory");
          if (arrived >= main_warps) break;
          __nanosleep(32);
        }
      }
      __syncthreads();
#ifdef BXS_OP_TRACE
      if (tid == 0 && g_op_trace) {
        unsigned long long t_;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));
        g_op_trace[(kFinTrace + blockIdx.x * 8 + 1) * 2] = t_;
      }
#endif
    }
    const unsigned long long wtot = __ldg(&hdr->wtot);
    const int4 recv = __ldg(reinterpret_cast<const int4*>(plan + wq_plan_rec_offset(N)) + n);
    SRec rec;
    rec.j0 = (short)recv.x; rec.j1 = (short)recv.y; rec.i0 = (short)recv.z; rec.i1 = (short)recv.w; rec.img = 0;
    const bool empty = rec.j0 > rec.j1;
    // ---- independent loads: this thread's row result and its column's per-item keys ----
    unsigned long long rp = 0ull;
    if (row_i < H) rp = __ldcg(ws.row_packed + (size_t)n * H + row_i);
    unsigned long long cp = 0ull;
    if (col_i < W) {
      const unsigned long long* src = ws.col_part + (size_t)n * S * W + col_i;
      for (int s0 = 0; s0 < S; s0 += 12) {               // all loads of a batch first: one round trip for S <= 12
        unsigned long long v[12];
#pragma unroll
        for (int j = 0; j < 12; ++j) v[j] = s0 + j < S ? __ldcg(src + (size_t)(s0 + j) * W) : 0ull;
#pragma unroll
        for (int j = 0; j < 12; ++j) cp = v[j] > cp ? v[j] : cp;  // larger key; on equal keys the earlier group (larger ~group)
      }
    }
#ifdef BXS_OP_TRACE
    if (real && tid == 32 && g_op_trace) {          // a column thread: its partial keys have arrived
      unsigned long long t_;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_) : "r"((unsigned)cp));
      g_op_trace[(kFinTrace + blockIdx.x * 8 + 4) * 2] = t_;
    }
#endif
    // ---- exact positions: first element of the float4 group / first row of the 4-row group equal to the maximum
    //      (indices are clamped into the map: the rehearsal reads whatever the buffers hold) ----
    const float xr = fkey_inv((unsigned)(rp >> 32)), xc = fkey_inv((unsigned)(cp >> 32));
    int ar = 0, ac = 0;
    if (row_i < H) {
      const int grp = max(min((int)(0xffffffffu - (unsigned)(rp & 0xffffffffull)), (W - 4) >> 2), 0);
      const float4 q = __ldcg(reinterpret_cast<const float4*>(xin + (size_t)row_i * W + 4 * grp));
      ar = 4 * grp + (q.x == xr ? 0 : (q.y == xr ? 1 : (q.z == xr ? 2 : 3)));
      ar = min(ar, W - 1);
    }
    if (col_i < W) {
      const int y4 = max(min(4 * (int)(0xffffffffu - (unsigned)(cp & 0xffffffffull)), H - 1), 0);
      const float v0 = __ldcg(xin + (size_t)y4 * W + col_i);
      const float v1 = y4 + 1 < H ? __ldcg(xin + (size_t)(y4 + 1) * W + col_i) : 0.f;
      const float v2 = y4 + 2 < H ? __ldcg(xin + (size_t)(y4 + 2) * W + col_i) : 0.f;
      ac = y4 + (v0 == xc ? 0 : (v1 == xc ? 1 : (v2 == xc ? 2 : 3)));
      ac = min(ac, H - 1);
    }
#ifdef BXS_OP_TRACE
    if (real && tid == 32 && g_op_trace) {          // its arg-max row is resolved (second dependent load phase)
      unsigned long long t_;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_) : "r"(ac));
      g_op_trace[(kFinTrace + blockIdx.x * 8 + 5) * 2] = t_;
    }
#endif
    // ---- dice terms ----
    const float sr = row_i < H ? sigmoid_exact(xr) : 0.f;
    const float sc = col_i < W ? sigmoid_exact(xc) : 0.f;
    const bool tr = !empty && row_i >= rec.j0 && row_i <= rec.j1, tc = !empty && col_i >= rec.i0 && col_i <= rec.i1;
    const float r0 = warp_sum(tr ? sr : 0.f), r1 = warp_sum(sr * sr), r2 = warp_sum(tc ? sc : 0.f), r3 = warp_sum(sc * sc);
    if (lane == 0) { s_f[0][wid] = r0; s_f[1][wid] = r1; s_f[2][wid] = r2; s_f[3][wid] = r3; }
    if (row_i < H) s_arow[row_i] = ar;
    if (col_i < W) s_acol[col_i] = ac;
    // the (scaled) pairwise gradient at the arg-max positions, loaded before the barrier
    float svr = 0.f, svc = 0.f;
    if (row_i < H) svr = __ldcg(ginst + (size_t)row_i * W + ar);
    if (col_i < W) svc = __ldcg(ginst + (size_t)ac * W + col_i);
    __syncthreads();
#ifdef BXS_OP_TRACE
    if (real && tid == 0 && g_op_trace) {
      unsigned long long t_;
      asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));
      g_op_trace[(kFinTrace + blockIdx.x * 8 + 3) * 2] = t_;
    }
#endif
    float Ir = 0.f, Xr = 0.f, Ic = 0.f, Xc = 0.f;
#pragma unroll
    for (int i = 0; i < NWF; ++i) { Ir += s_f[0][i]; Xr += s_f[1][i]; Ic += s_f[2][i]; Xc += s_f[3][i]; }
    const float inv_n = 1.f / (float)N;
    const float Ur = Xr + (empty ? 0.f : (float)(rec.j1 - rec.j0 + 1)) + kDiceEps;
    const float Uc = Xc + (empty ? 0.f : (float)(rec.i1 - rec.i0 + 1)) + kDiceEps;
    // This instance's loss term goes out NOW (one thread): the atomic's round trip overlaps the coefficient math and the
    // gradient stores below.  ONE atomic carries the term (low 48 bits, fixed point) and the arrival count (top 16 bits):
    // the CTA that sees count == N - 1 in the returned value knows the complete sum without another round trip.
    bool last_cta = false;
    long long prj_total_fx = 0;
    if (real && tid == 0) {
      const OpSpan sp = op_span<D>(rec, H, W);
      reinterpret_cast<int4*>(ws.span)[n] = make_int4(sp.y_lo, sp.y_hi, sp.c_lo, sp.c_hi);
      const float prj_n = (1.f - 2.f * Ir / Ur) + (1.f - 2.f * Ic / Uc);
      ws.inst_prj[n] = prj_n;
      const unsigned long long mine = (unsigned long long)__double2ll_rn((double)fmaxf(prj_n, 0.f) * WQ_PRJ_FX) + (1ull << 48);
      const unsigned long long before = atomicAdd(&sched->prj_fx, mine);
      last_cta = (before >> 48) == (unsigned long long)(N - 1);
      prj_total_fx = (long long)((before + mine) & ((1ull << 48) - 1));
    }
    // d dice / d s = -2 t / U + 4 I s / U^2 ; through the sigmoid: * s (1 - s); mean over N
    const float crow = inv_n * (-2.f * (tr ? 1.f : 0.f) / Ur + 4.f * Ir * sr / (Ur * Ur)) * sr * (1.f - sr);
    const float ccol = inv_n * (-2.f * (tc ? 1.f : 0.f) / Uc + 4.f * Ic * sc / (Uc * Uc)) * sc * (1.f - sc);
    if (row_i < H) s_coef[row_i] = crow;
    __syncthreads();               // all reads of the arg-max positions precede the writes below
    if (real && row_i < H) {
      if (s_acol[ar] != row_i) ginst[(size_t)row_i * W + ar] = svr + crow;
      ws.coef_row[(size_t)n * H + row_i] = crow; ws.arg_row[(size_t)n * H + row_i] = ar; ws.sv_row[(size_t)n * H + row_i] = svr;
    }
    if (real && col_i < W) {
      ginst[(size_t)ac * W + col_i] = s_arow[ac] == col_i ? (svc + s_coef[ac]) + ccol : svc + ccol;
      ws.coef_col[(size_t)n * W + col_i] = ccol; ws.arg_col[(size_t)n * W + col_i] = ac; ws.sv_col[(size_t)n * W + col_i] = svc;
    }
    if (real && tid == 0 && last_cta) {                              // every instance has added its term: the four scalars
      const float scale = fminf(iter_ptr[0] / warmup_iters, 1.f) / fmaxf((float)wtot, 1.f);
      const long long num_fx = (long long)*reinterpret_cast<volatile unsigned long long*>(&sched->num_fx);   // main kernel: complete
      const float pn = (float)((double)num_fx * (1.0 / WQ_NUM_FX));
      losses_out[0] = (float)((double)prj_total_fx * (1.0 / WQ_PRJ_FX)) * inv_n;
      losses_out[1] = pn * scale;
      losses_out[2] = pn;
      losses_out[3] = (float)wtot;
      sched->prj_fx = 0ull;
      sched->num_fx = 0ull;
      sched->next_s = 0u;          // every CTA passed its poll before it added its term: nobody reads these any more
      sched->next_p = 0u;
      sched->done = 0u;
    }
    __syncthreads();               // the shared tables are rewritten by the next pass
  }
#ifdef BXS_OP_TRACE
  if (tid == 0 && g_op_trace) {
    unsigned long long t_;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_));
    g_op_trace[(kFinTrace + blockIdx.x * 8 + 2) * 2] = t_;
  }
#endif
}

inline size_t wq_smem_bytes(int64_t W) { return (size_t)WQ_STREAMERS * WQ_RING * WQ_SUB * W * 4; }

template <int NCHUNK, int D, bool FULLW>
int wq_launch_main(cudaStream_t st, const float* logits, const uint8_t* edge_bits, unsigned char* plan, int N, int H, int W,
                   OpWorkspace ws, WqSched* sched, const float* iter_ptr, float warmup_iters, float* losses_out,
                   float* g_logits) {
  const size_t smem = wq_smem_bytes(W);
  auto kern = wq_main_kernel<NCHUNK, D, FULLW>;
  constexpr int kMaxDev = 64;
  static thread_local size_t configured[kMaxDev] = {};   // per instantiation and device: opted-in dynamic shared memory
  static thread_local int occ_dev = -1, occ = 0;
  static thread_local size_t occ_smem = 0;
  int dev = 0;
  cudaGetDevice(&dev);
  const bool tracked = dev >= 0 && dev < kMaxDev;
  if (!tracked || smem > configured[dev]) {
    if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) {
      set_last_error(cudaGetLastError());
      return BXS_ERR_UNSUPPORTED;
    }
    if (tracked) configured[dev] = smem;
  }
  if (dev != occ_dev || smem != occ_smem) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, WQ_NT, smem) != cudaSuccess || occ < 1) {
      set_last_error(cudaGetLastError());
      return BXS_ERR_UNSUPPORTED;
    }
    occ_dev = dev;
    occ_smem = smem;
  }
  // the pair-item count lives in the plan (device memory): size the grid for the machine, bounded by the largest
  // possible queue; warps beyond the queues leave at once
  const int64_t max_items = (int64_t)N * (wq_strips(H) + wq_max_chains(H, W, D));
  const int grid = (int)std::min<int64_t>(ceil_div(max_items, WQ_NW), (int64_t)sm_count() * occ);
  // streamers: as many as give every one the same number of stream items (k each), at most WQ_STREAMERS per CTA
  const int64_t T = (int64_t)N * wq_strips(H), slots = (int64_t)grid * WQ_STREAMERS;
  const int NS = (int)ceil_div(T, ceil_div(T, slots));
  op_launch_pdl(kern, dim3((unsigned)grid), dim3(WQ_NT), smem, st, logits, edge_bits, plan, N, H, W, NS, ws.row_packed,
                ws.col_part, sched, iter_ptr, warmup_iters, g_logits);
  int rc = check_launch();
  if (rc != BXS_OK) return rc;
  op_launch_pdl(wq_finalize_kernel<D>, dim3((unsigned)N), dim3(OP_FIN_NT), 0, st, logits, plan, N, H, W, ws, sched, iter_ptr,
                warmup_iters, losses_out, g_logits, 0 /* first_pass: 0 = rehearse once while waiting */, (unsigned)(grid * WQ_NW));
  return check_launch();
}

inline int wq_build_plan(cudaStream_t st, const uint8_t* edge_bits, const int32_t* rects, const int32_t* inst_gt,
                         const int32_t* gt_img, unsigned char* plan, int N, int H, int W, int dilation) {
  wq_count_kernel<<<N, 128, 0, st>>>(edge_bits, rects, inst_gt, gt_img, H, W, reinterpret_cast<unsigned*>(plan + 64));
  switch (dilation) {
    case 1: wq_build_kernel<1><<<1, 1024, 0, st>>>(rects, inst_gt, gt_img, N, H, W, plan); break;
    case 2: wq_build_kernel<2><<<1, 1024, 0, st>>>(rects, inst_gt, gt_img, N, H, W, plan); break;
    case 3: wq_build_kernel<3><<<1, 1024, 0, st>>>(rects, inst_gt, gt_img, N, H, W, plan); break;
    default: wq_build_kernel<4><<<1, 1024, 0, st>>>(rects, inst_gt, gt_img, N, H, W, plan); break;
  }
  return check_launch();
}

inline int wq_forward(cudaStream_t st, const float* logits, const uint8_t* edge_bits, unsigned char* plan,
                      const float* iter_ptr, float warmup_iters, OpWorkspace ws, WqSched* sched, float* losses_out,
                      float* g_logits, int N, int H, int W, int dilation) {
  int rc = BXS_ERR_UNSUPPORTED;
#define BXS_WQ_CASE(NC, DD)                                                                                            \
  rc = (W == NC * 128) ? wq_launch_main<NC, DD, true>(st, logits, edge_bits, plan, N, H, W, ws, sched, iter_ptr,        \
                                                      warmup_iters, losses_out, g_logits)                            \
                       : wq_launch_main<NC, DD, false>(st, logits, edge_bits, plan, N, H, W, ws, sched, iter_ptr,       \
                                                       warmup_iters, losses_out, g_logits);
#define BXS_WQ_D(NC)                                                  \
  switch (dilation) {                                                 \
    case 1: { BXS_WQ_CASE(NC, 1) } break;                             \
    case 2: { BXS_WQ_CASE(NC, 2) } break;                             \
    case 3: { BXS_WQ_CASE(NC, 3) } break;                             \
    default: { BXS_WQ_CASE(NC, 4) } break;                            \
  }
  if (W <= 128) { BXS_WQ_D(1) }
  else if (W <= 256) { BXS_WQ_D(2) }
  else { BXS_WQ_D(4) }
#undef BXS_WQ_D
#undef BXS_WQ_CASE
  return rc;
}
