// a6 (DiscoBox MIL form) + a17: the DiscoBox mask loss of one FPN level on 16-bit mask logits, forward and backward.
// Replaces, for float16 / bfloat16 predictions (the reference trains DiscoBox under autocast, discobox_head.py:1142),
// the chain of DiscoBoxSOLOv2Head.loss (:1266-1300) after the dynamic convolution: sigmoid, mil_loss + dice_loss
// (:542-562), max_pool2d of the target, s * enlarged and the teacher-student dice_loss, with the keep weights of the
// all-zero targets.  The pseudo-label comes from bxs_meanfield_forward_logits (meanfield.cu).
//
// Arithmetic (T = the logits' type): s = round_T(sigmoid(x)) exactly as torch computes it; the row / column profiles
// and their first arg-max are taken on the ROUNDED s (many logits round to one s, torch.max(dim) returns the first
// index); every sum is float32 in a fixed order.  The gradient d/ds is float32 and is rounded to T once, after the
// sigmoid backward: g_x = round_T(g_s * (1 - s) * s).
//
// Work split: a CTA owns a strip of kRows rows of one instance and a tile of kNT columns (one thread per column), so
// config C's 32 instances of 200x256 run on 416 CTAs.  A CTA writes partial row maxima (per tile), partial column maxima
// (per strip) and three partial dense sums; db_finalize_kernel merges them per instance in a fixed order, and
// db_total_kernel sums the instances.  No atomics, no state kept between calls: deterministic and graph capturable.
#include <algorithm>

#include "half_math.cuh"

namespace bxs {
namespace {

constexpr int kNT = 256;            // threads per CTA = columns per tile
constexpr int kRows = 16;           // rows per strip
constexpr float kEps = 1e-3f;       // dice_loss, discobox_head.py:548
constexpr int kInst = 5;            // per-instance record: mil, d_ts, keep, sum x_ts*p, dice denominator of d_ts

struct DbGeom {
  int64_t n;
  int h, w, strips, tiles;
};

struct DbWs {
  unsigned long long* row_part;   // [n][tiles][h]   pack_key(key of the tile's row max of s, its first column)
  uint8_t* row_tpart;             // [n][tiles][h]   any target pixel in the tile's part of the row
  unsigned long long* col_part;   // [n][strips][w]  pack_key(key of the strip's column max of s, its first row)
  uint8_t* col_tpart;             // [n][strips][w]
  float* dense_part;              // [n][strips*tiles][3]  sum x_ts*p, sum x_ts^2, sum p^2 over the CTA's pixels
  int* arg_row;                   // [n][h]  first column of the row max
  float* coef_row;                // [n][h]  d mil / d (row max)
  int* arg_col;                   // [n][w]
  float* coef_col;                // [n][w]
  float* inst;                    // [n][kInst]
  size_t total_bytes;
};

inline DbGeom make_geom(int64_t n, int64_t h, int64_t w) {
  return DbGeom{n, (int)h, (int)w, (int)ceil_div(h, kRows), (int)ceil_div(w, kNT)};
}

inline DbWs carve_db(void* base, const DbGeom& g) {
  DbWs p{};
  Carver c(base);
  const int64_t n = g.n, h = g.h, w = g.w;
  p.row_part = (unsigned long long*)c.take(8 * n * g.tiles * h);
  p.row_tpart = (uint8_t*)c.take(n * g.tiles * h);
  p.col_part = (unsigned long long*)c.take(8 * n * g.strips * w);
  p.col_tpart = (uint8_t*)c.take(n * g.strips * w);
  p.dense_part = (float*)c.take(4 * 3 * n * g.strips * g.tiles);
  p.arg_row = (int*)c.take(4 * n * h);
  p.coef_row = (float*)c.take(4 * n * h);
  p.arg_col = (int*)c.take(4 * n * w);
  p.coef_col = (float*)c.take(4 * n * w);
  p.inst = (float*)c.take(4 * kInst * n);
  p.total_bytes = c.off;
  return p;
}

// any target pixel among columns col-1..col+1 of row y (zero outside the map): one row of the 3x3 max pool
__device__ __forceinline__ uint8_t row3_any(const uint8_t* __restrict__ tg, int y, int col, const DbGeom& g) {
  if (y < 0 || y >= g.h) return 0;
  const uint8_t* r = tg + (int64_t)y * g.w;
  uint8_t v = __ldg(r + col);
  if (col > 0) v |= __ldg(r + col - 1);
  if (col + 1 < g.w) v |= __ldg(r + col + 1);
  return v;
}

struct Cta {
  int64_t n;
  int strip, tile, col, y0, y1;
};
__device__ __forceinline__ Cta cta_of(const DbGeom& g) {
  Cta c;
  const int64_t b = blockIdx.x;
  c.strip = (int)(b % g.strips);
  c.tile = (int)((b / g.strips) % g.tiles);
  c.n = b / ((int64_t)g.strips * g.tiles);
  c.col = c.tile * kNT + (int)threadIdx.x;
  c.y0 = c.strip * kRows;
  c.y1 = min(c.y0 + kRows, g.h);
  return c;
}

// One strip x tile of one instance: partial row / column maxima of s with their first arg-max, partial target
// profiles, and (with a pseudo-label) the partial sums of the teacher-student dice.
template <typename T>
__global__ void __launch_bounds__(kNT) db_forward_kernel(const T* __restrict__ x, const uint8_t* __restrict__ tg,
                                                         const uint8_t* __restrict__ pl, DbGeom g, DbWs ws) {
  __shared__ unsigned long long s_rk[kRows][kNT / 32];
  __shared__ uint8_t s_rt[kRows][kNT / 32];
  __shared__ float s_red[kNT / 32];
  const Cta c = cta_of(g);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool active = c.col < g.w;
  const int64_t base = c.n * g.h * g.w;
  const T* xn = x + base;
  const uint8_t* tn = tg + base;
  const uint8_t* pn = pl ? pl + base : nullptr;
  unsigned ckey = 0;
  int carg = c.y0;
  uint8_t ct = 0;
  float sxp = 0.f, sxx = 0.f, spp = 0.f;
  // enl = 3x3 max pool of the target: the OR of three row triples, slid down the strip
  uint8_t up = 0, mid = 0;
  if (pn && active) { up = row3_any(tn, c.y0 - 1, c.col, g); mid = row3_any(tn, c.y0, c.col, g); }
  for (int y = c.y0; y < c.y1; ++y) {
    const int64_t i = (int64_t)y * g.w + c.col;
    unsigned key = 0;
    bool t = false;
    float s = 0.f;
    if (active) {
      s = sigmoid_rounded(xn[i]);
      key = fkey(s);
      t = tn[i] != 0;
    }
    const unsigned kmax = __reduce_max_sync(kFull, key);
    const unsigned amin = __reduce_min_sync(kFull, (active && key == kmax) ? (unsigned)c.col : 0xffffffffu);
    const unsigned tany = __any_sync(kFull, t);
    if (lane == 0) {
      s_rk[y - c.y0][warp] = kmax ? pack_key(kmax, (int)amin) : 0ull;
      s_rt[y - c.y0][warp] = (uint8_t)tany;
    }
    if (key > ckey) { ckey = key; carg = y; }      // rows ascending: strict > keeps the first row
    ct |= (uint8_t)t;
    if (pn && active) {
      const uint8_t down = row3_any(tn, y + 1, c.col, g);
      const float p = pn[i] ? 1.f : 0.f;
      const float xts = (up | mid | down) ? s : 0.f;   // s * enlarged, exact
      sxp = fmaf(xts, p, sxp);
      sxx = fmaf(xts, xts, sxx);
      spp += p;
      up = mid;
      mid = down;
    }
  }
  __syncthreads();
  for (int r = threadIdx.x; r < c.y1 - c.y0; r += kNT) {
    unsigned long long k = 0;
    uint8_t t = 0;
#pragma unroll
    for (int q = 0; q < kNT / 32; ++q) { k = max(k, s_rk[r][q]); t |= s_rt[r][q]; }
    const int64_t o = (c.n * g.tiles + c.tile) * g.h + c.y0 + r;
    ws.row_part[o] = k;
    ws.row_tpart[o] = t;
  }
  if (active) {
    const int64_t o = (c.n * g.strips + c.strip) * g.w + c.col;
    ws.col_part[o] = ckey ? pack_key(ckey, carg) : 0ull;
    ws.col_tpart[o] = ct;
  }
  if (pn) {
    sxp = block_sum<float>(sxp, s_red);
    sxx = block_sum<float>(sxx, s_red);
    spp = block_sum<float>(spp, s_red);
    if (threadIdx.x == 0) {
      float* d = ws.dense_part + 3 * (c.n * g.strips * g.tiles + (int64_t)c.tile * g.strips + c.strip);
      d[0] = sxp; d[1] = sxx; d[2] = spp;
    }
  }
}

// merged row profile of row y: (max s, target bit, first column of the max), tiles in order
__device__ __forceinline__ void row_profile(const DbGeom& g, const DbWs& ws, int64_t n, int y, float& r, float& l, int& a) {
  unsigned long long k = 0;
  uint8_t t = 0;
  for (int q = 0; q < g.tiles; ++q) {
    const int64_t o = (n * g.tiles + q) * g.h + y;
    k = max(k, ws.row_part[o]);
    t |= ws.row_tpart[o];
  }
  r = fkey_inv((unsigned)(k >> 32));
  l = t ? 1.f : 0.f;
  a = (int)(0xffffffffu - (unsigned)(k & 0xffffffffull));
}
__device__ __forceinline__ void col_profile(const DbGeom& g, const DbWs& ws, int64_t n, int x, float& r, float& l, int& a) {
  unsigned long long k = 0;
  uint8_t t = 0;
  for (int q = 0; q < g.strips; ++q) {
    const int64_t o = (n * g.strips + q) * g.w + x;
    k = max(k, ws.col_part[o]);
    t |= ws.col_tpart[o];
  }
  r = fkey_inv((unsigned)(k >> 32));
  l = t ? 1.f : 0.f;
  a = (int)(0xffffffffu - (unsigned)(k & 0xffffffffull));
}

__device__ __forceinline__ float dice(float inter, float xx, float tt) {
  return 1.f - 2.f * inter / ((xx + kEps) + (tt + kEps));
}

// One CTA per instance: the MIL dice over both profiles, the teacher-student dice, the keep weight, and the gradient
// coefficient of every row / column maximum.
__global__ void __launch_bounds__(kNT) db_finalize_kernel(DbGeom g, DbWs ws, int has_pl) {
  __shared__ float s_red[kNT / 32];
  __shared__ float s_bc[4];
  const int64_t n = blockIdx.x;
  float ir = 0.f, xr = 0.f, tr = 0.f, ic = 0.f, xc = 0.f, tc = 0.f, it = 0.f, xt = 0.f, pt = 0.f;
  for (int y = threadIdx.x; y < g.h; y += kNT) {
    float r, l;
    int a;
    row_profile(g, ws, n, y, r, l, a);
    ir = fmaf(r, l, ir); xr = fmaf(r, r, xr); tr = fmaf(l, l, tr);
  }
  for (int x = threadIdx.x; x < g.w; x += kNT) {
    float r, l;
    int a;
    col_profile(g, ws, n, x, r, l, a);
    ic = fmaf(r, l, ic); xc = fmaf(r, r, xc); tc = fmaf(l, l, tc);
  }
  if (has_pl) {
    const int parts = g.strips * g.tiles;
    for (int q = threadIdx.x; q < parts; q += kNT) {
      const float* d = ws.dense_part + 3 * (n * parts + q);
      it += d[0]; xt += d[1]; pt += d[2];
    }
  }
  ir = block_sum<float>(ir, s_red); xr = block_sum<float>(xr, s_red); tr = block_sum<float>(tr, s_red);
  ic = block_sum<float>(ic, s_red); xc = block_sum<float>(xc, s_red); tc = block_sum<float>(tc, s_red);
  if (has_pl) { it = block_sum<float>(it, s_red); xt = block_sum<float>(xt, s_red); pt = block_sum<float>(pt, s_red); }
  if (threadIdx.x == 0) {
    const float ur = (xr + kEps) + (tr + kEps), uc = (xc + kEps) + (tc + kEps);
    float* rec = ws.inst + kInst * n;
    rec[0] = dice(ir, xr, tr) + dice(ic, xc, tc);                 // rows (x.max(2)) + columns (x.max(1)), :559-561
    rec[1] = has_pl ? dice(it, xt, pt) : 0.f;
    rec[2] = tr > 0.f ? 1.f : 0.f;                                  // an all-zero target has weight 0 (:1283-1287)
    rec[3] = it;
    rec[4] = (xt + kEps) + (pt + kEps);
    s_bc[0] = ir; s_bc[1] = ur; s_bc[2] = ic; s_bc[3] = uc;
  }
  __syncthreads();
  const float Ir = s_bc[0], Ur = s_bc[1], Ic = s_bc[2], Uc = s_bc[3];
  for (int y = threadIdx.x; y < g.h; y += kNT) {
    float r, l;
    int a;
    row_profile(g, ws, n, y, r, l, a);
    ws.arg_row[n * g.h + y] = a;
    ws.coef_row[n * g.h + y] = -2.f * l / Ur + 4.f * Ir * r / (Ur * Ur);
  }
  for (int x = threadIdx.x; x < g.w; x += kNT) {
    float r, l;
    int a;
    col_profile(g, ws, n, x, r, l, a);
    ws.arg_col[n * g.w + x] = a;
    ws.coef_col[n * g.w + x] = -2.f * l / Uc + 4.f * Ic * r / (Uc * Uc);
  }
}

// out = {sum keep * mil, sum keep * d_ts, sum keep} over the instances, in instance order
__global__ void __launch_bounds__(kNT) db_total_kernel(int64_t n, const float* __restrict__ inst, float* __restrict__ out) {
  __shared__ float s_red[kNT / 32];
  float a = 0.f, b = 0.f, k = 0.f;
  for (int64_t i = threadIdx.x; i < n; i += kNT) {
    const float* rec = inst + kInst * i;
    if (rec[2] != 0.f) { a += rec[0]; b += rec[1]; k += 1.f; }
  }
  a = block_sum<float>(a, s_red);
  b = block_sum<float>(b, s_red);
  k = block_sum<float>(k, s_red);
  if (threadIdx.x == 0) { out[0] = a; out[1] = b; out[2] = k; }
}

// g_x over one strip x tile: the MIL part at the arg-max positions plus the dense teacher part, scaled by the upstream
// gradients g_out = {d/d sum keep*mil, d/d sum keep*d_ts} in float32, through the sigmoid, rounded to T once.
template <typename T>
__global__ void __launch_bounds__(kNT) db_backward_kernel(const T* __restrict__ x, const uint8_t* __restrict__ tg,
                                                          const uint8_t* __restrict__ pl, DbGeom g, DbWs ws,
                                                          const float* __restrict__ g_out, T* __restrict__ g_x) {
  const Cta c = cta_of(g);
  if (c.col >= g.w) return;
  const int64_t base = c.n * g.h * g.w;
  const T* xn = x + base;
  T* gn = g_x + base;
  const float* rec = ws.inst + kInst * c.n;
  if (rec[2] == 0.f) {                                               // weight 0: exactly zero
    for (int y = c.y0; y < c.y1; ++y) gn[(int64_t)y * g.w + c.col] = Half16Ops<T>::round(0.f);
    return;
  }
  const uint8_t* tn = tg + base;
  const uint8_t* pn = pl ? pl + base : nullptr;
  const float gi = __ldg(g_out), gt = pn ? __ldg(g_out + 1) : 0.f;
  const float ut = rec[4];
  const float ca = -2.f / ut, cb = 4.f * rec[3] / (ut * ut);         // d d_ts / d x_ts = ca * p + cb * x_ts
  const int acol = ws.arg_col[c.n * g.w + c.col];
  const float ccol = ws.coef_col[c.n * g.w + c.col];
  uint8_t up = 0, mid = 0;
  if (pn) { up = row3_any(tn, c.y0 - 1, c.col, g); mid = row3_any(tn, c.y0, c.col, g); }
  for (int y = c.y0; y < c.y1; ++y) {
    const int64_t i = (int64_t)y * g.w + c.col;
    const float s = sigmoid_rounded(xn[i]);
    float gm = 0.f;
    if (__ldg(ws.arg_row + c.n * g.h + y) == c.col) gm += __ldg(ws.coef_row + c.n * g.h + y);
    if (acol == y) gm += ccol;
    float gs = gm * gi;
    if (pn) {
      const uint8_t down = row3_any(tn, y + 1, c.col, g);
      if (up | mid | down) gs = fmaf(gt, fmaf(cb, s, pn[i] ? ca : 0.f), gs);
      up = mid;
      mid = down;
    }
    gn[i] = Half16Ops<T>::round(gs * (1.f - s) * s);
  }
}

inline bool known_half(int dtype) { return dtype == BXS_F16 || dtype == BXS_BF16; }

// sizes the kernels index with 32-bit rows / columns and a 1-D grid
inline bool db_shape_ok(int64_t n, int64_t h, int64_t w) {
  if (h > INT32_MAX || w > INT32_MAX) return false;
  return n * ceil_div(h, kRows) * ceil_div(w, kNT) <= INT32_MAX;
}

template <typename T>
int db_forward(const T* x, const uint8_t* tg, const uint8_t* pl, void* workspace, float* out, int64_t n, int64_t h,
               int64_t w, cudaStream_t st) {
  const DbGeom g = make_geom(n, h, w);
  const DbWs ws = carve_db(workspace, g);
  if (n > 0) {
    db_forward_kernel<T><<<(unsigned)(n * g.strips * g.tiles), kNT, 0, st>>>(x, tg, pl, g, ws);
    db_finalize_kernel<<<(unsigned)n, kNT, 0, st>>>(g, ws, pl ? 1 : 0);
  }
  db_total_kernel<<<1, kNT, 0, st>>>(n, ws.inst, out);
  return check_launch();
}

template <typename T>
int db_backward(const T* x, const uint8_t* tg, const uint8_t* pl, const void* workspace, const float* g_out, T* g_x,
                int64_t n, int64_t h, int64_t w, cudaStream_t st) {
  const DbGeom g = make_geom(n, h, w);
  const DbWs ws = carve_db(const_cast<void*>(workspace), g);
  db_backward_kernel<T><<<(unsigned)(n * g.strips * g.tiles), kNT, 0, st>>>(x, tg, pl, g, ws, g_out, g_x);
  return check_launch();
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int64_t bxs_discobox_loss_workspace_bytes(int64_t n, int64_t h, int64_t w) {
  if (n < 0 || h <= 0 || w <= 0 || !db_shape_ok(n, h, w)) return 0;
  return (int64_t)carve_db(nullptr, make_geom(n, h, w)).total_bytes;
}

extern "C" int bxs_discobox_loss_forward(const void* s_logits, const uint8_t* targets, const uint8_t* pseudo, int dtype,
                                         void* workspace, float* out, int64_t n, int64_t h, int64_t w,
                                         bxs_stream_t stream) {
  if (!out || n < 0 || h <= 0 || w <= 0 || !known_half(dtype)) return BXS_ERR_INVALID_ARG;
  if (n > 0 && (!s_logits || !targets || !workspace)) return BXS_ERR_INVALID_ARG;
  if (!db_shape_ok(n, h, w)) return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  if (dtype == BXS_F16)
    return db_forward(static_cast<const __half*>(s_logits), targets, pseudo, workspace, out, n, h, w, st);
  return db_forward(static_cast<const __nv_bfloat16*>(s_logits), targets, pseudo, workspace, out, n, h, w, st);
}

extern "C" int bxs_discobox_loss_backward(const void* s_logits, const uint8_t* targets, const uint8_t* pseudo, int dtype,
                                          const void* workspace, const float* g_out, void* g_logits, int64_t n, int64_t h,
                                          int64_t w, bxs_stream_t stream) {
  if (n < 0 || h <= 0 || w <= 0 || !known_half(dtype)) return BXS_ERR_INVALID_ARG;
  if (n > 0 && (!s_logits || !targets || !workspace || !g_out || !g_logits)) return BXS_ERR_INVALID_ARG;
  if (!db_shape_ok(n, h, w)) return BXS_ERR_UNSUPPORTED;
  if (n == 0) return BXS_OK;
  cudaStream_t st = as_stream(stream);
  if (dtype == BXS_F16)
    return db_backward(static_cast<const __half*>(s_logits), targets, pseudo, workspace, g_out,
                       static_cast<__half*>(g_logits), n, h, w, st);
  return db_backward(static_cast<const __nv_bfloat16*>(s_logits), targets, pseudo, workspace, g_out,
                     static_cast<__nv_bfloat16*>(g_logits), n, h, w, st);
}
