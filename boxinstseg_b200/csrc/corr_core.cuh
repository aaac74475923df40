// f4: cores of DiscoBox's semantic-correspondence path (mmdet/models/dense_heads/discobox_head.py):
//
//   corr_solve    SemanticCorrSolver.solve (:369-411) after the cosine similarity: the window mask (eye -> max_pool2d ->
//                 transpose, :393-397), num_iter rounds of { num_smooth x (pass_message (:347-366) + row normalisation),
//                 C = Cu + votes, row normalisation } for ONE retrieved object, the whole [P,P] state in shared memory.
//                 The reference issues ~25 element-wise / slice-assign kernels per round on a [K,49,49] tensor.
//   corr_transfer corr_loss (:1087-1096) + superres_T (:851-865): T * softmax(Cu), row normalisation, the bilinear /
//                 trilinear 7x7 -> 28x28 super-resolution of both index pairs, the two thresholded mask products and the
//                 two [K,784,784] x [K,784,1] products -- for one (object, query pixel) per thread, without building any of
//                 the six [K,784,784] tensors (12 MB each) of the reference.
//
// Written as PHASES (`corr_phase(n, f)`: on the device a block-strided loop + __syncthreads, on the host a plain loop), each
// element written by exactly one phase item and every sum taken in a fixed order, so that tests/host_harness/corr_host.cpp
// runs the very same source on the CPU (the solve loop is the same sequence of correctly rounded operations on both sides;
// the transfer uses expf and lets the device compiler contract a*b+c, so it agrees to rounding only).  Both builds are
// checked against the oracle: the host build by the CPU suite, the device build by tests/test_corr_gpu.py; against the
// reference (whose row sums are ATen reductions in another order) the agreement is ~1e-6.
#pragma once
#include <stdint.h>

#include "assign_core.cuh"      // BXS_HD, BXS_FADD / FSUB / FMUL / FDIV

namespace bxs {

template <class F>
BXS_HD void corr_phase(int n, F f) {
#if defined(__CUDA_ARCH__)
  for (int i = threadIdx.x; i < n; i += blockDim.x) f(i);
  __syncthreads();
#else
  for (int i = 0; i < n; ++i) f(i);
#endif
}

// pass_message (:347-366) for one element i = p * P + q of a [P,P] = [h,w,h,w] table: the mean over the (dy,dx) in
// {-1,0,1}^2 for which BOTH the source cell p - (dy,dx) and the target cell q - (dy,dx) exist.  Accumulation order = the
// reference's loop order (dx outer, dy inner), starting from its zero tensor.
// CH, CW > 0: compile-time grid (the divisions become multiplications; 7 x 7 is the reference's configuration), else h_rt, w_rt.
template <int CH, int CW>
BXS_HD float corr_pass_message(const float* T, int h_rt, int w_rt, int i) {
  const int h = CH > 0 ? CH : h_rt, w = CW > 0 ? CW : w_rt;
  const int P = h * w;
  const int p = i / P, q = i - p * P;
  const int y = p / w, x = p - y * w, v = q / w, u = q - v * w;
  float acc = 0.f;
  int cnt = 0;
  for (int dx = -1; dx <= 1; ++dx)
    for (int dy = -1; dy <= 1; ++dy) {
      const int ys = y - dy, xs = x - dx, vs = v - dy, us = u - dx;
      if (ys < 0 || ys >= h || vs < 0 || vs >= h || xs < 0 || xs >= w || us < 0 || us >= w) continue;
      acc = BXS_FADD(acc, T[(ys * w + xs) * P + vs * w + us]);
      ++cnt;
    }
  return BXS_FDIV(acc, (float)cnt);
}

// dist_mask (:393-395): eye(P) viewed [P,h,w], max-pooled (kernel dk, stride 1, padding dk/2), transposed: 1 where the two
// cells are within dk/2 of each other in both coordinates (symmetric, so the transpose changes nothing).
BXS_HD bool corr_in_window(int p, int q, int w, int r) {
  const int dy = p / w - q / w, dx = p % w - q % w;
  return dy <= r && -dy <= r && dx <= r && -dx <= r;
}

// rows of a [P,P] table summed left to right (one phase item per row)
BXS_HD float corr_row_sum(const float* A, int P, int p) {
  float s = 0.f;
  for (int q = 0; q < P; ++q) s = BXS_FADD(s, A[p * P + q]);
  return s;
}

// The same sum in two fixed-order stages (kCorrLanes interleaved partial sums per row, then the partials in order): 1/8 of the
// dependent additions per phase item, identical on the host and on the device.  part: [kCorrLanes * P].
constexpr int kCorrLanes = 8;
BXS_HD void corr_row_sums(const float* A, float* part, float* rs, int P, float eps) {
  corr_phase(P * kCorrLanes, [&](int i) {
    const int p = i / kCorrLanes, j = i - p * kCorrLanes;
    float s = 0.f;
    for (int q = j; q < P; q += kCorrLanes) s = BXS_FADD(s, A[p * P + q]);
    part[i] = s;
  });
  corr_phase(P, [&](int p) {
    float s = part[p * kCorrLanes];
    for (int j = 1; j < kCorrLanes; ++j) s = BXS_FADD(s, part[p * kCorrLanes + j]);
    rs[p] = BXS_FADD(s, eps);
  });
}

// The solve loop for one object.  Cu: [P,P] cosine similarities (global or host memory); a, b: two [P,P] work tables,
// rs: [(1 + kCorrLanes) * P] row sums and their partials (shared memory on the device).  The result is left in `out`
// ([P,P], global).
template <int CH, int CW>
BXS_HD void corr_solve_t(const float* Cu, float* out, float* a, float* b, float* rs, int h_rt, int w_rt, int dist_kernel,
                         int num_iter, int num_smooth) {
  const int h = CH > 0 ? CH : h_rt, w = CW > 0 ? CW : w_rt;
  const int P = h * w, PP = P * P, r = dist_kernel / 2;
  float* cur = a;        // C
  float* nxt = b;
  corr_phase(PP, [&](int i) { cur[i] = corr_in_window(i / P, i % P, w, r) ? Cu[i] : BXS_FMUL(Cu[i], 0.f); });   // :396-397
  for (int it = 0; it < num_iter; ++it) {
    // votes = C.clone(); num_smooth x { pass_message; votes /= votes.sum(2) + 1e-4 }          (:399-403)
    // C = Cu + votes; C /= C.sum(2) + 1e-4                                                     (:407-408)
    for (int s = 0; s < num_smooth; ++s) {
      corr_phase(PP, [&](int i) { nxt[i] = corr_pass_message<CH, CW>(cur, h, w, i); });
      corr_row_sums(nxt, rs + P, rs, P, 1e-4f);
      corr_phase(PP, [&](int i) { nxt[i] = BXS_FDIV(nxt[i], rs[i / P]); });
      float* t = cur; cur = nxt; nxt = t;
    }
    corr_phase(PP, [&](int i) { cur[i] = BXS_FADD(Cu[i], cur[i]); });
    corr_row_sums(cur, rs + P, rs, P, 1e-4f);
    corr_phase(PP, [&](int i) { cur[i] = BXS_FDIV(cur[i], rs[i / P]); });
  }
  corr_phase(PP, [&](int i) { out[i] = cur[i]; });
}

BXS_HD void corr_solve(const float* Cu, float* out, float* a, float* b, float* rs, int h, int w, int dist_kernel, int num_iter,
                       int num_smooth) {
  if (h == 7 && w == 7)                 // obj_bank feat_height / feat_width of the reference's configs
    corr_solve_t<7, 7>(Cu, out, a, b, rs, h, w, dist_kernel, num_iter, num_smooth);
  else
    corr_solve_t<0, 0>(Cu, out, a, b, rs, h, w, dist_kernel, num_iter, num_smooth);
}

// ATen's align_corners=False linear tap for destination index d of an `in` -> `out` up-sampling (UpSample.h:
// area_pixel_compute_source_index, guard_index_and_lambda): i0, i1 and the weights l0 = 1 - l1, l1.
struct CorrTap { int i0, i1; float l0, l1; };
BXS_HD CorrTap corr_tap(int d, int in, int out) {
  CorrTap t;
  const float scale = (float)in / (float)out;
  float src = BXS_FSUB(BXS_FMUL(scale, BXS_FADD((float)d, 0.5f)), 0.5f);
  if (src < 0.f) src = 0.f;
  t.i0 = (int)src;
  if (t.i0 > in - 1) t.i0 = in - 1;
  t.i1 = t.i0 < in - 1 ? t.i0 + 1 : t.i0;
  t.l1 = BXS_FSUB(src, (float)t.i0);
  if (t.l1 < 0.f) t.l1 = 0.f;
  if (t.l1 > 1.f) t.l1 = 1.f;
  t.l0 = BXS_FSUB(1.f, t.l1);
  return t;
}

// T2 = T * softmax(Cu, 2); T2 /= T2.sum(2) + 1e-5 for one object, all in one [P,P] table (:1086-1090).
// e: [P,P] scratch (may alias nothing), rs: [P].  Uses expf: host and device agree to the last ulp only where libm and
// CUDA's expf do (both are within 2 ulp of the true value), so host-twin comparisons of this part carry a tolerance.
template <class Exp>
BXS_HD void corr_weighted(const float* T, const float* Cu, float* t2, float* rs, float* mx, int P, Exp ex) {
  const int PP = P * P;
  corr_phase(P, [&](int p) {
    float m = Cu[p * P];
    for (int q = 1; q < P; ++q) m = Cu[p * P + q] > m ? Cu[p * P + q] : m;
    mx[p] = m;
  });
  corr_phase(PP, [&](int i) { t2[i] = ex(BXS_FSUB(Cu[i], mx[i / P])); });
  corr_phase(P, [&](int p) { rs[p] = corr_row_sum(t2, P, p); });
  corr_phase(PP, [&](int i) { t2[i] = BXS_FMUL(T[i], BXS_FDIV(t2[i], rs[i / P])); });
  corr_phase(P, [&](int p) { mx[p] = BXS_FADD(corr_row_sum(t2, P, p), 1e-5f); });
  corr_phase(PP, [&](int i) { t2[i] = BXS_FDIV(t2[i], mx[i / P]); });
}

// One (object, query pixel pq = (Y,X) of the Hm x Wm mask grid): the row pq of the super-resolved table contracted with the
// two thresholded, clamped mask vectors of the object (:1094-1095).  t2: [P,P] of the object (shared / host memory), m0q =
// query mask at pq, m1: [Hm*Wm] mask of the object, R: P floats of scratch owned by the caller.
//   Tsr[pq][(V,U)] = scale * sum_{v,u} wV wU ( sum_{y,x} wY wX t2[(y,x)][(v,u)] ),   scale = P / (Hm*Wm)   (:851-865)
//   fg = sum_(V,U) Tsr * [m0q * m1 > 0.5] * clamp(m1, .1, .9),  bg = sum Tsr * [(1-m0q)(1-m1) > 0.5] * clamp(1-m1, .1, .9)
// tapV [Hm], tapU [Wm]: corr_tap(V, h, Hm) / corr_tap(U, w, Wm), computed once per CTA.
BXS_HD void corr_transfer_pixel(const float* t2, float m0q, const float* m1, float* R, const CorrTap* tapV, const CorrTap* tapU,
                                int h, int w, int Hm, int Wm, int pq, float* fg_out, float* bg_out) {
  const int P = h * w;
  const int Y = pq / Wm, X = pq - Y * Wm;
  const CorrTap ty = tapV[Y], tx = tapU[X];
  const float* r00 = t2 + (ty.i0 * w + tx.i0) * P;
  const float* r01 = t2 + (ty.i0 * w + tx.i1) * P;
  const float* r10 = t2 + (ty.i1 * w + tx.i0) * P;
  const float* r11 = t2 + (ty.i1 * w + tx.i1) * P;
  for (int c = 0; c < P; ++c)                                    // up-sampling of the SOURCE cell (the trilinear pass)
    R[c] = ty.l0 * (tx.l0 * r00[c] + tx.l1 * r01[c]) + ty.l1 * (tx.l0 * r10[c] + tx.l1 * r11[c]);
  const float scale = (float)P / (float)(Hm * Wm);
  const float n0q = BXS_FSUB(1.f, m0q);
  float fg = 0.f, bg = 0.f;
  for (int V = 0; V < Hm; ++V) {
    const CorrTap tv = tapV[V];
    for (int U = 0; U < Wm; ++U) {
      const CorrTap tu = tapU[U];
      const float val = tv.l0 * (tu.l0 * R[tv.i0 * w + tu.i0] + tu.l1 * R[tv.i0 * w + tu.i1]) +
                        tv.l1 * (tu.l0 * R[tv.i1 * w + tu.i0] + tu.l1 * R[tv.i1 * w + tu.i1]);
      const float m = m1[V * Wm + U], n = BXS_FSUB(1.f, m);
      const float mc = m < 0.1f ? 0.1f : (m > 0.9f ? 0.9f : m);
      const float nc = n < 0.1f ? 0.1f : (n > 0.9f ? 0.9f : n);
      if (BXS_FMUL(m0q, m) > 0.5f) fg += val * mc;
      if (BXS_FMUL(n0q, n) > 0.5f) bg += val * nc;
    }
  }
  *fg_out = fg * scale;
  *bg_out = bg * scale;
}

// ---------------------------------------------------------------------------------------------------------------------------
// corr_retrieve: get_similar_obj (:174-221) for every query object of a level at once, with the order dependence of the
// reference's per-object loop resolved on the device.  The bank is a packed store of num_class x L slots; object i of the
// level sees the bank of its class as the objects before it left it: slot s holds the LAST eligible earlier object of this
// level (same class, ring position (ptr[c] + rank) % L, rank = its index among those objects) that targets s, else the
// stored slot.  The class has a bank at query time if it had one before the level or an earlier object appended to it.
//
// Sources are int32: >= 0 a row of the store (class * L + slot), < 0 the level's own object -(src + 1) (its teacher RoI
// feature / mask / box, which is what its append stores).  tests/host_harness/corr_retrieve_host.cpp compiles this part for
// the host.
// ---------------------------------------------------------------------------------------------------------------------------
struct CorrBank {
  const float* feat;        // [num_class * L, C * P]
  const float* mask;        // [num_class * L, M]
  const float* box;         // [num_class * L, 4]
  const int32_t* ptr;       // [num_class] ring write pointer
  const int32_t* exists;    // [num_class] 1 once the class's first append happened
  int num_class, L;
};

struct CorrLevel {
  const float* q_feat;        // [n, C * P] student RoI features (the query's)
  const float* q_feat_first;  // [n, C * P] the same re-normalised (create_one :43): used by the first query the head sees
  const float* q_mask;        // [n, M] student RoI masks
  const float* t_feat;        // [n, C * P] teacher RoI features (what an append stores)
  const float* t_mask;        // [n, M]
  const float* box;           // [n, 4] x1, y1, x2, y2 (integer valued)
  const int32_t* label;       // [n]
  const int32_t* valid;       // [n] 0: the object takes no part (all-zero target)
  int n;
};

struct CorrRetrieveCfg {
  int C, h, w, Hm, Wm;
  float fg_thr, bg_thr, app_thr, ratio_lo, ratio_hi, min_size;
  int max_objs, min_objs;
};

// per-query outputs
struct CorrRetrieveOut {
  int32_t* src;        // [n, max(max_objs, 1)] the retrieved sources in ascending slot order (0 past `count`)
  int32_t* count;      // [n] number retrieved (<= max_objs)
  int32_t* kcount;     // [n] tables the loss uses: count if count >= min_objs, else 0
  int32_t* slot;       // [n] the slot the object's append writes, -1 when it does not append
  int32_t* exists;     // [n] the class had a bank at query time
};

BXS_HD bool corr_live(const CorrLevel& lv, int num_class, int j) {
  return lv.valid[j] != 0 && lv.label[j] >= 0 && lv.label[j] < num_class;
}

// :1056-1057 -- an object is appended when both sides of its box exceed min_size
BXS_HD bool corr_appends(const float* b, float min_size) {
  return BXS_FSUB(b[2], b[0]) > min_size && BXS_FSUB(b[3], b[1]) > min_size;
}

// ObjectElements.get_ratio (:103-105)
BXS_HD float corr_box_ratio(const float* b) {
  return BXS_FDIV(BXS_FSUB(b[2], b[0]), BXS_FADD(BXS_FSUB(b[3], b[1]), 1e-5f));
}

// a Hm x Wm mask at cell p of the h x w grid: F.interpolate(bilinear, align_corners=False) (:188-199)
BXS_HD float corr_mask_small(const float* m, int Hm, int Wm, int h, int w, int p) {
  const CorrTap ty = corr_tap(p / w, Hm, h), tx = corr_tap(p % w, Wm, w);
  return ty.l0 * (tx.l0 * m[ty.i0 * Wm + tx.i0] + tx.l1 * m[ty.i0 * Wm + tx.i1]) +
         ty.l1 * (tx.l0 * m[ty.i1 * Wm + tx.i0] + tx.l1 * m[ty.i1 * Wm + tx.i1]);
}

constexpr int kCorrSums = 6;   // A*B, [A+B >= 1], (1-A)(1-B), [2-A-B >= 1], f0 f1 a b, a b

// Scratch of one query (shared memory on the device): bytes of corr_retrieve_scratch(L, P).
BXS_HD int64_t corr_retrieve_scratch(int L, int P) {
  return (int64_t)4 * (L + 8 + P + (int64_t)L * P + (int64_t)L * kCorrSums * kCorrLanes + L);
}

// Query i of the level.  All threads of the CTA call it (phases synchronise); the host calls it query by query.
BXS_HD void corr_retrieve_query(const CorrBank& bk, const CorrLevel& lv, const CorrRetrieveCfg& cf, int first_flag, int i,
                                void* scratch, const CorrRetrieveOut& out) {
  const int L = bk.L, P = cf.h * cf.w, M = cf.Hm * cf.Wm, CP = cf.C * P, K = cf.max_objs > 0 ? cf.max_objs : 1;
  int32_t* src = static_cast<int32_t*>(scratch);     // [L]
  int32_t* st = src + L;                              // [8]: live, exists, first, slot, count
  float* a_small = reinterpret_cast<float*>(st + 8);  // [P]
  float* b_small = a_small + P;                       // [L, P]
  float* part = b_small + (int64_t)L * P;             // [L, kCorrSums, kCorrLanes]
  int32_t* pass = reinterpret_cast<int32_t*>(part + (int64_t)L * kCorrSums * kCorrLanes);   // [L]
  const bool live = corr_live(lv, bk.num_class, i);
  const int c = live ? lv.label[i] : 0;
  corr_phase(L, [&](int s) { src[s] = c * L + s; });
  corr_phase(1, [&](int) {                          // the appends of the earlier objects of this level, in order
    int rank = 0;
    bool earlier_live = false;
    for (int j = 0; j < i; ++j) {
      if (!corr_live(lv, bk.num_class, j)) continue;
      earlier_live = true;
      if (lv.label[j] != c || !corr_appends(lv.box + 4 * j, cf.min_size)) continue;
      src[(bk.ptr[c] + rank) % L] = -(j + 1);
      ++rank;
    }
    st[0] = live;
    st[1] = live && (bk.exists[c] != 0 || rank > 0);
    st[2] = live && first_flag != 0 && !earlier_live;
    st[3] = live && corr_appends(lv.box + 4 * i, cf.min_size) ? (bk.ptr[c] + rank) % L : -1;
    out.slot[i] = st[3];
    out.exists[i] = st[1];
  });
  if (!st[1]) {                                     // no bank: nothing retrieved (get_similar_obj returns None)
    corr_phase(K, [&](int k) { out.src[(int64_t)i * K + k] = 0; });
    corr_phase(1, [&](int) { out.count[i] = 0; out.kcount[i] = 0; });
    return;
  }
  const float* qf = (st[2] ? lv.q_feat_first : lv.q_feat) + (int64_t)i * CP;
  const float* qm = lv.q_mask + (int64_t)i * M;
  auto smask = [&](int s) { const int v = src[s]; return v >= 0 ? bk.mask + (int64_t)v * M : lv.t_mask + (int64_t)(-v - 1) * M; };
  auto sfeat = [&](int s) { const int v = src[s]; return v >= 0 ? bk.feat + (int64_t)v * CP : lv.t_feat + (int64_t)(-v - 1) * CP; };
  auto sbox = [&](int s) { const int v = src[s]; return v >= 0 ? bk.box + (int64_t)v * 4 : lv.box + (int64_t)(-v - 1) * 4; };
  corr_phase(P, [&](int p) { a_small[p] = corr_mask_small(qm, cf.Hm, cf.Wm, cf.h, cf.w, p); });
  corr_phase(L * P, [&](int e) { b_small[e] = corr_mask_small(smask(e / P), cf.Hm, cf.Wm, cf.h, cf.w, e % P); });
  // the six sums of every slot, kCorrLanes interleaved partials each (then reduced in lane order: a fixed order)
  corr_phase(L * kCorrLanes, [&](int e) {
    const int s = e / kCorrLanes, j = e - s * kCorrLanes;
    const float* B = smask(s);
    const float* f1 = sfeat(s);
    const float* bs = b_small + (int64_t)s * P;
    float ab = 0.f, un = 0.f, nab = 0.f, nun = 0.f, app = 0.f, den = 0.f;
    for (int q = j; q < M; q += kCorrLanes) {
      const float a = qm[q], b = B[q];
      ab = BXS_FADD(ab, BXS_FMUL(a, b));
      un = BXS_FADD(un, BXS_FADD(a, b) >= 1.f ? 1.f : 0.f);
      nab = BXS_FADD(nab, BXS_FMUL(BXS_FSUB(1.f, a), BXS_FSUB(1.f, b)));
      nun = BXS_FADD(nun, BXS_FSUB(BXS_FSUB(2.f, a), b) >= 1.f ? 1.f : 0.f);
    }
    for (int q = j; q < CP; q += kCorrLanes) {
      const int p = q % P;
      app = BXS_FADD(app, BXS_FMUL(BXS_FMUL(BXS_FMUL(qf[q], f1[q]), a_small[p]), bs[p]));
    }
    for (int p = j; p < P; p += kCorrLanes) den = BXS_FADD(den, BXS_FMUL(a_small[p], bs[p]));
    float* o = part + (int64_t)s * kCorrSums * kCorrLanes + j;
    o[0 * kCorrLanes] = ab; o[1 * kCorrLanes] = un; o[2 * kCorrLanes] = nab;
    o[3 * kCorrLanes] = nun; o[4 * kCorrLanes] = app; o[5 * kCorrLanes] = den;
  });
  // the four tests (:205-221).  NaN (0/0 of an all-zero slot) fails every comparison, an infinite ratio fails the upper bound.
  corr_phase(L, [&](int s) {
    float v[kCorrSums];
    for (int t = 0; t < kCorrSums; ++t) {
      const float* o = part + ((int64_t)s * kCorrSums + t) * kCorrLanes;
      float acc = o[0];
      for (int j = 1; j < kCorrLanes; ++j) acc = BXS_FADD(acc, o[j]);
      v[t] = acc;
    }
    const float fg = BXS_FDIV(v[0], v[1]), bg = BXS_FDIV(v[2], v[3]);
    const float app = BXS_FDIV(v[4], BXS_FADD(v[5], 1e-6f));
    const float ratio = BXS_FDIV(corr_box_ratio(lv.box + 4 * i), corr_box_ratio(sbox(s)));
    pass[s] = fg > cf.fg_thr && bg > cf.bg_thr && app > cf.app_thr && ratio >= cf.ratio_lo && ratio <= cf.ratio_hi;
  });
  corr_phase(1, [&](int) {                          // ascending slot order, at most max_objs
    int k = 0;
    for (int s = 0; s < L && k < cf.max_objs; ++s)
      if (pass[s]) out.src[(int64_t)i * K + k++] = src[s];
    for (int r = k; r < K; ++r) out.src[(int64_t)i * K + r] = 0;
    out.count[i] = k;
    out.kcount[i] = k >= cf.min_objs ? k : 0;
  });
}

}  // namespace bxs
