// a1: CondInst dynamic mask head -- per-instance 3-layer 1x1 FCN over [rel_x, rel_y, mask_feat]
// followed by the x f "aligned bilinear" upsample, forward and backward.
// Replaces CondInstMaskHead.forward + parse_dynamic_params + aligned_bilinear
// (mmdet/models/dense_heads/condinst_head.py:1120-1164, 146-167): the reference materialises
// feat[img_inds] ++ rel_coords as [N,18,h,w] (118 MB at config A) and runs three cuDNN grouped
// convs with K <= 18 plus a pad/interpolate/pad/slice chain.
//
// Design: HBM-bound op with tiny K, so SIMT with the per-instance weights in shared memory
// (transposed so that the 8 output channels of one input channel are two LDS.128 broadcasts).
//   forward : CTA = (instance, 16x32 low-res tile + 1px apron); low-res logits live only in shared
//             memory; the CTA writes the upsampled 32x64 output tile directly (float4 stores).
//   backward: CTA = (image, 8x32 low-res tile, instance group) looping over every GS-th instance of
//             that image, so d/d mask_feat is accumulated in registers across the group's instances and
//             written once per group (no atomics); the GS group partials are summed in a fixed order by a
//             second kernel (deterministic).  d/d params is an outer-product reduction over the tile in
//             shared memory -> per-tile partials -> a fixed-order second-stage sum.
// Layout of params[n] (condinst_head.py:1079-1088,1122-1123): [W1(8xCIN) | W2(8x8) | W3(1x8) | b1 | b2 | b3]
#include <algorithm>

#include "common.cuh"

namespace bxs {
namespace {

constexpr int CH = 8;            // dynamic_channels of every BoxInst/CondInst config in the reference
constexpr int NT = 256;
constexpr int MAX_CIN = 34;      // in_channels (<=32) + 2 relative coordinates

struct HeadDims {
  int N, B, C, h, w;             // C = mask_feat channels
  int cin;                       // C (+2 with relative coordinates)
  int stride;                    // in_stride
  int f;                         // in_stride / out_stride
  int rel;                       // 1 when relative coordinates are used
  int P;                         // parameters per instance
};

// shared-memory image of one instance's parameters, W1/W2 transposed to [in][out]
struct SmemParams {
  float w1t[MAX_CIN * CH];
  float w2t[CH * CH];
  float w3[CH];
  float b1[CH];
  float b2[CH];
  float b3;
  float cx, cy, soi;
};

__device__ __forceinline__ void load_params(SmemParams& sp, const float* __restrict__ params,
                                            const float* __restrict__ coors, const float* __restrict__ soi, int n,
                                            const HeadDims& d) {
  const float* p = params + (int64_t)n * d.P;
  const int o2 = CH * d.cin, o3 = o2 + CH * CH, ob1 = o3 + CH, ob2 = ob1 + CH, ob3 = ob2 + CH;
  for (int i = threadIdx.x; i < CH * d.cin; i += blockDim.x) {
    int j = i / d.cin, k = i - j * d.cin;            // W1[j][k] -> w1t[k][j]
    sp.w1t[k * CH + j] = p[i];
  }
  for (int i = threadIdx.x; i < CH * CH; i += blockDim.x) sp.w2t[(i % CH) * CH + i / CH] = p[o2 + i];
  if (threadIdx.x < CH) {
    sp.w3[threadIdx.x] = p[o3 + threadIdx.x];
    sp.b1[threadIdx.x] = p[ob1 + threadIdx.x];
    sp.b2[threadIdx.x] = p[ob2 + threadIdx.x];
  }
  if (threadIdx.x == 0) {
    sp.b3 = p[ob3];
    sp.cx = d.rel ? coors[2 * n] : 0.f;
    sp.cy = d.rel ? coors[2 * n + 1] : 0.f;
    sp.soi = d.rel ? soi[n] : 1.f;
  }
}

// inputs of one low-res pixel: in[0..1] = relative coordinates, in[2..] = mask features
// Register arrays are always laid out [rel_x, rel_y, feat_0 ..]; without relative coordinates the
// first two slots are zero and the weights are shifted by `o` when they are read (static indexing).
template <int CMAX>
__device__ __forceinline__ void gather_inputs(const float* __restrict__ feat_img, const SmemParams& sp,
                                              const HeadDims& d, int y, int x, float* in) {
  // locations = arange * stride + stride // 2 ; rel = (coor - loc) / soi   (condinst_head.py:1143-1153)
  in[0] = d.rel ? __fdiv_rn(sp.cx - (float)(x * d.stride + d.stride / 2), sp.soi) : 0.f;
  in[1] = d.rel ? __fdiv_rn(sp.cy - (float)(y * d.stride + d.stride / 2), sp.soi) : 0.f;
  const int64_t plane = (int64_t)d.h * d.w, pix = (int64_t)y * d.w + x;
#pragma unroll
  for (int c = 0; c < CMAX; ++c) in[2 + c] = c < d.C ? __ldg(feat_img + c * plane + pix) : 0.f;
}

template <int CMAX>
__device__ __forceinline__ float mlp_forward(const SmemParams& sp, const float* in, const HeadDims& d, float* x1,
                                             float* x2) {
#pragma unroll
  for (int j = 0; j < CH; ++j) x1[j] = sp.b1[j];
  const int skip = d.rel ? 0 : 2;                  // register slot k <-> weight row k - skip
#pragma unroll
  for (int k = 0; k < CMAX + 2; ++k) {
    if (k < skip || k - skip >= d.cin) continue;
    const float v = in[k];
    const float4 a = *reinterpret_cast<const float4*>(&sp.w1t[(k - skip) * CH]);
    const float4 b = *reinterpret_cast<const float4*>(&sp.w1t[(k - skip) * CH + 4]);
    x1[0] = fmaf(a.x, v, x1[0]); x1[1] = fmaf(a.y, v, x1[1]); x1[2] = fmaf(a.z, v, x1[2]); x1[3] = fmaf(a.w, v, x1[3]);
    x1[4] = fmaf(b.x, v, x1[4]); x1[5] = fmaf(b.y, v, x1[5]); x1[6] = fmaf(b.z, v, x1[6]); x1[7] = fmaf(b.w, v, x1[7]);
  }
#pragma unroll
  for (int j = 0; j < CH; ++j) { x1[j] = fmaxf(x1[j], 0.f); x2[j] = sp.b2[j]; }
#pragma unroll
  for (int k = 0; k < CH; ++k) {
    const float v = x1[k];
    const float4 a = *reinterpret_cast<const float4*>(&sp.w2t[k * CH]);
    const float4 b = *reinterpret_cast<const float4*>(&sp.w2t[k * CH + 4]);
    x2[0] = fmaf(a.x, v, x2[0]); x2[1] = fmaf(a.y, v, x2[1]); x2[2] = fmaf(a.z, v, x2[2]); x2[3] = fmaf(a.w, v, x2[3]);
    x2[4] = fmaf(b.x, v, x2[4]); x2[5] = fmaf(b.y, v, x2[5]); x2[6] = fmaf(b.z, v, x2[6]); x2[7] = fmaf(b.w, v, x2[7]);
  }
  float o = sp.b3;
#pragma unroll
  for (int j = 0; j < CH; ++j) { x2[j] = fmaxf(x2[j], 0.f); o = fmaf(sp.w3[j], x2[j], o); }
  return o;
}

// aligned_bilinear source of output index Y (condinst_head.py:146-167): position max(Y - f/2, 0)/f
__device__ __forceinline__ void up_src(int Y, int f, int len, int& i0, int& i1, float& fr) {
  if (f == 2) {                                    // every BoxInst/CondInst config: no integer / float division
    const int s = max(Y - 1, 0);
    i0 = s >> 1;
    fr = (s & 1) ? 0.5f : 0.f;
  } else {
    const int s = max(Y - f / 2, 0);
    i0 = s / f;
    fr = (float)(s - i0 * f) / (float)f;
  }
  i1 = min(i0 + 1, len - 1);
}

// ---------------------------------------------------------------------------------------
// forward
// ---------------------------------------------------------------------------------------
constexpr int FTY = 16, FTX = 32;                 // low-res tile of the forward kernel

template <int CMAX>
__global__ void __launch_bounds__(NT) head_fwd_kernel(const float* __restrict__ feat, const float* __restrict__ params,
                                                      const float* __restrict__ coors, const float* __restrict__ soi,
                                                      const int32_t* __restrict__ img_inds, float* __restrict__ out,
                                                      HeadDims d) {
  __shared__ __align__(16) SmemParams sp;
  __shared__ float s_low[FTY + 2][FTX + 2];
  const int n = blockIdx.z, ty0 = blockIdx.y * FTY, tx0 = blockIdx.x * FTX;
  load_params(sp, params, coors, soi, n, d);
  __syncthreads();
  const float* feat_img = feat + (int64_t)img_inds[n] * d.C * d.h * d.w;
  float in[CMAX + 2], x1[CH], x2[CH];
  for (int i = threadIdx.x; i < (FTY + 2) * (FTX + 2); i += NT) {
    const int r = i / (FTX + 2), c = i - r * (FTX + 2);
    const int y = min(max(ty0 - 1 + r, 0), d.h - 1), x = min(max(tx0 - 1 + c, 0), d.w - 1);
    gather_inputs<CMAX>(feat_img, sp, d, y, x, in);
    s_low[r][c] = mlp_forward<CMAX>(sp, in, d, x1, x2);
  }
  __syncthreads();
  const int OH = d.f * d.h, OW = d.f * d.w;
  const int oy0 = ty0 * d.f, ox0 = tx0 * d.f, th = FTY * d.f, tw = FTX * d.f;
  float* o = out + (int64_t)n * OH * OW;
  const int tw_shift = 31 - __clz(tw);             // tw = FTX * f is a power of two when f is (f = 2 -> 64)
  const bool tw_pow2 = (tw & (tw - 1)) == 0;
  for (int i = threadIdx.x; i < th * tw; i += NT) {
    const int ry = tw_pow2 ? (i >> tw_shift) : i / tw;
    const int Y = oy0 + ry, X = ox0 + (i - ry * tw);
    if (Y >= OH || X >= OW) continue;
    int y0, y1, x0, x1i;
    float fy, fx;
    up_src(Y, d.f, d.h, y0, y1, fy);
    up_src(X, d.f, d.w, x0, x1i, fx);
    const int r0 = y0 - (ty0 - 1), r1 = y1 - (ty0 - 1), c0 = x0 - (tx0 - 1), c1 = x1i - (tx0 - 1);
    const float top = s_low[r0][c0] * (1.f - fx) + s_low[r0][c1] * fx;
    const float bot = s_low[r1][c0] * (1.f - fx) + s_low[r1][c1] * fx;
    o[(int64_t)Y * OW + X] = top * (1.f - fy) + bot * fy;
  }
}

// ---------------------------------------------------------------------------------------
// backward
// ---------------------------------------------------------------------------------------
// stable counting sort of the instances by image (one CTA): order[N], start[B+1]
__global__ void group_by_image(const int32_t* __restrict__ img_inds, int N, int B, int* __restrict__ order,
                               int* __restrict__ start) {
  extern __shared__ int s_cnt[];               // B+1
  for (int b = threadIdx.x; b <= B; b += blockDim.x) s_cnt[b] = 0;
  __syncthreads();
  for (int n = threadIdx.x; n < N; n += blockDim.x) atomicAdd(&s_cnt[img_inds[n] + 1], 1);
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int b = 0; b < B; ++b) s_cnt[b + 1] += s_cnt[b];
    for (int b = 0; b <= B; ++b) start[b] = s_cnt[b];
    for (int n = 0; n < N; ++n) order[s_cnt[img_inds[n]]++] = n;      // stable, N is small
  }
}

constexpr int BTY = 8, BTX = 32;                  // 256 low-res pixels per CTA, one per thread
// per-pixel vectors for the outer products, [pixel][value] with odd pitches (bank-conflict free)
constexpr int PIT_8 = CH + 1;

template <int CMAX>
struct SmemBwd {
  static constexpr int PIT_IN = CMAX + 3;       // odd
  SmemParams sp;
  float in[NT * PIT_IN];       // layer-1 inputs (slot layout [rel_x, rel_y, feat..])
  float x1[NT * PIT_8];        // relu(layer 1)
  float x2[NT * PIT_8];        // relu(layer 2)
  float g1[NT * PIT_8];        // d/d pre-activation 1
  float g2[NT * PIT_8];        // d/d pre-activation 2
  float g3[NT];                // d/d low-res logit
};

template <int CMAX>
__global__ void __launch_bounds__(NT, 2) head_bwd_kernel(const float* __restrict__ feat, const float* __restrict__ params,
                                                      const float* __restrict__ coors, const float* __restrict__ soi,
                                                      const float* __restrict__ g_out, const int* __restrict__ order,
                                                      const int* __restrict__ start, float* __restrict__ g_feat,
                                                      float* __restrict__ g_params_partial, HeadDims d, int tiles,
                                                      int groups) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  using SB = SmemBwd<CMAX>;
  constexpr int PIT_IN = SB::PIT_IN;
  SB& S = *reinterpret_cast<SB*>(smem_raw);
  const int b = blockIdx.y, tile = blockIdx.x;
  const int tiles_x = (d.w + BTX - 1) / BTX;
  const int ty0 = (tile / tiles_x) * BTY, tx0 = (tile % tiles_x) * BTX;
  const int t = threadIdx.x;
  const int y = ty0 + t / BTX, x = tx0 + t % BTX;
  const bool live = y < d.h && x < d.w;
  const float* feat_img = feat + (int64_t)b * d.C * d.h * d.w;
  const int OH = d.f * d.h, OW = d.f * d.w;
  const int o = d.rel ? 2 : 0;                     // weight-row offset of the feature channels

  float gfeat[CMAX];
#pragma unroll
  for (int c = 0; c < CMAX; ++c) gfeat[c] = 0.f;
  float fin[CMAX + 2];                             // feature part is instance independent
#pragma unroll
  for (int c = 0; c < CMAX + 2; ++c) fin[c] = 0.f;
  if (live) {
    const int64_t plane = (int64_t)d.h * d.w, pix = (int64_t)y * d.w + x;
#pragma unroll
    for (int c = 0; c < CMAX; ++c)
      if (c < d.C) fin[2 + c] = __ldg(feat_img + c * plane + pix);
  }

  // transpose of the aligned upsample for factor 2 (every BoxInst/CondInst config): the weights of the 6 x 6 output
  // pixels that read this low-res pixel depend only on (y, x), not on the instance -> computed once per thread
  const bool f2 = d.f == 2;
  float wyv[6], wxv[6];
  const int Y0 = max(2 * (y - 1), 0), X0 = max(2 * (x - 1), 0);
#pragma unroll
  for (int a = 0; a < 6; ++a) {
    wyv[a] = 0.f; wxv[a] = 0.f;
    if (f2 && live) {
      int i0, i1; float fr;
      const int Y = Y0 + a, X = X0 + a;
      if (Y < min(2 * (y + 2), OH)) { up_src(Y, 2, d.h, i0, i1, fr); wyv[a] = (i0 == y ? 1.f - fr : 0.f) + (i1 == y ? fr : 0.f); }
      if (X < min(2 * (x + 2), OW)) { up_src(X, 2, d.w, i0, i1, fr); wxv[a] = (i0 == x ? 1.f - fr : 0.f) + (i1 == x ? fr : 0.f); }
    }
  }
  const int grp = blockIdx.z;                      // this CTA handles instances start[b] + grp, + groups, ...
  for (int it = start[b] + grp; it < start[b + 1]; it += groups) {
    const int n = order[it];
    __syncthreads();                               // previous instance fully consumed
    load_params(S.sp, params, coors, soi, n, d);
    __syncthreads();
    float x1[CH], x2[CH], g1[CH], g2[CH], g3 = 0.f;
    if (live) {
      // ---- d/d low-res logit: transpose of the aligned upsample (gather) ----
      const float* go = g_out + (int64_t)n * OH * OW;
      if (f2) {                                      // same terms, same order as the general loop below
#pragma unroll
        for (int a = 0; a < 6; ++a) {
          if (wyv[a] == 0.f) continue;
          const float* grow = go + (int64_t)(Y0 + a) * OW + X0;
          float rowacc = 0.f;
#pragma unroll
          for (int c = 0; c < 6; ++c)
            if (wxv[c] != 0.f) rowacc = fmaf(wxv[c], __ldg(grow + c), rowacc);
          g3 = fmaf(wyv[a], rowacc, g3);
        }
      } else {
        for (int Y = max(d.f * (y - 1), 0); Y < min(d.f * (y + 2), OH); ++Y) {
          int a0, a1; float fr;
          up_src(Y, d.f, d.h, a0, a1, fr);
          const float wy = (a0 == y ? 1.f - fr : 0.f) + (a1 == y ? fr : 0.f);
          if (wy == 0.f) continue;
          float rowacc = 0.f;
          for (int X = max(d.f * (x - 1), 0); X < min(d.f * (x + 2), OW); ++X) {
            int c0, c1; float fc;
            up_src(X, d.f, d.w, c0, c1, fc);
            const float wx = (c0 == x ? 1.f - fc : 0.f) + (c1 == x ? fc : 0.f);
            if (wx != 0.f) rowacc = fmaf(wx, __ldg(go + (int64_t)Y * OW + X), rowacc);
          }
          g3 = fmaf(wy, rowacc, g3);
        }
      }
      // ---- recompute the forward, then backpropagate through the three layers ----
      if (d.rel) {
        fin[0] = __fdiv_rn(S.sp.cx - (float)(x * d.stride + d.stride / 2), S.sp.soi);
        fin[1] = __fdiv_rn(S.sp.cy - (float)(y * d.stride + d.stride / 2), S.sp.soi);
      }
      mlp_forward<CMAX>(S.sp, fin, d, x1, x2);
#pragma unroll
      for (int j = 0; j < CH; ++j) g2[j] = x2[j] > 0.f ? g3 * S.sp.w3[j] : 0.f;
#pragma unroll
      for (int k = 0; k < CH; ++k) {                // g_x1[k] = sum_j W2[j][k] g2[j] ; w2t[k][j]
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < CH; ++j) acc = fmaf(S.sp.w2t[k * CH + j], g2[j], acc);
        g1[k] = x1[k] > 0.f ? acc : 0.f;
      }
#pragma unroll
      for (int c = 0; c < CMAX; ++c) {              // g_in[o+c] = sum_j W1[j][o+c] g1[j]
        if (c >= d.C) continue;
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < CH; ++j) acc = fmaf(S.sp.w1t[(o + c) * CH + j], g1[j], acc);
        gfeat[c] += acc;
      }
    } else {
#pragma unroll
      for (int j = 0; j < CH; ++j) { x1[j] = x2[j] = g1[j] = g2[j] = 0.f; }
    }
    // ---- stage the per-pixel vectors, then reduce the outer products over the tile ----
#pragma unroll
    for (int k = 0; k < CMAX + 2; ++k) S.in[t * PIT_IN + k] = live ? fin[k] : 0.f;
#pragma unroll
    for (int j = 0; j < CH; ++j) {
      S.x1[t * PIT_8 + j] = x1[j]; S.x2[t * PIT_8 + j] = x2[j];
      S.g1[t * PIT_8 + j] = g1[j]; S.g2[t * PIT_8 + j] = g2[j];
    }
    S.g3[t] = g3;
    __syncthreads();
    // output index q in [0,P): same layout as params
    const int o2 = CH * d.cin, o3 = o2 + CH * CH, ob1 = o3 + CH, ob2 = ob1 + CH, ob3 = ob2 + CH;
    for (int q = t; q < d.P; q += NT) {
      const float *A, *Bv;
      int pa, pb, ia, ib;                          // sum_p A[p*pa+ia] * B[p*pb+ib]
      const float* ones = nullptr;
      if (q < o2)        { A = S.g1; pa = PIT_8; ia = q / d.cin; Bv = S.in; pb = PIT_IN; ib = q % d.cin + (2 - o); }
      else if (q < o3)   { A = S.g2; pa = PIT_8; ia = (q - o2) / CH; Bv = S.x1; pb = PIT_8; ib = (q - o2) % CH; }
      else if (q < ob1)  { A = S.g3; pa = 1; ia = 0; Bv = S.x2; pb = PIT_8; ib = q - o3; }
      else if (q < ob2)  { A = S.g1; pa = PIT_8; ia = q - ob1; Bv = ones; pb = 0; ib = 0; }
      else if (q < ob3)  { A = S.g2; pa = PIT_8; ia = q - ob2; Bv = ones; pb = 0; ib = 0; }
      else               { A = S.g3; pa = 1; ia = 0; Bv = ones; pb = 0; ib = 0; }
      float acc = 0.f;
      if (Bv) {
#pragma unroll 8
        for (int p = 0; p < NT; ++p) acc = fmaf(A[p * pa + ia], Bv[p * pb + ib], acc);
      } else {
#pragma unroll 8
        for (int p = 0; p < NT; ++p) acc += A[p * pa + ia];
      }
      g_params_partial[((int64_t)n * tiles + tile) * d.P + q] = acc;
    }
  }
  if (live) {
    const int64_t plane = (int64_t)d.h * d.w, pix = (int64_t)y * d.w + x;
    // groups == 1: g_feat itself; else partial [grp][B][C][h*w] (g_feat then points at the partial buffer)
    float* gf = g_feat + ((int64_t)grp * d.B + b) * d.C * plane;
#pragma unroll
    for (int c = 0; c < CMAX; ++c)
      if (c < d.C) gf[c * plane + pix] = gfeat[c];
  }
}

// g_feat[i] = sum over groups of partial[g][i], fixed order
__global__ void feat_reduce_kernel(const float4* __restrict__ partial, float4* __restrict__ g_feat, int64_t n4, int groups) {
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 a = partial[i];
    for (int g = 1; g < groups; ++g) {
      const float4 v = partial[g * n4 + i];
      a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
    }
    g_feat[i] = a;
  }
}

__global__ void params_reduce_kernel(const float* __restrict__ partial, float* __restrict__ g_params, int N, int tiles,
                                     int P) {
  const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
  if (idx >= (int64_t)N * P) return;
  const int n = idx / P, q = idx % P;
  float acc = 0.f;
  for (int tle = 0; tle < tiles; ++tle) acc += partial[((int64_t)n * tiles + tle) * P + q];
  g_params[idx] = acc;
}

inline bool dims_ok(const HeadDims& d) {
  return d.N > 0 && d.N < 65536 && d.B > 0 && d.C > 0 && d.C <= MAX_CIN - 2 && d.h > 0 && d.w > 0 && d.f >= 1 &&
         d.f <= 8 && d.stride > 0 && d.P == CH * d.cin + CH * CH + CH + CH + CH + 1;
}

inline HeadDims make_dims(int64_t N, int64_t B, int64_t C, int64_t h, int64_t w, int in_stride, int factor, int rel,
                          int64_t P) {
  HeadDims d;
  d.N = (int)N; d.B = (int)B; d.C = (int)C; d.h = (int)h; d.w = (int)w; d.cin = (int)C + (rel ? 2 : 0);
  d.stride = in_stride; d.f = factor; d.rel = rel; d.P = (int)P;
  return d;
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_condinst_head_forward(const float* feat, const float* params, const float* coors, const float* soi,
                                         const int32_t* img_inds, float* out, int64_t N, int64_t B, int64_t C,
                                         int64_t h, int64_t w, int64_t P, int in_stride, int factor, int rel_coors,
                                         bxs_stream_t stream) {
  if (!feat || !params || !img_inds || !out || (rel_coors && (!coors || !soi))) return BXS_ERR_INVALID_ARG;
  HeadDims d = make_dims(N, B, C, h, w, in_stride, factor, rel_coors, P);
  if (!dims_ok(d)) return BXS_ERR_UNSUPPORTED;
  dim3 grid((unsigned)ceil_div(w, FTX), (unsigned)ceil_div(h, FTY), (unsigned)N);
  cudaStream_t st = as_stream(stream);
  if (C <= 8) head_fwd_kernel<8><<<grid, NT, 0, st>>>(feat, params, coors, soi, img_inds, out, d);
  else if (C <= 16) head_fwd_kernel<16><<<grid, NT, 0, st>>>(feat, params, coors, soi, img_inds, out, d);
  else head_fwd_kernel<32><<<grid, NT, 0, st>>>(feat, params, coors, soi, img_inds, out, d);
  return check_launch();
}

namespace bxs {
namespace {
constexpr int kMaxGroups = 8;
// instance groups per image of the backward grid: enough CTAs for ~4 per SM, at most kMaxGroups
inline int bwd_groups(int64_t N, int64_t B, int64_t tiles) {
  const int64_t want = ceil_div((int64_t)sm_count() * 4, tiles * B);
  return (int)std::max<int64_t>(1, std::min<int64_t>({want, (int64_t)kMaxGroups, ceil_div(N, B)}));
}
}  // namespace
}  // namespace bxs

extern "C" int64_t bxs_condinst_head_workspace_bytes(int64_t N, int64_t B, int64_t h, int64_t w, int64_t P) {
  const int64_t tiles = ceil_div(h, BTY) * ceil_div(w, BTX);
  const int64_t cin = (P - (CH * CH + 3 * CH + 1)) / CH;            // >= mask_feat channels
  return (N + B + 1) * 4 + 512 + N * tiles * P * 4 + (int64_t)kMaxGroups * B * cin * h * w * 4 + 16;
}

extern "C" int bxs_condinst_head_backward(const float* feat, const float* params, const float* coors, const float* soi,
                                          const int32_t* img_inds, const float* g_out, float* g_feat, float* g_params,
                                          void* workspace, int64_t N, int64_t B, int64_t C, int64_t h, int64_t w,
                                          int64_t P, int in_stride, int factor, int rel_coors, bxs_stream_t stream) {
  if (!feat || !params || !img_inds || !g_out || !g_feat || !g_params || !workspace ||
      (rel_coors && (!coors || !soi)))
    return BXS_ERR_INVALID_ARG;
  HeadDims d = make_dims(N, B, C, h, w, in_stride, factor, rel_coors, P);
  if (!dims_ok(d) || B > 8192) return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  const int tiles = (int)(ceil_div(h, BTY) * ceil_div(w, BTX));
  int* order = (int*)workspace;
  int* start = order + N;
  float* partial = (float*)((char*)workspace + ((N + B + 1) * 4 + 255) / 256 * 256);
  float* feat_partial = (float*)((char*)partial + ((size_t)N * tiles * P * 4 + 255) / 256 * 256);
  const int groups = bwd_groups(N, B, tiles);
  const bool vec4 = ((B * C * h * w) % 4 == 0) && ((reinterpret_cast<uintptr_t>(g_feat) & 15) == 0);
  const int use_groups = vec4 ? groups : 1;
  float* gf_target = use_groups > 1 ? feat_partial : g_feat;
  group_by_image<<<1, 256, (B + 1) * sizeof(int), st>>>(img_inds, (int)N, (int)B, order, start);
#define BXS_LAUNCH_BWD(CM)                                                                                   \
  do {                                                                                                       \
    if (opt_in_smem(head_bwd_kernel<CM>, sizeof(SmemBwd<CM>)) != BXS_OK) return BXS_ERR_LAUNCH;              \
    head_bwd_kernel<CM><<<dim3(tiles, (unsigned)B, (unsigned)use_groups), NT, sizeof(SmemBwd<CM>), st>>>(    \
        feat, params, coors, soi, g_out, order, start, gf_target, partial, d, tiles, use_groups);            \
  } while (0)
  if (C <= 8) BXS_LAUNCH_BWD(8);
  else if (C <= 16) BXS_LAUNCH_BWD(16);
  else BXS_LAUNCH_BWD(32);
#undef BXS_LAUNCH_BWD
  int rc = check_launch();
  if (rc) return rc;
  // images without instances never write their partials: zero-fill is not needed because every
  // instance belongs to exactly one image and that image's CTAs write all of its tiles.
  params_reduce_kernel<<<(unsigned)ceil_div(N * P, 256), 256, 0, st>>>(partial, g_params, (int)N, tiles, (int)P);
  if (use_groups > 1) {
    const int64_t n4 = B * C * h * w / 4;
    feat_reduce_kernel<<<(unsigned)std::min<int64_t>(ceil_div(n4, 256), (int64_t)sm_count() * 8), 256, 0, st>>>(
        reinterpret_cast<const float4*>(feat_partial), reinterpret_cast<float4*>(g_feat), n4, use_groups);
  }
  return check_launch();
}
