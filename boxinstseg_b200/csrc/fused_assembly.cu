// a14, a17, a18: the glue the reference leaves to eager PyTorch around its loss kernels, as kernels.
//
//   a18  bilinear resize, forward + deterministic backward -- F.interpolate(mode='bilinear') as called by
//        _scale_target (mmdet/models/utils/misc.py:75-86) and box2mask_head.py:232-233,300,315-317,323-324,329 /
//        box_solov2_head.py:213,412-415 (align_corners False) and discobox_head.py:1201 (align_corners True).
//        Same arithmetic as ATen's upsample_bilinear2d (source index, lambdas, the order of the four products);
//        the backward is a gather over the output pixels that touch an input pixel instead of ATen's atomicAdd
//        scatter, hence run-to-run deterministic.
//   a14  TreeFilter2D.build_edge_weight (mmdet/ops/tree_filter/modules/tree_filter.py:91-108): two [n,C,V] gathers +
//        squared distance + exp as ONE kernel, and its autograd (scatter to both end points of every tree edge) as
//        ONE gather kernel over (own edge, child edges).
//   a17  the level-set assembly of box_solov2_head.py:341-360 / box2mask_head.py:305-327: sigmoid, cat(s, 1-s) * box,
//        T * box, clamp(sum box, 1) and LevelsetLoss (levelset_loss.py:13-44) in ONE launch per call: a thread-block
//        cluster of 8 CTAs per instance, the two-pass dependency (means, then energy) resolved through distributed
//        shared memory, plus one backward launch that writes d/d logits and d/d T directly.
#include <cooperative_groups.h>

#include <algorithm>

#include "common.cuh"
#include "resize_core.cuh"

namespace cg = cooperative_groups;

namespace bxs {
namespace {

constexpr int NT = 256;

// ---------------------------------------------------------------------------------------
// a18: bilinear resize (ATen UpSample.cuh semantics; the arithmetic is in resize_core.cuh)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) resize_fwd_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t NC,
                                                        int h, int w, int H, int W, bool align) {
  const float sh = rs_scale(h, H, align), sw = rs_scale(w, W, align);
  const int64_t total = NC * H * W;
  for (int64_t i = blockIdx.x * (int64_t)NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    const int ox = (int)(i % W), oy = (int)((i / W) % H);
    const int64_t nc = i / ((int64_t)W * H);
    out[i] = rs_pixel(in + nc * h * w, h, w, sh, sw, oy, ox, align);
  }
}

// output indices whose taps can touch input index `ii`: a superset [lo, hi] (each candidate is re-checked exactly)
__device__ __forceinline__ void rs_candidates(float scale, int ii, int out, bool align, int& lo, int& hi) {
  if (scale <= 0.f) { lo = 0; hi = out - 1; return; }
  const float inv = 1.f / scale, off = align ? 0.f : 0.5f;
  lo = (int)floorf(((float)ii - 1.f + off) * inv - off) - 1;
  hi = (int)ceilf(((float)ii + 1.f + off) * inv - off) + 1;
  lo = max(lo, 0);
  hi = min(hi, out - 1);
}

__global__ void __launch_bounds__(NT) resize_bwd_kernel(const float* __restrict__ g_out, float* __restrict__ g_in,
                                                        int64_t NC, int h, int w, int H, int W, bool align) {
  const float sh = rs_scale(h, H, align), sw = rs_scale(w, W, align);
  const int64_t total = NC * h * w;
  for (int64_t i = blockIdx.x * (int64_t)NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    const int ix = (int)(i % w), iy = (int)((i / w) % h);
    const int64_t nc = i / ((int64_t)w * h);
    int ylo, yhi, xlo, xhi;
    rs_candidates(sh, iy, H, align, ylo, yhi);
    rs_candidates(sw, ix, W, align, xlo, xhi);
    const float* g = g_out + nc * H * W;
    float acc = 0.f;
    for (int oy = ylo; oy <= yhi; ++oy) {
      const RsTap ty = rs_tap(sh, oy, h, align);
      float wy = 0.f;                                  // both taps may land on iy (ip == 0 at the border)
      if (ty.i0 == iy) wy += ty.l0;
      if (ty.i0 + ty.ip == iy) wy += ty.l1;
      if (wy == 0.f) continue;
      float row = 0.f;
      for (int ox = xlo; ox <= xhi; ++ox) {
        const RsTap tx = rs_tap(sw, ox, w, align);
        float wx = 0.f;
        if (tx.i0 == ix) wx += tx.l0;
        if (tx.i0 + tx.ip == ix) wx += tx.l1;
        if (wx != 0.f) row = fmaf(wx, __ldg(g + (int64_t)oy * W + ox), row);
      }
      acc = fmaf(wy, row, acc);
    }
    g_in[i] = acc;
  }
}

// ---------------------------------------------------------------------------------------
// a14: tree edge weights  w[p] = exp(-|E(v_p) - E(v_par(p))|^2 / sigma)
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) edge_weight_fwd_kernel(const float* __restrict__ embed, const int32_t* __restrict__ idx,
                                                             const int32_t* __restrict__ par, float* __restrict__ w,
                                                             int64_t BG, int groups, int C, int V, float sigma) {
  const int64_t total = BG * V;
  for (int64_t i = blockIdx.x * (int64_t)NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    const int p = (int)(i % V);
    const int64_t bg = i / V, b = bg / groups;
    const int32_t* ib = idx + b * V;
    const int v = __ldg(ib + p), u = __ldg(ib + __ldg(par + b * V + p));
    const float* e = embed + bg * C * V;
    float d = 0.f;
    for (int c = 0; c < C; ++c) {
      const float t = __ldg(e + (int64_t)c * V + v) - __ldg(e + (int64_t)c * V + u);
      d += t * t;                                      // (diff * diff).sum(dim=1), tree_filter.py:83-84
    }
    w[i] = expf(-d / sigma);
  }
}

// d/d embed: vertex v at position p receives from its own edge (p, par) and from the edges of its children
__global__ void __launch_bounds__(NT) edge_weight_bwd_kernel(const float* __restrict__ embed, const int32_t* __restrict__ idx,
                                                             const int32_t* __restrict__ par, const int32_t* __restrict__ chd,
                                                             const float* __restrict__ w, const float* __restrict__ g_w,
                                                             float* __restrict__ g_embed, int64_t BG, int groups, int C,
                                                             int V, float sigma) {
  const int64_t total = BG * V;
  const float k = -2.f / sigma;
  for (int64_t i = blockIdx.x * (int64_t)NT + threadIdx.x; i < total; i += (int64_t)gridDim.x * NT) {
    const int p = (int)(i % V);
    const int64_t bg = i / V, b = bg / groups;
    const int32_t* ib = idx + b * V;
    const int v = __ldg(ib + p);
    const float* e = embed + bg * C * V;
    const float* wb = w + bg * V;
    const float* gb = g_w + bg * V;
    // neighbours of v in the tree: parent (own edge) and up to 4 children
    int nv[5];
    float coef[5];
    int cnt = 0;
    if (p > 0) { nv[cnt] = __ldg(ib + __ldg(par + b * V + p)); coef[cnt] = __ldg(gb + p) * __ldg(wb + p) * k; ++cnt; }
    const int32_t* cp = chd + (b * V + p) * 4;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int q = __ldg(cp + j);
      if (q > 0) { nv[cnt] = __ldg(ib + q); coef[cnt] = __ldg(gb + q) * __ldg(wb + q) * k; ++cnt; }
    }
    for (int c = 0; c < C; ++c) {
      const float ev = __ldg(e + (int64_t)c * V + v);
      float acc = 0.f;
      for (int j = 0; j < cnt; ++j) acc = fmaf(coef[j], ev - __ldg(e + (int64_t)c * V + nv[j]), acc);
      g_embed[(bg * C + c) * V + v] = acc;
    }
  }
}

// ---------------------------------------------------------------------------------------
// a17: level-set assembly, one cluster of 8 CTAs per instance
// ---------------------------------------------------------------------------------------
constexpr int LS_MAXC = 8;
constexpr int LS_CL = 8;            // CTAs per cluster (portable maximum)
constexpr int LS_NT = 512;
constexpr float kLsEps = 1e-5f;     // levelset_loss.py:36-37

struct LsfStats {                    // per instance: what the backward needs
  float den[2], z[2];
  float a[2][LS_MAXC], m[2][LS_MAXC], d[2][LS_MAXC];
  float pix, energy;
};

// FUSED: (a, b, T) of a pixel come from (logit, box, raw T): a = s m, b = (1 - s) m, T <- T m   (box2mask_head.py:305-312)
// else : (a, b) = the two channels of `scores2`, T as given                                   (levelset_loss.py:13-18)
template <bool FUSED>
struct LsfPixel {
  const float* x;      // FUSED: logits [hw]        else: scores channel 0
  const float* y;      // FUSED: box [hw]           else: scores channel 1
  const float* t;      // [C, hw]
  int64_t hw;
  __device__ __forceinline__ void ab(int64_t p, float& a, float& b, float& m) const {
    if (FUSED) {
      m = __ldg(y + p);
      const float s = 1.f / (1.f + expf(-__ldg(x + p)));             // torch.sigmoid in fp32
      a = s * m;
      b = (1.f - s) * m;
    } else {
      m = 1.f;
      a = __ldg(x + p);
      b = __ldg(y + p);
    }
  }
  __device__ __forceinline__ float tv(int c, int64_t p, float m) const {
    const float v = __ldg(t + (int64_t)c * hw + p);
    return FUSED ? v * m : v;
  }
};

// CTA-wide sums of NV values in a fixed order (warp shuffles, then the warps in order): thread i < NV ends up with the CTA's
// sum of value i in `v[i]`... as `own`; the other threads' values are left untouched.  (Round 2a had every thread add up all
// NV x 16 warp partials itself: 304 shared-memory loads per thread per pass -- two thirds of the kernel's 11 M instructions.)
template <int NV>
__device__ __forceinline__ float lsf_block_sum(const float (&v)[NV], float* s_warp /* [NV][LS_NT/32] */) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int i = 0; i < NV; ++i) {
    const float r = warp_sum(v[i]);
    if (lane == 0) s_warp[i * (LS_NT / 32) + wid] = r;
  }
  __syncthreads();
  float own = 0.f;
  if (threadIdx.x < NV) {
#pragma unroll
    for (int k = 0; k < LS_NT / 32; ++k) own += s_warp[threadIdx.x * (LS_NT / 32) + k];
  }
  return own;
}

// MC: compile-time bound of the channel loops (4 for C <= 4, else LS_MAXC): the loops are fully unrolled and predicated on c < C
template <bool FUSED, int MC>
__global__ void __cluster_dims__(LS_CL, 1, 1) __launch_bounds__(LS_NT)
lsf_forward_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ T,
                   const float* __restrict__ pixel_num, int C, int64_t hw, float loss_weight,
                   LsfStats* __restrict__ stats, float* __restrict__ loss) {
  constexpr int NV1 = 3 + 2 * MC, NV2 = 1 + 2 * MC;
  __shared__ float s_warp[NV1 * (LS_NT / 32)];
  __shared__ float s_part[NV1];                 // this CTA's partial sums, read by the whole cluster
  __shared__ float s_tot[NV1];                  // the cluster's totals of pass 1
  cg::cluster_group cluster = cg::this_cluster();
  const int n = blockIdx.x / LS_CL, rank = (int)cluster.block_rank();
  LsfPixel<FUSED> px;
  px.hw = hw;
  px.x = FUSED ? x + (int64_t)n * hw : x + (int64_t)n * 2 * hw;
  px.y = FUSED ? y + (int64_t)n * hw : x + (int64_t)n * 2 * hw + hw;
  px.t = T + (int64_t)n * C * hw;
  // ---- pass 1: z0, z1, pix, a0[c], a1[c] ----
  float acc[NV1];
#pragma unroll
  for (int i = 0; i < NV1; ++i) acc[i] = 0.f;
  for (int64_t p = (int64_t)rank * LS_NT + threadIdx.x; p < hw; p += (int64_t)LS_CL * LS_NT) {
    float a, b, m;
    px.ab(p, a, b, m);
    acc[0] += a; acc[1] += b; acc[2] += m;
#pragma unroll
    for (int c = 0; c < MC; ++c)
      if (c < C) {
        const float tv = px.tv(c, p, m);
        acc[3 + c] = fmaf(a, tv, acc[3 + c]);
        acc[3 + MC + c] = fmaf(b, tv, acc[3 + MC + c]);
      }
  }
  {
    const float own = lsf_block_sum<NV1>(acc, s_warp);
    if (threadIdx.x < NV1) s_part[threadIdx.x] = own;
  }
  cluster.sync();
  // thread i < NV1 of every CTA sums value i of the 8 partials in rank order (identical statistics in every CTA, no broadcast
  // needed) and publishes it to its own CTA
  if (threadIdx.x < NV1) {
    float t = 0.f;
    for (int r = 0; r < LS_CL; ++r) t += cluster.map_shared_rank(s_part, r)[threadIdx.x];
    s_tot[threadIdx.x] = t;
  }
  cluster.sync();                                 // s_part is rewritten below; s_tot is complete
  float tot[NV1];
#pragma unroll
  for (int i = 0; i < NV1; ++i) tot[i] = s_tot[i];
  float den[2], mean[2][MC];
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    den[k] = fmaxf(tot[k], kLsEps);
#pragma unroll
    for (int c = 0; c < MC; ++c) mean[k][c] = c < C ? tot[3 + k * MC + c] / den[k] : 0.f;
  }
  // ---- pass 2: C * energy, r0[c] = sum (T - m0) a, r1[c] ----
  float acc2[NV2];
#pragma unroll
  for (int i = 0; i < NV2; ++i) acc2[i] = 0.f;
  for (int64_t p = (int64_t)rank * LS_NT + threadIdx.x; p < hw; p += (int64_t)LS_CL * LS_NT) {
    float a, b, m;
    px.ab(p, a, b, m);
#pragma unroll
    for (int c = 0; c < MC; ++c)
      if (c < C) {
        const float tv = px.tv(c, p, m);
        const float d0 = tv - mean[0][c], d1 = tv - mean[1][c];
        acc2[0] = fmaf(d0 * d0, a, acc2[0]);
        acc2[0] = fmaf(d1 * d1, b, acc2[0]);
        acc2[1 + c] = fmaf(d0, a, acc2[1 + c]);
        acc2[1 + MC + c] = fmaf(d1, b, acc2[1 + MC + c]);
      }
  }
  {
    const float own = lsf_block_sum<NV2>(acc2, s_warp);
    if (threadIdx.x < NV2) s_part[threadIdx.x] = own;
  }
  cluster.sync();
  if (rank == 0) {
    if (threadIdx.x < NV2) {                      // value i of the 8 partials, rank order
      float t = 0.f;
      for (int r = 0; r < LS_CL; ++r) t += cluster.map_shared_rank(s_part, r)[threadIdx.x];
      s_tot[threadIdx.x] = t;
    }
    __syncthreads();
  }
  if (rank == 0 && threadIdx.x == 0) {
    float tot2[NV2];
    for (int i = 0; i < NV2; ++i) tot2[i] = s_tot[i];
    LsfStats st;
    for (int k = 0; k < 2; ++k) {
      st.z[k] = tot[k];
      st.den[k] = den[k];
      for (int c = 0; c < LS_MAXC; ++c) {
        const bool in = c < C && c < MC;
        st.a[k][c] = in ? tot[3 + k * MC + (c < MC ? c : 0)] : 0.f;
        st.m[k][c] = in ? mean[k][c < MC ? c : 0] : 0.f;
        st.d[k][c] = in ? -2.f / (float)C * tot2[1 + k * MC + (c < MC ? c : 0)] : 0.f;
      }
    }
    st.energy = tot2[0] / (float)C;
    st.pix = FUSED ? fmaxf(tot[2], 1.f) : pixel_num[n];           // clamp(sum box, min=1), box2mask_head.py:309-310
    stats[n] = st;
    loss[n] = loss_weight * st.energy / st.pix;
  }
  cluster.sync();                                 // rank 0 reads the other CTAs' shared memory until here
}

// d/d (a, b) and d/d T of loss_n = w E / pix, chained to d/d logits (through a = s m, b = (1 - s) m) and d/d raw T
// (through T m) when FUSED.  The clamp(sum S_k, min=eps) passes no gradient while it is active.  Instance n0 + blockIdx.y.
template <bool FUSED>
__global__ void __launch_bounds__(NT)
lsf_backward_kernel(const float* __restrict__ x, const float* __restrict__ y, const float* __restrict__ T, int C, int64_t hw,
                    const LsfStats* __restrict__ stats, float loss_weight, const float* __restrict__ g_loss,
                    float* __restrict__ g_x, float* __restrict__ g_T, int64_t n0) {
  __shared__ LsfStats st;
  const int64_t n = n0 + blockIdx.y;            // instances go over launches of at most 65535 (gridDim.y)
  if (threadIdx.x == 0) st = stats[n];
  __syncthreads();
  const float scale = g_loss[n] * loss_weight / st.pix;
  const float inv_c = 1.f / (float)C;
  LsfPixel<FUSED> px;
  px.hw = hw;
  px.x = FUSED ? x + (int64_t)n * hw : x + (int64_t)n * 2 * hw;
  px.y = FUSED ? y + (int64_t)n * hw : x + (int64_t)n * 2 * hw + hw;
  px.t = T + (int64_t)n * C * hw;
  float off[2] = {0.f, 0.f};
  for (int k = 0; k < 2; ++k)
    if (st.z[k] > kLsEps)
      for (int c = 0; c < C; ++c) off[k] -= st.d[k][c] * st.a[k][c] / (st.den[k] * st.den[k]);
  for (int64_t p = blockIdx.x * (int64_t)NT + threadIdx.x; p < hw; p += (int64_t)gridDim.x * NT) {
    float a, b, m;
    px.ab(p, a, b, m);
    float g0 = off[0], g1 = off[1];
#pragma unroll
    for (int c = 0; c < LS_MAXC; ++c)
      if (c < C) {
        const float tv = px.tv(c, p, m);
        const float d0 = tv - st.m[0][c], d1 = tv - st.m[1][c];
        g0 += d0 * d0 * inv_c + st.d[0][c] * tv / st.den[0];
        g1 += d1 * d1 * inv_c + st.d[1][c] * tv / st.den[1];
        if (g_T) {
          const float gt = scale * (2.f * inv_c * (d0 * a + d1 * b) + st.d[0][c] * a / st.den[0] + st.d[1][c] * b / st.den[1]);
          g_T[((int64_t)n * C + c) * hw + p] = FUSED ? gt * m : gt;
        }
      }
    if (g_x) {
      if (FUSED) {
        const float s = 1.f / (1.f + expf(-__ldg(px.x + p)));
        g_x[(int64_t)n * hw + p] = scale * (g0 - g1) * m * s * (1.f - s);
      } else {
        g_x[(int64_t)n * 2 * hw + p] = scale * g0;
        g_x[(int64_t)n * 2 * hw + hw + p] = scale * g1;
      }
    }
  }
}

}  // namespace
}  // namespace bxs

using namespace bxs;

extern "C" int bxs_bilinear_resize_forward(const float* in, float* out, int64_t NC, int64_t h, int64_t w, int64_t H, int64_t W,
                                           int align_corners, bxs_stream_t stream) {
  if (!in || !out || NC <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0) return BXS_ERR_INVALID_ARG;
  if (h >= (1 << 24) || w >= (1 << 24) || H >= (1 << 24) || W >= (1 << 24)) return BXS_ERR_UNSUPPORTED;
  resize_fwd_kernel<<<grid_for(NC * H * W, NT, 16), NT, 0, as_stream(stream)>>>(in, out, NC, (int)h, (int)w, (int)H, (int)W,
                                                                                  align_corners != 0);
  return check_launch();
}

extern "C" int bxs_bilinear_resize_backward(const float* g_out, float* g_in, int64_t NC, int64_t h, int64_t w, int64_t H,
                                            int64_t W, int align_corners, bxs_stream_t stream) {
  if (!g_out || !g_in || NC <= 0 || h <= 0 || w <= 0 || H <= 0 || W <= 0) return BXS_ERR_INVALID_ARG;
  if (h >= (1 << 24) || w >= (1 << 24) || H >= (1 << 24) || W >= (1 << 24)) return BXS_ERR_UNSUPPORTED;
  resize_bwd_kernel<<<grid_for(NC * h * w, NT, 16), NT, 0, as_stream(stream)>>>(g_out, g_in, NC, (int)h, (int)w, (int)H,
                                                                                  (int)W, align_corners != 0);
  return check_launch();
}

extern "C" int bxs_tree_edge_weight_forward(const float* embed, const int32_t* sorted_index, const int32_t* sorted_parent,
                                            float* edge_weight, int64_t B, int64_t groups, int64_t C, int64_t V, float sigma,
                                            bxs_stream_t stream) {
  if (!embed || !sorted_index || !sorted_parent || !edge_weight || B <= 0 || groups <= 0 || C <= 0 || V <= 0 ||
      V >= (int64_t(1) << 31) || !(sigma > 0.f))
    return BXS_ERR_INVALID_ARG;
  edge_weight_fwd_kernel<<<grid_for(B * groups * V, NT, 16), NT, 0, as_stream(stream)>>>(
      embed, sorted_index, sorted_parent, edge_weight, B * groups, (int)groups, (int)C, (int)V, sigma);
  return check_launch();
}

extern "C" int bxs_tree_edge_weight_backward(const float* embed, const int32_t* sorted_index, const int32_t* sorted_parent,
                                             const int32_t* sorted_child, const float* edge_weight, const float* g_weight,
                                             float* g_embed, int64_t B, int64_t groups, int64_t C, int64_t V, float sigma,
                                             bxs_stream_t stream) {
  if (!embed || !sorted_index || !sorted_parent || !sorted_child || !edge_weight || !g_weight || !g_embed || B <= 0 ||
      groups <= 0 || C <= 0 || V <= 0 || V >= (int64_t(1) << 31) || !(sigma > 0.f))
    return BXS_ERR_INVALID_ARG;
  edge_weight_bwd_kernel<<<grid_for(B * groups * V, NT, 16), NT, 0, as_stream(stream)>>>(
      embed, sorted_index, sorted_parent, sorted_child, edge_weight, g_weight, g_embed, B * groups, (int)groups, (int)C, (int)V,
      sigma);
  return check_launch();
}

extern "C" int64_t bxs_levelset_fused_workspace_bytes(int64_t n) { return n <= 0 ? 0 : (int64_t)(sizeof(LsfStats) * n); }

// mode 0: x = scores2 [n,2,h,w], y unused, pixel_num [n] given (LevelsetLoss.forward as the reference calls it)
// mode 1: x = logits [n,h,w], y = box mask [n,h,w], T raw [n,C,h,w]; sigmoid / cat / * box / clamp(sum box, 1) inside
extern "C" int bxs_levelset_fused_forward(const float* x, const float* y, const float* T, const float* pixel_num, float* loss,
                                          void* workspace, int64_t n, int64_t C, int64_t h, int64_t w, float loss_weight,
                                          int mode, bxs_stream_t stream) {
  if (!x || !T || !loss || !workspace || n <= 0 || n > INT32_MAX / LS_CL || h <= 0 || w <= 0 || (mode == 0 && !pixel_num) ||
      (mode == 1 && !y) || (mode != 0 && mode != 1))
    return BXS_ERR_INVALID_ARG;
  if (C < 1 || C > LS_MAXC) return BXS_ERR_UNSUPPORTED;
  cudaStream_t st = as_stream(stream);
  LsfStats* stats = reinterpret_cast<LsfStats*>(workspace);
  if (mode == 1)
    if (C <= 4) lsf_forward_kernel<true, 4><<<(unsigned)(n * LS_CL), LS_NT, 0, st>>>(x, y, T, pixel_num, (int)C, h * w, loss_weight, stats, loss);
    else lsf_forward_kernel<true, LS_MAXC><<<(unsigned)(n * LS_CL), LS_NT, 0, st>>>(x, y, T, pixel_num, (int)C, h * w, loss_weight, stats, loss);
  else
    if (C <= 4) lsf_forward_kernel<false, 4><<<(unsigned)(n * LS_CL), LS_NT, 0, st>>>(x, y, T, pixel_num, (int)C, h * w, loss_weight, stats, loss);
    else lsf_forward_kernel<false, LS_MAXC><<<(unsigned)(n * LS_CL), LS_NT, 0, st>>>(x, y, T, pixel_num, (int)C, h * w, loss_weight, stats, loss);
  return check_launch();
}

extern "C" int bxs_levelset_fused_backward(const float* x, const float* y, const float* T, const void* workspace,
                                           const float* g_loss, float* g_x, float* g_T, int64_t n, int64_t C, int64_t h,
                                           int64_t w, float loss_weight, int mode, bxs_stream_t stream) {
  if (!x || !T || !workspace || !g_loss || (!g_x && !g_T) || n <= 0 || h <= 0 || w <= 0 ||
      (mode == 1 && !y) || (mode != 0 && mode != 1))
    return BXS_ERR_INVALID_ARG;
  if (C < 1 || C > LS_MAXC) return BXS_ERR_UNSUPPORTED;
  const int64_t hw = h * w;
  const int chunks = (int)std::max<int64_t>(1, std::min<int64_t>(ceil_div(hw, NT), ceil_div((int64_t)sm_count() * 8, n)));
  const LsfStats* stats = reinterpret_cast<const LsfStats*>(workspace);
  constexpr int64_t kMaxGridY = 65535;
  for (int64_t n0 = 0; n0 < n; n0 += kMaxGridY) {
    const dim3 grid(chunks, (unsigned)std::min(n - n0, kMaxGridY));
    if (mode == 1)
      lsf_backward_kernel<true><<<grid, NT, 0, as_stream(stream)>>>(x, y, T, (int)C, hw, stats, loss_weight, g_loss, g_x, g_T, n0);
    else
      lsf_backward_kernel<false><<<grid, NT, 0, as_stream(stream)>>>(x, y, T, (int)C, hw, stats, loss_weight, g_loss, g_x, g_T, n0);
  }
  return check_launch();
}
