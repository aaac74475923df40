/*
 * boxseg_b200 -- C ABI of the H100 (sm_90a) box-supervised mask-loss hot path.
 *
 * This is the drop-in boundary (SURVEY.md section 8b): every entry point takes raw DEVICE
 * pointers + sizes + the CUDA stream to launch on, allocates nothing, keeps no state and
 * returns 0 or a negative bxs_status.  No torch types.  The Python package
 * `boxinstseg_b200` binds it with ctypes and re-creates the reference's own operator
 * signatures (mmdet/ops/pairwise, mmdet/ops/tree_filter, the LOSSES/HEADS classes) on top.
 *
 * For each entry point the reference interface it replaces is cited (paths relative to
 * the reference checkout).  Tensors are dense, row-major ("contiguous"), fp32 unless noted.
 */
#ifndef BOXSEG_B200_H_
#define BOXSEG_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* bxs_stream_t; /* cudaStream_t */

typedef enum {
  BXS_OK = 0,
  BXS_ERR_INVALID_ARG = -1,   /* null pointer, non-positive size, unsupported neighbourhood */
  BXS_ERR_LAUNCH = -2,        /* cudaGetLastError() != cudaSuccess after the launch */
  BXS_ERR_UNSUPPORTED = -3,   /* shape outside what the kernel was built for */
  BXS_ERR_NO_DEVICE = -4
} bxs_status;

/* library identity / environment ---------------------------------------------------------- */
int bxs_version(void);                       /* 10000*major + 100*minor + patch */
const char* bxs_last_error(void);            /* text of the last CUDA error seen by this thread */
int bxs_device_sm_count(void);               /* multiprocessor count of the current device */
int bxs_flush_l2(void* scratch, int64_t bytes, bxs_stream_t stream); /* bench helper: overwrite scratch */

/* ---------------------------------------------------------------------------------------
 * a7  pairwise -log P(same label)            replaces pairwise_ext.pairwise_nlog_forward /
 *     pairwise_nlog_backward   (mmdet/ops/pairwise/csrc/pairwise/bind.cpp:15-36,
 *     kernels pairwise.cu:68-149, Python wrapper mmdet/ops/pairwise/pairwise.py:6-26)
 * logits [B,1,H,W] -> out [B,k*k-1,H,W];  dtype: 0 = float32, 1 = float64.
 * backward is a deterministic gather (no atomics): g_logits is fully overwritten.
 * --------------------------------------------------------------------------------------- */
int bxs_pairwise_nlog_forward(const void* logits, void* out, int64_t B, int64_t H, int64_t W,
                              int size, int dilation, int dtype, bxs_stream_t stream);
int bxs_pairwise_nlog_backward(const void* logits, const void* g_out, void* g_logits, int64_t B,
                               int64_t H, int64_t W, int size, int dilation, int dtype,
                               bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a5  BoxInst targets      replaces CondInstMaskHead.get_targets / get_bitmasks_from_boxes /
 *     get_original_image / get_image_color_similarity
 *     (mmdet/models/dense_heads/condinst_head.py:170-246, 1345-1448) incl. the host round trips
 *     through mmcv.tensor2imgs and skimage.color.rgb2lab.
 *
 * bxs_boxinst_lab: img [B,3,Hp,Wp] normalised RGB -> lab [B,3,Hp/s,Wp/s] (float32) and
 *   valid [B,Hp/s,Wp/s] (uint8).  img_hw [B,2] int32 = (img_h, img_w) of each image,
 *   removed_rows [B] int32 = int(bottom_pixels_removed*img_h/ori_h) (host integers),
 *   mean/std: 3 floats each (host pointers, read at call time).
 * bxs_boxinst_similarity: lab, valid -> sim [B,k*k-1,H,W] float32 (may be NULL) and, for
 *   size==3, edge_bits [B,H,W] uint8 with bit c = (sim[c] >= thresh) (may be NULL).
 * bxs_boxinst_rects: boxes [G,4] float xyxy -> rects [G,4] int32 (j0,j1,i0,i1 inclusive grid
 *   ranges of the centre-sampled bitmask; empty when j0>j1 or i0>i1); Python slice semantics
 *   of condinst_head.py:1429-1432 are kept.
 * bxs_boxinst_bitmasks: rects -> dense bitmasks [G,H,W] float32 (API parity only).
 * --------------------------------------------------------------------------------------- */
int bxs_boxinst_lab(const float* img, const int32_t* img_hw, const int32_t* removed_rows,
                    const float* mean3_host, const float* std3_host, float* lab, uint8_t* valid,
                    int64_t B, int64_t Hp, int64_t Wp, int stride, bxs_stream_t stream);
int bxs_boxinst_similarity(const float* lab, const uint8_t* valid, float* sim, uint8_t* edge_bits,
                           int64_t B, int64_t H, int64_t W, int size, int dilation, float thresh,
                           bxs_stream_t stream);
int bxs_boxinst_rects(const float* boxes, int32_t* rects, int64_t G, int64_t Hp, int64_t Wp,
                      int stride, bxs_stream_t stream);
int bxs_boxinst_bitmasks(const int32_t* rects, float* bitmasks, int64_t G, int64_t H, int64_t W,
                         bxs_stream_t stream);

/* The whole target build of a batch (bxs_boxinst_lab + bxs_boxinst_rects + the GT -> image index + bxs_boxinst_similarity) in
 * two launches, with the per-image metadata passed BY VALUE from host arrays (img_hw_host [B,2] = (h, w) of img_shape,
 * removed_rows_host [B], num_gts_host [B]; B <= 64, else BXS_ERR_UNSUPPORTED): no host-to-device copies, capturable in a CUDA
 * graph.  boxes [sum num_gts, 4] xyxy (device, image-major), rects [G,4] / gt_img [G] outputs (may be NULL when G == 0);
 * sim / edge_bits as in bxs_boxinst_similarity.  Replaces CondInstMaskHead.get_targets' host round trip
 * (condinst_head.py:170-246, 1345-1448). */
int bxs_boxinst_targets_forward(const float* img, const float* boxes, const int32_t* img_hw_host,
                                const int32_t* removed_rows_host, const int32_t* num_gts_host, const float* mean3_host,
                                const float* std3_host, float* lab, uint8_t* valid, float* sim, uint8_t* edge_bits,
                                int32_t* rects, int32_t* gt_img, int64_t B, int64_t Hp, int64_t Wp, int stride, int size,
                                int dilation, float thresh, bxs_stream_t stream);

/* CIE-LAB (float64 evaluation of scikit-image's rgb2lab, cast to float32) of n packed uint8 RGB triplets: lab [n,3].
 * The colour conversion of the target build on its own, so that it can be checked over all 2^24 colours. */
int bxs_rgb_u8_to_lab(const uint8_t* rgb, float* lab, int64_t n, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a6+a7+a8  fused BoxInst mask loss     replaces the arithmetic of CondInstMaskHead.loss
 *     (condinst_head.py:1288-1343): sigmoid, compute_project_term (:134-143), pairwise_nlog,
 *     colour-threshold weights and the normalised reduction, plus their backward.
 *
 * logits [N,1,H,W]; edge_bits [B,H,W]; rects [G,4]; inst_gt [N] int32 (GT of each instance);
 * gt_img [G] int32 (image of each GT); iter_ptr: device float holding CondInstMaskHead._iter
 * (after the increment); warmup_iters: pairwise_warmup.
 * workspace: device scratch of bxs_boxinst_loss_workspace_bytes(N,H,W) bytes; it carries the
 * arg-max positions and gradient coefficients from forward to backward.
 * losses_out: device float[4] = {loss_prj, loss_pairwise, pairwise numerator, weight sum}.
 * backward: g_losses device float[2] = upstream d/d loss_prj, d/d loss_pairwise;
 * g_logits [N,1,H,W] fully overwritten (deterministic, no atomics).
 * --------------------------------------------------------------------------------------- */
int64_t bxs_boxinst_loss_workspace_bytes(int64_t N, int64_t H, int64_t W);
int bxs_boxinst_loss_forward(const float* logits, const uint8_t* edge_bits, const int32_t* rects,
                             const int32_t* inst_gt, const int32_t* gt_img, const float* iter_ptr,
                             float warmup_iters, void* workspace, float* losses_out, int64_t N,
                             int64_t H, int64_t W, int dilation, bxs_stream_t stream);
int bxs_boxinst_loss_backward(const float* logits, const uint8_t* edge_bits, const int32_t* rects,
                              const int32_t* inst_gt, const int32_t* gt_img, const void* workspace,
                              const float* g_losses, float* g_logits, int64_t N, int64_t H,
                              int64_t W, int dilation, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a6+a7+a8, single pass: the same loss (condinst_head.py:1288-1343) AND d/d logits from ONE
 * read of the logits (boxinst_onepass.cu).  The pairwise normaliser is logit-independent and the
 * projection term reaches only H + W arg-max positions per instance, so the dense gradient is
 * written while the logits stream through the SM; HBM traffic = read logits once + write the
 * gradient once.  Use when a gradient is wanted (training); the two-call API above remains for
 * forward-only use and for shapes outside bxs_boxinst_loss_fused_supported().
 *
 * forward: computes losses_out (as above) and writes g_logits [N,1,H,W] = d(loss_prj +
 *   loss_pairwise)/d logits, i.e. the gradient for upstream gradients (1, 1).
 * backward: g_prj / g_pair are device floats (upstream gradients).  When both are 1 the kernel
 *   returns at once (g_logits already holds the answer); otherwise g_logits is converted IN
 *   PLACE to g_prj * d loss_prj + g_pair * d loss_pairwise (exact: the pairwise part at the
 *   arg-max positions is kept in the workspace).  Call it at most once per forward.
 * workspace: bxs_boxinst_loss_fused_workspace_bytes(N,H,W) bytes, no initial state needed.
 * sched_state: bxs_boxinst_loss_fused_sched_bytes() bytes of device memory that MUST be zero
 *   before the first call and is owned by one stream at a time (the kernel's work-item counter,
 *   per-instance completion counters, finalize ticket and fixed-point loss sums live there; each call that runs to
 *   completion leaves it zeroed again -- after a failed launch, zero it with cudaMemsetAsync before the next call).
 * Returns BXS_ERR_UNSUPPORTED outside the supported envelope (W % 4 == 0, W,H <= 512,
 * 1 <= dilation <= 4, N <= 2048, 16-byte aligned logits / g_logits).
 * --------------------------------------------------------------------------------------- */
int bxs_boxinst_loss_fused_supported(int64_t N, int64_t H, int64_t W, int dilation);
int64_t bxs_boxinst_loss_fused_workspace_bytes(int64_t N, int64_t H, int64_t W);
int64_t bxs_boxinst_loss_fused_sched_bytes(void);
int bxs_boxinst_loss_fused_forward(const float* logits, const uint8_t* edge_bits, const int32_t* rects,
                                   const int32_t* inst_gt, const int32_t* gt_img, const float* iter_ptr,
                                   float warmup_iters, void* workspace, void* sched_state,
                                   float* losses_out, float* g_logits, int64_t N, int64_t H, int64_t W,
                                   int dilation, bxs_stream_t stream);
int bxs_boxinst_loss_fused_backward(const void* workspace, const float* g_prj, const float* g_pair,
                                    float* g_logits, int64_t N, int64_t H, int64_t W,
                                    bxs_stream_t stream);

/* The work plan of the single-pass kernel: instance records, every work item (32-byte descriptor, in queue
 * order) and the logit-independent weight total of condinst_head.py:1318-1319, derived from the TARGETS only
 * (edge_bits, rects, the instance->GT assignment).  Build it once per target set and pass it to
 * bxs_boxinst_loss_fused_forward_planned(); bxs_boxinst_loss_fused_forward() (no plan argument) builds one in the
 * tail of its workspace on every call.  plan: bxs_boxinst_loss_plan_bytes() bytes, 16-byte aligned, read-only for
 * the loss kernels. */
int64_t bxs_boxinst_loss_plan_bytes(int64_t N, int64_t H, int64_t W, int dilation);
int bxs_boxinst_loss_plan(const uint8_t* edge_bits, const int32_t* rects, const int32_t* inst_gt,
                          const int32_t* gt_img, void* plan, int64_t N, int64_t H, int64_t W, int dilation,
                          bxs_stream_t stream);
int bxs_boxinst_loss_fused_forward_planned(const float* logits, const uint8_t* edge_bits, void* plan,
                                           const float* iter_ptr, float warmup_iters, void* workspace,
                                           void* sched_state, float* losses_out, float* g_logits, int64_t N,
                                           int64_t H, int64_t W, int dilation, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a1  CondInst dynamic mask head       replaces CondInstMaskHead.forward + parse_dynamic_params +
 *     aligned_bilinear (mmdet/models/dense_heads/condinst_head.py:1120-1164, 146-167).
 * feat [B,C,h,w]; params [N,P] laid out [W1(8 x cin) | W2(8x8) | W3(1x8) | b1 | b2 | b3] with
 * cin = C + 2*rel_coors; coors [N,2] (x,y); soi [N] = sizes_of_interest[level_inds] as float;
 * img_inds [N] int32; out [N,1,factor*h,factor*w].  dynamic_channels == 8, dynamic_convs == 3,
 * C <= 32 (BXS_ERR_UNSUPPORTED otherwise).
 * backward: g_out [N,1,fh,fw] -> g_feat [B,C,h,w] and g_params [N,P], both fully overwritten,
 * deterministic (no atomics).  workspace: bxs_condinst_head_workspace_bytes(...) device bytes.
 * --------------------------------------------------------------------------------------- */
int bxs_condinst_head_forward(const float* feat, const float* params, const float* coors, const float* soi,
                              const int32_t* img_inds, float* out, int64_t N, int64_t B, int64_t C,
                              int64_t h, int64_t w, int64_t P, int in_stride, int factor, int rel_coors,
                              bxs_stream_t stream);
int64_t bxs_condinst_head_workspace_bytes(int64_t N, int64_t B, int64_t h, int64_t w, int64_t P);
int bxs_condinst_head_backward(const float* feat, const float* params, const float* coors, const float* soi,
                               const int32_t* img_inds, const float* g_out, float* g_feat, float* g_params,
                               void* workspace, int64_t N, int64_t B, int64_t C, int64_t h, int64_t w,
                               int64_t P, int in_stride, int factor, int rel_coors, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a6 (dense)  box-projection dice loss on arbitrary maps     replaces BoxProjectionLoss.forward
 *     (mmdet/models/losses/box_projection_loss.py:11-42; eps = 1e-5), DiscoBox mil_loss+dice_loss
 *     (mmdet/models/dense_heads/discobox_head.py:542-562; eps = 2e-3).
 * scores, targets [n,h,w] -> loss [n] = loss_weight * (dice(row profiles) + dice(col profiles)),
 * dice = 1 - 2<x,t>/(|x|^2 + |t|^2 + eps).  backward: g_loss [n] -> g_scores [n,h,w] (gradient goes
 * to the first arg-max of each row / column, as torch.max(dim) does).
 * --------------------------------------------------------------------------------------- */
int64_t bxs_projection_workspace_bytes(int64_t n, int64_t h, int64_t w);
int bxs_projection_loss_forward(const float* scores, const float* targets, float* loss, void* workspace,
                                int64_t n, int64_t h, int64_t w, float eps, float loss_weight,
                                bxs_stream_t stream);
int bxs_projection_loss_backward(const void* workspace, const float* g_loss, float* g_scores, int64_t n,
                                 int64_t h, int64_t w, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a9  region level-set energy        replaces LevelsetLoss / region_levelset
 *     (mmdet/models/losses/levelset_loss.py:7-44).
 * scores2 [n,2,h,w], targets [n,C,h,w] (C <= 8), pixel_num [n] -> loss [n] = w * E / pixel_num.
 * backward writes g_scores2 and/or g_targets (either may be NULL).  workspace carries the
 * region means from forward to backward: bxs_levelset_workspace_bytes(n).
 * a10 length regulariser (levelset_loss.py:47-60): scores [n,C,h,w] -> out [n]; workspace n*64 floats.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_levelset_workspace_bytes(int64_t n);
int bxs_levelset_loss_forward(const float* scores2, const float* targets, const float* pixel_num, float* loss,
                              void* workspace, int64_t n, int64_t C, int64_t h, int64_t w, float loss_weight,
                              bxs_stream_t stream);
int bxs_levelset_loss_backward(const float* scores2, const float* targets, const float* pixel_num,
                               const void* workspace, const float* g_loss, float* g_scores2, float* g_targets,
                               int64_t n, int64_t C, int64_t h, int64_t w, float loss_weight,
                               bxs_stream_t stream);
int bxs_length_reg_forward(const float* scores, float* out, void* workspace, int64_t n, int64_t C, int64_t h,
                           int64_t w, bxs_stream_t stream);
int bxs_length_reg_backward(const float* scores, const float* g_out, float* g_scores, int64_t n, int64_t C,
                            int64_t h, int64_t w, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a11  Local Consistency Module (Box2Mask)     replaces LCM / LocalConsistencyModule
 *     (mmdet/models/losses/levelset_loss.py:64-126).
 * imgs [n,C,h,w], phis [n,1,h,w], box [n,1,h,w] -> loss_out device float[1]
 *   = sum |phi_T - phi_0| box / max(sum box, 1) after num_iter affinity-propagation rounds.
 * workspace (bxs_lcm_workspace_bytes) carries affinity + phi_T to the backward, which writes
 * g_phis [n,1,h,w] = g_loss * d loss / d phi_0 (deterministic gather form).
 * --------------------------------------------------------------------------------------- */
int64_t bxs_lcm_workspace_bytes(int64_t n, int64_t h, int64_t w);
int bxs_lcm_forward(const float* imgs, const float* phis, const float* box, float* loss_out, void* workspace,
                    int64_t n, int64_t C, int64_t h, int64_t w, int dilation, int num_iter, bxs_stream_t stream);
int bxs_lcm_backward(const float* phis, const float* box, const void* workspace, const float* g_loss,
                     float* g_phis, int64_t n, int64_t h, int64_t w, int dilation, int num_iter,
                     bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a16  DiscoBox mean-field CRF (forward only, as in the reference)     replaces MeanField
 *     (mmdet/models/dense_heads/discobox_head.py:585-651).
 * bxs_meanfield_kernel: feature [B,C,h,w] -> K [B,k*k,h,w] bilateral kernel (incl. centre tap).
 * bxs_meanfield_forward: x, targets [n,1,h,w]; obj_img [n] int32 (image of each object, may be NULL
 *   when B == 1); neglog4_host = {-log U_fg(bit0), -log U_fg(bit1), -log U_bg(bit0), -log U_bg(bit1)}
 *   (4 host floats computed by the caller with the reference's float32 arithmetic);
 *   ret [n,1,h,w] in {0,1}, valid [n].  workspace: bxs_meanfield_workspace_bytes (large maps only).
 * --------------------------------------------------------------------------------------- */
int bxs_meanfield_kernel(const float* feature, float* K, int64_t B, int64_t C, int64_t h, int64_t w,
                         int kernel_size, float two_theta0_sq, float two_theta1_sq, float alpha0,
                         bxs_stream_t stream);
int64_t bxs_meanfield_workspace_bytes(int64_t n, int64_t h, int64_t w);
int bxs_meanfield_forward(const float* K, const int32_t* obj_img, const float* x, const float* targets,
                          const float* neglog4_host, float* ret, float* valid, void* workspace, int64_t n,
                          int64_t h, int64_t w, int kernel_size, int num_iter, bxs_stream_t stream);
/* same with the inter-image term of corr_loss (discobox_head.py:616,643-644): inter_img_mask f32 [n,2,h,w] (background,
 * foreground), f += inter_img_mask * gamma before the target product; NULL = the call above. */
int bxs_meanfield_forward_inter(const float* K, const int32_t* obj_img, const float* x, const float* targets,
                                const float* inter_img_mask, float gamma, const float* neglog4_host, float* ret,
                                float* valid, void* workspace, int64_t n, int64_t h, int64_t w, int kernel_size,
                                int num_iter, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a12-a15  tree filter      replaces the pybind module tree_filter_cuda
 *     (mmdet/ops/tree_filter/src/tree_filter.cpp:7-13: mst_forward, bfs_forward, refine_forward,
 *      refine_backward_feature, refine_backward_weight).
 *
 * bxs_mst_forward: edge_index int32 [B,E,2], edge_weight f32 [B,E] -> edge_out int32 [B,V-1,2]: the unique
 *   minimum spanning tree under the strict total order (weight, edge id) -- the same edge SET the reference's
 *   CPU Boruvka returns (src/mst/boruvka.cpp:74-80) -- emitted in ascending edge id.  Runs on the GPU.
 * bxs_bfs_forward: tree edges -> sorted_index [B,V] (position -> vertex), sorted_parent [B,V] (position of
 *   the parent, root 0), sorted_child [B,V,4] (positions, 0 terminated) exactly as src/bfs/bfs.cu:46-98 defines
 *   them, plus level_start [B,V+1] / num_levels [B]: the order is level-contiguous and deterministic.
 * bxs_tree_levels: recovers level_start / num_levels from a level-contiguous sorted_parent (scratch 16*B*V bytes).
 * bxs_refine_forward: feature f32 [B,C,V] (vertex order), edge_weight f32 [B,V] (sorted order; entry 0 is
 *   ignored = 0 and NOT overwritten, unlike refine.cu:43-46) -> feature_out, aggr [B,C,V], aggr_up [B,C,V],
 *   wsum [B,V], wsum_up [B,V] (the five tensors of refine.cu:201-249).  scratch: bxs_refine_scratch_bytes.
 * bxs_refine_backward_feature / _weight: refine.cu:251-370.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_mst_workspace_bytes(int64_t B, int64_t E, int64_t V);
int bxs_mst_forward(const int32_t* edge_index, const float* edge_weight, int32_t* edge_out, void* workspace,
                    int64_t B, int64_t E, int64_t V, bxs_stream_t stream);
int64_t bxs_bfs_workspace_bytes(int64_t B, int64_t V);
int bxs_bfs_forward(const int32_t* tree_edges, int32_t* sorted_index, int32_t* sorted_parent,
                    int32_t* sorted_child, int32_t* level_start, int32_t* num_levels, void* workspace,
                    int64_t B, int64_t V, int max_adj, bxs_stream_t stream);
/* same, rooted at vertex `root` instead of vertex 0 (the filter's result does not depend on the root; the number of
 * dependent levels of every pass does: about half from the centre of the map) */
int bxs_bfs_forward_rooted(const int32_t* tree_edges, int32_t* sorted_index, int32_t* sorted_parent,
                    int32_t* sorted_child, int32_t* level_start, int32_t* num_levels, void* workspace,
                    int64_t B, int64_t V, int max_adj, int64_t root, bxs_stream_t stream);
int bxs_tree_levels(const int32_t* sorted_parent, int32_t* level_start, int32_t* num_levels, void* scratch,
                    int64_t B, int64_t V, bxs_stream_t stream);
int64_t bxs_refine_scratch_bytes(int64_t B, int64_t C, int64_t V);
int bxs_refine_forward(const float* feature, const float* edge_weight, const int32_t* sorted_index,
                       const int32_t* sorted_parent, const int32_t* sorted_child, const int32_t* level_start,
                       const int32_t* num_levels, float* feature_out, float* aggr, float* aggr_up, float* wsum,
                       float* wsum_up, void* scratch, int64_t B, int64_t C, int64_t V, bxs_stream_t stream);
int bxs_refine_backward_feature(const float* edge_weight, const int32_t* sorted_index,
                                const int32_t* sorted_parent, const int32_t* sorted_child,
                                const int32_t* level_start, const int32_t* num_levels, const float* wsum,
                                const float* grad_out, float* grad_feature, void* scratch, int64_t B, int64_t C,
                                int64_t V, bxs_stream_t stream);
int bxs_refine_backward_weight(const float* edge_weight, const int32_t* sorted_index,
                               const int32_t* sorted_parent, const int32_t* sorted_child,
                               const int32_t* level_start, const int32_t* num_levels, const float* feature_out,
                               const float* aggr, const float* aggr_up, const float* wsum, const float* wsum_up,
                               const float* grad_out, float* grad_weight, void* scratch, int64_t B, int64_t C,
                               int64_t V, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a2/a3/a4  dense dynamic 1x1 convolution on the Hopper tensor cores (wgmma, TMA fed)
 *     replaces F.conv2d(feature.view(1,B*C,h,w), kernel[B*S*S,C,1,1], groups=B)
 *       (mmdet/models/dense_heads/box_solov2_head.py:209-211),
 *     F.conv2d(mask_feat[1,C,h,w], kernels[I,C,1,1]) (mmdet/models/dense_heads/discobox_head.py:1219) and
 *     einsum('bqc,bchw->bqhw') (mmdet/models/dense_heads/box2mask_head.py:345).
 * feat [B,C,P] (P = h*w), kernels [B,I,C] -> out [B,I,P]; TF32 operands (as cuDNN's default for the
 * reference's conv2d on Ampere+), FP32 accumulation.  C % 32 == 0, C <= 256, P % 4 == 0, 16-byte aligned.
 * --------------------------------------------------------------------------------------- */
int bxs_dynconv1x1_forward(const float* feat, const float* kernels, float* out, int64_t B, int64_t C, int64_t P,
                           int64_t I, bxs_stream_t stream);

/* Backward of the dynamic 1x1 convolution (autograd of the same call sites; the reference gets it from cuDNN / cuBLAS):
 *   g_feat    [B,C,P] = kernels^T . g_out   (wgmma: the forward kernel with the operand roles swapped; I <= 256)
 *   g_kernels [B,I,C] = g_out . feat^T      (wgmma split-K over the pixels + an ordered reduction: deterministic)
 * Either output may be NULL (not needed).  TF32 inputs, FP32 accumulation.  workspace:
 * bxs_dynconv1x1_backward_workspace_bytes(B, C, P, I) bytes.  BXS_ERR_UNSUPPORTED: the forward's shape rules, or g_feat with
 * I > 256. */
int64_t bxs_dynconv1x1_backward_workspace_bytes(int64_t B, int64_t C, int64_t P, int64_t I);
int bxs_dynconv1x1_backward(const float* feat, const float* kernels, const float* g_out, float* g_feat, float* g_kernels,
                            void* workspace, int64_t B, int64_t C, int64_t P, int64_t I, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * (SURVEY 8f rank 1)  projection profiles of a bilinearly resized map, never materialised.
 *     replaces, for BoxMatchingCost (mmdet/core/bbox/match_costs/match_cost.py:400-425), the F.interpolate of
 *     the query masks to GT resolution (mmdet/models/dense_heads/box2mask_head.py:157-161) + max(dim).
 * x [n,h,w] -> row_prof [n,H] (max over columns), col_prof [n,W] (max over rows) of resize(x, (H,W), bilinear,
 * align_corners=False); sigmoid_act applies the (monotone) sigmoid to the profiles.  workspace: 4*n*(H+W) bytes.
 * --------------------------------------------------------------------------------------- */
int bxs_upsampled_rowcol_max(const float* x, float* row_prof, float* col_prof, void* workspace, int64_t n,
                             int64_t h, int64_t w, int64_t H, int64_t W, int sigmoid_act, bxs_stream_t stream);

/* Grouped forms of the three refine entry points: n instances share G trees (tree_of [n] int32 -> group), as the
 * heads use them -- the instances of one image share the image's tree (box_solov2_head.py:300-305,353;
 * box2mask_head.py:271-276).  edge_weight / sorted_* / level_start / num_levels / wsum / wsum_up are per GROUP
 * ([G,...]); feature, feature_out, aggr, aggr_up, grad_* are per INSTANCE ([n,...]).  The normaliser is computed once
 * per group.  bxs_refine_backward_weight_grouped returns d/d edge_weight per instance [n,V]; the caller sums the
 * rows of a group.  scratch: bxs_refine_scratch_bytes(max(n, G), C, V). */
int bxs_refine_forward_grouped(const float* feature, const float* edge_weight, const int32_t* sorted_index,
                               const int32_t* sorted_parent, const int32_t* sorted_child,
                               const int32_t* level_start, const int32_t* num_levels, const int32_t* tree_of,
                               float* feature_out, float* aggr, float* aggr_up, float* wsum, float* wsum_up,
                               void* scratch, int64_t n, int64_t G, int64_t C, int64_t V, bxs_stream_t stream);
int bxs_refine_backward_feature_grouped(const float* edge_weight, const int32_t* sorted_index,
                                        const int32_t* sorted_parent, const int32_t* sorted_child,
                                        const int32_t* level_start, const int32_t* num_levels,
                                        const int32_t* tree_of, const float* wsum, const float* grad_out,
                                        float* grad_feature, void* scratch, int64_t n, int64_t G, int64_t C,
                                        int64_t V, bxs_stream_t stream);
int bxs_refine_backward_weight_grouped(const float* edge_weight, const int32_t* sorted_index,
                                       const int32_t* sorted_parent, const int32_t* sorted_child,
                                       const int32_t* level_start, const int32_t* num_levels,
                                       const int32_t* tree_of, const float* feature_out, const float* aggr,
                                       const float* aggr_up, const float* wsum, const float* wsum_up,
                                       const float* grad_out, float* grad_weight, void* scratch, int64_t n,
                                       int64_t G, int64_t C, int64_t V, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a18  bilinear resize      replaces F.interpolate(mode='bilinear') as the heads call it:
 *     _scale_target (mmdet/models/utils/misc.py:75-86), box2mask_head.py:232-233,300,315-317,323-324,329,
 *     box_solov2_head.py:213,412-415 (align_corners=False); discobox_head.py:1201 (align_corners=True).
 * in [NC,h,w] -> out [NC,H,W] with ATen's upsample_bilinear2d arithmetic; backward g_out [NC,H,W] -> g_in [NC,h,w]
 * fully overwritten, deterministic gather (ATen scatters with atomicAdd).
 * --------------------------------------------------------------------------------------- */
int bxs_bilinear_resize_forward(const float* in, float* out, int64_t NC, int64_t h, int64_t w, int64_t H,
                                int64_t W, int align_corners, bxs_stream_t stream);
int bxs_bilinear_resize_backward(const float* g_out, float* g_in, int64_t NC, int64_t h, int64_t w, int64_t H,
                                 int64_t W, int align_corners, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a14  tree edge weights     replaces TreeFilter2D.build_edge_weight with the default norm2 distance
 *     (mmdet/ops/tree_filter/modules/tree_filter.py:72-108) and its autograd.
 * embed [B*groups, C, V] (vertex order; a [B, groups*C, V] tensor viewed per group), sorted_index / sorted_parent
 * [B,V], sorted_child [B,V,4] (bfs_forward) -> edge_weight [B*groups, V], w[p] = exp(-|E(v_p)-E(v_par(p))|^2 / sigma)
 * (sigma = 1 gives exp(-dist), the low_tree=False form).  backward: g_weight -> g_embed, fully overwritten,
 * deterministic (each vertex gathers its own edge and its children's edges).
 * --------------------------------------------------------------------------------------- */
int bxs_tree_edge_weight_forward(const float* embed, const int32_t* sorted_index, const int32_t* sorted_parent,
                                 float* edge_weight, int64_t B, int64_t groups, int64_t C, int64_t V, float sigma,
                                 bxs_stream_t stream);
int bxs_tree_edge_weight_backward(const float* embed, const int32_t* sorted_index, const int32_t* sorted_parent,
                                  const int32_t* sorted_child, const float* edge_weight, const float* g_weight,
                                  float* g_embed, int64_t B, int64_t groups, int64_t C, int64_t V, float sigma,
                                  bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a17 + a9  level-set assembly in one launch    replaces the eager chain around LevelsetLoss in
 *     box_solov2_head.py:341-360 and box2mask_head.py:305-327 (sigmoid, cat(s, 1-s) * box, T * box,
 *     clamp(sum box, 1)) together with LevelsetLoss.forward / region_levelset (levelset_loss.py:13-44).
 * mode 1: x = mask logits [n,h,w], y = box mask [n,h,w], T = raw targets [n,C,h,w]; pixel_num ignored.
 * mode 0: x = scores2 [n,2,h,w], T [n,C,h,w], pixel_num [n] (the dense LevelsetLoss signature), y ignored.
 * One thread-block cluster of 8 CTAs per instance; the means -> energy dependency goes through distributed
 * shared memory.  loss [n] = loss_weight * E / pixel_num.  workspace: bxs_levelset_fused_workspace_bytes(n),
 * carries the statistics to the backward.  backward: g_loss [n] -> g_x (mode 1: d/d logits [n,h,w]; mode 0:
 * d/d scores2 [n,2,h,w]) and/or g_T [n,C,h,w] (mode 1: d/d raw T, i.e. already multiplied by the box mask).
 * C <= 8.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_levelset_fused_workspace_bytes(int64_t n);
int bxs_levelset_fused_forward(const float* x, const float* y, const float* T, const float* pixel_num, float* loss,
                               void* workspace, int64_t n, int64_t C, int64_t h, int64_t w, float loss_weight,
                               int mode, bxs_stream_t stream);
int bxs_levelset_fused_backward(const float* x, const float* y, const float* T, const void* workspace,
                                const float* g_loss, float* g_x, float* g_T, int64_t n, int64_t C, int64_t h,
                                int64_t w, float loss_weight, int mode, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * f2  FCOS point assignment    replaces CondInstBoxHead.get_targets + _get_target_single
 *     (mmdet/models/dense_heads/condinst_head.py:477-548, 550-633) for a whole batch in one launch.
 * points f32 [P,2] (all levels concatenated, level l = [level_off[l], level_off[l+1])), gt_boxes f32 [sum G,4] and
 * gt_labels i64 [sum G] (the images' ground truths concatenated; may be null when sum G = 0).  The *_host arrays are HOST
 * arrays, copied into the kernel parameters (no H2D copy: the call can be captured in a CUDA graph): gt_off_host i64
 * [B+1] (image b owns [gt_off[b], gt_off[b+1]) of the concatenated list), level_off_host i64 [num_levels+1], and per
 * level regress_ranges, strides[l] * center_sample_radius (rounded to f32), strides[l].
 * Outputs in the reference's layout, level-major and image-major inside a level (what torch.cat of its per-level
 * lists gives): labels i64 [B*P] (num_classes = background), bbox_targets f32 [B*P,4] (divided by the level's stride
 * when norm_on_bbox), gt_inds i64 [B*P] (index into the CONCATENATED ground truths, -1 = none).
 * Bit-exact: every value is one correctly rounded fp32 operation of the reference, in its order.  num_levels <= 8,
 * B <= 256.
 * --------------------------------------------------------------------------------------- */
int bxs_fcos_targets(const float* points, const float* gt_boxes, const int64_t* gt_labels, const int64_t* gt_off_host,
                     int64_t* labels, float* bbox_targets, int64_t* gt_inds, int64_t B, int64_t num_levels,
                     const int64_t* level_off_host, const float* range_lo_host, const float* range_hi_host,
                     const float* stride_radius_host, const float* stride_host, int center_sampling,
                     int norm_on_bbox, int64_t num_classes, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * f4  DiscoBox semantic correspondence    replaces the inner part of SemanticCorrSolver.solve
 *     (mmdet/models/dense_heads/discobox_head.py:393-410, with pass_message :347-366) and the transfer of
 *     corr_loss (:1086-1096, with superres_T :851-865).
 * bxs_corr_solve: Cu f32 [K,P,P] (cosine similarities of the query cells x the cells of K retrieved objects,
 *   P = h*w) -> T [K,P,P]: C = Cu * window(dist_kernel), then num_iter x { votes = C; num_smooth x (pass_message,
 *   rows /= sum + 1e-4); C = Cu + votes; rows /= sum + 1e-4 }.  One CTA per object, state in shared memory;
 *   dist_kernel odd; (2 P^2 + 9 P) * 4 bytes <= 200 KB (P <= 156).
 * bxs_corr_transfer: T, Cu [K,P,P], m0 f32 [Hm*Wm] (query RoI mask), m1 f32 [K,Hm*Wm] (masks of the objects) ->
 *   fg_ci, bg_ci f32 [Hm*Wm]: T2 = T * softmax(Cu, 2), rows /= sum + 1e-5, super-resolution h x w -> Hm x Wm of both
 *   index pairs (x P / (Hm Wm)), contraction with [m0 m1 > .5] clamp(m1, .1, .9) resp. [(1-m0)(1-m1) > .5]
 *   clamp(1-m1, .1, .9), mean over the K objects (fixed order).  workspace: bxs_corr_transfer_workspace_bytes.
 * --------------------------------------------------------------------------------------- */
int bxs_corr_solve(const float* Cu, float* T, int64_t K, int64_t h, int64_t w, int dist_kernel, int num_iter,
                   int num_smooth, bxs_stream_t stream);
int64_t bxs_corr_transfer_workspace_bytes(int64_t K, int64_t Hm, int64_t Wm);
int bxs_corr_transfer(const float* T, const float* Cu, const float* m0, const float* m1, float* fg_ci, float* bg_ci,
                      void* workspace, int64_t K, int64_t h, int64_t w, int64_t Hm, int64_t Wm, bxs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* BOXSEG_B200_H_ */
