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
 * bxs_boxinst_targets_forward: the whole target build of a batch.  img [B,3,Hp,Wp] normalised RGB ->
 *   lab [B,3,H,W] float32 and valid [B,H,W] uint8 (H = Hp/s, W = Wp/s);
 *   sim [B,k*k-1,H,W] float32 (may be NULL) and, for size==3, edge_bits [B,H,W] uint8 with
 *   bit c = (sim[c] >= thresh) (may be NULL; not both);
 *   boxes [G,4] float xyxy (device, image-major, G = sum num_gts) -> rects [G,4] int32 (j0,j1,i0,i1
 *   inclusive grid ranges of the centre-sampled bitmask; empty when j0>j1 or i0>i1; Python slice
 *   semantics of condinst_head.py:1429-1432) and gt_img [G] int32, the image of each GT
 *   (boxes / rects / gt_img may be NULL when G == 0).
 *   Host arrays, read at call time: img_hw_host [B,2] = (img_h, img_w) of img_shape,
 *   removed_rows_host [B] = int(bottom_pixels_removed*img_h/ori_h), num_gts_host [B], mean/std:
 *   3 floats each.  The per-image metadata is passed BY VALUE in the kernel parameters: no
 *   host-to-device copies, capturable in a CUDA graph.  Two launches for up to 64 images, one
 *   more per further 64.
 * bxs_boxinst_bitmasks: rects -> dense bitmasks [G,H,W] float32 (API parity only).
 * --------------------------------------------------------------------------------------- */
int bxs_boxinst_bitmasks(const int32_t* rects, float* bitmasks, int64_t G, int64_t H, int64_t W,
                         bxs_stream_t stream);
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
 * a10 length regulariser (levelset_loss.py:47-60): scores [n,C,h,w] -> out [n]; workspace n*64 floats.
 *     (a9, the region level-set energy of LevelsetLoss / region_levelset, is bxs_levelset_fused_* mode 0.)
 * --------------------------------------------------------------------------------------- */
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
 * bxs_meanfield_forward_inter: x, targets [n,1,h,w]; obj_img [n] int32 (image of each object, may be NULL
 *   when B == 1); neglog4_host = {-log U_fg(bit0), -log U_fg(bit1), -log U_bg(bit0), -log U_bg(bit1)}
 *   (4 host floats computed by the caller with the reference's float32 arithmetic);
 *   ret [n,1,h,w] in {0,1}, valid [n].  workspace: bxs_meanfield_workspace_bytes (large maps only).
 *   inter_img_mask f32 [n,2,h,w] (background, foreground) is the inter-image term of corr_loss
 *   (discobox_head.py:616,643-644): f += inter_img_mask * gamma before the target product; NULL = no such term
 *   (MeanField.forward without it).
 * --------------------------------------------------------------------------------------- */
int bxs_meanfield_kernel(const float* feature, float* K, int64_t B, int64_t C, int64_t h, int64_t w,
                         int kernel_size, float two_theta0_sq, float two_theta1_sq, float alpha0,
                         bxs_stream_t stream);
int64_t bxs_meanfield_workspace_bytes(int64_t n, int64_t h, int64_t w);
int bxs_meanfield_forward_inter(const float* K, const int32_t* obj_img, const float* x, const float* targets,
                                const float* inter_img_mask, float gamma, const float* neglog4_host, float* ret,
                                float* valid, void* workspace, int64_t n, int64_t h, int64_t w, int kernel_size,
                                int num_iter, bxs_stream_t stream);

/* The mean field of the DiscoBox mask loss on 16-bit predictions (the reference under autocast, discobox_head.py:1142):
 * s_logits, t_logits [n,h,w] of the type `dtype` (a bxs_half_t) names; t_logits NULL = no independent teacher (t = s);
 * targets uint8 [n,h,w].  The initial state is x = (t + s) / 2 with s = round(sigmoid(s_logits)), t = round(sigmoid(
 * t_logits)) and every step rounded to `dtype`, as torch computes it; the rounds are those of
 * bxs_meanfield_forward_inter, and the result equals it on x.float() and the targets as float32, bit for bit.
 * pseudo: uint8 [n,h,w] in {0,1}; no `valid` (the loss does not read it).  workspace: bxs_meanfield_workspace_bytes(n,h,w)
 * bytes, or NULL for the per-object schedule (bit maps in shared memory, 2*h*w bytes <= 200 KB).
 * BXS_ERR_INVALID_ARG: a NULL pointer (with n > 0), a negative n, a non-positive h / w, an even kernel size, a negative
 * num_iter, an unknown dtype, or no workspace for a map too large for shared memory.  BXS_ERR_UNSUPPORTED: h*w >= 2^30.
 * All checks run before any device call; n == 0 does nothing. */
int bxs_meanfield_forward_logits(const float* K, const int32_t* obj_img, const void* s_logits, const void* t_logits,
                                 const uint8_t* targets, int dtype, const float* neglog4_host, uint8_t* pseudo,
                                 void* workspace, int64_t n, int64_t h, int64_t w, int kernel_size, int num_iter,
                                 bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a6 + a17  DiscoBox mask loss of one level on 16-bit logits     replaces, under autocast, the chain of
 *     DiscoBoxSOLOv2Head.loss (discobox_head.py:1266-1300): sigmoid, mil_loss + dice_loss (:542-562), max_pool2d of
 *     the target, s * enlarged and the teacher-student dice_loss against the mean-field pseudo-label.
 * s_logits [n,h,w] of the type `dtype` names; targets uint8 [n,h,w] (non-zero = object); pseudo uint8 [n,h,w] from
 * bxs_meanfield_forward_logits, or NULL without the teacher-student term.  s = round(sigmoid(s_logits)) as torch computes
 * it; the row / column maxima and their first arg-max are taken on the rounded s; sums are float32 in a fixed order.
 * forward: out float[3] on the device = {sum keep * mil, sum keep * d_ts, sum keep} over the n instances, keep = 0 for
 *   an all-zero target, else 1 (d_ts = 0 without a pseudo-label).  For n == 0 out is zeroed.
 * backward: g_out float[2] on the device = upstream d/d out[0], d/d out[1]; g_logits [n,h,w] of `dtype`, fully
 *   overwritten: round(g_s * (1 - s) * s) with g_s in float32, exactly 0 for keep = 0.  Pass the inputs of the forward.
 * workspace: bxs_discobox_loss_workspace_bytes(n,h,w) bytes, written by the forward and read by the backward.
 * Deterministic (no atomics), no host synchronisation.  BXS_ERR_INVALID_ARG: a NULL pointer, a negative n, a non-positive
 * h / w, an unknown dtype; BXS_ERR_UNSUPPORTED: h or w above INT32_MAX, or more than INT32_MAX CTAs.  All checks run
 * before any device call.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_discobox_loss_workspace_bytes(int64_t n, int64_t h, int64_t w);
int bxs_discobox_loss_forward(const void* s_logits, const uint8_t* targets, const uint8_t* pseudo, int dtype,
                              void* workspace, float* out, int64_t n, int64_t h, int64_t w, bxs_stream_t stream);
int bxs_discobox_loss_backward(const void* s_logits, const uint8_t* targets, const uint8_t* pseudo, int dtype,
                               const void* workspace, const float* g_out, void* g_logits, int64_t n, int64_t h,
                               int64_t w, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a12-a15  tree filter      replaces the pybind module tree_filter_cuda
 *     (mmdet/ops/tree_filter/src/tree_filter.cpp:7-13: mst_forward, bfs_forward, refine_forward,
 *      refine_backward_feature, refine_backward_weight).
 *
 * bxs_mst_forward: edge_index int32 [B,E,2], edge_weight f32 [B,E] -> edge_out int32 [B,V-1,2]: the unique
 *   minimum spanning tree under the strict total order (weight, edge id) -- the same edge SET the reference's
 *   CPU Boruvka returns (src/mst/boruvka.cpp:74-80) -- emitted in ascending edge id.  Runs on the GPU.
 * bxs_bfs_forward_rooted: tree edges -> sorted_index [B,V] (position -> vertex), sorted_parent [B,V] (position of
 *   the parent, root 0), sorted_child [B,V,4] (positions, 0 terminated) exactly as src/bfs/bfs.cu:46-98 defines
 *   them, plus level_start [B,V+1] / num_levels [B]: the order is level-contiguous and deterministic.  The tree is
 *   rooted at vertex `root` (the reference: always vertex 0).  The filter's result does not depend on the root; the
 *   number of dependent levels of every pass does: about half from the centre of the map.
 * bxs_refine_forward_grouped: feature f32 [n,C,V] (vertex order), edge_weight f32 [G,V] (sorted order; entry 0 is
 *   ignored = 0 and NOT overwritten, unlike refine.cu:43-46) -> feature_out, aggr [n,C,V], aggr_up [n,C,V],
 *   wsum [G,V], wsum_up [G,V] (the five tensors of refine.cu:201-249).
 * bxs_refine_backward_feature_grouped / _weight_grouped: refine.cu:251-370.
 * The refine entry points take n instances that share G trees: tree_of [n] int32 -> tree.  The instances of one image
 * share the image's tree in the heads (box_solov2_head.py:300-305,353; box2mask_head.py:271-276).  tree_of == NULL:
 * instance i uses tree i (the reference's one tree per batch entry); n must equal G.  edge_weight / sorted_* /
 * level_start / num_levels / wsum / wsum_up are per TREE ([G,...]); feature, feature_out, aggr, aggr_up, grad_* are
 * per INSTANCE ([n,...]).  The normaliser is computed once per tree.  bxs_refine_backward_weight_grouped returns d/d
 * edge_weight per instance [n,V]; with a tree_of table the caller sums the rows of a tree.
 * scratch: bxs_refine_scratch_bytes(max(n, G), C, V).
 * --------------------------------------------------------------------------------------- */
int64_t bxs_mst_workspace_bytes(int64_t B, int64_t E, int64_t V);
int bxs_mst_forward(const int32_t* edge_index, const float* edge_weight, int32_t* edge_out, void* workspace,
                    int64_t B, int64_t E, int64_t V, bxs_stream_t stream);
int64_t bxs_bfs_workspace_bytes(int64_t B, int64_t V);
int bxs_bfs_forward_rooted(const int32_t* tree_edges, int32_t* sorted_index, int32_t* sorted_parent,
                    int32_t* sorted_child, int32_t* level_start, int32_t* num_levels, void* workspace,
                    int64_t B, int64_t V, int max_adj, int64_t root, bxs_stream_t stream);
int64_t bxs_refine_scratch_bytes(int64_t B, int64_t C, int64_t V);
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

/* a2  the dynamic convolution of the POSITIVE grid cells only, all levels and images in one launch
 *     replaces F.interpolate(F.conv2d(feature_pred, kernel_pred[l] cells, groups=B), (2h_l, 2w_l))[positives]
 *     (box_solov2_head.py:204-216 followed by the boolean indexing of :317-320).
 * Level l (n_levels) convolves operand level_op_host[l] (operands [B,C,op_size_host[o]] float32, e.g. feature_pred and
 * its bilinear resizes to the levels' output sizes; the levels of one operand are consecutive, level_op_host runs
 * 0, ..., n_ops-1 without gaps) with the positive cells of its raw kernel grid kernels_host[l] [B,C,S_l,S_l]
 * (S_l = grid_host[l]).  counts_host [n_levels*B]: positives of (level, image).  cells i32 [sum counts] on the device:
 * the cell index (gy*S_l + gx) of every positive, level-major, then image-major, ascending within a (level, image).
 * out_host[l] -> [n_l, op_size] with the rows in that order: exactly the rows the reference's boolean indexing keeps.
 * A problem is (operand, image): each operand is read once per image for all its levels.  The kernels are gathered
 * from the raw grids by a pack launch (K-major, in the workspace); then one TMA + wgmma launch (TF32, FP32 accumulate).
 * Backward: g_out_host[l] [n_l, op_size] ->
 *   g_operands_host[o] [B,C,op_size] (the roles-swapped product per problem; NULL: not needed) and
 *   g_kernels_host[l] [B,C,S_l,S_l] (split-K + an ordered reduce: positive cells get their gradient, every other cell 0;
 *   NULL: not needed).  Deterministic, no atomics.  Both need cells ascending within each (level, image).
 * A cell outside [0, S_l^2) acts as a zero kernel.  The *_host arrays are HOST arrays, copied into kernel parameters.
 * Limits: n_levels <= 8, n_ops <= 4, B <= 16, C % 32 == 0, C <= 256, op_size % 4 == 0, 16-byte aligned operands and
 * output gradients; d/d operand also needs sum over a problem's levels of round_up(count, 32) <= 256.
 * BXS_ERR_UNSUPPORTED outside them, BXS_ERR_INVALID_ARG for NULL pointers the shapes need, non-positive sizes, a count
 * outside [0, S_l^2] or a level_op_host that is not as described.  All checks run before any device call. */
int64_t bxs_dynconv1x1_cells_forward_workspace_bytes(const int64_t* counts_host, int64_t n_levels, int64_t B, int64_t C);
int bxs_dynconv1x1_cells_forward(const float* const* operands_host, const int64_t* op_size_host,
                                 const float* const* kernels_host, const int64_t* grid_host, const int64_t* level_op_host,
                                 const int64_t* counts_host, const int32_t* cells, float* const* out_host, void* workspace,
                                 int64_t n_levels, int64_t n_ops, int64_t B, int64_t C, bxs_stream_t stream);
int64_t bxs_dynconv1x1_cells_backward_workspace_bytes(const int64_t* op_size_host, const int64_t* grid_host,
                                                      const int64_t* level_op_host, const int64_t* counts_host,
                                                      int64_t n_levels, int64_t n_ops, int64_t B, int64_t C);
int bxs_dynconv1x1_cells_backward(const float* const* operands_host, const int64_t* op_size_host,
                                  const float* const* kernels_host, const int64_t* grid_host, const int64_t* level_op_host,
                                  const int64_t* counts_host, const int32_t* cells, const float* const* g_out_host,
                                  float* const* g_operands_host, float* const* g_kernels_host, void* workspace,
                                  int64_t n_levels, int64_t n_ops, int64_t B, int64_t C, bxs_stream_t stream);

/* a3  DiscoBox's dynamic kernels of the covered cells, packed for one dense convolution per network
 *     replaces the gather kernel_preds[l][b].view(C, -1)[:, grid_order] (discobox_head.py:1180-1189) of every (level, image):
 *     all levels of image b convolve the same s_ins_pred[b], so bxs_dynconv1x1_forward / _half_forward on the packed
 *     [B,I_pad,C] operand computes every (level, image) convolution of :1214-1227 in one call.
 * grids_host[l] [B,C,S_l,S_l] (S_l = grid_host[l]) of the element type dtype (0 float32, 1 float16, 2 bfloat16);
 * counts_host [n_levels*B]: rows of (level, image); cells i32 [n_cells] on the device: the cell (gy*S_l + gx) of every row,
 * level-major, then image-major, each (level, image) in the order given (repeats allowed: DiscoBox appends a cell once per
 * ground truth that covers it, :1511-1520).  packed [B,I_pad,C]: the rows of image b level by level, zeros past its total.
 * status (device i32, may be NULL): set to BXS_ERR_INVALID_ARG when a cell lies outside [0, S_l^2); that row is packed as
 * zeros and nothing outside the grids is read.  The caller zeroes it; the call never clears it.
 * unpack_grad: g_packed [B,I_pad,C] -> g_grids_host[l] [B,C,S_l,S_l]: every (cell, channel) gets the sum over the rows of
 * its (level, image) that name the cell, in row order, in FP32, rounded once to dtype; every other cell 0.  No atomics:
 * bit-identical from run to run.  Neither needs a workspace.  No host synchronisation.
 * Limits: n_levels <= 8, B <= 16, S_l <= 64, I_pad <= 2048 (BXS_ERR_UNSUPPORTED).  BXS_ERR_INVALID_ARG: a NULL pointer the
 * shapes need, a non-positive size, an unknown dtype, a negative count, counts whose sum is not n_cells, an image whose
 * rows exceed I_pad.  All checks run on the host before any device call. */
int bxs_disco_cells_pack(const void* const* grids_host, const int64_t* grid_host, const int64_t* counts_host,
                         const int32_t* cells, int64_t n_cells, void* packed, int32_t* status, int64_t n_levels, int64_t B,
                         int64_t C, int64_t I_pad, int dtype, bxs_stream_t stream);
int bxs_disco_cells_unpack_grad(const void* g_packed, const int64_t* grid_host, const int64_t* counts_host,
                                const int32_t* cells, int64_t n_cells, void* const* g_grids_host, int64_t n_levels, int64_t B,
                                int64_t C, int64_t I_pad, int dtype, bxs_stream_t stream);

/* The same three products with 16-bit operands, for callers that run under torch.autocast (the reference's DiscoBox
 * configs train in FP16): feat, kernels, out, g_out, g_feat and g_kernels are all of the type `dtype` names, and the
 * tensor cores accumulate in FP32.  Each result is rounded to `dtype` once, at the end; d/d kernel keeps FP32 split-K
 * partials in the workspace and rounds only after their ordered (deterministic) reduction.  No TF32 step: the operands
 * are multiplied exactly.
 * BXS_ERR_INVALID_ARG: a NULL pointer (both gradient outputs NULL in the backward), a non-positive size or an unknown
 * dtype.  BXS_ERR_UNSUPPORTED: C % 32 != 0, C > 256, P % 8 != 0 (the tensor maps need 16-byte row strides), a base
 * that is not 16-byte aligned, or g_feat with I > 256.  All checks run before any device call.
 * workspace: bxs_dynconv1x1_half_backward_workspace_bytes(B, C, P, I, dtype) bytes (0 for an empty shape or an unknown
 * dtype). */
typedef enum { BXS_F16 = 0, BXS_BF16 = 1 } bxs_half_t;
int bxs_dynconv1x1_half_forward(const void* feat, const void* kernels, void* out, int64_t B, int64_t C, int64_t P,
                                int64_t I, int dtype, bxs_stream_t stream);
int64_t bxs_dynconv1x1_half_backward_workspace_bytes(int64_t B, int64_t C, int64_t P, int64_t I, int dtype);
int bxs_dynconv1x1_half_backward(const void* feat, const void* kernels, const void* g_out, void* g_feat, void* g_kernels,
                                 void* workspace, int64_t B, int64_t C, int64_t P, int64_t I, int dtype,
                                 bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * (SURVEY 8f rank 1)  projection profiles of a bilinearly resized map, never materialised.
 *     replaces, for BoxMatchingCost (mmdet/core/bbox/match_costs/match_cost.py:400-425), the F.interpolate of
 *     the query masks to GT resolution (mmdet/models/dense_heads/box2mask_head.py:157-161) + max(dim).
 * x [n,h,w] -> row_prof [n,H] (max over columns), col_prof [n,W] (max over rows) of resize(x, (H,W), bilinear,
 * align_corners=False); sigmoid_act applies the (monotone) sigmoid to the profiles.  workspace: 4*n*(H+W) bytes.
 * --------------------------------------------------------------------------------------- */
int bxs_upsampled_rowcol_max(const float* x, float* row_prof, float* col_prof, void* workspace, int64_t n,
                             int64_t h, int64_t w, int64_t H, int64_t W, int sigmoid_act, bxs_stream_t stream);

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
 * a4  Box2Mask cross-attention mask    replaces the attention-mask lines of Box2MaskHead.forward_head
 *     (mmdet/models/dense_heads/box2mask_head.py:346-355) and, with reset_full_rows, the reset of its forward loop (:397).
 * mask_pred [B,Q,H,W] of the type `dtype` names -> attn uint8 [B*heads, Q, h*w] (0 / 1: the bytes of a torch.bool tensor),
 * row (b*heads + k, q) = row (b, q) for every head k.  Bit = sigmoid(r) < 0.5 with r the bilinear resize to (h, w),
 * align_corners False, in the arithmetic of bxs_bilinear_resize_forward; 16-bit inputs are interpolated in float32 and
 * rounded to `dtype`, their sigmoid is computed in float32 and rounded to `dtype` again (torch's rounding points).  NaN gives
 * 0.  reset_full_rows != 0: a (b, q) row whose bits are all 1 is written as all 0 (no count leaves the kernel).
 * Sync-free, no workspace; B*Q == 0 is a no-op.  BXS_ERR_INVALID_ARG: a NULL pointer, a negative B or Q, a non-positive
 * H, W, h, w, heads < 1, an unknown dtype.  BXS_ERR_UNSUPPORTED: a side >= 2^24, H*W or heads*h*w above INT32_MAX, an
 * element count above INT64_MAX, or a row h*w above 1.6 M pixels (8 CTAs x 200 KB of shared memory).  All checks run
 * before any device call.
 * --------------------------------------------------------------------------------------- */
typedef enum { BXS_ATTN_F32 = 0, BXS_ATTN_F16 = 1, BXS_ATTN_BF16 = 2 } bxs_attn_dtype_t;
int bxs_box2mask_attn_mask(const void* mask_pred, uint8_t* attn, int64_t B, int64_t Q, int64_t H, int64_t W, int64_t h,
                           int64_t w, int64_t heads, int dtype, int reset_full_rows, bxs_stream_t stream);

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
 * C <= 8.  n: any count up to INT32_MAX / 8 (the forward's grid is n clusters of 8 CTAs in x); the backward launches
 * over groups of at most 65535 instances, so its grid limit is not visible to the caller.
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
 *   dist_kernel odd; (2 P^2 + 9 P) * 4 bytes <= 200 KB (P <= 156); K <= 65535.
 * bxs_corr_solve_batched: the same for n queries of kmax tables each (Cu, T [n*kmax,P,P]); counts i32 [n] (NULL: all):
 *   table j of query q is solved only when j < counts[q], the others are zero-filled (and cost no solve).
 * bxs_corr_transfer: T, Cu [K,P,P], m0 f32 [Hm*Wm] (query RoI mask), m1 f32 [K,Hm*Wm] (masks of the objects) ->
 *   fg_ci, bg_ci f32 [Hm*Wm]: T2 = T * softmax(Cu, 2), rows /= sum + 1e-5, super-resolution h x w -> Hm x Wm of both
 *   index pairs (x P / (Hm Wm)), contraction with [m0 m1 > .5] clamp(m1, .1, .9) resp. [(1-m0)(1-m1) > .5]
 *   clamp(1-m1, .1, .9), mean over the K objects (fixed order).  workspace: bxs_corr_transfer_workspace_bytes.
 * bxs_corr_transfer_batched: the same for n queries in one launch pair: T, Cu [n*kmax,P,P], m0 [n,Hm*Wm], m1
 *   [n*kmax,Hm*Wm], counts i32 [n] (NULL: kmax each) -> fg_ci, bg_ci [n,Hm*Wm], the mean over query q's first counts[q]
 *   tables (0 when it has none); workspace bxs_corr_transfer_workspace_bytes(n*kmax, Hm, Wm).  n, kmax <= 65535.
 *   bxs_corr_transfer is its n = 1 case.
 * bxs_corr_retrieve: get_similar_obj (:174-221) for the n query objects of a level at once, each against the bank of its
 *   class as the objects before it in the level leave it.  Bank: a packed store of num_class x L slots, feat f32
 *   [num_class*L, C*h*w], mask f32 [num_class*L, Hm*Wm], box f32 [num_class*L, 4], ptr / exists i32 [num_class];
 *   first i32 [1]: the head has not seen a query yet (the first live query then uses q_feat_first, the create_one
 *   re-normalisation :43).  Level: q_feat, q_feat_first, t_feat f32 [n, C*h*w], q_mask, t_mask f32 [n, Hm*Wm], box f32
 *   [n,4] (integer valued), label, valid i32 [n] (valid 0 or a label outside [0, num_class): the object takes no part).
 *   An object appends when both box sides exceed min_size; the j-th appending object of class c in the level writes slot
 *   (ptr[c] + j) % L.  Outputs per query: src i32 [n, max(max_objs, 1)] the passing slots in ascending order, at most
 *   max_objs (>= 0: store row class*L + slot; < 0: the level's object -(src+1), i.e. its t_feat / t_mask / box; 0 past
 *   count), count i32 [n], kcount i32 [n] (count when count >= min_objs, else 0), slot i32 [n] (append slot or -1),
 *   exists i32 [n] (the class had a bank at query time).  One CTA per query; shared memory corr_retrieve_scratch(L, h*w)
 *   <= 200 KB (L = 100, 7 x 7: 40 KB).  Reads the bank, writes nothing of it.
 * bxs_corr_paste: fg, bg f32 [n,Hm,Wm], box f32 [n,4], counts i32 [n] -> for every query with counts > 0 and a
 *   non-empty box, iiu f32 [2n,H,W] planes 2q / 2q+1 over the box = the bilinear resize (align_corners False, the
 *   arithmetic of bxs_bilinear_resize_forward) of bg / fg to the box; everything else of iiu is left unchanged.
 * bxs_corr_bank_append: the ordered ring append of the level after bxs_corr_retrieve: every object with slot >= 0
 *   copies t_feat / t_mask / box to row label*L + slot unless a later object of the level writes the same row; ptr[c]
 *   = last slot + 1 mod L and exists[c] = 1 for every class that appended; first = 0 if the level had a live object.
 * All four are sync-free; n == 0 is a no-op.  BXS_ERR_INVALID_ARG: a NULL pointer, a non-positive size;
 * BXS_ERR_UNSUPPORTED: a dimension above INT32_MAX or the shared-memory bound.
 * --------------------------------------------------------------------------------------- */
int bxs_corr_solve(const float* Cu, float* T, int64_t K, int64_t h, int64_t w, int dist_kernel, int num_iter,
                   int num_smooth, bxs_stream_t stream);
int bxs_corr_solve_batched(const float* Cu, float* T, const int32_t* counts, int64_t n, int64_t kmax, int64_t h, int64_t w,
                           int dist_kernel, int num_iter, int num_smooth, bxs_stream_t stream);
int64_t bxs_corr_transfer_workspace_bytes(int64_t K, int64_t Hm, int64_t Wm);
int bxs_corr_transfer(const float* T, const float* Cu, const float* m0, const float* m1, float* fg_ci, float* bg_ci,
                      void* workspace, int64_t K, int64_t h, int64_t w, int64_t Hm, int64_t Wm, bxs_stream_t stream);
int bxs_corr_transfer_batched(const float* T, const float* Cu, const float* m0, const float* m1, const int32_t* counts,
                              float* fg_ci, float* bg_ci, void* workspace, int64_t n, int64_t kmax, int64_t h, int64_t w,
                              int64_t Hm, int64_t Wm, bxs_stream_t stream);
int bxs_corr_retrieve(const float* bank_feat, const float* bank_mask, const float* bank_box, const int32_t* bank_ptr,
                      const int32_t* bank_exists, const int32_t* first, const float* q_feat, const float* q_feat_first,
                      const float* q_mask, const float* t_feat, const float* t_mask, const float* box, const int32_t* label,
                      const int32_t* valid, int32_t* src, int32_t* count, int32_t* kcount, int32_t* slot, int32_t* exists,
                      int64_t n, int64_t num_class, int64_t L, int64_t C, int64_t h, int64_t w, int64_t Hm, int64_t Wm,
                      float fg_thr, float bg_thr, float app_thr, float ratio_lo, float ratio_hi, float min_size, int max_objs,
                      int min_objs, bxs_stream_t stream);
int bxs_corr_paste(const float* fg, const float* bg, const float* box, const int32_t* counts, float* iiu, int64_t n, int64_t Hm,
                   int64_t Wm, int64_t H, int64_t W, bxs_stream_t stream);
int bxs_corr_bank_append(float* bank_feat, float* bank_mask, float* bank_box, int32_t* bank_ptr, int32_t* bank_exists,
                         int32_t* first, const float* t_feat, const float* t_mask, const float* box, const int32_t* label,
                         const int32_t* valid, const int32_t* slot, int64_t n, int64_t num_class, int64_t L, int64_t CP,
                         int64_t M, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * f1  Hungarian matching    replaces scipy.optimize.linear_sum_assignment in MaskHungarianAssigner.assign step 3
 *     (mmdet/core/bbox/assigners/mask_hungarian_assigner.py:113-123) for a batch of independent problems.
 * Problem p is the rows_host[p] x cols_host[p] row-major matrix at element offset_host[p] of `cost` (f32 or f64, as
 * `dtype` names; widened to f64 exactly).  The *_host arrays are HOST arrays, copied into the kernel parameters in chunks
 * (no H2D copy, no host read: the call can be captured in a CUDA graph).
 * match i32 [sum rows]: problem p's rows follow those of the problems before it; entry = the matched column, or -1.
 * status i32 [num_problems] on the device: 0 ok, 1 a NaN or -inf entry, 2 infeasible; a failed problem leaves its rows
 * at -1.  The result equals scipy's (row_ind = the rows with match >= 0, col_ind = their match), ties included.
 * workspace: bxs_lsap_workspace_bytes(rows_host, cols_host, num_problems) bytes (0 when every problem is empty).
 * BXS_ERR_INVALID_ARG: a NULL pointer that the shapes need, a negative size or offset, an unknown dtype;
 * BXS_ERR_UNSUPPORTED: a dimension above INT32_MAX.  All checks run before any device call.
 * --------------------------------------------------------------------------------------- */
typedef enum { BXS_LSAP_F32 = 0, BXS_LSAP_F64 = 1 } bxs_lsap_dtype_t;
int64_t bxs_lsap_workspace_bytes(const int64_t* rows_host, const int64_t* cols_host, int64_t num_problems);
int bxs_lsap_solve(const void* cost, const int64_t* offset_host, const int64_t* rows_host, const int64_t* cols_host,
                   int64_t num_problems, int dtype, int32_t* match, int32_t* status, void* workspace,
                   bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * a2  BoxSOLOv2's category loss over every level    replaces the permute / reshape / cat of the category maps and
 *     FocalLoss(use_sigmoid=True)(preds, labels, avg_factor=num_ins + 1) (box_solov2_head.py:370-383,
 *     mmdet/models/losses/focal_loss.py, utils.py weight_reduce_loss).
 * Level l (n_levels): logits_host[l] f32 [B,C,S_l,S_l] in its own NCHW layout (S_l = grid_host[l]), labels_host[l] i64
 * [B,S_l^2]; a label outside [0, C) makes its cell all-negative (C is the background label).  avg_factor: f32 scalar on the
 * DEVICE.  loss (device f32 scalar) = loss_weight * sum FL(x, t) / (avg_factor + FLT_EPSILON), with FL the numerically
 * stable form of py_sigmoid_focal_loss: BCE-with-logits (softplus) * (alpha t + (1-alpha)(1-t)) * pt^gamma.
 * grad_host[l] f32 [B,C,S_l,S_l] (grad_host NULL: not needed) = d loss / d logits in the same pass:
 *   -alpha (1-p)^gamma (1 - p - gamma p log p) for a positive, -(1-alpha) p^gamma (gamma (1-p) log(1-p) - p) for a
 *   negative, times loss_weight / (avg_factor + FLT_EPSILON).
 * Two launches: one CTA per (level, image, 64-cell tile) leaves an FP32 partial, a one-CTA launch sums them in a fixed
 * order: bit-identical from run to run, no atomics, no host synchronisation.  The *_host arrays are HOST arrays, copied
 * into kernel parameters.  workspace: bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(grid_host, n_levels, B) bytes
 * (0 for invalid arguments).  BXS_ERR_INVALID_ARG: a NULL pointer, n_levels, B, C or an S_l <= 0, gamma < 0 or NaN.
 * BXS_ERR_UNSUPPORTED: n_levels > 8, S_l > 32768.  All checks run before any device call.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_sigmoid_focal_loss_levels_forward_workspace_bytes(const int64_t* grid_host, int64_t n_levels, int64_t B);
int bxs_sigmoid_focal_loss_levels_forward(const float* const* logits_host, const int64_t* const* labels_host,
                                          const int64_t* grid_host, float* const* grad_host, const float* avg_factor,
                                          float* loss, void* workspace, int64_t n_levels, int64_t B, int64_t C, float gamma,
                                          float alpha, float loss_weight, bxs_stream_t stream);

/* The same loss on rectangular levels (CondInstBoxHead's FCOS levels, condinst_head.py:404-445): cells_host[l] = H_l * W_l,
 * logits_host[l] f32 [B,C,H_l,W_l], labels_host[l] i64 [B,H_l*W_l] (cell y*W_l + x).  Everything else as above; the
 * square-grid form is this one with cells_host[l] = S_l^2.  BXS_ERR_INVALID_ARG: as above with a cell count <= 0;
 * BXS_ERR_UNSUPPORTED: n_levels > 8, a cell count above 2^30. */
int64_t bxs_sigmoid_focal_loss_cells_forward_workspace_bytes(const int64_t* cells_host, int64_t n_levels, int64_t B);
int bxs_sigmoid_focal_loss_cells_forward(const float* const* logits_host, const int64_t* const* labels_host,
                                         const int64_t* cells_host, float* const* grad_host, const float* avg_factor,
                                         float* loss, void* workspace, int64_t n_levels, int64_t B, int64_t C, float gamma,
                                         float alpha, float loss_weight, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * Box2Mask's classification loss over every decoder layer    replaces, per layer, mmdet's
 *     CrossEntropyLoss(use_sigmoid=False, reduction='mean', class_weight=w)(cls_scores.flatten(0, 1), labels.flatten(0, 1),
 *     avg_factor=w[labels].sum()) (box2mask_head.py:248-258, cross_entropy_loss.py, utils.py weight_reduce_loss).
 * Layer l (L layers): scores_host[l] f32 [B,Q,K] in its own layout (K = num_classes + 1); labels i64 [L,B,Q] on the device;
 * class_weight f32 [K] on the device (NULL: all ones).  loss f32 [L] on the device:
 *   loss[l] = loss_weight * sum_i w[y_i] (logsumexp(x_i) - x_{i,y_i}) / (sum_i w[y_i] + FLT_EPSILON),
 * with a max-subtracted logsumexp in float32.  avg_factor (the denominator's sum) is computed on the device from the labels.
 * A label outside [0, K) adds nothing to the loss, to avg_factor or to the gradient (torch asserts on such a label; the
 * head never produces one).  grad_host[l] f32 [B,Q,K] (grad_host NULL: not needed) = d loss[l] / d scores_host[l], written
 * in the same pass: loss_weight * w[y_i] (softmax(x_i) - onehot(y_i)) / (avg_factor + FLT_EPSILON).
 * Two launches: one CTA per (layer, 32 query rows) leaves an FP32 partial, a one-CTA-per-layer launch sums them in a fixed
 * order: bit-identical from run to run, no atomics, no host synchronisation.  workspace:
 * bxs_softmax_cross_entropy_layers_forward_workspace_bytes(L, B, Q) bytes (0 for invalid sizes).
 * backward: g_loss f32 [L] on the device (upstream gradients); grad_host[l] is scaled IN PLACE by g_loss[l], and a layer
 *   whose upstream gradient is exactly 1 returns at once.  Call it at most once per forward.
 * The *_host arrays are HOST arrays, copied into kernel parameters.  BXS_ERR_INVALID_ARG: a NULL pointer the call needs,
 * L, B, Q or K <= 0.  BXS_ERR_UNSUPPORTED: L > 16, B*Q or K above INT32_MAX.  All checks run before any device call.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_softmax_cross_entropy_layers_forward_workspace_bytes(int64_t L, int64_t B, int64_t Q);
int bxs_softmax_cross_entropy_layers_forward(const float* const* scores_host, const int64_t* labels, const float* class_weight,
                                             float* const* grad_host, float* loss, void* workspace, int64_t L, int64_t B,
                                             int64_t Q, int64_t K, float loss_weight, bxs_stream_t stream);
int bxs_softmax_cross_entropy_layers_backward(float* const* grad_host, const float* g_loss, int64_t L, int64_t B, int64_t Q,
                                              int64_t K, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * CondInstBoxHead's regression and centerness losses over every FCOS level and image    replaces the permute / cat of
 *     bbox_pred and centerness, nonzero(), the gathers, centerness_target, distance2bbox, GIoULoss(reduction='mean') with
 *     weight = centerness targets and avg_factor = max(reduce_mean(sum ct), 1e-6), and CrossEntropyLoss(use_sigmoid=True)
 *     with avg_factor = max(reduce_mean(num_pos), 1) (condinst_head.py:437-469).
 * Level l (n_levels <= 8, H_l = height_host[l], W_l = width_host[l], P_l = H_l*W_l, stride_host[l] > 0): labels_host[l] i64
 * [B*P_l] and targets_host[l] f32 [B*P_l,4] as bxs_fcos_targets writes them (point b*P_l + y*W_l + x; a label in [0, C) is
 * a positive), pred_host[l] f32 [B,4,H_l,W_l] (l, t, r, b distances), ctr_host[l] f32 [B,1,H_l,W_l] (logits).  The point
 * is ((x + 0.5) * stride, (y + 0.5) * stride); ct = sqrt(min(l,r)/max(l,r) * min(t,b)/max(t,b)) of the target.
 * stats: stats f32 [2] on the device = (number of positives, sum of their ct).
 * forward: den f32 [2] on the device = (max(reduce_mean(num_pos), 1), max(reduce_mean(sum ct), 1e-6));
 *   loss_bbox = lw_bbox * sum ct (1 - GIoU) / (den[1] + FLT_EPSILON) and
 *   loss_ctr = lw_ctr * sum BCE(ctr, ct) / (den[0] + FLT_EPSILON), f32 scalars on the device,
 *   GIoU with eps 1e-6 in the reference's operation order.  g_pred_host[l] f32 [B,4,H_l,W_l] and g_ctr_host[l] f32
 *   [B,1,H_l,W_l] (either array NULL: not needed) = d loss_bbox / d pred and d loss_ctr / d ctr, zero at every point that is
 *   not a positive.  At ties the gradient is autograd's for the reference's lines: half to each side of an elementwise
 *   max / min, clamp(min=0) passes at 0.
 * backward: g_pred [n_pred] *= *g_loss_bbox and g_ctr [n_ctr] *= *g_loss_ctr IN PLACE (device scalars; a NULL buffer is
 *   skipped, an upstream gradient of exactly 1 returns at once).  Call it at most once per forward.
 * stats and forward launch one kernel of one thread per point and a one-CTA sum of its per-CTA partials in a fixed order:
 * bit-identical from run to run, no atomics, no host synchronisation.  No vector loads: any 4-byte aligned base works.
 * workspace: bxs_fcos_loss_workspace_bytes(height_host, width_host, n_levels, B) bytes (0 for invalid arguments), for
 * stats and forward alike.  The *_host arrays are HOST arrays, copied into kernel parameters.  BXS_ERR_INVALID_ARG: a NULL
 * pointer the call needs, n_levels, B, C, an H_l or W_l <= 0, a stride not positive and finite, a negative n.
 * BXS_ERR_UNSUPPORTED: n_levels > 8, C or B * sum P_l above INT32_MAX.  All checks run before any device call.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_fcos_loss_workspace_bytes(const int64_t* height_host, const int64_t* width_host, int64_t n_levels, int64_t B);
int bxs_fcos_loss_stats(const int64_t* const* labels_host, const float* const* targets_host, const int64_t* height_host,
                        const int64_t* width_host, const float* stride_host, float* stats, void* workspace, int64_t n_levels,
                        int64_t B, int64_t C, bxs_stream_t stream);
int bxs_fcos_loss_forward(const float* const* pred_host, const float* const* ctr_host, const int64_t* const* labels_host,
                          const float* const* targets_host, float* const* g_pred_host, float* const* g_ctr_host,
                          const int64_t* height_host, const int64_t* width_host, const float* stride_host, const float* den,
                          float* loss_bbox, float* loss_ctr, void* workspace, int64_t n_levels, int64_t B, int64_t C, float lw_bbox, float lw_ctr,
                          bxs_stream_t stream);
int bxs_fcos_loss_backward(float* g_pred, int64_t n_pred, const float* g_loss_bbox, float* g_ctr, int64_t n_ctr,
                           const float* g_loss_ctr, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * SOLOv2 inference    replaces the body of get_seg_single of BoxSOLOv2Head (box_solov2_head.py:503-590) and
 *     DiscoBoxSOLOv2Head (discobox_head.py:1559-1660): thresholding, mask areas and scores, mask_matrix_nms
 *     (mmdet/core/post_processing/matrix_nms.py:5-121) and the two F.interpolate passes of the mask paste.
 * Rows: src_host[s] (n_src <= 8, a HOST array of device pointers) holds src_rows_host[s] rows of hw (h*w) elements of `dtype`
 *   (0 float32, 1 float16), dense; a row id indexes the concatenation of the sources (BoxSOLOv2: the levels' [B*S_l^2, h, w]
 *   probabilities of forward(eval=True) as they lie; DiscoBox: its candidate convolution).  logits != 0: an element is a logit
 *   and p = sigmoid(x) as torch computes it for that dtype; else p is the element.  A row id outside the sources reads as
 *   an all-zero row.  mask_thr is rounded to `dtype` first: torch compares a tensor with a Python float in the tensor's dtype.
 * bxs_solo_mask_stats: for each of n_rows ids in rows i64 -> bits u32 [n_rows, ceil(hw/32)] (bit k of word w: p[32w+k] >
 *   mask_thr), area i32 [n_rows] (its popcount), masked_sum f32 [n_rows] = sum of p over the set bits (accumulated in float64
 *   in a fixed order, rounded once).  One CTA per row.
 * bxs_matrix_nms: for B images of N candidate slots each, sorted by score (descending; the first min(n_valid[b], N) slots are
 *   the valid ones): row i64 [B,N] (the slot's row of bits), label i64 [B,N], area f32 [B,N], score f32 [B,N], n_valid i64
 *   [B] on the device -> out_score f32 [B,N] = score * decay coefficient (kernel 0 gaussian with sigma, 1 linear; the
 *   reference's lines in its operation order), -inf for an invalid slot or, with filter_thr > 0, a score below filter_thr.
 *   half_inter != 0 rounds each intersection count to float16 once (the reference's torch.mm under autocast).
 *   workspace: bxs_matrix_nms_workspace_bytes(B, N) bytes (B*N*N IoUs and B*N column maxima).  Two launches and a memset.
 * bxs_solo_paste_masks: for n row ids -> out u8 [n, H_ori, W_ori] (the bytes of a torch.bool tensor) =
 *   interpolate(interpolate(p, (4h, 4w))[:H_img, :W_img], (H_ori, W_ori)) > mask_thr, bilinear with align_corners=False in
 *   the arithmetic of bxs_bilinear_resize_forward; a float16 row is rounded to float16 after each stage and compared in
 *   float16, as ATen computes on a float16 tensor, or with interp_f32 != 0 interpolated and compared in float32 without
 *   rounding (torch.autocast runs upsample_bilinear2d in float32).  H_img <= 4h, W_img <= 4w.
 * bxs_maskformer_paste_masks (MaskFormerFusionHead.instance_postprocess after Box2MaskHead.simple_test's upsample): for n
 *   row ids of LOGITS (no sigmoid before the resizes) -> out u8 [n, H_out, W_out] = interpolate(interpolate(x, (H_pad,
 *   W_pad))[:H_img, :W_img], (H_out, W_out)) > 0, bilinear with align_corners=False in the arithmetic of
 *   bxs_bilinear_resize_forward, a float16 row rounded to float16 after each stage.  The first stage is skipped when (h, w)
 *   == (H_pad, W_pad), the second when rescale == 0 (then (H_out, W_out) == (H_img, W_img)): the value is read, as ATen
 *   copies, not lerped.  In the same pass, per row: area i32 [n] = the set pixels, masked_sum f32 [n] = the sum of
 *   sigmoid(v) over them (torch's sigmoid for the dtype, accumulated in float64 in a fixed order, rounded once), box f32
 *   [n,4] = [x_min, y_min, x_max + 1, y_max + 1] of them (mask2bbox), zeros for an empty mask.  h <= H_pad, w <= W_pad,
 *   H_img <= H_pad, W_img <= W_pad.  workspace: bxs_maskformer_paste_workspace_bytes(n) bytes, 8-byte aligned.  Two launches.
 * bxs_mask_extents (format_results of SingleStageBoxInsDetector / SingleStageWSInsDetector: seg_mask.sum() and the min / max
 *   of torch.where(seg_mask)): for n masks u8 [n, H, W] (bool or uint8 bytes, dense; any non-zero byte is set) -> area i32
 *   [n] = the set pixels, box f32 [n,4] = [x_min, y_min, x_max + 1, y_max + 1] of them, zeros for an empty mask.  Rows are
 *   read 16 bytes at a time when W % 16 == 0 and masks is 16-byte aligned, else byte by byte.  workspace:
 *   bxs_mask_extents_workspace_bytes(n, H, W) bytes, 8-byte aligned.  Two launches; n == 0 is a no-op.  masks may be NULL
 *   when H * W == 0.  BXS_ERR_INVALID_ARG: a negative size, a NULL pointer with n > 0; BXS_ERR_UNSUPPORTED: H * W above
 *   INT32_MAX.
 * No host synchronisation, deterministic.  BXS_ERR_INVALID_ARG: a NULL pointer the call needs, a negative count, a
 * non-positive size, an unknown dtype or kernel.  BXS_ERR_UNSUPPORTED: n_src > 8, more than INT32_MAX rows or pixels per
 * plane, more than 65535 images or 65535 * 32 slots.  All checks run before any device call.
 * --------------------------------------------------------------------------------------- */
int bxs_solo_mask_stats(const void* const* src_host, const int64_t* src_rows_host, int64_t n_src, int64_t hw, int dtype,
                        int logits, const int64_t* rows, int64_t n_rows, float mask_thr, uint32_t* bits, int32_t* area,
                        float* masked_sum, bxs_stream_t stream);
int64_t bxs_matrix_nms_workspace_bytes(int64_t B, int64_t N);
int bxs_matrix_nms(const uint32_t* bits, int64_t words, const int64_t* row, const int64_t* label, const float* area,
                   const float* score, const int64_t* n_valid, int64_t B, int64_t N, int kernel, float sigma, float filter_thr,
                   int half_inter, void* workspace, float* out_score, bxs_stream_t stream);
int bxs_solo_paste_masks(const void* const* src_host, const int64_t* src_rows_host, int64_t n_src, int64_t h, int64_t w,
                         int dtype, int logits, int interp_f32, const int64_t* rows, int64_t n, int64_t H_img, int64_t W_img,
                         int64_t H_ori, int64_t W_ori, float mask_thr, uint8_t* out, bxs_stream_t stream);
int64_t bxs_maskformer_paste_workspace_bytes(int64_t n);
int bxs_maskformer_paste_masks(const void* const* src_host, const int64_t* src_rows_host, int64_t n_src, int64_t h, int64_t w,
                               int dtype, const int64_t* rows, int64_t n, int64_t H_pad, int64_t W_pad, int64_t H_img,
                               int64_t W_img, int rescale, int64_t H_out, int64_t W_out, void* workspace, uint8_t* out,
                               int32_t* area, float* masked_sum, float* box, bxs_stream_t stream);
int64_t bxs_mask_extents_workspace_bytes(int64_t n, int64_t H, int64_t W);
int bxs_mask_extents(const uint8_t* masks, int64_t n, int64_t H, int64_t W, void* workspace, int32_t* area, float* box,
                     bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * CondInst inference   replaces the level loop of CondInstBoxHead._get_bboxes (condinst_head.py:762-813), the NMS of
 *     nms_with_others (:18-83: mmcv's batched_nms with type 'nms') and the mask lines of CondInstMaskHead.simple_test
 *     (:1261-1281: sigmoid, aligned_bilinear, crop, F.interpolate, > 0.5).
 * Level table: for each of n_levels <= 8 levels, cls_host[l] / ctr_host[l] / bbox_host[l] / param_host[l] (HOST arrays of
 *   device pointers) are float32 [B,C,H,W] / [B,1,H,W] / [B,4,H,W] / [B,P,H,W] read in place with the element strides
 *   *_strides_host[4l .. 4l+3] (any layout); height_host / width_host / stride_host give H_l, W_l and the level's stride.
 *   k_host[l] is the number of points the level keeps (H_l*W_l: all, in point order; less: the first k_host[l] of the
 *   level's row of `order`).  The slots of an image are the kept points, level after level: S = sum k_host.  B <= 32.
 * bxs_condinst_point_scores -> key f32 [B, n_levels, P_max] = max_c sigmoid(cls_c) * sigmoid(ctr) (a NaN wins), -inf past
 *   H_l*W_l.  P_max >= every H_l*W_l.
 * bxs_condinst_decode: order i64 [B, n_levels, P_max] (the per-level ranking of the keys; may be NULL when no level is cut),
 *   img_hw_host f32 [B,2] (img_shape[:2]), scale_host f32 [B,4] (scale_factor, or NULL: no rescale) -> for each slot g of
 *   [B,S]: box f32 [B,S,4] (distance2bbox with the per-image clamp, then / scale_factor), ctr f32 [B,S] = sigmoid(ctr),
 *   point i64 [B,S] (y*W_l + x), and per class cand u8 [B,S,C] = sigmoid(cls) > score_thr, score f32 [B,S,C] =
 *   sigmoid(cls) * sigmoid(ctr), sig f32 [B,S,C] = sigmoid(cls) (optional).
 * bxs_condinst_gather: for n slot ids rows i64 (b*S + s) -> params f32 [n,P], coors f32 [n,2] (the point), level i64 [n].
 * bxs_box_nms: N boxes f32 [N,4] (16-byte aligned; batched_nms's offset boxes) sorted into n_seg segments, segment s being
 *   the rows seg_start[s] .. seg_start[s+1]-1 (i64 [n_seg+1] on the device) in descending score order; mask_off i64 [n_seg]
 *   = the exclusive prefix sum of n_s * ceil(n_s / 64); max_seg >= every n_s -> keep u8 [N]: greedy NMS within every
 *   segment with mmcv's test interS > iou_thr * (Sa + Sb - interS).  workspace: bxs_box_nms_workspace_bytes(n_s host
 *   array, n_seg) bytes, 8-byte aligned.  Two launches.
 * bxs_condinst_paste_masks: logits f32 [n, h, w] (dense) -> out u8 [n, H_out, W_out] (the bytes of a torch.bool tensor) =
 *   aligned_bilinear(sigmoid(logits), factor)[:H_img, :W_img] > 0.5, or with rescale != 0 that crop resized to
 *   (H_out, W_out) (bilinear, align_corners=False) first; in the arithmetic of bxs_bilinear_resize_forward.  H_img <=
 *   factor*h, W_img <= factor*w; without rescale (H_out, W_out) == (H_img, W_img).
 * No host synchronisation, no atomics: deterministic.  BXS_ERR_INVALID_ARG: a NULL pointer the call needs, a negative count,
 *   a non-positive size, k_host[l] outside [0, H_l*W_l], P_max below a level's size.  BXS_ERR_UNSUPPORTED: more than 8
 *   levels or 32 images, more than INT32_MAX points per level or pixels per plane, a segment of more than 393216 boxes.
 *   All checks run before any device call.
 * --------------------------------------------------------------------------------------- */
int bxs_condinst_point_scores(const float* const* cls_host, const int64_t* cls_strides_host, const float* const* ctr_host,
                              const int64_t* ctr_strides_host, const int64_t* height_host, const int64_t* width_host,
                              int64_t n_levels, int64_t B, int64_t C, int64_t P_max, float* key, bxs_stream_t stream);
int bxs_condinst_decode(const float* const* cls_host, const int64_t* cls_strides_host, const float* const* ctr_host,
                        const int64_t* ctr_strides_host, const float* const* bbox_host, const int64_t* bbox_strides_host,
                        const int64_t* height_host, const int64_t* width_host, const float* stride_host, const int64_t* k_host,
                        int64_t n_levels, int64_t B, int64_t C, const int64_t* order, int64_t P_max, const float* img_hw_host,
                        const float* scale_host, float score_thr, float* box, float* ctr, int64_t* point, uint8_t* cand,
                        float* score, float* sig, bxs_stream_t stream);
int bxs_condinst_gather(const float* const* param_host, const int64_t* param_strides_host, const int64_t* height_host,
                        const int64_t* width_host, const float* stride_host, const int64_t* k_host, int64_t n_levels, int64_t B,
                        int64_t P, const int64_t* point, const int64_t* rows, int64_t n, float* params, float* coors,
                        int64_t* level, bxs_stream_t stream);
int64_t bxs_box_nms_workspace_bytes(const int64_t* seg_count_host, int64_t n_seg);
int bxs_box_nms(const float* boxes, const int64_t* seg_start, const int64_t* mask_off, int64_t N, int64_t n_seg, int64_t max_seg,
                float iou_thr, void* workspace, uint8_t* keep, bxs_stream_t stream);
int bxs_condinst_paste_masks(const float* logits, int64_t n, int64_t h, int64_t w, int64_t factor, int64_t H_img, int64_t W_img,
                             int64_t H_out, int64_t W_out, int rescale, uint8_t* out, bxs_stream_t stream);

/* ---------------------------------------------------------------------------------------
 * COCO RLE of instance masks   replaces pycocotools' mask.encode in mmdet's encode_mask_results (mmdet/core/mask/utils.py:
 *     38-65): rleEncode + rleToString of maskApi.c, byte for byte.
 * masks: n masks u8 [n, H, W] (the bytes of a bool or uint8 tensor, dense, row-major).  Walked in column-major order
 *   j = x * H + y with the previous byte starting at 0, a run closes wherever a byte differs from the one before it
 *   (byte values, not set / not set: in a uint8 mask 1 -> 2 closes a run, as in pycocotools).
 * bxs_mask_rle_runs -> offsets i64 [n + 1]: the first count of each mask, offsets[n] = R, the total count (each mask has
 *   its boundaries + 1 counts).  It leaves the boundaries of every segment in the workspace for bxs_mask_rle_counts.
 * bxs_mask_rle_counts: the same masks, the workspace and offsets as bxs_mask_rle_runs left them -> counts u32 [R]: mask k's
 *   uncompressed RLE at offsets[k] .. offsets[k + 1] - 1 (the first is 0 when the first byte is non-zero; an all-zero
 *   mask gives [H * W]).  workspace: bxs_mask_rle_counts_workspace_bytes(n, H, W) bytes, 8-byte aligned, for both calls.
 * bxs_mask_rle_strings: counts u32 [R] and offsets i64 [n + 1] as above -> chars u8 [<= 6 R]: the strings of rleToString
 *   (no terminator), mask k's at char_offsets[k] .. char_offsets[k + 1] - 1 of i64 [n + 1].  workspace:
 *   bxs_mask_rle_strings_workspace_bytes(n, R) bytes, 8-byte aligned.
 * The caller reads R between bxs_mask_rle_runs and bxs_mask_rle_counts to size counts and chars.  Three launches per call
 *   (one memset for the counts when H * W == 0).  No host synchronisation, no atomics: deterministic.  n == 0 is a no-op;
 *   masks may be NULL when H * W == 0.  BXS_ERR_INVALID_ARG: a negative size, a NULL pointer with n > 0, R < n.
 *   BXS_ERR_UNSUPPORTED: H * W >= 2^29 (every delta then fits 6 characters, pycocotools' own buffer).  All checks run
 *   before any device call.
 * --------------------------------------------------------------------------------------- */
int64_t bxs_mask_rle_counts_workspace_bytes(int64_t n, int64_t H, int64_t W);
int bxs_mask_rle_runs(const uint8_t* masks, int64_t n, int64_t H, int64_t W, void* workspace, int64_t* offsets,
                      bxs_stream_t stream);
int bxs_mask_rle_counts(const uint8_t* masks, int64_t n, int64_t H, int64_t W, const void* workspace, const int64_t* offsets,
                        uint32_t* counts, bxs_stream_t stream);
int64_t bxs_mask_rle_strings_workspace_bytes(int64_t n, int64_t R);
int bxs_mask_rle_strings(const uint32_t* counts, const int64_t* offsets, int64_t n, int64_t R, void* workspace,
                         uint8_t* chars, int64_t* char_offsets, bxs_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* BOXSEG_B200_H_ */
