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

#ifdef __cplusplus
}
#endif
#endif /* BOXSEG_B200_H_ */
