/* esb200.h — C ABI of libesb200.so, the sm_90a kernel library behind the EmbodiedScan hot path.
 *
 * The reference (OpenRobotLab/EmbodiedScan) has no FFI of its own: its kernels live in MinkowskiEngine, mmcv._ext and
 * pytorch3d._C. Each entry point below names the reference call site / upstream operator it replaces.
 *
 * Conventions
 *  - plain pointers and sizes only; all pointers are DEVICE pointers unless the name ends in _host.
 *  - the caller owns every buffer it passes (inputs, outputs, workspace); `*_workspace_bytes` returns the scratch size of
 *    the paired call. The one memory the library takes itself is the stream-ordered scratch of its deterministic
 *    reductions (per-block partial sums, added in a fixed order instead of with float atomics): it comes from one
 *    library-owned memory pool per device, created on first use, and is freed on the same stream within the call.
 *  - every call is asynchronous on `stream` (a cudaStream_t passed as void*), no implicit synchronisation.
 *    Data-dependent output sizes are written to a device int32 the caller reads after synchronising.
 *  - return 0 on success, negative ESB_E* otherwise; esb_last_error() gives a thread-local message.
 *  - dtype: 0 = fp32, 1 = bf16 (feature storage; accumulation is always fp32).
 *  - coordinates are int32 (N,4) rows [batch, x, y, z]; |x|,|y|,|z| < 32768, batch < 65535.
 */
#ifndef ESB200_H
#define ESB200_H
#include <stddef.h>
#ifdef __cplusplus
extern "C" {
#endif

#define ESB_OK 0
#define ESB_EINVAL (-1)
#define ESB_ECUDA (-2)
#define ESB_ENOMEM (-3)
#define ESB_ERANGE (-4)
#define ESB_F32 0
#define ESB_BF16 1
/* chamfer criteria (per coordinate, summed over coordinates): |x|, x^2, smooth-L1 with beta = 1 */
#define ESB_CD_L1 0
#define ESB_CD_L2 1
#define ESB_CD_SMOOTH_L1 2

const char* esb_last_error(void);

/* ---- voxelisation hashing / coordinate maps -------------------------------------------------------------
 * ME.utils.batch_sparse_collate + ME.SparseTensor(coordinates=, features=) at
 * embodiedscan/models/detectors/sparse_featfusion_single_stage.py:109-118 ; CoordinateManager stride / kernel-map
 * construction inside every ME.MinkowskiConvolution / MaxPooling / GenerativeConvolutionTranspose used by
 * embodiedscan/models/backbones/mink_resnet.py:58-69,104-108 and embodiedscan/models/dense_heads/fcaf3d_head.py:919-946. */
int esb_voxelize_points(const float* points, long long n, int pstride, int batch, float inv_voxel, int* coords,
                        void* stream);
long long esb_hash_capacity(long long n);
size_t esb_coord_unique_workspace_bytes(long long n);
int esb_coord_unique(const int* coords_in, long long n, int div, unsigned long long* keys, int* vals, long long cap,
                     int* out_coords, int* in2out, int* count_dev, void* ws, size_t ws_bytes, void* stream);
int esb_hash_build(const int* coords, long long n, unsigned long long* keys, int* vals, long long cap, void* stream);
int esb_hash_lookup(const int* query, long long nq, const unsigned long long* keys, const int* vals, long long cap,
                    int* out, void* stream);
/* ME `features_at_coordinates` at integer query coordinates (fcaf3d_head.py:1091-1114 `_prune`): multilinear interpolation of
 * the rows of the stride-`ts` tensor whose hash table is (keys, vals); out (nq, C) fp32; absent lattice points contribute 0. */
int esb_interp_features(const int* query, long long nq, const unsigned long long* keys, const int* vals, long long cap,
                        const void* feats, int C, int ts, int dtype, float* out, void* stream);
int esb_kernel_map(const int* out_coords, long long n_out, const int* offsets_host, int K,
                   const unsigned long long* keys, const int* vals, long long cap, int* nbr, void* stream);
int esb_kernel_map_transpose(const int* nbr_out, int K, long long n_out, long long n_in, int* nbr_in, void* stream);
size_t esb_kmap_pairs_workspace_bytes(int K, long long n_out);
int esb_kmap_pairs(const int* nbr, int K, long long n_out, int* pair_in, int* pair_out, int* k_offsets, void* ws,
                   size_t ws_bytes, void* stream);
int esb_generative_children(const int* coords_in, long long n_in, int half_stride, int* out_coords, void* stream);

/* ---- sparse convolution (ME.MinkowskiConvolution fwd/bwd; mink_resnet.py:58-62, fcaf3d_head.py:919-946) -------- */
int esb_spconv_fwd(const void* x, const void* w, const int* nbr, void* y, long long n_out, int cin, int cout, int K,
                   int w_transposed, int dtype, void* stream);
int esb_spconv_wgrad(const void* x, const void* dy, const int* pair_in, const int* pair_out, const int* k_offsets,
                     float* dw, long long n_pairs_hint, int cin, int cout, int K, int dtype, void* stream);
/* *_wgrad: dw += the gradient, the add chain starting from dw. *_wgrad_slot: dw = dw + the finished gradient, one rounded add
 * per element (gradient slots accumulating backward passes, as autograd's `grad += fresh`); equal on a zeroed dw. */
int esb_spconv_wgrad_slot(const void* x, const void* dy, const int* pair_in, const int* pair_out, const int* k_offsets,
                          float* dw, long long n_pairs_hint, int cin, int cout, int K, int dtype, void* stream);

/* bf16 tensor-core (wgmma) path of the same operator; masks from esb_kmap_tile_masks;
 * w_layout 0: w (K,cout,cin), 1: w (K,cin,cout) — forward and dgrad read the SAME stored bf16 kernel, no transpose */
int esb_kmap_tile_masks(const int* nbr, int K, long long n, unsigned* masks, void* stream);
int esb_spconv_tc_fwd(const void* x, const void* wt, const int* nbr, const unsigned* masks, void* y, long long n_out,
                      int cin, int cout, int K, int w_layout, void* stream);
int esb_spconv_tc_wgrad(const void* x, const void* dy, const int* pair_in, const int* pair_out, const int* k_offsets,
                        float* dw, long long n_pairs_hint, int cin, int cout, int K, void* stream);
int esb_spconv_tc_wgrad_slot(const void* x, const void* dy, const int* pair_in, const int* pair_out, const int* k_offsets,
                             float* dw, long long n_pairs_hint, int cin, int cout, int K, void* stream);

/* ---- pooling / normalisation / activation (ME.MinkowskiMaxPooling, InstanceNorm, BatchNorm, ReLU, ELU;
 * mink_resnet.py:64-69, fcaf3d_head.py:923,942,947) -------------------------------------------------------------- */
int esb_maxpool_fwd(const void* x, const int* nbr, void* y, int* arg, long long n_out, int C, int K, int dtype,
                    void* stream);
int esb_maxpool_bwd(const void* dy, const int* arg, void* dx, long long n_out, int C, int dtype, void* stream);
int esb_norm_fwd(const void* x, const void* res, const int* seg_off, const int* row_seg, int S, long long N,
                 int max_seg_rows, int C, const float* gamma, const float* beta, float eps, float* running_mean,
                 float* running_var, float momentum, int act, float* mean, float* rstd, void* y, int dtype,
                 void* stream);
/* BatchNorm (one segment) forward in two launches: one shifted single-pass statistics kernel + one apply kernel that derives
 * mean / rstd on the fly. stats (4,C) fp32 = [sum v, sum v^2, mean, rstd]; rows 2, 3 are what esb_norm_bwd takes as mean / rstd. */
int esb_batchnorm_fwd_fused(const void* x, const void* res, long long N, int C, const float* gamma, const float* beta, float eps,
                            float* running_mean, float* running_var, float momentum, int act, float* stats, void* y, int dtype,
                            void* stream);
int esb_norm_apply(const void* x, const void* res, const int* row_seg, long long N, int C, const float* mean,
                   const float* rstd, const float* gamma, const float* beta, int act, void* y, int dtype, void* stream);
/* zero_sums 1: sg / sgx (S,C) receive this pass's column sums. zero_sums 0 (S == 1): sg / sgx are gradient slots
 * (d beta, d gamma) that may hold earlier passes; dx uses this pass's sums only, and each slot becomes slot + sum. */
int esb_norm_bwd(const void* x, const void* y, const void* dy, const int* seg_off, const int* row_seg, int S,
                 long long N, int max_seg_rows, int C, const float* mean, const float* rstd, const float* gamma, int act,
                 float* sg, float* sgx, void* dx, void* dres, int zero_sums, int dtype, void* stream);
/* fused epilogue of the folded conv+BN blocks of the per-view 2D ResNet: y = act(x + bias[c] + res) on NHWC rows */
int esb_bias_act_fwd(const void* x, const float* bias, const void* res, void* y, long long rows, int C, int act,
                     int dtype, void* stream);
int esb_act_bwd(const void* dy, const void* y, void* dx, long long n, int act, int dtype, void* stream);
/* out (n,C) = a[ia] + b[ib] row-wise; a negative index contributes zeros. ia NULL = identity on the first na rows; b/ib NULL =
 * plain gather. The union `A + B` of sparse tensors on different coordinate maps (ME `__add__`, fcaf3d_head.py:1011) and the
 * row gathers of its backward. C % 8 == 0. */
int esb_gather2_rows(const void* a, const int* ia, long long na, const void* b, const int* ib, void* out, long long n, int C,
                     int dtype, void* stream);
/* The per-view 2D backbone's convolution as a persistent TMA + wgmma implicit GEMM (csrc/conv_tma.cu): activations,
 * filter and output move with cp.async.bulk.tensor tiles (zero padding = TMA out-of-bounds fill, stride = tensor-map element
 * strides), accumulators live in registers, bias + residual + ReLU are fused into the epilogue. Replaces the cuDNN call behind
 * mmdet.ResNet (embodiedscan/models/detectors/sparse_featfusion_single_stage.py:130-136). x (n_img,H,W,cin) bf16 NHWC;
 * w_ohwi (cout,kh,kw,cin) bf16; bias (cout) fp32 or NULL; residual / y (n_img,Ho,Wo,cout) bf16 NHWC, residual may be NULL.
 * cin, cout in {16, 32, 64, 128, 256, 512, ...}. */
int esb_conv2d_tma_fwd(const void* x, const void* w_ohwi, const float* bias, const void* residual, void* y, int n_img,
                       int H, int W, int cin, int cout, int kh, int kw, int stride, int pad, int relu, void* stream);
/* Weight gradient, TMA-fed (pixels = reduction dimension, both operands arrive as [pixel][channel] boxes = MN-major wgmma
 * operands): dw_t (kh*kw*cin, cout) fp32 += the gradient (zeroed by the caller), dW[co,ci,ky,kx] = dw_t[(ky*kw+kx)*cin+ci, co]. */
int esb_conv2d_tma_wgrad(const void* x, const void* dy, float* dw_t, int n_img, int H, int W, int cin, int cout, int kh,
                         int kw, int stride, int pad, void* stream);
/* Input gradient (stride 1 or 2) with the same kernel: dx (n_img,H,W,cin) from dy (n_img,Ho,Wo,cout) and the forward filter as
 * stored (filter read as the MN-major B operand: no transposed copy). Stride 1: flipped taps. Stride 2: one launch per parity
 * class of dx, stored through a tensor map that skips every other pixel; every dx element is written exactly once. */
int esb_conv2d_tma_dgrad(const void* dy, const void* w_ohwi, void* dx, int n_img, int H, int W, int cin, int cout, int kh,
                         int kw, int stride, int pad, void* stream);
/* The same three kernels on (n,D,H,W,C) volumes through rank-5 tensor maps: the dense Conv3d stack of the occupancy neck
 * (embodiedscan/models/necks/imvoxel_neck.py:86-129; †upstream nn.Conv3d). x / y / dy NDHWC bf16, w_odhwi (cout,k,k,k,cin) bf16,
 * dw_t (k*k*k*cin, cout) fp32 zeroed by the caller. */
int esb_conv3d_tma_fwd(const void* x, const void* w_odhwi, const float* bias, const void* residual, void* y, int n, int D, int H,
                       int W, int cin, int cout, int k, int stride, int pad, int relu, void* stream);
int esb_conv3d_tma_dgrad(const void* dy, const void* w_odhwi, void* dx, int n, int D, int H, int W, int cin, int cout, int k,
                         int stride, int pad, void* stream);
int esb_conv3d_tma_wgrad(const void* x, const void* dy, float* dw_t, int n, int D, int H, int W, int cin, int cout, int k,
                         int stride, int pad, void* stream);
/* The 7x7/2 stem on the 3-channel image as a wgmma implicit GEMM with the im2col rows built in shared memory
 * (csrc/conv_tma.cu::stem7x7_tc_kernel). x (n_img,H,W,3) bf16 NHWC, w_ohwi (16,7,7,3) bf16, bias (16) fp32, y (n_img,Ho,Wo,16). */
int esb_stem7x7_tc(const void* x, const void* w_ohwi, const float* bias, void* y, int n_img, int H, int W, int relu,
                   void* stream);
/* Direct (SIMT, fp32-accumulate) NHWC convolution and its gradients (csrc/conv2d_direct.cu): the fp32 parity arithmetic of
 * every 2D convolution of the image backbone, and the 7x7/2 stem on the 3-channel image in either dtype. x (n_img,H,W,cin),
 * w_ohwi (cout,kh,kw,cin), y / residual (n_img,Ho,Wo,cout) in `dtype` (ESB_F32 / ESB_BF16); bias fp32 or NULL. */
int esb_conv2d_direct_fwd(const void* x, const void* w_ohwi, const float* bias, const void* residual, void* y, int n_img,
                          int H, int W, int cin, int cout, int kh, int kw, int stride, int pad, int relu, int dtype,
                          void* stream);
int esb_conv2d_direct_dgrad(const void* dy, const void* w_ohwi, void* dx, int n_img, int H, int W, int cin, int cout, int kh,
                            int kw, int stride, int pad, int dtype, void* stream);
/* dw_ohwi (cout,kh,kw,cin) fp32, zeroed by the caller (pixel slices accumulate through fp32 atomics) */
int esb_conv2d_direct_wgrad(const void* x, const void* dy, float* dw_ohwi, int n_img, int H, int W, int cin, int cout, int kh,
                            int kw, int stride, int pad, int dtype, void* stream);
/* k x k / stride / pad max pooling on NHWC (the stem's F.max_pool2d(3, 2, 1)); forward only (the stem is frozen) */
int esb_maxpool2d_nhwc(const void* x, void* y, int n_img, int H, int W, int C, int k, int stride, int pad, int dtype,
                       void* stream);

/* ---- attention core of the grounding decoder (self-, text- and 3D cross-attention of
 * embodiedscan/models/layers/ground_transformer/decoder.py:89-95,151-177; †upstream nn.MultiheadAttention) as flash-attention
 * tiles on wgmma fed by TMA (csrc/attn_tc.cu). Head dimension 32. q (B,H,Lq,32), k / v (B,H,Lk,32), o bf16 contiguous;
 * key_pad (B,Lk) uint8 (1 = ignore) or NULL; lse (B,H,Lq) fp32. Backward: delta (B,H,Lq) fp32 workspace, dq (B,H,Lq,32) fp32
 * += the gradient (zeroed by the caller; key tiles add in order), dk / dv (B,H,Lk,32) bf16 written once. ------------------- */
int esb_attn_fwd(const void* q, const void* k, const void* v, const unsigned char* key_pad, void* o, float* lse, int B, int H,
                 int Lq, int Lk, float scale, void* stream);
int esb_attn_bwd(const void* q, const void* k, const void* v, const unsigned char* key_pad, const void* o, const void* dout,
                 const float* lse, float* delta, float* dq, void* dk, void* dv, int B, int H, int Lq, int Lk, float scale,
                 void* stream);

/* ---- point painting (batch_point_sample + apply_3d_transformation + batch_points_cam2img + F.grid_sample;
 * embodiedscan/models/layers/fusion_layers/point_fusion.py:208-311, structures/bbox_3d/utils.py:289-332) -------- */
int esb_paint_meta_bytes(void);
/* points: voxel rows `coords` (xyz * voxel_size) or, when fpts != NULL, explicit fp32 locations fpts (N,3) of scans
 * fbatch (N) (NULL: scan 0) — the prior grid of the occupancy model (dense_fusion_occ.py:156-202) */
int esb_paint_fwd(const int* coords, const float* fpts, const int* fbatch, long long N, float voxel_size,
                  const void* metas, const float* proj, int V,
                  const void* feat, int Hf, int Wf, int C, float pad_h, float pad_w, void* out, int* valid_count,
                  int dtype, void* stream);
int esb_paint_bwd(const int* coords, const float* fpts, const int* fbatch, long long N, float voxel_size,
                  const void* metas, const float* proj, int V,
                  const void* dout, int Hf, int Wf, int C, float pad_h, float pad_w, float* dfeat, int dtype,
                  void* stream);

/* ---- FCAF3D head: target assignment (fcaf3d_head.py:1578-1664) and sigmoid focal loss (mmcv.ops.sigmoid_focal_loss
 * through mmdet.FocalLoss, cfg :46-52) --------------------------------------------------------------------------- */
size_t esb_fcaf3d_targets_workspace_bytes(int L, int NgT, int B);
int esb_fcaf3d_targets(const float* points, const int* level_off, int L, int Np, const int* pt_batch,
                       const float* boxes, const float* rneg, const long long* labels, const int* box_off, int B, int NgT,
                       int max_ng, int assign_thr, int center_thr, float* center_t, float* bbox_t, long long* cls_t,
                       int* box_idx, void* ws, size_t ws_bytes, void* stream);
int esb_focal_loss_fwd(const void* logits, const long long* target, long long n, int C, float gamma, float alpha,
                       const float* row_w, float* loss_sum, int dtype, void* stream);
int esb_focal_loss_bwd(const void* logits, const long long* target, long long n, int C, float gamma, float alpha,
                       const float* row_w, const float* scale_dev, void* grad, int dtype, void* stream);

/* box regression: _bbox_pred_to_bbox + 4 decoupled BBoxCDLoss terms (fcaf3d_head.py:1224-1281,1454-1525;
 * chamfer_distance.py:160-285) for all positives, value and gradient in one launch.
 * mode: ESB_CD_*; group: 8 (every source corner searches all 8 target corners) or 4 (corners 0-3 and 4-7 search their
 * own half); norm_decouple != 0 divides the three decoupled terms of a row by clamp(|target size|, 0.1). */
int esb_bbox_cd_loss(const float* points, const float* bbox_pred, const float* targets, const float* row_w,
                     const float* w4_host, int P, int mode, int group, int norm_decouple, float* loss_out, float* grad,
                     void* stream);

/* ---- point-set chamfer distance (chamfer_distance.py:13-79) ---------------------------------------------------------
 * src (B,N,C), dst (B,M,C) fp32, 1 <= C <= 8, mode ESB_CD_*. dist1 (B,N) / idx1 (B,N) int64: per source point the
 * smallest criterion distance to dst and its index (lowest index on ties); dist2 / idx2 (B,M) the same from dst to src. */
int esb_chamfer_fwd(const float* src, const float* dst, int B, int N, int M, int C, int mode, float* dist1,
                    float* dist2, long long* idx1, long long* idx2, void* stream);
/* grad_src (B,N,C) / grad_dst (B,M,C) fp32 (overwritten) from g1 = dL/d dist1 and g2 = dL/d dist2 (either may be NULL):
 * each point's own term plus the terms of every point whose nearest neighbour it is, summed in index order. */
int esb_chamfer_bwd(const float* src, const float* dst, const long long* idx1, const long long* idx2, const float* g1,
                    const float* g2, int B, int N, int M, int C, int mode, float* grad_src, float* grad_dst,
                    void* stream);

/* ---- rotated BEV IoU + NMS (mmcv.ops.nms3d / nms3d_normal; fcaf3d_head.py:1666-1725) ---------------------------- */
int esb_nms_bev_segmented(const float* boxes, const int* seg_off, int S, int max_seg, float iou_thr, int rotated,
                          unsigned char* keep, void* stream);
int esb_iou_bev_pairwise(const float* a, int na, const float* b, int nb, int rotated, float* out, void* stream);

/* ---- exact 9-DoF box IoU (pytorch3d.ops.box3d_overlap via EulerInstance3DBoxes.overlaps, euler_box3d.py:103-135) ---- */
int esb_box3d_overlap(const float* corners1, int n1, const float* corners2, int n2, float* vol, float* iou,
                      void* stream);
/* Best same-range overlap: query i is compared with the targets tidx[qbeg[i] .. qend[i]) only (qcorners (m,8,3),
 * tcorners (g,8,3) fp32, tidx int32 into the g targets). best[i] = max IoU over the range (-inf when it is empty), arg[i] =
 * the target index that gives it (-1 when empty); a NaN IoU wins, ties go to the smallest target index (torch.max's
 * choice). Every pair is the arithmetic of esb_box3d_overlap, bit for bit; one thread per query, no atomics. */
int esb_box3d_best_overlap(const float* qcorners, int m, const float* tcorners, const int* tidx, const int* qbeg,
                           const int* qend, float* best, int* arg, void* stream);

/* ---- differentiable rotated 3D IoU of one-to-one box pairs (mmcv.ops.diff_iou_rotated_3d, the IoU behind
 * RotatedIoU3DLoss, rotated_iou_loss.py:14-91). a (n, lda), b (n, ldb) fp32 rows (x, y, z, w, l, h, alpha, ...), z the
 * box centre, lda, ldb >= 7; columns past 7 are ignored. fwd writes iou (n). bwd recomputes the geometry and writes
 * grad_a / grad_b (n, 7) = grad_iou * d iou / d (x, y, z, w, l, h, alpha); grad_b may be NULL. One thread per pair, no
 * atomics: bit-reproducible. ---- */
int esb_rotated_iou3d_fwd(const float* a, int lda, const float* b, int ldb, long long n, float* iou, void* stream);
int esb_rotated_iou3d_bwd(const float* a, int lda, const float* b, int ldb, long long n, const float* grad_iou,
                          float* grad_a, float* grad_b, void* stream);

/* ---- greedy NMS on the exact 9-DoF 3D IoU (the demo's final box filter `nms_filter`, demo/demo.py:84-130), batched over
 * S segments. boxes9 (M,9) = centre, size, ZXY Euler angles; scores (M); labels (M) in [0, num_classes); seg_off (S+1).
 * Candidates are already score-descending inside each segment. Walking a segment in order, a candidate is skipped when
 * its label already has topk_per_class kept boxes, when score < score_thr, or when its IoU with a kept box exceeds
 * iou_thr (>= 0); skipped candidates suppress nothing. Segment s writes the kept positions (indices into the M rows) to
 * keep[seg_off[s] ..) in selection order and their count to n_keep[s]. A box with a size <= 0 or a non-finite value has
 * IoU 0 with every box: it can be kept, never suppresses and is never suppressed. A label outside [0, num_classes) is
 * never kept. After the call the first 3*S unsigned long long of ws hold, per segment, the pairs tested, the pairs
 * left by the bounding-sphere test and the pairs left by the separating-axis test (those ran the exact clipping). */
size_t esb_nms3d_9dof_workspace_bytes(int M, int S, int max_seg);
int esb_nms3d_9dof(const float* boxes9, const float* scores, const int* labels, const int* seg_off, int S, int max_seg,
                   float iou_thr, float score_thr, int topk_per_class, int num_classes, int* keep, int* n_keep, void* ws,
                   size_t ws_bytes, void* stream);

/* ---- batched one-to-one assignment (HungarianAssigner3D.assign: hungarian_assigner.py:110-126 -> scipy
 * linear_sum_assignment on the host, 7 layers x batch times per iteration from grounding_head.py:398).
 * cost: (n_problems, n_pred, ld_gt) fp32, problem p uses columns [0, n_gt[p]); n_gt[p] <= ld_gt <= n_pred.
 * NaN/+inf -> 100, -inf -> -100 as torch.nan_to_num in the reference. pred_to_gt: (n_problems, n_pred) int32, the
 * 0-based target matched to each prediction or -1; gt_to_pred (nullable): (n_problems, ld_gt) int32, the inverse map
 * (-1 beyond n_gt[p]). One launch, one CTA per problem. ---- */
int esb_hungarian_batch(const float* cost, const int* n_gt, int n_problems, int n_pred, int ld_gt, int* pred_to_gt,
                        int* gt_to_pred, void* stream);

/* ---- input side: Det3DDataPreprocessor image path (data_preprocessor.py:249-264, utils.py:9-63) and the
 * depth->points unprojection (datasets/transforms/points.py:30-81, multiview.py:139-169) ------------------------- */
int esb_img_normalize(const unsigned char* src, int n_img, int H, int W, int Hp, int Wp, const float* mean3_host,
                      const float* std3_host, int bgr_to_rgb, int channels_last, void* dst, int dtype, void* stream);
/* MultiViewPipeline's `Resize(scale=(w, h), keep_ratio=False)` (cv2.resize INTER_LINEAR through mmcv imresize, bit for
 * bit, including cv2's switch to INTER_AREA at an exact 2x downscale on both axes and its copy at an unchanged size):
 * src (V,H,W,3) uint8 as decoded -> dst (V,3,h,w) uint8, channel order unchanged. One launch for all V views
 * (V <= 65535). */
int esb_img_resize_linear_u8(const unsigned char* src, int V, int H, int W, int h, int w, unsigned char* dst,
                             void* stream);
size_t esb_unproject_depth_workspace_bytes(int V, int H, int W);
int esb_unproject_depth(const unsigned short* depth, int V, int H, int W, float depth_shift, const float* mats,
                        float* out, int* view_of, int* count_dev, void* ws, size_t ws_bytes, void* stream);

/* ---- optimiser step over the flat parameter arena (AdamW + clip_grad; cfg :219-223) -----------------------------
 * esb_adamw_step_groups: one launch. lr_wd_host: n_groups (lr, weight_decay) pairs in host memory, copied into the
 * launch (1 <= n_groups <= 2048, else ESB_EINVAL). group_of: (n,) uint16 group of every element, each < n_groups; null
 * exactly when n_groups == 1. Elements of a group whose lr is 0 are left untouched (parameter and moments).
 * grad_scale * clip_state[2] (esb_grad_clip_coef) scales the gradient. */
int esb_grad_clip_coef(const float* grad, long long n, float max_norm, float world_scale, float* state, void* stream);
int esb_adamw_step_groups(float* param, const float* grad, float* exp_avg, float* exp_avg_sq,
                          const unsigned short* group_of, const float* lr_wd_host, int n_groups, long long n,
                          float beta1, float beta2, float eps, int step, float grad_scale, const float* clip_state,
                          void* stream);
int esb_cast_f32_to_bf16(const float* src, void* dst, long long n, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ESB200_H */
