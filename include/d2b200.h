/*
 * d2b200.h -- C ABI of the H100-native detection hot path (libd2b200.so).
 *
 * This is the drop-in boundary: plain pointers, sizes and a CUDA stream, no torch types.
 * Every entry point cites the reference interface it replaces (paths relative to the
 * detectron2 source tree).  The Python host (detectron2_b200/) binds these with ctypes and
 * re-exports the reference's `detectron2.layers` operator surface on top; INTEGRATION.md shows
 * the binding a detectron2 maintainer would add.
 *
 * Conventions
 *   - all tensor pointers are DEVICE pointers on the current device, dense row-major
 *     ("contiguous" NCHW unless stated); the caller owns every buffer (no hidden allocation:
 *     scratch comes in through explicit workspace pointers whose size is queried first);
 *   - `stream` is a cudaStream_t passed as void*; launches are asynchronous, there are no
 *     internal device synchronisations;
 *   - return value: 0 = ok, <0 = invalid argument (D2B_E*), >0 = cudaError_t from a launch;
 *   - stateless and re-entrant.
 */
#ifndef D2B200_H_
#define D2B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define D2B_OK 0
#define D2B_EINVAL (-1)      /* bad shape / null pointer / unsupported parameter */
#define D2B_EWORKSPACE (-2)  /* workspace too small */
#define D2B_EUNSUPPORTED (-3)

#define D2B_ABI_VERSION 4
int d2b_abi_version(void);
/* compile-time facts, replaces detectron2._C.get_cuda_version / has_cuda (csrc/vision.cpp:23-49,86-88) */
int d2b_cuda_version(void);
const char* d2b_arch(void); /* "sm_90a" */

/* ---- RoIAlign, axis-aligned -------------------------------------------------------------
 * Replaces torchvision::roi_align / torchvision::_roi_align_backward as reached from
 * detectron2/layers/roi_align.py:58-65 (forward) and its autograd (backward).
 * input [N,C,H,W] fp32, rois [K,5] = (batch_idx,x1,y1,x2,y2) fp32, out [K,C,PH,PW] fp32.
 * sampling_ratio <= 0 -> adaptive ceil(roi/pooled) grid.  aligned: 0/1. */
int d2b_roi_align_forward(const float* input, int N, int C, int H, int W, const float* rois, int K,
                          float spatial_scale, int pooled_h, int pooled_w, int sampling_ratio,
                          int aligned, float* out, void* stream);
/* grad_in [N,C,H,W] is fully written (zero-filled inside, then accumulated with atomics). */
int d2b_roi_align_backward(const float* grad_out, const float* rois, int K, float spatial_scale,
                           int pooled_h, int pooled_w, int N, int C, int H, int W,
                           int sampling_ratio, int aligned, float* grad_in, void* stream);

/* ---- Multi-level RoI pooler (fused) --------------------------------------------------------
 * Replaces the per-level loop of detectron2/modeling/poolers.py:206-263 (ROIPooler.forward with
 * pooler_type "ROIAlign"/"ROIAlignV2"): level assignment (poolers.py:23-59,
 * floor(canonical_level + log2(sqrt(area)/canonical_box_size + 1e-8)) clamped), the per-level
 * nonzero / gather / roi_align / index_put_ -- one launch, no host synchronisation.
 * feat[l] is [N,C,H[l],W[l]] fp32 (level min_level + l), scale[l] its spatial scale; grad[l] is
 * only read by the backward (fully written: zero-filled inside, then accumulated).
 * rois [K,5] in image coordinates, out / grad_out [K,C,PH,PW]. */
#define D2B_MAX_LEVELS 8
typedef struct {
  int num_levels;
  const float* feat[D2B_MAX_LEVELS];
  float* grad[D2B_MAX_LEVELS];
  int H[D2B_MAX_LEVELS], W[D2B_MAX_LEVELS];
  float scale[D2B_MAX_LEVELS];
  int min_level, max_level, canonical_level;
  float canonical_box_size;
  /* Optional [K,5] boxes the FPN level is assigned from (NULL: the sampling rois).  The reference assigns levels from the
   * fp32 boxes (poolers.py:245) but samples half-precision feature maps with rois cast to the feature dtype
   * (layers/roi_align.py:60): a host that reproduces that hands the rounded rois as `rois` and the fp32 ones here. */
  const float* level_rois;
} d2b_pyramid;
int d2b_roi_pooler_forward(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int pooled_h,
                           int pooled_w, int sampling_ratio, int aligned, float* out, void* stream);
int d2b_roi_pooler_backward(const d2b_pyramid* pyr, int N, int C, const float* grad_out, const float* rois,
                            int K, int pooled_h, int pooled_w, int sampling_ratio, int aligned, void* stream);

/* Channels-last variants.  torchvision::roi_align calls input.contiguous() (a hidden NCHW copy) when it is handed a
 * torch.channels_last feature map; these entry points consume the NHWC storage directly: feat[l] / input is
 * [N,H,W,C] fp32 (the storage of a channels_last [N,C,H,W] tensor), C % 4 == 0, H*W*C < 2^31 per image.
 * Same results contract as d2b_roi_align_forward / d2b_roi_pooler_forward, out stays [K,C,PH,PW]. */
int d2b_roi_align_forward_nhwc(const float* input, int N, int C, int H, int W, const float* rois, int K,
                               float spatial_scale, int pooled_h, int pooled_w, int sampling_ratio,
                               int aligned, float* out, void* stream);
int d2b_roi_pooler_forward_nhwc(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int pooled_h,
                                int pooled_w, int sampling_ratio, int aligned, float* out, void* stream);
/* Layout change of a whole pyramid in ONE launch: pyr->feat[l] [N,C,H,W] -> dst[l] [N,H,W,C] (dst: host array of
 * pyr->num_levels device pointers, caller-owned).  Used by the host when a large pooler call on NCHW features is
 * cheaper as transform + channels-last pooling (detectron2_b200/ops.py). */
int d2b_pyramid_nchw_to_nhwc(const d2b_pyramid* pyr, int N, int C, float* const* dst, void* stream);
/* The inverse: pyr->feat[l] [N,H,W,C] -> dst[l] [N,C,H,W], one launch. */
int d2b_pyramid_nhwc_to_nchw(const d2b_pyramid* pyr, int N, int C, float* const* dst, void* stream);
/* Half-precision activations / gradients (dtype codes below): the same kernels read or write fp16 / bf16 elements in place
 * of fp32 ones -- fp32 arithmetic, no separate cast pass.  The reference up-casts such tensors before its fp32 kernels
 * (torchvision's autocast wrapper of roi_align; layers/roi_align_rotated.py:81-83) and casts the result back.
 *   d2b_pyramid_nchw_to_nhwc_t   pyr->feat[l] point to [N,C,H,W] elements of `src_dtype`; dst[l] are fp32 [N,H,W,C]
 *   d2b_pyramid_nhwc_to_nchw_t   pyr->feat[l] fp32 [N,H,W,C]; dst[l] [N,C,H,W] elements of `dst_dtype`
 *   d2b_roi_pooler_forward_nhwc_t    out [K,C,PH,PW] elements of `out_dtype`
 *   d2b_roi_pooler_backward_nhwc_t   grad_out [K,C,PH,PW] elements of `grad_dtype`; pyr->grad[l] stay fp32 (accumulators) */
#define D2B_F32 0
#define D2B_F16 1
#define D2B_BF16 2
int d2b_pyramid_nchw_to_nhwc_t(const d2b_pyramid* pyr, int N, int C, float* const* dst, int src_dtype, void* stream);
int d2b_pyramid_nhwc_to_nchw_t(const d2b_pyramid* pyr, int N, int C, void* const* dst, int dst_dtype, void* stream);
int d2b_roi_pooler_forward_nhwc_t(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int pooled_h,
                                  int pooled_w, int sampling_ratio, int aligned, void* out, int out_dtype, void* stream);
int d2b_roi_pooler_backward_nhwc_t(const d2b_pyramid* pyr, int N, int C, const void* grad_out, int grad_dtype,
                                   const float* rois, int K, int pooled_h, int pooled_w, int sampling_ratio, int aligned,
                                   void* stream);
/* Channels-last backward (autograd of the two forwards above): grad_in / pyr->grad[l] are [N,H,W,C] fp32, 16-byte aligned,
 * fully written (zero-filled inside, then accumulated with one 128-bit vector reduction per footprint pixel and 4 channels).
 * grad_out stays [K,C,PH,PW].  Same results contract as d2b_roi_align_backward / d2b_roi_pooler_backward. */
int d2b_roi_align_backward_nhwc(const float* grad_out, const float* rois, int K, float spatial_scale,
                                int pooled_h, int pooled_w, int N, int C, int H, int W,
                                int sampling_ratio, int aligned, float* grad_in, void* stream);
int d2b_roi_pooler_backward_nhwc(const d2b_pyramid* pyr, int N, int C, const float* grad_out, const float* rois,
                                 int K, int pooled_h, int pooled_w, int sampling_ratio, int aligned, void* stream);

/* ---- RoIAlign, rotated ------------------------------------------------------------------
 * Replaces torch.ops.detectron2.roi_align_rotated_forward / _backward
 * (csrc/vision.cpp:118-119, csrc/ROIAlignRotated/ROIAlignRotated.h:50-113).
 * rois [K,6] = (batch_idx,cx,cy,w,h,angle_degrees). */
int d2b_roi_align_rotated_forward(const float* input, int N, int C, int H, int W, const float* rois,
                                  int K, float spatial_scale, int pooled_h, int pooled_w,
                                  int sampling_ratio, float* out, void* stream);
int d2b_roi_align_rotated_backward(const float* grad_out, const float* rois, int K,
                                   float spatial_scale, int pooled_h, int pooled_w, int N, int C,
                                   int H, int W, int sampling_ratio, float* grad_in, void* stream);
/* Channels-last variants (input / grad_in are [N,H,W,C] fp32 storage, 16-byte aligned, C % 4 == 0); out / grad_out stay
 * [K,C,PH,PW].  Same results contract. */
int d2b_roi_align_rotated_forward_nhwc(const float* input, int N, int C, int H, int W, const float* rois,
                                       int K, float spatial_scale, int pooled_h, int pooled_w,
                                       int sampling_ratio, float* out, void* stream);
int d2b_roi_align_rotated_backward_nhwc(const float* grad_out, const float* rois, int K,
                                        float spatial_scale, int pooled_h, int pooled_w, int N, int C,
                                        int H, int W, int sampling_ratio, float* grad_in, void* stream);

/* ---- Multi-level rotated RoI pooler (fused) ------------------------------------------------
 * Replaces the per-level loop of detectron2/modeling/poolers.py:245-263 for pooler_type "ROIAlignRotated" (nonzero /
 * gather / roi_align_rotated / index_put_ per level): one launch per direction, no host synchronisation.  Level rule of
 * d2b_roi_pooler_forward with area = w*h of the (batch_idx,cx,cy,w,h,angle_degrees) row (RotatedBoxes.area,
 * structures/rotated_boxes.py:236-245); a negative or NaN area matches no level: zero output, no gradient.
 * rois [K,6]; pyr->level_rois must be NULL (the reference samples rotated RoIs in fp32 whatever the feature dtype,
 * layers/roi_align_rotated.py:81-83).  pyr->grad[l] are fully written by the backward (all levels zero-filled by one launch,
 * then accumulated).  Every argument is checked before anything is launched.
 *   d2b_roi_pooler_rotated_forward / _backward            feat[l] / grad[l] NCHW fp32, out / grad_out [K,C,PH,PW] fp32
 *   d2b_roi_pooler_rotated_forward_nhwc_t / _backward_nhwc_t
 *       feat[l] / grad[l] fp32 [N,H,W,C] storage, 16-byte aligned, C % 4 == 0; out / grad_out [K,C,PH,PW] elements of
 *       out_dtype / grad_dtype (D2B_F32 / D2B_F16 / D2B_BF16 above; fp32 arithmetic, grad[l] stay fp32); D2B_EUNSUPPORTED
 *       when a [128][PH*PW] fp32 tile exceeds 150 KB of shared memory (use the NCHW form).
 * N == 0 with K > 0 is D2B_EINVAL (RoIs of images that do not exist). */
int d2b_roi_pooler_rotated_forward(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int pooled_h,
                                   int pooled_w, int sampling_ratio, float* out, void* stream);
int d2b_roi_pooler_rotated_backward(const d2b_pyramid* pyr, int N, int C, const float* grad_out, const float* rois,
                                    int K, int pooled_h, int pooled_w, int sampling_ratio, void* stream);
int d2b_roi_pooler_rotated_forward_nhwc_t(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int pooled_h,
                                          int pooled_w, int sampling_ratio, void* out, int out_dtype, void* stream);
int d2b_roi_pooler_rotated_backward_nhwc_t(const d2b_pyramid* pyr, int N, int C, const void* grad_out, int grad_dtype,
                                           const float* rois, int K, int pooled_h, int pooled_w, int sampling_ratio,
                                           void* stream);

/* ---- NMS --------------------------------------------------------------------------------
 * Replaces torchvision::nms reached from detectron2/layers/nms.py:5-22 (nms, batched_nms) and
 * torch.ops.detectron2.nms_rotated (csrc/vision.cpp:116, csrc/nms_rotated/nms_rotated.h:22-37).
 * Greedy NMS in stable descending-score order (equal scores: lower index first), the order of
 * torch.sort(scores, descending=True, stable=True): a NaN score of either sign ranks above +inf, NaNs among
 * themselves by index; -0.0 and +0.0 are equal scores.
 *   boxes  [M,4] xyxy fp32 (rotated: [M,5] cx,cy,w,h,angle_deg), scores [M] fp32
 *   idxs   [M] int64 category ids or NULL (plain nms).  When non-NULL the reference's coordinate
 *          trick is applied on the fly:  axis-aligned  box + idx*(max_coord+1)   (torchvision
 *          ops/boxes.py _batched_nms_coordinate_trick);  rotated  centre + idx*(max-min+1)
 *          (detectron2/layers/nms.py:137-146), all in fp32 like the reference.  The range propagates
 *          NaN like torch's max / min: a NaN coordinate makes every offset box NaN, so nothing is suppressed.
 *          Boxes of different categories meet in the reference's single NMS with IoU 0, so a threshold that 0 passes
 *          (rotated thr <= 0, axis-aligned thr < 0) suppresses across categories too; that case runs as one segment
 *          of all non-ignored boxes (max_segment must then bound their number).
 *          The range covers the non-ignored boxes only (see below); torchvision has no ignored ids and
 *          treats a negative id as an ordinary category, so public batched_nms callers pass ids >= 0.
 *   keep   [M] int64 out: kept ORIGINAL indices, score-descending; num_keep [1] int64 out (device).
 * Suppression rule: axis-aligned  iou >  thr (torchvision);  rotated  iou >= thr (nms_rotated_cpu.cpp:54).
 * flags: D2B_NMS_ROTATED selects the rotated variant; D2B_NMS_NO_OFFSET makes `idxs` pure segment ids -- the
 *        coordinates are used as given (the caller already applied whatever offsets it wants, e.g. the per-image offsets
 *        of a multi-image RPN batch, detectron2_b200/proposal_utils.py).
 *   idxs   negative category ids mark boxes to be IGNORED: they suppress nothing and are never kept (callers with a
 *          fixed-capacity candidate list park their empty slots there instead of compacting the list).
 * max_segment: upper bound on the number of boxes of one category (0 = unknown, i.e. M).  It sizes the IoU bitmask
 *        ((max_segment/64 + 2) words per box instead of M/64), so a batched caller that knows its per-category limit (RPN:
 *        pre_nms_topk per image and level) keeps memory and work linear in the batch size.  If a category turns out larger,
 *        nothing is written out of bounds and num_keep is set to -1.
 *   keep   entries past num_keep are 0.
 * workspace: d2b_nms_workspace_bytes(M, flags, max_segment) bytes of device scratch. */
#define D2B_NMS_ROTATED 1
#define D2B_NMS_NO_OFFSET 2
size_t d2b_nms_workspace_bytes(int64_t M, int flags, int64_t max_segment);
int d2b_nms(const float* boxes, const float* scores, const int64_t* idxs, int64_t M,
            double iou_threshold, int flags, int64_t max_segment, int64_t* keep, int64_t* num_keep,
            void* workspace, size_t workspace_bytes, void* stream);

/* ---- Batched RPN proposal selection around the NMS (SURVEY 8f-2) ----------------------------------------
 * Replaces the per-image Python loop of detectron2/modeling/proposal_generator/proposal_utils.py:96-133 (boolean filtering,
 * `.item()` sync, per-image batched_nms, slicing) by a fixed-capacity launch sequence for ALL images:
 *   torch.topk per level (library)  ->  d2b_rpn_prepare  ->  d2b_nms(category = image*L + level, D2B_NMS_NO_OFFSET,
 *   max_segment = pre_nms_topk)  ->  d2b_rpn_select.
 * d2b_rpn_prepare: lv->proposals[l] [N,A_l,4] decoded boxes, lv->topk_idx[l] / topk_scores[l] [N,k_l] (the per-level top-k of
 *   the objectness logits), image_hw [N,2] (h, w) on the device.  T = sum_l k_l candidates per image.  Writes, for all N*T
 *   candidates: flat_boxes (clipped to the image; zeros for removed ones), nms_boxes (+ torchvision's per-image
 *   level offsets when use_offsets), nms_scores (-inf for removed), raw_scores, cat_ids (image*L + level, or -1 = removed:
 *   non-finite or not larger than min_box_size after clipping), nonfinite[1] (1 if any candidate was non-finite).
 * d2b_rpn_select: keep / num_keep as returned by d2b_nms over the N*T candidates; out_boxes [N,post_nms_topk,4],
 *   out_scores / out_index [N,post_nms_topk] (0-padded), counts [N] int64. */
typedef struct {
  int num_levels;
  const float* proposals[D2B_MAX_LEVELS];
  const int64_t* topk_idx[D2B_MAX_LEVELS];
  const float* topk_scores[D2B_MAX_LEVELS];
  int A[D2B_MAX_LEVELS], k[D2B_MAX_LEVELS];
} d2b_rpn_levels;
int d2b_rpn_prepare(const d2b_rpn_levels* lv, int N, const float* image_hw, float min_box_size, int use_offsets,
                    float* flat_boxes, float* nms_boxes, float* nms_scores, float* raw_scores, int64_t* cat_ids,
                    int* nonfinite, void* stream);
int d2b_rpn_select(const int64_t* keep, const int64_t* num_keep, int N, int T, int post_nms_topk,
                   const float* flat_boxes, const float* raw_scores, const int64_t* cat_ids, float* out_boxes,
                   float* out_scores, int64_t* out_index, int64_t* counts, void* stream);

/* ---- Fast R-CNN and dense-head (RetinaNet) inference candidates around the NMS (SURVEY 8f-2) -----------------
 * Replace the per-image Python loops of detectron2/modeling/roi_heads/fast_rcnn.py:46-173 (`fast_rcnn_inference`:
 * boolean filtering, `nonzero()` sync, per-image batched_nms, slicing) and of meta_arch/dense_detector.py:186-258 +
 * meta_arch/retinanet.py:256-308 (per-level filter / top-k / apply_deltas, per-image batched_nms) by
 *   d2b_frcnn_prepare | (torch.topk per level ->) d2b_dense_prepare  ->  d2b_nms(category = image*(K+1) + class,
 *   D2B_NMS_NO_OFFSET)  ->  d2b_rpn_select (the same per-image first-topk selection).
 * d2b_frcnn_prepare: boxes [Rtot, kreg*4] predicted boxes (kreg = 1 class-agnostic or K), scores [Rtot, K+1] (last column =
 *   background) of N <= D2B_MAX_IMAGES images concatenated; row_start [N+1] HOST array of the images' first rows;
 *   image_hw [N,2] on the device.  Per image the (row, class) pairs with score > score_thresh of the rows whose box and
 *   score entries are all finite are written in row-major order into `cap` slots: cand_boxes (clipped), nms_boxes
 *   (+ torchvision's class * (max coordinate + 1) offsets), nms_scores (-inf in dead slots), raw_scores, cand_flat
 *   (row_in_image * K + class), cat_ids (image*(K+1) + class, -1 = dead); n_cand [N] = the image's candidate count (larger
 *   than cap: the list was truncated and the caller must redo that image); row_map [Rtot] = index of a row among its image's
 *   valid rows (-1 for dropped rows) -- what the reference returns as kept row indices.
 * d2b_dense_prepare: per level l anchors [R_l,4], deltas [N,R_l,4], and the batched top-k of the thresholded scores
 *   (topk_idx [N,k_l] = anchor*K + class, topk_scores [N,k_l] with -inf in dead slots); weights[4] (HOST) and scale_clamp of
 *   Box2BoxTransform.  Writes for all N*T candidates (T = sum k_l): flat_boxes (decoded), nms_boxes (+ offsets while the
 *   image has <= 25 000 live candidates, as torchvision), nms_scores, raw_scores, classes, cat_ids. */
#define D2B_MAX_IMAGES 64
typedef struct {
  int num_levels;
  const float* anchors[D2B_MAX_LEVELS];
  const float* deltas[D2B_MAX_LEVELS];
  const int64_t* topk_idx[D2B_MAX_LEVELS];
  const float* topk_scores[D2B_MAX_LEVELS];
  int R[D2B_MAX_LEVELS], k[D2B_MAX_LEVELS];
} d2b_dense_levels;
int d2b_frcnn_prepare(const float* boxes, const float* scores, const int* row_start, int N, int num_classes, int kreg,
                      const float* image_hw, float score_thresh, int cap, float* cand_boxes, float* nms_boxes,
                      float* nms_scores, float* raw_scores, int64_t* cand_flat, int64_t* cat_ids, int64_t* n_cand,
                      int64_t* row_map, void* stream);
int d2b_dense_prepare(const d2b_dense_levels* lv, int N, int num_classes, const float* weights, float scale_clamp,
                      float* flat_boxes, float* nms_boxes, float* nms_scores, float* raw_scores, int64_t* classes,
                      int64_t* cat_ids, void* stream);

/* ---- Mask-head training targets + loss (SURVEY 8f-4) ------------------------------------------------------
 * Replaces, for one image, BitMasks.crop_and_resize (detectron2/structures/masks.py:193-224) + the class gather and
 * binary_cross_entropy_with_logits of mask_rcnn_loss (modeling/roi_heads/mask_head.py:60-112).
 *   logits [K,C,S,S] fp32 mask-head outputs of the image's K sampled proposals; gt_masks [G,H,W] bytes (0 / non-0);
 *   boxes [K,4] proposal boxes; mask_index [K] int64 ground-truth mask of every proposal (NULL: proposal k uses mask k, the
 *   reference's per-proposal BitMasks); classes [K] int64 (NULL: class-agnostic, channel 0).
 *   loss_per_roi [K]: sum over the S*S bins of the BCE of the proposal's class channel (the caller sums and divides by the
 *   total number of elements, "mean" reduction); targets [K,S,S] bytes: the 0/1 targets.
 * Backward: grad_scale [K] = d loss / d loss_per_roi; grad_logits [K,C,S,S] fully written: (sigmoid(x) - t) * grad_scale[k]
 * on the class channel, 0 elsewhere. */
int d2b_mask_loss_forward(const float* logits, int K, int C, int S, const uint8_t* gt_masks, int G, int H, int W,
                          const float* boxes, const int64_t* mask_index, const int64_t* classes,
                          float* loss_per_roi, uint8_t* targets, void* stream);
int d2b_mask_loss_backward(const float* logits, int K, int C, int S, const uint8_t* targets, const int64_t* classes,
                           const float* grad_scale, float* grad_logits, void* stream);

/* ---- Rotated-box IoU --------------------------------------------------------------------
 * Replaces torch.ops.detectron2.box_iou_rotated (csrc/vision.cpp:117,
 * csrc/box_iou_rotated/box_iou_rotated.h:20-33).  boxes1 [N,5], boxes2 [M,5] fp32 -> ious [N,M] fp32. */
int d2b_box_iou_rotated(const float* boxes1, int64_t N, const float* boxes2, int64_t M, float* ious,
                        void* stream);

/* ---- Deformable convolution v1 / v2 -----------------------------------------------------
 * Replaces detectron2._C.deform_conv_forward / deform_conv_backward_input /
 * deform_conv_backward_filter / modulated_deform_conv_forward / modulated_deform_conv_backward
 * (csrc/vision.cpp:90-102, csrc/deformable/deform_conv.h:116-375).  One description for both:
 * mask == NULL -> DCNv1, bias == NULL -> no bias.
 *   x [N,Cin,H,W], offset [N,2*DG*kh*kw,Ho,Wo] (channel 2k = dy, 2k+1 = dx of kernel point k),
 *   mask [N,DG*kh*kw,Ho,Wo], weight [Cout,Cin/G,kh,kw], bias [Cout], out [N,Cout,Ho,Wo]; all fp32.
 */
typedef struct {
  int N, Cin, H, W, Cout, kh, kw, stride_h, stride_w, pad_h, pad_w, dil_h, dil_w, groups,
      deformable_groups;
} d2b_dcn_params;

/* precision: 0 = fp32 FFMA (parity path), 1 = bf16x3 split on wgmma (fp32-class accuracy, <= 1e-4 rel), 2 = plain bf16
 * operands on wgmma (autocast path), -1 = auto (1 when the tensor-core kernels take the shape, else 0).
 * flags: D2B_DCN_X_NHWC -- x (and grad_x) are channels-last storage [N,H,W,Cin] (the storage of a torch.channels_last
 *        tensor), 16-byte aligned; tensor-core precisions only.  Without it the tensor-core path re-lays x out once per call.
 * The tensor-core path needs scratch (NHWC copy of x, pre-tiled bf16 operands): query the size first; 256-byte aligned.
 * d2b_deform_conv_tc_shape_supported: 1 when precision 1/2 is available for the shape (backward: both gradient kernels). */
#define D2B_DCN_X_NHWC 1
int d2b_deform_conv_tc_shape_supported(const d2b_dcn_params* p, int backward);
size_t d2b_deform_conv_forward_workspace_bytes(const d2b_dcn_params* p, int precision, int flags);
/* Saved columns (training).  `cols` (optional, d2b_deform_conv_cols_bytes() bytes, 16-byte aligned, tensor-core precisions
 * only) receives the sampled columns the forward builds anyway -- bf16 hi [| lo] tiles in the tensor core's operand layout;
 * handed to the backward, the weight-gradient kernel streams them back instead of sampling x a second time (the reference
 * re-runs deformable_im2col in deform_conv_backward_parameters, deform_conv_cuda.cu:586-610).  The buffer is opaque and only
 * valid for the same params / precision.  d2b_deform_conv_cols_bytes returns 0 when the shape has no tensor-core path. */
size_t d2b_deform_conv_cols_bytes(const d2b_dcn_params* p, int precision);
int d2b_deform_conv_forward(const float* x, const float* offset, const float* mask,
                            const float* weight, const float* bias, const d2b_dcn_params* p,
                            int precision, int flags, float* out, void* cols, void* workspace,
                            size_t workspace_bytes, void* stream);
/* Backward.  Any of the grad outputs may be NULL to skip it.  Outputs are fully written (zero-filled inside, then
 * accumulated); need_data = any of grad_x / grad_offset / grad_mask, need_weight = grad_weight. */
size_t d2b_deform_conv_backward_workspace_bytes(const d2b_dcn_params* p, int precision, int flags, int need_data,
                                                int need_weight);
int d2b_deform_conv_backward(const float* x, const float* offset, const float* mask,
                             const float* weight, const float* grad_out, const d2b_dcn_params* p,
                             int precision, int flags, const void* cols, float* grad_x, float* grad_offset,
                             float* grad_mask, float* grad_weight, float* grad_bias, void* workspace,
                             size_t workspace_bytes, void* stream);

/* conv2 of a DeformBottleneckBlock fused (detectron2/modeling/backbone/resnet.py:305-318): `offset_mask`
 * [N, 3*DG*kh*kw, Ho, Wo] is the raw conv2_offset output (chunk / cat / sigmoid of :307-311 applied while the sampling taps
 * are built), y = relu(conv * scale[oc] + shift[oc]) (FrozenBatchNorm folded, or scale NULL and shift = bias; relu 0/1) is
 * applied in the accumulator epilogue.  Tensor-core precisions only (1, 2 or -1); workspace sizes are those of
 * d2b_deform_conv_forward / backward_workspace_bytes.  The backward takes y (to gate the ReLU) and returns the gradient of
 * the fused offset_mask tensor (mask part through the sigmoid). */
int d2b_deform_conv_fused_forward(const float* x, const float* offset_mask, const float* weight, const float* scale,
                                  const float* shift, int relu, const d2b_dcn_params* p, int precision, int flags,
                                  float* out, void* cols, void* workspace, size_t workspace_bytes, void* stream);
int d2b_deform_conv_fused_backward(const float* x, const float* offset_mask, const float* weight, const float* scale,
                                   int relu, const float* y, const float* grad_out, const d2b_dcn_params* p,
                                   int precision, int flags, const void* cols, float* grad_x, float* grad_offset_mask,
                                   float* grad_weight, void* workspace, size_t workspace_bytes, void* stream);

/* ---- paste_masks_in_image ---------------------------------------------------------------
 * Replaces detectron2/layers/mask_ops.py:74-147 (GPU branch: every pixel of the image for every mask).
 * masks [N,M,M] fp32, boxes [N,4] xyxy fp32 -> out [N,H,W] uint8: (v >= threshold) as 0/1 when
 * threshold >= 0, else (uint8)(v*255). */
int d2b_paste_masks(const float* masks, const float* boxes, int N, int M, int H, int W,
                    float threshold, uint8_t* out, void* stream);
/* The boolean result (threshold >= 0 only) bit-packed: out [N,H,ceil(W/32)] uint32, bit b of word w of row y = pixel
 * (y, 32 w + b), unused bits of a row's last word zero.  Identical decisions to d2b_paste_masks; 1/8 of the bytes for the
 * device -> host copy that follows the paste in inference post-processing. */
int d2b_paste_masks_packed(const float* masks, const float* boxes, int N, int M, int H, int W,
                           float threshold, uint32_t* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* D2B200_H_ */
