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

#define D2B_ABI_VERSION 7
int d2b_abi_version(void);
/* compile-time facts, replaces detectron2._C.get_cuda_version / has_cuda (csrc/vision.cpp:23-49,86-88) */
int d2b_cuda_version(void);
const char* d2b_arch(void); /* "sm_90a" */

/* ---- RoIAlign and the multi-level RoI pooler (fused) ---------------------------------------
 * One forward and one backward entry point serve every RoIAlign call, axis-aligned or rotated, NCHW or channels-last.
 * A single-level op is a one-level pyramid: feat[0] / grad[0] = its input / grad_in, H[0], W[0], scale[0] = spatial_scale
 * (a one-level pyramid skips the level assignment).  Replaces:
 *   - torchvision::roi_align / torchvision::_roi_align_backward as reached from detectron2/layers/roi_align.py:58-65 and its
 *     autograd: rois [K,5] = (batch_idx,x1,y1,x2,y2);
 *   - torch.ops.detectron2.roi_align_rotated_forward / _backward (csrc/vision.cpp:118-119,
 *     csrc/ROIAlignRotated/ROIAlignRotated.h:50-113): rois [K,6] = (batch_idx,cx,cy,w,h,angle_degrees), flag D2B_ROI_ROTATED;
 *   - the per-level loop of detectron2/modeling/poolers.py:206-263 (ROIPooler.forward with pooler_type "ROIAlign",
 *     "ROIAlignV2" or "ROIAlignRotated"): level assignment (poolers.py:23-59, floor(canonical_level +
 *     log2(sqrt(area)/canonical_box_size + 1e-8)) clamped), the per-level nonzero / gather / roi_align / index_put_ -- one
 *     launch per direction, no host synchronisation.  area = (x2-x1)*(y2-y1), or w*h of a rotated row (RotatedBoxes.area,
 *     structures/rotated_boxes.py:236-245); a negative or NaN area matches no level: zero output, no gradient.
 * feat[l] is level min_level + l, [N,C,H[l],W[l]] fp32, scale[l] its spatial scale; rois are in image coordinates, fp32;
 * out / grad_out are [K,C,PH,PW].  sampling_ratio <= 0 -> adaptive ceil(roi/pooled) grid.  aligned: 0/1 (ignored when
 * rotated).  The backward fully writes every grad[l] (all levels zero-filled by one launch, then accumulated with atomics);
 * feat[] is not read by it. */
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
   * (layers/roi_align.py:60): a host that reproduces that hands the rounded rois as `rois` and the fp32 ones here.  Must be
   * NULL when rotated: the reference samples rotated RoIs in fp32 whatever the feature dtype (layers/roi_align_rotated.py:81-83). */
  const float* level_rois;
} d2b_pyramid;
/* Element types of out / grad_out and of the layout changes below.  fp16 / bf16 are read or written in place of fp32 --
 * fp32 arithmetic, no separate cast pass; the reference up-casts such tensors before its fp32 kernels (torchvision's
 * autocast wrapper of roi_align; layers/roi_align_rotated.py:81-83) and casts the result back. */
#define D2B_F32 0
#define D2B_F16 1
#define D2B_BF16 2
/* flags */
#define D2B_ROI_ROTATED 1  /* rois [K,6]; `aligned` is ignored                                     */
#define D2B_ROI_BACKWARD 2 /* d2b_roi_pooler_nhwc_supported only                                  */
#define D2B_ROI_NHWC 4     /* feat[l] / grad[l] are channels-last [N,H,W,C] fp32 storage (the storage of a torch.channels_last
                            * [N,C,H,W] tensor, which torchvision::roi_align would .contiguous() first), 16-byte aligned;
                            * out / grad_out stay [K,C,PH,PW].  Without it out_dtype / grad_dtype must be D2B_F32.      */
/* Arguments are checked in this order, and nothing is launched before every check has passed:
 *   forward:  1. K == 0 or C == 0: D2B_OK (nothing to compute).
 *             2. D2B_EINVAL: a flag bit other than ROTATED | NHWC; an invalid pyramid (num_levels outside 1..D2B_MAX_LEVELS,
 *                an H[l] or W[l] below 1, or more than one level and max_level - min_level + 1 != num_levels); level_rois
 *                with ROTATED; N < 1, C < 0 or K < 0; pooled_h or pooled_w below 1; rois, out or a feat[l] NULL; out_dtype
 *                not a D2B_F* code, or not D2B_F32 without NHWC; with NHWC, a feat[l] that is not 16-byte aligned.
 *             3. With NHWC, D2B_EUNSUPPORTED when d2b_roi_pooler_nhwc_supported refuses the shape.
 *   backward: 1. D2B_EINVAL: the flag bits, the pyramid, level_rois with ROTATED; N, C or K below 0; N == 0 with K > 0 (RoIs
 *                of images that do not exist); the dtype rule of the forward for grad_dtype.
 *             2. N == 0 or C == 0: D2B_OK (no gradient element to write).
 *             3. D2B_EINVAL: a grad[l] NULL or, with NHWC, not 16-byte aligned; when K > 0, grad_out or rois NULL, or
 *                pooled_h or pooled_w below 1.
 *             4. With NHWC and K > 0, D2B_EUNSUPPORTED when d2b_roi_pooler_nhwc_supported refuses the shape.
 *             5. The zero-fill, then (K > 0) the accumulation. */
int d2b_roi_pooler_forward(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int pooled_h, int pooled_w,
                           int sampling_ratio, int aligned, int flags, void* out, int out_dtype, void* stream);
int d2b_roi_pooler_backward(const d2b_pyramid* pyr, int N, int C, const void* grad_out, int grad_dtype, const float* rois,
                            int K, int pooled_h, int pooled_w, int sampling_ratio, int aligned, int flags, void* stream);
/* Which shapes the channels-last kernels take: D2B_OK, or D2B_EUNSUPPORTED where the pooler entry points above return
 * D2B_EUNSUPPORTED with D2B_ROI_NHWC -- use the NCHW form then.  The entry points ask the same function, so the answer
 * cannot disagree with them.  Reads pyr->num_levels, H[] and W[] only: pointer alignment stays the caller's check.
 * Host-only, no CUDA call (safe during graph capture).  flags: D2B_ROI_ROTATED for the rotated kernels, | D2B_ROI_BACKWARD
 * for the backward.  The limits: C % 4 == 0, H*W*C < 2^30 per level and image, and a bound on PH*PW from each kernel's
 * shared-memory tile (rotated: a [128][PH*PW] fp32 tile within 150 KB). */
int d2b_roi_pooler_nhwc_supported(const d2b_pyramid* pyr, int C, int pooled_h, int pooled_w, int flags);
/* Layout change of a whole pyramid in ONE launch (dst: host array of pyr->num_levels device pointers, caller-owned).  Used by
 * the host when a large pooler call on NCHW features is cheaper as transform + channels-last pooling
 * (detectron2_b200/ops.py), and to bring gradients accumulated channels-last back to NCHW.
 *   d2b_pyramid_nchw_to_nhwc   pyr->feat[l] [N,C,H,W] elements of `src_dtype` -> dst[l] fp32 [N,H,W,C], 16-byte aligned
 *   d2b_pyramid_nhwc_to_nchw   pyr->feat[l] fp32 [N,H,W,C], 16-byte aligned -> dst[l] [N,C,H,W] elements of `dst_dtype` */
int d2b_pyramid_nchw_to_nhwc(const d2b_pyramid* pyr, int N, int C, float* const* dst, int src_dtype, void* stream);
int d2b_pyramid_nhwc_to_nchw(const d2b_pyramid* pyr, int N, int C, void* const* dst, int dst_dtype, void* stream);

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

/* ---- Inference candidate selection around the NMS (SURVEY 8f-2) -------------------------------------------------------
 * Replaces the per-image Python loops of detectron2/modeling/proposal_generator/proposal_utils.py:96-133 and rrpn.py:20-127
 * (find_top_rpn_proposals / find_top_rrpn_proposals: boolean filtering, `.item()` sync, per-image batched_nms, slicing),
 * of modeling/roi_heads/fast_rcnn.py:46-173 and rotated_fast_rcnn.py:46-132 (fast_rcnn_inference[_rotated]: boolean
 * filtering, `nonzero()` sync, per-image batched_nms, slicing) and of meta_arch/dense_detector.py:186-258 +
 * meta_arch/retinanet.py:256-308 / fcos.py:253-301 (per-level filter / top-k / apply_deltas, per-image batched_nms) by a
 * fixed-capacity launch sequence for ALL images:
 *   d2b_rpn_prepare | d2b_frcnn_prepare | (torch.topk per level ->) d2b_dense_prepare  ->  d2b_nms(D2B_NMS_NO_OFFSET, and
 *   D2B_NMS_ROTATED for rotated boxes; category = image*L + level | image*(K+1) + class, -1 = removed; max_segment =
 *   pre_nms_topk for the RPN)  ->  d2b_rpn_select (the same per-image first-topk selection for all three).
 * flags, one namespace for the four entry points:
 *   D2B_SELECT_ROTATED (rpn, frcnn, select): boxes are (cx, cy, w, h, angle_deg), D = 5 floats per box, no alignment
 *     requirement.  The prepares apply RotatedBoxes.clip(image, clip_angle_threshold = 1) -- every angle normalised to
 *     (a + 180) % 360 - 180 (torch's float remainder), boxes with |angle| <= 1 clipped as xyxy boxes -- and
 *     batched_nms_rotated's per-image offsets category * (max - min + 1) on the centre (layers/nms.py:137-146).  Without it
 *     boxes are xyxy, D = 4, and the box arrays must be 16-byte aligned (float4 access); the offsets are torchvision's
 *     category * (max coordinate + 1).  Offsets are computed over the image's surviving boxes, in fp32.
 *   D2B_SELECT_SEG_PER_IMAGE (rpn, frcnn; with ROTATED only): every surviving candidate of image n gets NMS category n,
 *     offsets unchanged.  Pass it for iou_threshold <= 0, which IoU 0 passes (the reference's single NMS then suppresses
 *     across categories too); the NMS max_segment must then bound the image's slot count.
 *   D2B_SELECT_NO_OFFSETS (rpn, without ROTATED only): nms_boxes are not shifted, as torchvision's batched_nms past 25 000
 *     boxes per image.  The rotated offsets are always applied.
 *   D2B_SELECT_LINEAR (dense only): the Box2BoxTransformLinear.apply_deltas decode of FCOS (box_regression.py:275-307,
 *     normalize_by_size): relu(deltas) times the anchor's (width, height), then the centre minus (l, t), plus (r, b);
 *     weights and scale_clamp are unused and weights may be NULL.
 * d2b_rpn_prepare: lv->proposals[l] [N,A_l,D] decoded boxes, lv->topk_idx[l] / topk_scores[l] [N,k_l] (the per-level top-k of
 *   the objectness logits), image_hw [N,2] (h, w) on the device.  T = sum_l k_l candidates per image.  Writes, for all N*T
 *   candidates: flat_boxes [N*T,D] (clipped to the image; zeros for removed ones), nms_boxes [N*T,D] (+ the per-image level
 *   offsets), nms_scores (-inf for removed), raw_scores, cat_ids (image*L + level, or -1 = removed: non-finite, or width or
 *   height not larger than min_box_size after clipping), nonfinite[1] (1 if any candidate was non-finite).
 * d2b_frcnn_prepare: boxes [Rtot, kreg*D] predicted boxes (kreg = 1 class-agnostic or K), scores [Rtot, K+1] (last column =
 *   background) of N <= D2B_MAX_IMAGES images concatenated; row_start [N+1] HOST array of the images' first rows;
 *   image_hw [N,2] on the device.  Per image the (row, class) pairs with score > score_thresh of the rows whose box and
 *   score entries are all finite are written in row-major order into `cap` slots: cand_boxes [N*cap,D] (clipped), nms_boxes
 *   (+ the class offsets), nms_scores (-inf in dead slots), raw_scores, cand_flat (row_in_image * K + class), cat_ids
 *   (image*(K+1) + class, -1 = dead); n_cand [N] = the image's candidate count (larger than cap: the list was truncated and
 *   the caller must redo that image); row_map [Rtot] = index of a row among its image's valid rows (-1 for dropped rows) --
 *   what the reference returns as kept row indices.
 * d2b_dense_prepare: per level l anchors [R_l,4], deltas [N,R_l,4], and the batched top-k of the thresholded scores
 *   (topk_idx [N,k_l] = anchor*K + class, topk_scores [N,k_l] with -inf in dead slots); weights[4] (HOST) and scale_clamp of
 *   Box2BoxTransform.  Writes for all N*T candidates (T = sum k_l): flat_boxes (decoded), nms_boxes (+ offsets while the
 *   image has <= 25 000 live candidates, as torchvision), nms_scores, raw_scores, classes, cat_ids.  xyxy boxes only.
 * d2b_rpn_select: keep / num_keep as returned by d2b_nms over the N*T candidates (T = cap after d2b_frcnn_prepare),
 *   flat_boxes [N*T,D]; out_boxes [N,post_nms_topk,D], out_scores / out_index [N,post_nms_topk] (0-padded), counts [N] int64.
 * Arguments are checked in this order, and nothing is launched or written before every check has passed:
 *   all four:  1. D2B_EINVAL: a flag bit the entry point does not take, SEG_PER_IMAGE without ROTATED, NO_OFFSETS with it.
 *   rpn_prepare:  2. D2B_EINVAL: lv or nonfinite NULL, num_levels outside 1..D2B_MAX_LEVELS, N < 0; per level A_l < 0,
 *                    k_l < 0 or k_l > A_l, a level pointer NULL when N > 0 and k_l > 0, or (xyxy) proposals[l] not 16-byte
 *                    aligned; T > INT_MAX; when N > 0 and T > 0, image_hw or an output NULL; (xyxy) flat_boxes or
 *                    nms_boxes not 16-byte aligned.
 *                 3. nonfinite is zeroed, even when there is no candidate; N == 0 or T == 0: D2B_OK.
 *   frcnn_prepare: 2. D2B_EINVAL: N < 0 or N > D2B_MAX_IMAGES, num_classes < 1, kreg neither 1 nor num_classes, cap < 0,
 *                    row_start NULL.
 *                 3. N == 0: D2B_OK.
 *                 4. D2B_EINVAL: row_start[0] < 0 or row_start decreasing; image_hw or n_cand NULL; when the images have
 *                    rows, boxes, scores or row_map NULL; when cap > 0, an output NULL; (xyxy) cand_boxes or nms_boxes not
 *                    16-byte aligned.
 *   dense_prepare: 2. D2B_EINVAL: lv NULL, num_levels outside 1..D2B_MAX_LEVELS, N < 0, num_classes < 1, weights NULL
 *                    without LINEAR.
 *                 3. N == 0: D2B_OK.
 *                 4. D2B_EINVAL: per level R_l < 0 or k_l < 0, a level pointer NULL when k_l > 0, or anchors[l] or
 *                    deltas[l] not 16-byte aligned; T > INT_MAX.
 *                 5. T == 0: D2B_OK.
 *                 6. D2B_EINVAL: an output NULL, or flat_boxes or nms_boxes not 16-byte aligned.
 *   rpn_select:    2. D2B_EINVAL: N, T or post_nms_topk below 0.
 *                 3. N == 0: D2B_OK.
 *                 4. D2B_EINVAL: counts NULL; when T > 0 and post_nms_topk > 0, another pointer NULL, or (xyxy)
 *                    flat_boxes or out_boxes not 16-byte aligned.
 *                 5. T == 0 or post_nms_topk == 0: counts zeroed, D2B_OK. */
#define D2B_SELECT_ROTATED 1
#define D2B_SELECT_SEG_PER_IMAGE 2
#define D2B_SELECT_NO_OFFSETS 4
#define D2B_SELECT_LINEAR 8
#define D2B_MAX_IMAGES 64
typedef struct {
  int num_levels;
  const float* proposals[D2B_MAX_LEVELS];
  const int64_t* topk_idx[D2B_MAX_LEVELS];
  const float* topk_scores[D2B_MAX_LEVELS];
  int A[D2B_MAX_LEVELS], k[D2B_MAX_LEVELS];
} d2b_rpn_levels;
typedef struct {
  int num_levels;
  const float* anchors[D2B_MAX_LEVELS];
  const float* deltas[D2B_MAX_LEVELS];
  const int64_t* topk_idx[D2B_MAX_LEVELS];
  const float* topk_scores[D2B_MAX_LEVELS];
  int R[D2B_MAX_LEVELS], k[D2B_MAX_LEVELS];
} d2b_dense_levels;
int d2b_rpn_prepare(const d2b_rpn_levels* lv, int N, const float* image_hw, float min_box_size, int flags, float* flat_boxes,
                    float* nms_boxes, float* nms_scores, float* raw_scores, int64_t* cat_ids, int* nonfinite, void* stream);
int d2b_frcnn_prepare(const float* boxes, const float* scores, const int* row_start, int N, int num_classes, int kreg,
                      const float* image_hw, float score_thresh, int cap, int flags, float* cand_boxes, float* nms_boxes,
                      float* nms_scores, float* raw_scores, int64_t* cand_flat, int64_t* cat_ids, int64_t* n_cand,
                      int64_t* row_map, void* stream);
int d2b_dense_prepare(const d2b_dense_levels* lv, int N, int num_classes, const float* weights, float scale_clamp, int flags,
                      float* flat_boxes, float* nms_boxes, float* nms_scores, float* raw_scores, int64_t* classes,
                      int64_t* cat_ids, void* stream);
int d2b_rpn_select(const int64_t* keep, const int64_t* num_keep, int N, int T, int post_nms_topk, int flags,
                   const float* flat_boxes, const float* raw_scores, const int64_t* cat_ids, float* out_boxes,
                   float* out_scores, int64_t* out_index, int64_t* counts, void* stream);

/* ---- Anchor / proposal matching for the training targets -------------------------------------------------------
 * Replaces the per-image pairwise_iou + Matcher loops of RPN / RRPN.label_and_sample_anchors, RetinaNet.label_anchors,
 * (R)ROIHeads.label_and_sample_proposals and CascadeROIHeads._match_and_label_boxes up to their sampling step, for all
 * images at once and without the G x A IoU matrix (structures/boxes.py:312-358, modeling/matcher.py:61-127).
 *   gt_boxes [N,Gmax,D] fp32 with gt_count [N] (device, int64; clamped to [0, Gmax]); D = 4 xyxy, or 5 (cx,cy,w,h,angle_deg)
 *   with D2B_MATCH_ROTATED.  pred_boxes [A,D] shared by every image (pred_image_stride 0, anchors) or [N,stride,D] per image
 *   (pred_image_stride >= Pmax rows); pred_count [N] (device, int64, clamped to [0, Pmax]) or NULL for Pmax.
 *   D2B_MATCH_APPEND_GT: the image's GT boxes follow its pred_count predictions (add_ground_truth_to_proposals); output row
 *   p >= pred_count[n] is GT p - pred_count[n].  Output rows per image P = Pmax (+ Gmax with D2B_MATCH_APPEND_GT).
 *   thresholds[num_thresholds] (HOST, compared in fp32) and labels[num_thresholds + 1] (HOST) as Matcher(thresholds, labels):
 *   thresholds[0] > 0, ascending, labels in {-1, 0, 1}, 1 <= num_thresholds <= D2B_MATCH_MAX_THRESHOLDS.
 *   D2B_MATCH_LOW_QUALITY = allow_low_quality_matches.  boundary_thresh >= 0 (axis-aligned only): after the matcher, rows
 *   whose box is not Boxes.inside_box(image_hw[n], boundary_thresh) get label -1; image_hw [N,2] (h, w) fp32 device.
 * Outputs [N,P]: matches (int64, first GT on ties), match_labels (int8), matched_gt_boxes [N,P,D] (NULL-able; zeros for an
 *   image without GT), classes (NULL-able; needs gt_classes [N,Gmax] int64: label 1 -> gt_classes[match], 0 -> num_classes,
 *   -1 -> -1, an image without GT -> num_classes).  Rows past pred_count (+ gt_count) are padding: match 0, label -1, zero
 *   box, class -1.  An image without GT gets matches 0 and label labels[0], as the reference.  status [N] int32:
 *   D2B_MATCH_STATUS_INVALID_IOU when an IoU of the image is negative or NaN (the reference's assertion; the image's other
 *   outputs are then unspecified).  workspace: d2b_match_workspace_bytes(N, Gmax, P) bytes, no initialisation needed.
 * No host synchronisation, static shapes: capturable in a CUDA graph.  All arguments are checked before the first CUDA call. */
#define D2B_MATCH_ROTATED 1
#define D2B_MATCH_LOW_QUALITY 2
#define D2B_MATCH_APPEND_GT 4
#define D2B_MATCH_MAX_THRESHOLDS 8
#define D2B_MATCH_STATUS_INVALID_IOU 1
size_t d2b_match_workspace_bytes(int N, int Gmax, int P);
int d2b_match_boxes(const float* gt_boxes, const int64_t* gt_count, int N, int Gmax, const float* pred_boxes,
                    int64_t pred_image_stride, const int64_t* pred_count, int Pmax, const double* thresholds,
                    int num_thresholds, const int* labels, int flags, const float* image_hw, double boundary_thresh,
                    const int64_t* gt_classes, int64_t num_classes, int64_t* matches, int8_t* match_labels,
                    float* matched_gt_boxes, int64_t* classes, int* status, void* workspace, size_t workspace_bytes,
                    void* stream);

/* ---- FCOS point assignment -------------------------------------------------------------------------------------------
 * Replaces FCOS._match_anchors + label_anchors (meta_arch/fcos.py:97-191) for all images in one launch, without the
 * reference's [G,R,2] / [G,R,4] tensors.  anchors [R,4] fp32: the point boxes of every level concatenated (R = sum of the
 * level_counts[num_levels], HOST, 1 <= num_levels <= D2B_MAX_LEVELS); gt_boxes [N,Gmax,4] fp32 with gt_count [N] (device,
 * int64, clamped to [0, Gmax]; rows past it are never read), gt_classes [N,Gmax] int64.
 * Per point (fp32): centre (a[:2] + a[2:]) / 2, size a[2] - a[0], lower bound 4 * size (0 on the first level), upper bound
 * 8 * size (+inf on the last level; on every point when the last level is empty, as the reference's [-0:] slice).
 * Per GT g: quality = float(max(|centre - centre_g|) < radius * size && min(l, t, r, b) > 0 && lower < max(l, t, r, b)
 *   < upper) * (1e8 - area_g), radius = center_sampling_radius rounded to fp32, (l, t, r, b) the distances of the centre to
 *   g's edges.  Boxes whose areas differ by less than the fp32 spacing at 1e8 tie; a GT with a non-finite area has NaN
 *   quality at every point.
 * Outputs [N,R]: matches int64 = torch.max(dim=0)'s argmax over GT (NaN beats every number, first index on ties), -1 when
 *   the maximum is < 1e-5 (a NaN maximum is matched) or the image has no GT; labels int64 = gt_classes[match], num_classes
 *   when unmatched; matched_gt_boxes [N,R,4] = gt_boxes[max(match, 0)] (GT 0 for the unmatched points of an image with GT,
 *   zeros for an image without GT).
 * No host synchronisation, static shapes: capturable in a CUDA graph.  All arguments are checked before the first CUDA call. */
int d2b_fcos_assign(const float* anchors, const int* level_counts, int num_levels, const float* gt_boxes,
                    const int64_t* gt_count, int N, int Gmax, const int64_t* gt_classes, int64_t num_classes,
                    double center_sampling_radius, int64_t* matches, int64_t* labels, float* matched_gt_boxes, void* stream);

/* ---- Sampling of the training labels --------------------------------------------------------------------------------
 * Replaces subsample_labels (modeling/sampling.py:9-54) and the per-image loops around it in RPN._subsample_labels
 * (proposal_generator/rpn.py:286-303, rrpn.py:184) and ROIHeads._sample_proposals (roi_heads/roi_heads.py:181-217,
 * rotated_fast_rcnn.py:218-270), for all images at once, without the reference's nonzero() host syncs.
 *   labels [N,P] of label_kind (D2B_LABELS_I8: int8, e.g. the match_labels of d2b_match_boxes; D2B_LABELS_I64: int64, e.g.
 *   its classes).  Per image: positive = label != -1 && label != bg_label, negative = label == bg_label (padding rows, label
 *   -1, are never sampled).  max_pos = int(num_samples * positive_fraction), computed by the caller (HOST, sampling.py:41);
 *   k_pos = min(#pos, max_pos), k_neg = min(#neg, num_samples - k_pos).
 *   Keys: mix = the SplitMix64 finaliser, arithmetic mod 2^64; s_n = mix(*seed + (n+1) * 0xD1B54A32D192ED03),
 *   key(n, i) = mix(s_n + (i+1) * 0x9E3779B97F4A7C15).  The sample is the k_pos smallest-key positives, then the k_neg
 *   smallest-key negatives, each in ascending key order (unsigned compare): the reference's law (a uniform random subset
 *   in uniform random order), not torch.randperm's random stream.  seed: one uint64 in device memory.
 * Outputs (NULL-able, not both NULL): out_labels [N,P] int8 in the RPN form (1 sampled positive, 0 sampled negative, -1
 *   otherwise; must not alias labels); sampled [N,num_samples] int64: the k_pos positive indices, then the k_neg negative
 *   ones, then -1.  num_pos / num_neg [N] int64 (device): k_pos, k_neg.
 * 0 <= num_samples <= D2B_SAMPLE_MAX_SAMPLES, 0 <= max_pos <= num_samples, N <= 65535.  workspace:
 *   d2b_sample_labels_workspace_bytes(N, P, num_samples) bytes, 256-byte aligned, no initialisation needed.
 * Exact for every input (a radix select on the keys, refined until the threshold bin fits its buffer).  Five launches on
 * `stream`, no allocation, no host synchronisation: capturable in a CUDA graph.  All arguments are checked before the first
 * CUDA call. */
#define D2B_SAMPLE_MAX_SAMPLES 8192
size_t d2b_sample_labels_workspace_bytes(int N, int P, int num_samples);
int d2b_sample_labels(const void* labels, int label_kind, int N, int P, int64_t bg_label, int num_samples, int max_pos,
                      const uint64_t* seed, int8_t* out_labels, int64_t* sampled, int64_t* num_pos, int64_t* num_neg,
                      void* workspace, size_t workspace_bytes, void* stream);

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

/* ---- Polygon ground-truth masks (DESIGN.md f-4) ------------------------------------------------------------------------
 * PolygonMasks.crop_and_resize (detectron2/structures/masks.py:396-420, rasterize_polygons_within_box :39-85) and
 * polygons_to_bitmask / BitMasks.from_polygon_masks (:22-36, :166-180), bit-exact to pycocotools' rleFrPoly + merge +
 * decode, for a whole batch without a host round trip.
 * A batch's polygons (polygon_masks.pack_polygons): coords [V,2] float64 (x, y) vertices; poly_start [P+1] int32, polygon p
 *   = vertices [poly_start[p], poly_start[p+1]); inst_start [G+1] int32, instance g = polygons [inst_start[g],
 *   inst_start[g+1]).  An instance's mask is the union of its polygons' masks; an instance without polygons is all zeros.
 * Contracts for input the reference rejects or leaves undefined: an instance index outside [0, G) gives an all-zero mask;
 *   an instance range out of order or past P is empty, and so is a polygon range out of order or past V (nothing outside
 *   the arrays is read); a polygon with a non-finite vertex, or a lattice coordinate 5 x' + 0.5 outside (-2^30, 2^30), adds
 *   nothing; so does every polygon of a proposal whose box is not finite.
 *
 * d2b_polygons_crop_and_resize: boxes [K,4] fp32 proposal boxes; mask_index [K] int64 instance of each proposal (NULL:
 *   proposal k uses instance k) -> out [K,S,S] uint8 0/1, row-major.  Per proposal, each vertex becomes
 *   x' = (x - x0) * ratio_w (float64), ratio_w = S / (x1 - x0) in fp32 when x1 - x0 >= 0.1, else S / 0.1 in float64
 *   (y likewise), and is rasterized on the S x S grid.  One CTA per proposal.
 *   Checks, in order (nothing is launched before all pass):
 *     1. D2B_EINVAL: K < 0, S < 1 or S > D2B_POLYGON_MAX_S, V, P or G below 0.
 *     2. K == 0: D2B_OK.
 *     3. D2B_EINVAL: boxes or out NULL; inst_start NULL with G > 0, poly_start NULL with P > 0, coords NULL with V > 0.
 * d2b_polygons_to_bitmask: out [G,H,W] uint8 0/1, every instance rasterized on the full H x W image (no transform).  CTAs
 *   tile the columns and rows, and each edge visits only the columns it crosses.
 *   Checks, in order:
 *     1. D2B_EINVAL: V, P or G below 0, H or W below 1, H * W > INT_MAX, more than INT_MAX tiles.
 *     2. G == 0: D2B_OK.
 *     3. D2B_EINVAL: out or inst_start NULL, poly_start NULL with P > 0, coords NULL with V > 0.
 * d2b_mask_loss_polygons_forward: d2b_mask_loss_forward with the targets of d2b_polygons_crop_and_resize, rasterized inside
 *   the proposal's CTA: the same loss_per_roi and targets outputs, for all K proposals of a batch in one launch (mask_index
 *   holds batch-wide instance indices).  The backward is d2b_mask_loss_backward on these targets.
 *   Checks, in order:
 *     1. D2B_EINVAL: K < 0, C < 1, S < 1 or S > D2B_POLYGON_MAX_S, V, P or G below 0.
 *     2. K == 0: D2B_OK.
 *     3. D2B_EINVAL: logits, boxes, loss_per_roi or targets NULL; inst_start NULL with G > 0, poly_start NULL with P > 0,
 *        coords NULL with V > 0.
 * No host synchronisation, no allocation: capturable in a CUDA graph. */
#define D2B_POLYGON_MAX_S 256
int d2b_polygons_crop_and_resize(const double* coords, int V, const int* poly_start, int P, const int* inst_start, int G,
                                 const float* boxes, const int64_t* mask_index, int K, int S, uint8_t* out, void* stream);
int d2b_polygons_to_bitmask(const double* coords, int V, const int* poly_start, int P, const int* inst_start, int G, int H,
                            int W, uint8_t* out, void* stream);
int d2b_mask_loss_polygons_forward(const float* logits, int K, int C, int S, const double* coords, int V,
                                   const int* poly_start, int P, const int* inst_start, int G, const float* boxes,
                                   const int64_t* mask_index, const int64_t* classes, float* loss_per_roi,
                                   uint8_t* targets, void* stream);

/* ---- Keypoint head: heatmap decoding (inference) ----------------------------------------------------------------
 * Replaces the per-detection loop of heatmaps_to_keypoints (detectron2/structures/keypoints.py:164-235), reached from
 * keypoint_rcnn_inference (modeling/roi_heads/keypoint_head.py:99-132).
 *   maps [R,K,S,S] fp32 logits, rois [R,4] xyxy fp32 -> out [R,K,4] fp32 (x, y, logit, score), 16-byte aligned.
 * Per ROI: w = max(x2 - x1, 1), h = max(y2 - y1, 1), Wo = ceil(w), Ho = ceil(h); the (Ho, Wo) bicubic resize of each map with
 * PyTorch's CUDA upsample_bicubic2d arithmetic (align_corners = False, A = -0.75, source indices clamped to [0, S-1]) is
 * evaluated on the fly, never stored.  x = (x_int + 0.5) * (w / Wo) + x1, y likewise, logit = the resized map at the argmax,
 * score = 1 / sum_{S x S} exp(maps - logit).
 * Argmax rule (torch.argmax / max on CUDA): ties go to the smallest linear index y * Wo + x; a NaN beats every number and the
 * first NaN wins (logit NaN); -0.0 and +0.0 are equal.
 * A ROI with a non-finite coordinate difference, or more than 2^32 output pixels, gets a NaN row (the reference raises
 * in int(); the condition is detected on the device, without a host synchronisation).
 * 1 <= S <= D2B_KEYPOINTS_MAX_S (the map is staged in shared memory), K >= 1.  workspace: d2b_keypoints_workspace_bytes(R, K)
 * bytes, 8-byte aligned, no initialisation needed.  Three launches, no host synchronisation: capturable in a CUDA graph. */
#define D2B_KEYPOINTS_MAX_S 241
size_t d2b_keypoints_workspace_bytes(int R, int K);
int d2b_keypoints_from_heatmaps(const float* maps, int R, int K, int S, const float* rois, float* out, void* workspace,
                                size_t workspace_bytes, void* stream);

/* ---- Keypoint head: training targets + loss --------------------------------------------------------------------
 * Replaces keypoint_rcnn_loss (modeling/roi_heads/keypoint_head.py:40-96): the per-image Keypoints.to_heatmap
 * (_keypoints_to_heatmap, structures/keypoints.py:105-161), the nonzero() host sync, the gather of the valid logit rows and
 * F.cross_entropy, for all images of the batch in one launch.
 *   logits [N,K,S,S] of `dtype` (D2B_F32 / D2B_F16 / D2B_BF16, read in place, fp32 arithmetic); keypoints [N,K,3] fp32
 *   (x, y, v) matched ground truth of every proposal; boxes [N,4] fp32 proposal boxes.
 *   target [N,K] int64 = y * S + x of the keypoint's heatmap cell, 0 when not valid; valid [N,K] uint8: the cell is inside
 *   the S x S map and v > 0.  Cell: floor((c - x1) * (S / (x2 - x1))) with S / t evaluated as reciprocal(t) * S, each
 *   operation rounded on its own; c == x2 gives S - 1 (y likewise); a NaN cell (a NaN coordinate, or 0 * inf at c == x1
 *   of a subnormal-width box) is not valid, as PyTorch's CUDA float-to-int64 conversion gives INT64_MIN for NaN.
 *   loss_per_kp [N,K] fp32: logsumexp(row) - row[target] on valid rows, 0 elsewhere; num_valid [1] int64 (zeroed inside).
 *   logits and loss_per_kp may both be NULL: the targets alone (Keypoints.to_heatmap).
 * Backward: grad_scale [N,K] fp32 = d loss / d loss_per_kp; grad_logits [N,K,S,S] of `dtype`, fully written:
 * (softmax(row) - onehot(target)) * grad_scale on valid rows, 0 elsewhere. */
int d2b_keypoint_loss_forward(const void* logits, int dtype, int N, int K, int S, const float* keypoints,
                              const float* boxes, int64_t* target, uint8_t* valid, float* loss_per_kp, int64_t* num_valid,
                              void* stream);
int d2b_keypoint_loss_backward(const void* logits, int dtype, int N, int K, int S, const int64_t* target,
                               const uint8_t* valid, const float* grad_scale, void* grad_logits, void* stream);

/* ---- Panoptic FPN inference: semantic labels and the thing / stuff combine --------------------------------------------
 * Replace the per-image loop of PanopticFPN.inference (modeling/meta_arch/panoptic_fpn.py:159-179): sem_seg_postprocess
 * (modeling/postprocessing.py:77-100) + argmax(dim=0), and combine_semantic_and_instance_outputs (panoptic_fpn.py:184-269),
 * for N <= D2B_MAX_IMAGES images of different sizes, without host reads.  Images are described per image (pointers and
 * sizes), so a batch of differently sized detector_postprocess outputs needs no concatenation.
 *
 * d2b_sem_seg_labels: logits [N,C,Hp,Wp] of `dtype` (D2B_F32 / D2B_F16 / D2B_BF16, read in place); per image the crop
 *   (h[n], w[n]) <= (Hp, Wp) of the top-left corner and the output size (H[n], W[n]); labels[n] [H[n],W[n]] int64 out =
 *   argmax over the channels of the bilinear resize of the crop (align_corners = False, no scale factor: PyTorch's CUDA
 *   upsample_bilinear2d arithmetic, a plain copy when the sizes are equal), each channel's value rounded to `dtype` before
 *   the comparison.  Argmax as torch.argmax on CUDA: the first maximal channel wins; a NaN beats every number and the first
 *   NaN wins; -0.0 == +0.0.  The C x H x W map is never stored.  One launch.
 *   Checks, in order (nothing is launched before all pass):
 *     1. D2B_EINVAL: img NULL, N < 0 or N > D2B_MAX_IMAGES, dtype not a D2B_F* code, C < 1, Hp < 1 or Wp < 1.
 *     2. N == 0: D2B_OK.
 *     3. D2B_EINVAL: logits NULL; per image h outside 1..Hp, w outside 1..Wp, H or W below 1, H * W > INT_MAX, labels NULL.
 *
 * d2b_panoptic_combine: per image n, R[n] instances: scores[n] [R] fp32, classes[n] [R] int64, masks[n] [R,H,W] uint8 (any
 *   nonzero byte is "in"); labels[n] [H,W] int64 in [0, C); num_instances [N] int64 (device, NULL = R[n]; clamped to
 *   [0, R[n]]: rows at or past it are ignored).  Per image, restating panoptic_fpn.py:206-267:
 *     1. the instances ordered by ascending -score: a NaN (either sign) goes last, ties to the lower index (the reference's
 *        argsort is not stable; this is the documented tie rule).  Not the NMS order, where NaN comes first;
 *     2. walked in that order, stopping at the first with (double)score < instances_score_thresh (a NaN never stops it);
 *     3. area = the instance's nonzero pixels; area == 0: skipped, no id consumed;
 *     4. inter = its pixels already painted; (double)inter / (double)area > overlap_threshold: skipped;
 *     5. otherwise the next id (from 1) paints its unpainted pixels, and the record (id, isthing 1, classes[i], instance i,
 *        area = the pixels painted; score = scores[i]) is written;
 *     6. then every label present anywhere in labels[n], ascending, label 0 skipped: a = its still unpainted pixels;
 *        (double)a < stuff_area_thresh: skipped; otherwise the next id paints them, record (id, isthing 0, label, -1, a;
 *        score 0).  With stuff_area_thresh <= 0 a present but fully covered label becomes a zero-area segment.
 *   Outputs: panoptic[n] [H,W] int32, every pixel written (0 = unassigned); num_segments [N] int64; seg_info [N,S,5] int64
 *   (id, isthing, category, instance, area) and seg_score [N,S] fp32, S = max_n R[n] + C slots, those past num_segments[n]
 *   zero; status [N] int32: D2B_PANOPTIC_STATUS_BAD_LABEL when a label of the image is outside [0, C) (the image's other
 *   outputs are then unspecified).  Integer decisions, double threshold comparisons: bitwise reproducible.
 *   workspace: d2b_panoptic_workspace_bytes(img, N, C) bytes, 256-byte aligned, no initialisation needed (0 for an invalid
 *   description).  Four launches: bit-packing of the masks, one CTA per image for the ordered walk (the instances are ranked
 *   by counting, hence R[n] <= D2B_PANOPTIC_MAX_INSTANCES), the stuff histogram of the unpainted pixels, the stuff ids.
 *   Checks, in order (nothing is launched before all pass):
 *     1. D2B_EINVAL: img NULL, N < 0 or N > D2B_MAX_IMAGES, C < 1 or C > D2B_PANOPTIC_MAX_CLASSES.
 *     2. N == 0: D2B_OK.
 *     3. D2B_EINVAL: per image H or W below 1, H * W > INT_MAX, R < 0 or R > D2B_PANOPTIC_MAX_INSTANCES, labels or panoptic
 *        NULL, or, when R > 0, scores, classes or masks NULL; num_segments, seg_info, seg_score, status or workspace NULL;
 *        workspace not 256-byte aligned.
 *     4. D2B_EWORKSPACE: workspace_bytes below d2b_panoptic_workspace_bytes(img, N, C). */
#define D2B_PANOPTIC_MAX_INSTANCES 4096
#define D2B_PANOPTIC_MAX_CLASSES 1024
#define D2B_PANOPTIC_STATUS_BAD_LABEL 1
typedef struct {
  int h[D2B_MAX_IMAGES], w[D2B_MAX_IMAGES];  /* crop of the logits */
  int H[D2B_MAX_IMAGES], W[D2B_MAX_IMAGES];  /* output size */
  int64_t* labels[D2B_MAX_IMAGES];
} d2b_sem_seg_images;
typedef struct {
  int R[D2B_MAX_IMAGES], H[D2B_MAX_IMAGES], W[D2B_MAX_IMAGES];
  const float* scores[D2B_MAX_IMAGES];
  const int64_t* classes[D2B_MAX_IMAGES];
  const uint8_t* masks[D2B_MAX_IMAGES];
  const int64_t* labels[D2B_MAX_IMAGES];
  int32_t* panoptic[D2B_MAX_IMAGES];
} d2b_panoptic_images;
int d2b_sem_seg_labels(const void* logits, int dtype, int N, int C, int Hp, int Wp, const d2b_sem_seg_images* img,
                       void* stream);
size_t d2b_panoptic_workspace_bytes(const d2b_panoptic_images* img, int N, int C);
int d2b_panoptic_combine(const d2b_panoptic_images* img, int N, int C, const int64_t* num_instances,
                         double overlap_threshold, double stuff_area_thresh, double instances_score_thresh,
                         int64_t* num_segments, int64_t* seg_info, float* seg_score, int* status, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---- Semantic segmentation loss: bilinear upsampling fused into the pixel cross-entropy ------------------------------
 * Replaces SemSegFPNHead.losses (modeling/meta_arch/semantic_seg.py:255-267), the "cross_entropy" losses of
 * DeepLabV3PlusHead / DeepLabV3Head and DeepLabCE (projects/DeepLab/deeplab/loss.py) as Panoptic-DeepLab's semantic head
 * uses it: F.interpolate(logits.float(), scale_factor=stride, mode="bilinear", align_corners=False) followed by the
 * per-pixel cross-entropy, without storing the [N,C,H,W] upsampled map or its log_softmax.
 *   logits [N,C,Hp,Wp] of `dtype` (D2B_F32 / D2B_F16 / D2B_BF16, read in place, each value converted to fp32 first);
 *   H = Hp * stride, W = Wp * stride, 1 <= stride <= D2B_SEMSEG_MAX_STRIDE.  Every upsampled value is bitwise PyTorch's
 *   CUDA upsample_bilinear2d with the scale factor's source scale (float)(1.0 / stride) (not h / H); stride 1 is a copy.
 *   targets [N,H,W] int64: a pixel equal to ignore_value (any int64) is skipped; another value outside [0, C) sets
 *   D2B_SEMSEG_STATUS_BAD_LABEL in status and is skipped as well (the reference raises; the loss is then unspecified).
 *   Per valid pixel p: lse(p) = logsumexp_c v_c(p), loss(p) = lse(p) - v_target(p).  As in F.log_softmax, lse(p) is NaN
 *   when some v_c(p) is NaN or +inf, and so are loss(p) and every gradient term of p; a -inf v_c(p) adds nothing to the
 *   sum (a -inf v_target(p) gives loss(p) = +inf).
 * reduction D2B_SEMSEG_MEAN (nn.CrossEntropyLoss(reduction="mean", ignore_index)): loss_sum = sum of loss(p) over the valid
 *   pixels; weights must be NULL.  The caller's loss is loss_sum / count (NaN with no valid pixel, as torch).
 * reduction D2B_SEMSEG_TOP_K (DeepLabCE with top_k_percent_pixels in [0, 1], no class weight): the per-pixel values
 *   x(p) = loss(p) (0 on ignored pixels), times weights[p] when weights [N,H,W] fp32 is given; k = (int64)(top_k_percent_pixels
 *   * N*H*W), as Python's int(); the caller's loss is loss_sum / k.
 *     top_k_percent_pixels == 1.0: loss_sum = the sum of every x(p), no selection (DeepLabCE's mean over all pixels).
 *     Otherwise loss_sum = the sum of the k largest x(p): a radix select over an order-preserving uint32 image of the values
 *     (every NaN above +inf, as torch.topk orders them; -0.0 == +0.0) finds the k-th largest t, loss_sum = sum_{x > t} x +
 *     (k - #{x > t}) * t.  Pixels tied at t are taken in ascending flat index (the reference's choice among ties is
 *     unspecified; it changes only the gradient of the tied pixels).  selected [N,H,W] uint8 receives 1 for the k pixels
 *     taken.  k == 0: loss_sum 0, nothing selected.
 * Forward outputs (device, no host read): lse [N,H,W] fp32 (0 on skipped pixels), loss_sum [1] fp32, count [1] int64 = the
 *   valid pixels, status [1] int32; selected as above.  Reductions are per-CTA partials added in a fixed order by a
 *   finish launch (no float atomics): bitwise reproducible.  workspace: d2b_sem_seg_loss_workspace_bytes(...) bytes,
 *   256-byte aligned, no initialisation needed; the query makes no CUDA call and returns 0 for arguments that fail rule 1
 *   below (weights aside), otherwise at least 256.  Launches: 2 (MEAN, TOP_K 1.0) or 8 (TOP_K below 1.0).
 * Backward: grad_sum [1] fp32 (device) = d loss / d loss_sum.  grad_logits [N,C,Hp,Wp] of `dtype` is written once, every
 *   element (no zero fill, no atomics): each low-res logit gathers, in a fixed order, over the output pixels p whose two
 *   row taps and two column taps reach it, tap weight * g(p) * (exp(v_c(p) - lse(p)) - [target(p) = c]), with v_c(p)
 *   recomputed and g(p) = grad_sum * weights[p] (1 when NULL) on valid pixels whose selected[p] is 1 (all when NULL), 0
 *   elsewhere.  At the last row / column both taps fall on the same logit and both weights go to it.  Pass the forward's
 *   weights and selected.  One launch.  No host synchronisation in either direction: capturable in a CUDA graph.
 * Arguments are checked in this order, and nothing is launched or written before every check has passed:
 *   forward:  1. D2B_EINVAL: N < 0 or N > 65535, C < 1, Hp < 1, Wp < 1, stride outside 1..D2B_SEMSEG_MAX_STRIDE, dtype
 *                not a D2B_F* code, N*H*W > INT_MAX - 1024 or C*Hp*Wp > INT_MAX; reduction not a D2B_SEMSEG_* code; MEAN
 *                with weights; TOP_K with top_k_percent_pixels NaN or outside [0, 1].
 *             2. D2B_EINVAL: loss_sum, count or status NULL; when N > 0, logits, targets or lse NULL; TOP_K below 1.0 with
 *                selected NULL.
 *             3. D2B_EINVAL: workspace NULL or not 256-byte aligned; D2B_EWORKSPACE: workspace_bytes below the query.
 *             4. The launches; N == 0 runs the finish alone (loss_sum 0, count 0, status 0).
 *   backward: 1. D2B_EINVAL: the shape and dtype rules of the forward's rule 1.
 *             2. N == 0: D2B_OK, nothing written.
 *             3. D2B_EINVAL: logits, targets, lse, grad_sum or grad_logits NULL. */
#define D2B_SEMSEG_MEAN 0
#define D2B_SEMSEG_TOP_K 1
#define D2B_SEMSEG_MAX_STRIDE 32
#define D2B_SEMSEG_STATUS_BAD_LABEL 1
size_t d2b_sem_seg_loss_workspace_bytes(int N, int C, int Hp, int Wp, int stride, int dtype, int reduction,
                                        double top_k_percent_pixels);
int d2b_sem_seg_loss_forward(const void* logits, int dtype, int N, int C, int Hp, int Wp, int stride,
                             const int64_t* targets, int64_t ignore_value, int reduction, double top_k_percent_pixels,
                             const float* weights, float* lse, uint8_t* selected, float* loss_sum, int64_t* count,
                             int* status, void* workspace, size_t workspace_bytes, void* stream);
int d2b_sem_seg_loss_backward(const void* logits, int dtype, int N, int C, int Hp, int Wp, int stride,
                              const int64_t* targets, int64_t ignore_value, const float* weights, const uint8_t* selected,
                              const float* lse, const float* grad_sum, void* grad_logits, void* stream);

/* ---- Box-branch training losses: RPN / RRPN, RetinaNet, Fast R-CNN ------------------------------------------------
 * Replace RPN.losses (proposal_generator/rpn.py:366-429), RetinaNet.losses (meta_arch/retinanet.py:160-210) and
 * FastRCNNOutputLayers.losses / box_reg_loss / _log_classification_stats (roi_heads/fast_rcnn.py:88-115, 307-352, 424-463)
 * for all images at once, without the reference's host reads (.item(), nonzero, get_deltas' assertion).
 * Box targets: Box2BoxTransform.get_deltas (modeling/box_regression.py:43-76) for box_dim 4 (x1, y1, x2, y2), and
 * Box2BoxTransformRotated.get_deltas (:145-180) for box_dim 5 (cx, cy, w, h, angle_deg); weights[box_dim] (HOST).
 * Regression, summed: loss_type D2B_LOSS_SMOOTH_L1 = fvcore smooth_l1_loss with `beta` (|d| for beta < 1e-5) of the deltas
 * against the get_deltas targets; D2B_LOSS_GIOU (box_dim 4 only) = fvcore giou_loss (eps 1e-7) of the boxes decoded by
 * Box2BoxTransform.apply_deltas (:78-116, dw / dh clamped at scale_clamp; the gradient passes the clamp at equality, is 0
 * above it) against the GT boxes.  Predictions (logits, scores, deltas) are
 * elements of `dtype` (D2B_F32 / D2B_F16 / D2B_BF16) read in place, fp32 arithmetic; boxes are fp32.
 * Reductions are per-CTA partials added in a fixed order by a second launch (no float atomics): bitwise reproducible.
 * status [1] int32, OR of D2B_LOSS_STATUS_*: INVALID_BOX when a source box width is not > 0 (the reference's assertion in
 * get_deltas: every anchor for the dense losses, the foreground proposals for Fast R-CNN); INVALID_CLASS when a Fast R-CNN
 * gt class is outside [0, K] or a dense int64 label outside [-1, K] (int8: outside {-1, 0, 1}); INVALID_BOX_ORDER (GIoU)
 * when a decoded or GT box of a regressed row fails fvcore's x2 >= x1 and y2 >= y1 (NaN included); with GIoU the
 * get_deltas assertion does not apply, as in the reference (nor with LINEAR_GIOU).  No host synchronisation, static
 * shapes: capturable in a CUDA graph.
 *
 * Dense: lv->logits[l] [N,R_l,K] (16-byte aligned), lv->deltas[l] [N,R_l,box_dim] -- the reference's per-level lists, no cat;
 *   anchors [R,box_dim] shared by the images (R = sum R_l), gt_boxes [N,R,box_dim] matched GT boxes, labels [N,R]:
 *     D2B_LABELS_I8   int8 {-1, 0, 1} (RPN gt_labels), K must be 1: target = label;
 *     D2B_LABELS_I64  int64 {-1, 0..K-1, K = background} (RetinaNet gt_labels): target = one_hot(label)[:K].
 *   Classification: fvcore sigmoid_focal_loss(gamma, alpha; alpha < 0 = no weighting) summed over the rows with label >= 0;
 *   gamma = 0 and alpha < 0 is binary_cross_entropy_with_logits.  Rows with label -1 are not read.  Regression over the
 *   positive rows (I8: label 1, I64: 0 <= label < K).
 *   D2B_LOSS_LINEAR_GIOU (box_dim 4, D2B_LABELS_I64) is FCOS.losses + compute_ctrness_targets (meta_arch/fcos.py:193-251):
 *   the regression is fvcore giou_loss of the deltas decoded by Box2BoxTransformLinear (relu(deltas) * stride; the relu
 *   gradient is 0 at <= 0), and the positive rows add the centerness term: binary_cross_entropy_with_logits of
 *   lv->ctr[l] [N,R_l] (`dtype`, read in place) against sqrt((min(l,r) / max(l,r)) * (min(t,b) / max(t,b))),
 *   (l,t,r,b) = Box2BoxTransformLinear.get_deltas(anchor, gt box).  weights and scale_clamp are not read (weights may be
 *   NULL).
 *   Outputs (device): sums [3] fp32 = classification, regression, centerness (0 unless LINEAR_GIOU); counts [2] int64 =
 *   num_pos, num_neg (I8: label 0, I64: label K); status [1].  workspace: d2b_dense_loss_workspace_bytes(lv, N, K, dtype)
 *   bytes, 16-byte aligned.
 *   Backward: grad_sums [3] (device) = d loss / d sums (the third is read with LINEAR_GIOU only); lv->grad_logits[l]
 *   (16-byte aligned), lv->grad_deltas[l] and, with LINEAR_GIOU, lv->grad_ctr[l] [N,R_l] are fully written in `dtype` (0 on
 *   ignored / non-positive rows).
 * Fast R-CNN: scores [R,K+1], deltas [R,kreg*box_dim] (kreg = K class-specific, gathered at the gt class, or 1), proposals
 *   and gt_boxes [R,box_dim] fp32, gt_classes [R] int64.  Outputs (device): sums [2] fp32 = cross_entropy over all rows,
 *   regression over the foreground rows (0 <= class < K); counts [4] int64 = num_fg, num_accurate, fg_num_accurate,
 *   num_false_negative of _log_classification_stats (argmax: first index on ties, NaN wins); status [1].
 *   workspace: d2b_frcnn_loss_workspace_bytes(R) bytes, 16-byte aligned.  Backward: grad_sums [2] (device) = d loss / d sums;
 *   grad_scores / grad_deltas fully written.
 * Workspace queries (host only, no CUDA call): d2b_dense_loss_workspace_bytes returns 0 for N < 0, K < 1 or a dtype that is
 *   not a D2B_F* code, then for a level table that fails the forward's rule 2 below (without the ctr rules, which need the
 *   loss type); d2b_frcnn_loss_workspace_bytes returns 0 for R <= 0.
 * Arguments are checked in this order, and nothing is launched or written before every check has passed:
 *   dense:  1. D2B_EINVAL: N < 0, K < 1, box_dim neither 4 nor 5, dtype not a D2B_F* code, weights NULL without
 *              LINEAR_GIOU; label_kind not a D2B_LABELS_* code, or I8 with K != 1; gamma < 0, beta < 0 or either NaN, alpha
 *              NaN; loss_type not a D2B_LOSS_* type, GIOU with box_dim 5, LINEAR_GIOU with box_dim 5 or I8 labels.
 *           2. D2B_EINVAL: the level table -- lv NULL, num_levels outside 1..D2B_MAX_LEVELS, R_l < 0, R > INT_MAX; on a
 *              level with rows (N * R_l > 0) logits[l] or deltas[l] NULL or logits[l] not 16-byte aligned, in the backward
 *              grad_logits[l] or grad_deltas[l] NULL or grad_logits[l] not 16-byte aligned; with LINEAR_GIOU ctr[l] NULL
 *              on a level with rows, in the backward grad_ctr[l] too; with another loss type ctr[l] or grad_ctr[l] set.
 *           3. D2B_EINVAL: when there are rows (N * R > 0), anchors, gt_boxes or labels NULL.
 *           4. D2B_EINVAL: more than INT_MAX CTAs.
 *           forward:  5. D2B_EINVAL: sums, counts or status NULL.
 *                     6. When there are rows, D2B_EINVAL for a NULL or not 16-byte aligned workspace, then D2B_EWORKSPACE
 *                        when workspace_bytes is below the query's size.
 *                     7. The loss launch (when there are rows), then the finish, which writes the outputs even
 *                        without rows.
 *           backward: 5. D2B_EINVAL: grad_sums NULL.
 *                     6. No row: D2B_OK, nothing written.
 *   frcnn:  1. D2B_EINVAL: R < 0, K < 1, kreg neither 1 nor K, box_dim neither 4 nor 5, dtype not a D2B_F* code, weights
 *              NULL; beta < 0 or NaN, kreg * box_dim > INT_MAX / 2, loss_type neither SMOOTH_L1 nor GIOU, GIOU with
 *              box_dim 5.
 *           2. D2B_EINVAL: when R > 0, scores, deltas, proposals, gt_boxes or gt_classes NULL.
 *           forward:  3. D2B_EINVAL: sums, counts or status NULL.
 *                     4. When R > 0, D2B_EINVAL for a NULL or not 16-byte aligned workspace, then D2B_EWORKSPACE when
 *                        workspace_bytes is below d2b_frcnn_loss_workspace_bytes(R).
 *                     5. The loss launch (when R > 0), then the finish, which writes the outputs even for R = 0.
 *           backward: 3. R == 0: D2B_OK, nothing written.
 *                     4. D2B_EINVAL: grad_sums, grad_scores or grad_deltas NULL. */
#define D2B_LABELS_I8 0
#define D2B_LABELS_I64 1
#define D2B_LOSS_STATUS_INVALID_BOX 1
#define D2B_LOSS_STATUS_INVALID_CLASS 2
#define D2B_LOSS_STATUS_INVALID_BOX_ORDER 4
#define D2B_LOSS_SMOOTH_L1 0
#define D2B_LOSS_GIOU 1
#define D2B_LOSS_LINEAR_GIOU 2 /* dense only */
typedef struct {
  int num_levels;
  const void* logits[D2B_MAX_LEVELS];
  const void* deltas[D2B_MAX_LEVELS];
  void* grad_logits[D2B_MAX_LEVELS];
  void* grad_deltas[D2B_MAX_LEVELS];
  const void* ctr[D2B_MAX_LEVELS];   /* LINEAR_GIOU only: centerness logits [N,R_l] */
  void* grad_ctr[D2B_MAX_LEVELS];
  int R[D2B_MAX_LEVELS];
} d2b_dense_loss_levels;
size_t d2b_dense_loss_workspace_bytes(const d2b_dense_loss_levels* lv, int N, int K, int dtype);
int d2b_dense_loss_forward(const d2b_dense_loss_levels* lv, int N, int K, int box_dim, int dtype, const float* anchors,
                           const float* gt_boxes, const void* labels, int label_kind, float gamma, float alpha, float beta,
                           int loss_type, float scale_clamp, const float* weights, float* sums, int64_t* counts,
                           int* status, void* workspace, size_t workspace_bytes, void* stream);
int d2b_dense_loss_backward(const d2b_dense_loss_levels* lv, int N, int K, int box_dim, int dtype, const float* anchors,
                            const float* gt_boxes, const void* labels, int label_kind, float gamma, float alpha, float beta,
                            int loss_type, float scale_clamp, const float* weights, const float* grad_sums, void* stream);
size_t d2b_frcnn_loss_workspace_bytes(int R);
int d2b_frcnn_loss_forward(const void* scores, const void* deltas, int R, int K, int kreg, int box_dim, int dtype,
                           const float* proposals, const float* gt_boxes, const int64_t* gt_classes, float beta,
                           int loss_type, float scale_clamp, const float* weights, float* sums, int64_t* counts,
                           int* status, void* workspace, size_t workspace_bytes, void* stream);
int d2b_frcnn_loss_backward(const void* scores, const void* deltas, int R, int K, int kreg, int box_dim, int dtype,
                            const float* proposals, const float* gt_boxes, const int64_t* gt_classes, float beta,
                            int loss_type, float scale_clamp, const float* weights, const float* grad_sums,
                            void* grad_scores, void* grad_deltas, void* stream);

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
 * threshold >= 0, else (uint8)(v*255).  A box whose sample coordinates are not finite (zero or negative extent where a pixel
 * centre meets x0, NaN or infinite corners) gives v = 0 there.  Any N >= 0.
 *   1. D2B_OK without a launch when N, H or W is 0.
 *   2. D2B_EINVAL: masks, boxes or out NULL, N, H or W below 0, M below 1 (the packed form: also threshold below 0 or NaN).
 *   3. D2B_EUNSUPPORTED: M > 64, or H * W >= 2^30. */
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
