// Batched anchor / proposal matching for the training targets (SURVEY.md 8f): pairwise IoU + Matcher + the label / box /
// class gathers of
//   RPN.label_and_sample_anchors          (detectron2/modeling/proposal_generator/rpn.py:307-363, up to the sampling)
//   RRPN.label_and_sample_anchors         (proposal_generator/rrpn.py:151-195)
//   RetinaNet.label_anchors               (meta_arch/retinanet.py:213-255)
//   ROIHeads.label_and_sample_proposals   (roi_heads/roi_heads.py:220-302, with proposal_append_gt; up to the sampling)
//   RROIHeads.label_and_sample_proposals  (roi_heads/rotated_fast_rcnn.py:218-270)
//   CascadeROIHeads._match_and_label_boxes (roi_heads/cascade_rcnn.py:209-256)
// for all images in one launch sequence, without the G x A IoU matrix the reference materialises per image:
//   one zero-fill launch (status + per-GT maxima) -> match_kernel -> match_label_kernel.
//
//   match_kernel        one thread per prediction, the image's GT boxes staged through shared memory in tiles: the IoU with
//                       every GT, the max and FIRST argmax over GT (torch's max(dim=0)), "IoU < 0 or NaN" into the image's
//                       status (the reference's `assert torch.all(matrix >= 0)`), and the per-GT maximum over predictions
//                       published with atomicMax on the float bits (valid IoUs are >= 0 and never -0, so the bit order is
//                       the value order; the maxima start at 0, so the zero pairs -- nearly all of them -- publish nothing);
//   match_label_kernel  the threshold labels (fp32 compares, later intervals win, as Matcher.__call__), the low-quality
//                       matches (set_low_quality_matches_: every prediction whose IoU with GT g equals g's maximum, ties
//                       included; only GTs whose maximum is <= the prediction's best IoU can qualify, and only those pairs
//                       are recomputed -- same code, same bits; a maximum of 0 qualifies every prediction without a
//                       recomputation, the reference's quirk for a GT that overlaps nothing), Boxes.inside_box
//                       (structures/boxes.py:245-262) after the matcher, then the int8 labels, the gathered GT boxes and
//                       the classes (1 -> gt_classes[match], 0 -> num_classes, -1 -> -1; an image without GT: num_classes).
//
// The box type is a template policy (XyxyBox: pairwise_iou of structures/boxes.py:312-358 op for op; RotBox: the rotated IoU
// of nms.cu; boxes.cuh).  Compiled with -fmad=false like nms.cu / postproc.cu: bit-exact IoUs.
//
// d2b_fcos_assign (FCOS._match_anchors + label_anchors, meta_arch/fcos.py:97-191) shares the GT tiling: one launch,
// fcos_assign_kernel, one thread per (image, point), no G x R matrix; the quality and its argmax are bit-exact.
#include <climits>

#include "boxes.cuh"
#include "common.cuh"

namespace {

constexpr int kThreads = 256;  // predictions per CTA
constexpr int kTile = 256;     // GT boxes staged per shared-memory tile

struct MatchArgs {
  const float* gt;               // [N, Gmax, D]
  const long long* gt_count;     // [N]
  int Gmax;
  const float* pred;             // [A, D] (pred_stride 0) or [N, pred_stride, D]
  long long pred_stride;         // rows between images of `pred`
  const long long* pred_count;   // [N] or NULL (= Pmax)
  int Pmax, P;                   // P = output rows per image = Pmax (+ Gmax with append_gt)
  int append_gt, low_quality, boundary;
  int nthr;
  float thr[D2B_MATCH_MAX_THRESHOLDS];
  int lab[D2B_MATCH_MAX_THRESHOLDS + 1];
  const float* image_hw;         // [N, 2] (h, w)
  double boundary_thresh;
  const long long* gt_classes;   // [N, Gmax] or NULL
  long long num_classes;
  long long* matches;            // [N, P]
  signed char* labels;           // [N, P]
  float* out_boxes;              // [N, P, D] or NULL
  long long* classes;            // [N, P] or NULL
  int* status;                   // [N]
  unsigned* best;                // [N, Gmax] per-GT maximum IoU (float bits), zeroed
  float* mval;                   // [N, P] per-prediction maximum IoU
};

struct ImageRows {
  int G, pc, valid;
};

__device__ __forceinline__ ImageRows image_rows(const MatchArgs& a, int n) {
  ImageRows r;
  r.G = (int)min(max(a.gt_count[n], 0LL), (long long)a.Gmax);
  r.pc = a.pred_count ? (int)min(max(a.pred_count[n], 0LL), (long long)a.Pmax) : a.Pmax;
  r.valid = r.pc + (a.append_gt ? r.G : 0);
  return r;
}

// Row p of image n: a prediction, or (proposal_append_gt, proposal_utils.py:184-205) GT p - pc after the image's predictions.
template <class Box>
__device__ __forceinline__ void load_row(const MatchArgs& a, int n, int p, int pc, float* box) {
  const float* src = p < pc ? a.pred + ((size_t)n * a.pred_stride + p) * Box::D
                            : a.gt + ((size_t)n * a.Gmax + (p - pc)) * Box::D;
#pragma unroll
  for (int q = 0; q < Box::D; ++q) box[q] = src[q];
}

template <class Box>
__device__ __forceinline__ void stage_gt(const MatchArgs& a, int n, int g0, int ng, float* __restrict__ s_gt) {
  const float* src = a.gt + ((size_t)n * a.Gmax + g0) * Box::D;
  for (int t = threadIdx.x; t < ng * Box::D; t += kThreads) s_gt[t] = src[t];
}

template <class Box>
__global__ void __launch_bounds__(kThreads) match_kernel(const MatchArgs a) {
  constexpr int D = Box::D;
  __shared__ float s_gt[kTile * D];
  __shared__ unsigned s_best[kTile];
  const int n = blockIdx.y, tid = threadIdx.x;
  const ImageRows r = image_rows(a, n);
  const int p0 = blockIdx.x * kThreads;
  if (p0 >= r.valid || r.G == 0) return;  // whole CTA: match_label_kernel writes these rows
  const int p = p0 + tid;
  const bool live = p < r.valid;
  float box[D];
  if (live) load_row<Box>(a, n, p, r.pc, box);
  float best = -1.f;
  int arg = 0, bad = 0;
  for (int g0 = 0; g0 < r.G; g0 += kTile) {
    const int ng = min(kTile, r.G - g0);
    __syncthreads();  // previous tile consumed
    stage_gt<Box>(a, n, g0, ng, s_gt);
    for (int t = tid; t < ng; t += kThreads) s_best[t] = 0u;
    __syncthreads();
    if (live) {
      for (int j = 0; j < ng; ++j) {
        const float v = Box::iou(s_gt + j * D, box);
        if (v > best) {  // strict: the first GT wins ties
          best = v;
          arg = g0 + j;
        }
        bad |= (v >= 0.f) ? 0 : 1;
        if (v > 0.f) atomicMax(&s_best[j], __float_as_uint(v));
      }
    }
    __syncthreads();
    for (int t = tid; t < ng; t += kThreads)
      if (s_best[t]) atomicMax(&a.best[(size_t)n * a.Gmax + g0 + t], s_best[t]);
  }
  if (live) {
    const size_t o = (size_t)n * a.P + p;
    a.mval[o] = best;
    a.matches[o] = arg;
  }
  if (__syncthreads_or(bad) && tid == 0) atomicOr(&a.status[n], D2B_MATCH_STATUS_INVALID_IOU);
}

template <class Box>
__global__ void __launch_bounds__(kThreads) match_label_kernel(const MatchArgs a) {
  constexpr int D = Box::D;
  __shared__ float s_gt[kTile * D];
  __shared__ float s_best[kTile];
  const int n = blockIdx.y, tid = threadIdx.x;
  const ImageRows r = image_rows(a, n);
  const int p = blockIdx.x * kThreads + tid;
  const bool live = p < r.valid;
  float box[D];
  if (live) load_row<Box>(a, n, p, r.pc, box);
  const size_t o = (size_t)n * a.P + p;
  long long m = 0;
  int lab = -1;
  float v = 0.f;
  if (live) {
    if (r.G == 0) {
      lab = a.lab[0];  // Matcher on an empty matrix: matches 0, labels[0]
    } else {
      m = a.matches[o];
      v = a.mval[o];
      lab = 1;
      for (int i = 0; i <= a.nthr; ++i) {  // (v >= low) & (v < high) over [-inf, thr..., inf]; later intervals win
        const bool ge = i == 0 || v >= a.thr[i - 1];
        const bool lt = i == a.nthr || v < a.thr[i];
        if (ge && lt) lab = a.lab[i];
      }
    }
  }
  // set_low_quality_matches_: only predictions that are not positive yet can change
  bool need = a.low_quality && live && r.G > 0 && lab != 1;
  if (__syncthreads_or(need)) {
    for (int g0 = 0; g0 < r.G; g0 += kTile) {
      const int ng = min(kTile, r.G - g0);
      __syncthreads();
      stage_gt<Box>(a, n, g0, ng, s_gt);
      for (int t = tid; t < ng; t += kThreads) s_best[t] = __uint_as_float(a.best[(size_t)n * a.Gmax + g0 + t]);
      __syncthreads();
      for (int j = 0; need && j < ng; ++j) {
        const float bg = s_best[j];
        // IoU(g, p) <= v, so IoU(g, p) == bg needs bg <= v; bg == 0 is every IoU of g, so it needs no recomputation
        if (bg <= v && (bg == 0.f || Box::iou(s_gt + j * D, box) == bg)) {
          lab = 1;
          need = false;
        }
      }
      if (!__syncthreads_or(need)) break;
    }
  }
  if (!live) {  // rows past the image's valid count: matches 0, labels -1, zero boxes, classes -1
    if (p < a.P) {
      a.matches[o] = 0;
      a.labels[o] = -1;
      if (a.out_boxes)
#pragma unroll
        for (int q = 0; q < D; ++q) a.out_boxes[o * D + q] = 0.f;
      if (a.classes) a.classes[o] = -1;
    }
    return;
  }
  if constexpr (!Box::kRotated) {
    if (a.boundary) {  // anchors.inside_box(image_size, thresh): fp32 compares against -thresh and size + thresh
      const float ih = a.image_hw[2 * n], iw = a.image_hw[2 * n + 1];
      const float lo = (float)(-a.boundary_thresh);
      const float xhi = (float)((double)iw + a.boundary_thresh), yhi = (float)((double)ih + a.boundary_thresh);
      if (!(box[0] >= lo && box[1] >= lo && box[2] < xhi && box[3] < yhi)) lab = -1;
    }
  }
  a.matches[o] = m;
  a.labels[o] = (signed char)lab;
  if (a.out_boxes) {
    const float* src = a.gt + ((size_t)n * a.Gmax + m) * D;
#pragma unroll
    for (int q = 0; q < D; ++q) a.out_boxes[o * D + q] = r.G > 0 ? src[q] : 0.f;
  }
  if (a.classes)
    a.classes[o] = r.G == 0 ? a.num_classes
                            : (lab == 1 ? a.gt_classes[(size_t)n * a.Gmax + m] : (lab == 0 ? a.num_classes : -1LL));
}

// ---- FCOS point assignment (FCOS._match_anchors + label_anchors, meta_arch/fcos.py:97-191) -------------------------
// One thread per (image, point), the image's GT boxes staged in shared memory with their centre and 1e8 - area.  The
// quality of GT g at point p is float(centre test && inside test && scale test) * (1e8 - area_g), every value rounded in
// fp32 as the reference's tensor ops; the argmax over g is torch.max(dim=0)'s (a NaN beats every number, the first NaN
// wins, ties go to the lowest index).  Unmatched (q < 1e-5; a NaN maximum is matched) points keep GT 0's box and get
// label K, as the reference's `matched_idxs.clip(min=0)` gathers.
struct FcosArgs {
  const float* anchors;          // [R, 4]
  int R, lvl0_end, last_begin;   // points [0, lvl0_end): lower bound 0; [last_begin, R): upper bound +inf
  float radius;
  const float* gt;               // [N, Gmax, 4]
  const long long* gt_count;     // [N]
  int Gmax;
  const long long* gt_classes;   // [N, Gmax]
  long long num_classes;
  long long* matches;            // [N, R]
  long long* labels;             // [N, R]
  float* out_boxes;              // [N, R, 4]
};

constexpr int kFcosGt = 7;  // x0, y0, x1, y1, centre x, centre y, 1e8 - area

__global__ void __launch_bounds__(kThreads) fcos_assign_kernel(const FcosArgs a) {
  __shared__ float s_gt[kTile * kFcosGt];
  const int n = blockIdx.y, tid = threadIdx.x;
  const int p = blockIdx.x * kThreads + tid;
  const int G = (int)min(max(a.gt_count[n], 0LL), (long long)a.Gmax);
  const bool live = p < a.R;
  float cx = 0.f, cy = 0.f, rs = 0.f, lo = 0.f, hi = 0.f;
  if (live) {
    const float* an = a.anchors + (size_t)p * 4;
    cx = (an[0] + an[2]) / 2.f;  // Boxes.get_centers
    cy = (an[1] + an[3]) / 2.f;
    const float size = an[2] - an[0];
    rs = a.radius * size;
    lo = p < a.lvl0_end ? 0.f : size * 4.f;
    hi = p >= a.last_begin ? INFINITY : size * 8.f;
  }
  float best = -INFINITY;
  int arg = 0;
  const float* gt = a.gt + (size_t)n * a.Gmax * 4;
  for (int g0 = 0; g0 < G; g0 += kTile) {
    const int ng = min(kTile, G - g0);
    __syncthreads();  // previous tile consumed
    for (int t = tid; t < ng; t += kThreads) {
      const float* b = gt + (size_t)(g0 + t) * 4;
      float* s = s_gt + t * kFcosGt;
      s[0] = b[0];
      s[1] = b[1];
      s[2] = b[2];
      s[3] = b[3];
      s[4] = (b[0] + b[2]) / 2.f;
      s[5] = (b[1] + b[3]) / 2.f;
      s[6] = 1e8f - (b[2] - b[0]) * (b[3] - b[1]);  // 1e8 - Boxes.area()
    }
    __syncthreads();
    if (live) {
      for (int j = 0; j < ng; ++j) {
        const float* s = s_gt + j * kFcosGt;
        bool in = nan_max(fabsf(cx - s[4]), fabsf(cy - s[5])) < rs;               // centre sampling
        // pairwise_point_box_distance: (x - x0, y - y0, x1 - x, y1 - y)
        const float l = cx - s[0], t = cy - s[1], r = s[2] - cx, b = s[3] - cy;
        in = in && nan_min(nan_min(l, t), nan_min(r, b)) > 0.f;                   // inside the box
        const float m = nan_max(nan_max(l, t), nan_max(r, b));
        in = in && m > lo && m < hi;                                              // the level's scale range
        const float q = (in ? 1.f : 0.f) * s[6];
        if (q != q ? best == best : q > best) {  // GreaterOrNan, strict: the first index wins ties and NaNs
          best = q;
          arg = g0 + j;
        }
      }
    }
  }
  if (!live) return;
  const size_t o = (size_t)n * a.R + p;
  const bool matched = G > 0 && !(best < 1e-5f);
  a.matches[o] = matched ? arg : -1;
  a.labels[o] = matched ? a.gt_classes[(size_t)n * a.Gmax + arg] : a.num_classes;
  const int src = matched ? arg : 0;
#pragma unroll
  for (int q = 0; q < 4; ++q) a.out_boxes[o * 4 + q] = G > 0 ? gt[(size_t)src * 4 + q] : 0.f;
}

size_t align256(size_t b) { return (b + 255) & ~(size_t)255; }

template <class Box>
int launch(const MatchArgs& a, int N, cudaStream_t stream) {
  void* ptrs[2] = {a.best, a.status};
  size_t bytes[2] = {sizeof(unsigned) * (size_t)N * a.Gmax, sizeof(int) * (size_t)N};
  const int rc = d2b_zero_buffers(ptrs, bytes, 2, stream);
  if (rc) return rc;
  const dim3 grid((unsigned)d2b_cdiv(a.P, kThreads), (unsigned)N);
  match_kernel<Box><<<grid, kThreads, 0, stream>>>(a);
  D2B_CHECK_LAUNCH();
  match_label_kernel<Box><<<grid, kThreads, 0, stream>>>(a);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

}  // namespace

D2B_API size_t d2b_match_workspace_bytes(int N, int Gmax, int P) {
  if (N <= 0 || P <= 0) return 0;
  return align256(sizeof(unsigned) * (size_t)N * (size_t)(Gmax > 0 ? Gmax : 0)) + align256(sizeof(float) * (size_t)N * P);
}

D2B_API int d2b_match_boxes(const float* gt_boxes, const int64_t* gt_count, int N, int Gmax, const float* pred_boxes,
                            int64_t pred_image_stride, const int64_t* pred_count, int Pmax, const double* thresholds,
                            int num_thresholds, const int* labels, int flags, const float* image_hw, double boundary_thresh,
                            const int64_t* gt_classes, int64_t num_classes, int64_t* matches, int8_t* match_labels,
                            float* matched_gt_boxes, int64_t* classes, int* status, void* workspace, size_t workspace_bytes,
                            void* stream) {
  // Matcher.__init__ (modeling/matcher.py:49-57): thresholds[0] > 0, ascending, labels in {-1, 0, 1}, one more label
  if (num_thresholds < 1 || num_thresholds > D2B_MATCH_MAX_THRESHOLDS || !thresholds || !labels) return D2B_EINVAL;
  if (!(thresholds[0] > 0.0)) return D2B_EINVAL;
  for (int i = 1; i < num_thresholds; ++i)
    if (!(thresholds[i - 1] <= thresholds[i])) return D2B_EINVAL;
  for (int i = 0; i <= num_thresholds; ++i)
    if (labels[i] < -1 || labels[i] > 1) return D2B_EINVAL;
  if (flags & ~(D2B_MATCH_ROTATED | D2B_MATCH_LOW_QUALITY | D2B_MATCH_APPEND_GT)) return D2B_EINVAL;
  const bool rotated = (flags & D2B_MATCH_ROTATED) != 0, append = (flags & D2B_MATCH_APPEND_GT) != 0;
  const bool boundary = boundary_thresh >= 0.0;  // `if self.anchor_boundary_thresh >= 0` (NaN: off)
  if (N < 0 || N > 65535 || Gmax < 0 || Pmax < 0) return D2B_EINVAL;
  const long long P = (long long)Pmax + (append ? Gmax : 0);
  if (P > INT_MAX - kThreads) return D2B_EINVAL;
  if (pred_image_stride != 0 && pred_image_stride < Pmax) return D2B_EINVAL;
  if (boundary && rotated) return D2B_EINVAL;  // RRPN has no boundary rule
  if (N == 0 || P == 0) return D2B_OK;
  if (!gt_count || !matches || !match_labels || !status || !workspace) return D2B_EINVAL;
  if (Gmax > 0 && !gt_boxes) return D2B_EINVAL;
  if (Pmax > 0 && !pred_boxes) return D2B_EINVAL;
  if (boundary && !image_hw) return D2B_EINVAL;
  if (classes && Gmax > 0 && !gt_classes) return D2B_EINVAL;
  if (workspace_bytes < d2b_match_workspace_bytes(N, Gmax, (int)P)) return D2B_EINVAL;

  MatchArgs a = {};
  a.gt = gt_boxes;
  a.gt_count = (const long long*)gt_count;
  a.Gmax = Gmax;
  a.pred = pred_boxes;
  a.pred_stride = pred_image_stride;
  a.pred_count = (const long long*)pred_count;
  a.Pmax = Pmax;
  a.P = (int)P;
  a.append_gt = append;
  a.low_quality = (flags & D2B_MATCH_LOW_QUALITY) != 0;
  a.boundary = boundary;
  a.nthr = num_thresholds;
  for (int i = 0; i < num_thresholds; ++i) a.thr[i] = (float)thresholds[i];  // the tensor compares run in fp32
  for (int i = 0; i <= num_thresholds; ++i) a.lab[i] = labels[i];
  a.image_hw = image_hw;
  a.boundary_thresh = boundary_thresh;
  a.gt_classes = (const long long*)gt_classes;
  a.num_classes = num_classes;
  a.matches = (long long*)matches;
  a.labels = (signed char*)match_labels;
  a.out_boxes = matched_gt_boxes;
  a.classes = (long long*)classes;
  a.status = status;
  a.best = (unsigned*)workspace;
  a.mval = (float*)((char*)workspace + align256(sizeof(unsigned) * (size_t)N * Gmax));
  return rotated ? launch<RotBox>(a, N, (cudaStream_t)stream)
                 : launch<XyxyBox>(a, N, (cudaStream_t)stream);
}

D2B_API int d2b_fcos_assign(const float* anchors, const int* level_counts, int num_levels, const float* gt_boxes,
                            const int64_t* gt_count, int N, int Gmax, const int64_t* gt_classes, int64_t num_classes,
                            double center_sampling_radius, int64_t* matches, int64_t* labels, float* matched_gt_boxes,
                            void* stream) {
  if (num_levels < 1 || num_levels > D2B_MAX_LEVELS || !level_counts) return D2B_EINVAL;
  long long R = 0;
  for (int l = 0; l < num_levels; ++l) {
    if (level_counts[l] < 0) return D2B_EINVAL;
    R += level_counts[l];
  }
  if (R > INT_MAX - kThreads || N < 0 || N > 65535 || Gmax < 0 || num_classes < 0) return D2B_EINVAL;
  if (N == 0 || R == 0) return D2B_OK;
  if (!anchors || !gt_count || !matches || !labels || !matched_gt_boxes) return D2B_EINVAL;
  if (Gmax > 0 && (!gt_boxes || !gt_classes)) return D2B_EINVAL;
  FcosArgs a = {};
  a.anchors = anchors;
  a.R = (int)R;
  a.lvl0_end = level_counts[0];
  // upper_bound[-R_last:] = inf: with an empty last level that slice is the whole tensor
  const int last = level_counts[num_levels - 1];
  a.last_begin = last == 0 ? 0 : (int)R - last;
  a.radius = (float)center_sampling_radius;  // the python float meets an fp32 tensor: rounded to fp32
  a.gt = gt_boxes;
  a.gt_count = (const long long*)gt_count;
  a.Gmax = Gmax;
  a.gt_classes = (const long long*)gt_classes;
  a.num_classes = num_classes;
  a.matches = (long long*)matches;
  a.labels = (long long*)labels;
  a.out_boxes = matched_gt_boxes;
  const dim3 grid((unsigned)d2b_cdiv(R, kThreads), (unsigned)N);
  fcos_assign_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(a);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
