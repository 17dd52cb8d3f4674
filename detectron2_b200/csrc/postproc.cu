// Batched RPN proposal selection around the NMS (SURVEY.md 8f-2): the two data-dependent stages of
// detectron2/modeling/proposal_generator/proposal_utils.py:22-135 (find_top_rpn_proposals) and rrpn.py:20-127
// (find_top_rrpn_proposals) as fixed-capacity kernels, one CTA per image.
//
//   d2b_rpn_prepare   gather the per-level top-k candidates, clip them to the image (Boxes.clip, :112 /
//                     RotatedBoxes.clip), mark non-finite (:104-110) and too-small (:115-119) boxes as IGNORED (category -1)
//                     instead of removing them, and apply the batched-NMS coordinate offsets per image -- torchvision's
//                     level * (max coordinate + 1), or batched_nms_rotated's level * (max - min + 1) on the centres, over
//                     that image's surviving boxes, fp32 -- so that every IoU rounds like the reference's;
//   d2b_rpn_select    walks the score-ordered keep list of ONE NMS over all images and hands every image its first
//                     post_nms_topk survivors (:129) in a fixed [N, post_nms_topk] layout + a count.
//
// Together with d2b_nms (category = image * L + level, per-category bound = pre_nms_topk) the whole selection is a
// sync-free launch sequence with static shapes: capturable in a CUDA graph; the reference loops over images in Python
// with boolean indexing and one `.item()` per image.  Compiled with -fmad=false like nms.cu (bit-exact clip / offsets).
//
// The box type is a template policy (XyxyBox / RotBox, boxes.cuh) of every candidate and selection kernel in this file:
// rpn_prepare_kernel, frcnn_prepare_kernel and rpn_select_kernel.  Each entry point picks the instantiation from its
// D2B_SELECT_* flags; the rotated calls run d2b_nms with D2B_NMS_ROTATED | D2B_NMS_NO_OFFSET.
#include <climits>
#include <type_traits>

#include "boxes.cuh"
#include "common.cuh"
#include "polygon_raster.cuh"

namespace {

constexpr int kThreads = 1024;

struct RpnLevels {
  int L;
  const float* proposals[D2B_MAX_LEVELS];    // [N, A_l, Box::D]
  const int64_t* topk_idx[D2B_MAX_LEVELS];   // [N, k_l]
  const float* topk_scores[D2B_MAX_LEVELS];  // [N, k_l]
  int A[D2B_MAX_LEVELS], k[D2B_MAX_LEVELS], t0[D2B_MAX_LEVELS + 1];  // t0: prefix of k
};

__device__ __forceinline__ bool finitef(float v) { return fabsf(v) <= 3.402823466e38f; }  // false for inf and NaN

// D = 4: xyxy boxes, D = 5: rotated boxes (D2B_SELECT_ROTATED).
template <int D>
__global__ void __launch_bounds__(kThreads) rpn_select_kernel(const long long* __restrict__ keep,
                                                              const long long* __restrict__ num_keep, int T, int post_topk,
                                                              const float* __restrict__ flat_boxes,
                                                              const float* __restrict__ raw_scores,
                                                              const long long* __restrict__ cat_ids,
                                                              float* __restrict__ out_boxes, float* __restrict__ out_scores,
                                                              long long* __restrict__ out_index, long long* __restrict__ counts) {
  using Box = std::conditional_t<D == 4, XyxyBox, RotBox>;
  __shared__ int warp_tot[32];
  const int n = blockIdx.x, tid = threadIdx.x;
  const long long nk = max(0LL, *num_keep);
  int have = 0;
  for (long long j0 = 0; j0 < nk && have < post_topk; j0 += kThreads) {
    const long long j = j0 + tid;
    long long kidx = -1;
    int mine = 0;
    if (j < nk) {
      kidx = keep[j];
      mine = (kidx / T == n && cat_ids[kidx] >= 0) ? 1 : 0;
    }
    int total;
    __syncthreads();  // the previous scan is done reading warp_tot
    const int rank = have + block_exclusive_scan(mine, warp_tot, total);
    if (mine && rank < post_topk) {
      const size_t o = (size_t)n * post_topk + rank;
      store_box(out_boxes + o * D, load_box_aligned<Box>(flat_boxes + (size_t)kidx * D));
      out_scores[o] = raw_scores[kidx];
      out_index[o] = kidx;
    }
    have += total;
  }
  const int cnt = min(have, post_topk);
  for (int r = cnt + tid; r < post_topk; r += kThreads) {  // deterministic padding
    const size_t o = (size_t)n * post_topk + r;
    store_box(out_boxes + o * D, zero_box<Box>());
    out_scores[o] = 0.f;
    out_index[o] = 0;
  }
  if (tid == 0) counts[n] = cnt;
}

}  // namespace

namespace {

// A flag bit the entry point does not take (`allowed`), SEG_PER_IMAGE without ROTATED, or NO_OFFSETS with it.
bool bad_flags(int flags, int allowed) {
  const bool rot = (flags & D2B_SELECT_ROTATED) != 0;
  return (flags & ~allowed) != 0 || ((flags & D2B_SELECT_SEG_PER_IMAGE) && !rot) || ((flags & D2B_SELECT_NO_OFFSETS) && rot);
}

bool misaligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) != 0; }  // xyxy boxes: float4 access

}  // namespace

D2B_API int d2b_rpn_select(const int64_t* keep, const int64_t* num_keep, int N, int T, int post_nms_topk, int flags,
                           const float* flat_boxes, const float* raw_scores, const int64_t* cat_ids, float* out_boxes,
                           float* out_scores, int64_t* out_index, int64_t* counts, void* stream) {
  const bool rot = (flags & D2B_SELECT_ROTATED) != 0;
  if (bad_flags(flags, D2B_SELECT_ROTATED) || N < 0 || T < 0 || post_nms_topk < 0) return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  if (!counts) return D2B_EINVAL;
  if (T == 0 || post_nms_topk == 0) {
    D2B_CUDA(cudaMemsetAsync(counts, 0, sizeof(int64_t) * N, (cudaStream_t)stream));
    return D2B_OK;
  }
  if (!keep || !num_keep || !flat_boxes || !raw_scores || !cat_ids || !out_boxes || !out_scores || !out_index) return D2B_EINVAL;
  if (!rot && (misaligned16(flat_boxes) || misaligned16(out_boxes))) return D2B_EINVAL;
  const auto kernel = rot ? rpn_select_kernel<5> : rpn_select_kernel<4>;
  kernel<<<N, kThreads, 0, (cudaStream_t)stream>>>((const long long*)keep, (const long long*)num_keep, T, post_nms_topk,
                                                   flat_boxes, raw_scores, (const long long*)cat_ids, out_boxes, out_scores,
                                                   (long long*)out_index, (long long*)counts);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// ================================================================================================ Fast R-CNN / dense-head candidates
// The candidate stages of the two inference post-processors that sit on the same NMS (SURVEY.md 8f-2), as fixed-capacity
// kernels with one CTA per image; d2b_rpn_select above then hands every image its first `topk` survivors.
//
//   d2b_frcnn_prepare   fast_rcnn_inference_single_image (detectron2/modeling/roi_heads/fast_rcnn.py:117-173) up to the NMS:
//                       rows with a non-finite box or score are dropped (:137-140), the (row, class) pairs with
//                       score > score_thresh (:150-154) are written IN ROW-MAJOR ORDER (the order `nonzero()` gives the
//                       reference; it decides ties inside NMS) by an ordered block compaction -- no nonzero(), no sync --
//                       with their box clipped to the image (:146-147) and torchvision's batched-NMS coordinate offsets.
//   d2b_dense_prepare   DenseDetector._decode_per_level_predictions (meta_arch/dense_detector.py:186-235) after the per-level
//                       top-k: Box2BoxTransform.apply_deltas (box_regression.py:78-116, same fp32 expression order) on the
//                       selected (anchor, class) pairs only, class ids, coordinate offsets.  With D2B_SELECT_LINEAR the
//                       same for FCOS (meta_arch/fcos.py:253-301): Box2BoxTransformLinear.apply_deltas
//                       (box_regression.py:275-307) as the decode.
namespace {

struct FrcnnImages {
  int N;
  int row_start[D2B_MAX_IMAGES + 1];
};

__device__ __forceinline__ float block_max(float v, float* s_red, float* s_out) {
  const int tid = threadIdx.x;
  for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();  // s_red reuse
  if ((tid & 31) == 0) s_red[tid >> 5] = v;
  __syncthreads();
  if (tid < 32) {
    v = s_red[tid];
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    if (tid == 0) *s_out = v;
  }
  __syncthreads();
  return *s_out;
}

// Box = RotBox: rotated_fast_rcnn.py:84-122, the same steps on RotatedBoxes, with `seg_per_image` for thresholds that IoU 0
// passes: every candidate of the image in one NMS segment.
template <class Box>
__global__ void __launch_bounds__(kThreads) frcnn_prepare_kernel(const FrcnnImages I, const float* __restrict__ boxes,
                                                                 const float* __restrict__ scores, int K, int kreg,
                                                                 const float* __restrict__ image_hw, float score_thresh, int cap,
                                                                 int seg_per_image, float* __restrict__ cand_boxes,
                                                                 float* __restrict__ nms_boxes, float* __restrict__ nms_scores,
                                                                 float* __restrict__ raw_scores, long long* __restrict__ cand_flat,
                                                                 long long* __restrict__ cat_ids, long long* __restrict__ n_cand,
                                                                 long long* __restrict__ row_map) {
  constexpr int D = Box::D;
  __shared__ int warp_tot[32];
  __shared__ float s_red[32];
  __shared__ float s_max, s_min;
  const int n = blockIdx.x, tid = threadIdx.x;
  const int rs = I.row_start[n], R = I.row_start[n + 1] - rs;
  const float ih = image_hw[2 * n], iw = image_hw[2 * n + 1];
  const size_t obase = (size_t)n * cap;
  int have = 0, have_rows = 0;
  float mx = -INFINITY, mn = INFINITY;
  for (int r0 = 0; r0 < R; r0 += kThreads) {
    const int r = r0 + tid;
    int cnt = 0, valid = 0;
    const float* __restrict__ srow = scores + (size_t)(rs + (r < R ? r : 0)) * (K + 1);
    const float* __restrict__ brow = boxes + (size_t)(rs + (r < R ? r : 0)) * kreg * D;
    if (r < R) {
      valid = 1;
      for (int c = 0; c <= K; ++c) valid &= finitef(srow[c]) ? 1 : 0;
      for (int c = 0; c < kreg * D; ++c) valid &= finitef(brow[c]) ? 1 : 0;
      if (valid)
        for (int c = 0; c < K; ++c) cnt += srow[c] > score_thresh ? 1 : 0;
    }
    int total, total_rows;
    __syncthreads();  // the previous scan is done reading warp_tot
    const int off = have + block_exclusive_scan(cnt, warp_tot, total);
    __syncthreads();
    const int vrank = have_rows + block_exclusive_scan(valid, warp_tot, total_rows);
    if (r < R) row_map[rs + r] = valid ? vrank : -1;  // index of the row among the valid rows (:138-140)
    if (cnt) {
      int pos = off;
      for (int c = 0; c < K && pos < cap; ++c) {
        const float sc = srow[c];
        if (!(sc > score_thresh)) continue;
        Box b = load_box<Box>(brow + (kreg == 1 ? 0 : c * D));
        b.clip(ih, iw);
        store_box(cand_boxes + (obase + pos) * D, b);
        raw_scores[obase + pos] = sc;
        nms_scores[obase + pos] = sc;
        cand_flat[obase + pos] = (long long)r * K + c;
        cat_ids[obase + pos] = (long long)n * (K + 1) + c;
        mx = fmaxf(mx, b.hi());
        if constexpr (Box::kRotated) mn = fminf(mn, b.lo());
        ++pos;
      }
    }
    have += total;
    have_rows += total_rows;
  }
  if (tid == 0) n_cand[n] = have;  // > cap: the list was truncated, the caller redoes the image
  const int live = min(have, cap);
  mx = block_max(mx, s_red, &s_max);
  if constexpr (Box::kRotated) mn = -block_max(-mn, s_red, &s_min);
  const float scale = Box::scale(live > 0, mx, mn);  // idxs * (max + 1) (torchvision) or idxs * (max - min + 1) (rotated)
  __threadfence_block();
  for (int t = tid; t < cap; t += kThreads) {
    const size_t o = obase + t;
    if (t < live) {
      Box b = load_box_aligned<Box>(cand_boxes + o * D);
      b.shift((float)(cat_ids[o] - (long long)n * (K + 1)) * scale);
      store_box(nms_boxes + o * D, b);
      if constexpr (Box::kRotated)
        if (seg_per_image) cat_ids[o] = n;
    } else {  // dead slot: ignored by the NMS kernels
      store_box(cand_boxes + o * D, zero_box<Box>());
      store_box(nms_boxes + o * D, zero_box<Box>());
      raw_scores[o] = 0.f;
      nms_scores[o] = -INFINITY;
      cand_flat[o] = 0;
      cat_ids[o] = -1;
    }
  }
}

// find_top_rpn_proposals (proposal_utils.py:60-122) / find_top_rrpn_proposals (rrpn.py:59-113) up to the NMS, one CTA
// per image: the per-level top-k gather, the finiteness check (:104-110), the box type's clip (:112) and nonempty test
// (width and height larger than min_box_size, :115-119), and the per-image batched-NMS offsets over the surviving boxes.
// Removed boxes get category -1.  use_offsets = 0 leaves nms_boxes unshifted (torchvision's batched_nms over more than
// 25 000 boxes per image); seg_per_image (rotated only) puts every surviving box of image n in NMS category n.
template <class Box>
__global__ void __launch_bounds__(kThreads) rpn_prepare_kernel(const RpnLevels P, int T, const float* __restrict__ image_hw,
                                                               float min_box_size, int use_offsets, int seg_per_image,
                                                               float* __restrict__ flat_boxes, float* __restrict__ nms_boxes,
                                                               float* __restrict__ nms_scores, float* __restrict__ raw_scores,
                                                               long long* __restrict__ cat_ids, int* __restrict__ nonfinite) {
  constexpr int D = Box::D;
  __shared__ float s_red[32];
  __shared__ float s_max, s_min;
  const int n = blockIdx.x, tid = threadIdx.x;
  const float ih = image_hw[2 * n], iw = image_hw[2 * n + 1];
  float mx = -INFINITY, mn = INFINITY;
  int bad = 0, any = 0;
  for (int t = tid; t < T; t += kThreads) {
    int l = 0;
    while (l + 1 < P.L && t >= P.t0[l + 1]) ++l;
    const int j = t - P.t0[l];
    const long long a = P.topk_idx[l][(size_t)n * P.k[l] + j];
    const float s = P.topk_scores[l][(size_t)n * P.k[l] + j];
    Box b = load_box_aligned<Box>(P.proposals[l] + ((size_t)n * P.A[l] + a) * D);
    bool fin = finitef(s);
#pragma unroll
    for (int q = 0; q < D; ++q) fin = fin && finitef(b.v[q]);
    b.clip(ih, iw);
    const bool valid = fin && Box::width(b.v) > min_box_size && Box::height(b.v) > min_box_size;
    const size_t o = (size_t)n * T + t;
    store_box(flat_boxes + o * D, valid ? b : zero_box<Box>());
    raw_scores[o] = s;
    nms_scores[o] = valid ? s : -INFINITY;
    cat_ids[o] = valid ? (long long)n * P.L + l : -1LL;
    if (valid) {
      mx = fmaxf(mx, b.hi());
      if constexpr (Box::kRotated) mn = fminf(mn, b.lo());
      any = 1;
    }
    bad |= fin ? 0 : 1;
  }
  if (bad) atomicOr(nonfinite, 1);
  any = __syncthreads_or(any);
  mx = block_max(mx, s_red, &s_max);
  if constexpr (Box::kRotated) mn = -block_max(-mn, s_red, &s_min);
  const float scale = Box::scale(any != 0, mx, mn);
  for (int t = tid; t < T; t += kThreads) {
    int l = 0;
    while (l + 1 < P.L && t >= P.t0[l + 1]) ++l;
    const size_t o = (size_t)n * T + t;
    Box b = load_box_aligned<Box>(flat_boxes + o * D);
    if (cat_ids[o] >= 0) {
      if (use_offsets) b.shift((float)l * scale);
      if constexpr (Box::kRotated)
        if (seg_per_image) cat_ids[o] = n;
    }
    store_box(nms_boxes + o * D, b);
  }
}

struct DenseLevels {
  int L;
  const float* anchors[D2B_MAX_LEVELS];      // [R_l, 4]
  const float* deltas[D2B_MAX_LEVELS];       // [N, R_l, 4]
  const int64_t* topk_idx[D2B_MAX_LEVELS];   // [N, k_l]  flat (anchor * K + class)
  const float* topk_scores[D2B_MAX_LEVELS];  // [N, k_l]  -inf = dead slot
  int R[D2B_MAX_LEVELS], k[D2B_MAX_LEVELS], t0[D2B_MAX_LEVELS + 1];
};

// kLinear: Box2BoxTransformLinear.apply_deltas (FCOS) instead of Box2BoxTransform.apply_deltas (weights unused)
template <bool kLinear>
__global__ void __launch_bounds__(kThreads) dense_prepare_kernel(const DenseLevels P, int T, int K, float wx, float wy, float ww,
                                                                 float wh, float scale_clamp, float* __restrict__ flat_boxes,
                                                                 float* __restrict__ nms_boxes, float* __restrict__ nms_scores,
                                                                 float* __restrict__ raw_scores, long long* __restrict__ classes,
                                                                 long long* __restrict__ cat_ids) {
  __shared__ float s_red[32];
  __shared__ int s_redi[32];
  __shared__ float s_max;
  __shared__ int s_live;
  const int n = blockIdx.x, tid = threadIdx.x;
  float mx = -INFINITY;
  int nlive = 0;
  for (int t = tid; t < T; t += kThreads) {
    int l = 0;
    while (l + 1 < P.L && t >= P.t0[l + 1]) ++l;
    const int j = t - P.t0[l];
    const long long f = P.topk_idx[l][(size_t)n * P.k[l] + j];
    const float s = P.topk_scores[l][(size_t)n * P.k[l] + j];
    const bool live = s > -INFINITY;
    const long long a = f / K;
    const long long cls = f - a * K;
    const float4 an = *reinterpret_cast<const float4*>(P.anchors[l] + (size_t)a * 4);
    const float4 d = *reinterpret_cast<const float4*>(P.deltas[l] + ((size_t)n * P.R[l] + a) * 4);
    float x1, y1, x2, y2;
    if constexpr (kLinear) {
      const LinearBox lb = apply_deltas_linear(an, d);
      x1 = lb.x1, y1 = lb.y1, x2 = lb.x2, y2 = lb.y2;
    } else {
      const DecodedBox db = apply_deltas(an, d, wx, wy, ww, wh, scale_clamp);
      x1 = db.x1, y1 = db.y1, x2 = db.x2, y2 = db.y2;
    }
    const size_t o = (size_t)n * T + t;
    *reinterpret_cast<float4*>(flat_boxes + o * 4) = make_float4(x1, y1, x2, y2);
    raw_scores[o] = s;
    nms_scores[o] = live ? s : -INFINITY;
    classes[o] = cls;
    cat_ids[o] = live ? (long long)n * (K + 1) + cls : -1LL;
    if (live) {
      mx = fmaxf(mx, fmaxf(fmaxf(x1, y1), fmaxf(x2, y2)));
      ++nlive;
    }
  }
  for (int o = 16; o; o >>= 1) nlive += __shfl_xor_sync(0xffffffffu, nlive, o);
  if ((tid & 31) == 0) s_redi[tid >> 5] = nlive;
  mx = block_max(mx, s_red, &s_max);
  if (tid < 32) {
    int v = s_redi[tid];
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    if (tid == 0) s_live = v;
  }
  __syncthreads();
  // torchvision/ops/boxes.py batched_nms: coordinate trick while the image has at most 100 000 box elements on CUDA
  const bool trick = (long long)s_live * 4 <= 100000;
  const float scale = (s_live > 0 ? mx : 0.f) + 1.0f;
  for (int t = tid; t < T; t += kThreads) {
    const size_t o = (size_t)n * T + t;
    float4 b = make_float4(0.f, 0.f, 0.f, 0.f);
    if (cat_ids[o] >= 0) {
      b = *reinterpret_cast<const float4*>(flat_boxes + o * 4);
      if (trick) {
        const float offv = (float)classes[o] * scale;
        b.x += offv;
        b.y += offv;
        b.z += offv;
        b.w += offv;
      }
    }
    *reinterpret_cast<float4*>(nms_boxes + o * 4) = b;
  }
}

}  // namespace

D2B_API int d2b_rpn_prepare(const d2b_rpn_levels* lv, int N, const float* image_hw, float min_box_size, int flags,
                            float* flat_boxes, float* nms_boxes, float* nms_scores, float* raw_scores, int64_t* cat_ids,
                            int* nonfinite, void* stream) {
  const bool rot = (flags & D2B_SELECT_ROTATED) != 0;
  if (bad_flags(flags, D2B_SELECT_ROTATED | D2B_SELECT_SEG_PER_IMAGE | D2B_SELECT_NO_OFFSETS) || !lv || lv->num_levels < 1 ||
      lv->num_levels > D2B_MAX_LEVELS || N < 0 || !nonfinite)
    return D2B_EINVAL;
  RpnLevels P = {};
  P.L = lv->num_levels;
  long long T = 0;
  for (int l = 0; l < P.L; ++l) {
    if (lv->A[l] < 0 || lv->k[l] < 0 || lv->k[l] > lv->A[l]) return D2B_EINVAL;
    if (N > 0 && lv->k[l] > 0 && (!lv->proposals[l] || !lv->topk_idx[l] || !lv->topk_scores[l])) return D2B_EINVAL;
    if (!rot && misaligned16(lv->proposals[l])) return D2B_EINVAL;
    P.proposals[l] = lv->proposals[l];
    P.topk_idx[l] = lv->topk_idx[l];
    P.topk_scores[l] = lv->topk_scores[l];
    P.A[l] = lv->A[l];
    P.k[l] = lv->k[l];
    P.t0[l] = (int)T;
    T += lv->k[l];
  }
  if (T > INT_MAX) return D2B_EINVAL;
  P.t0[P.L] = (int)T;
  if (N > 0 && T > 0 && (!image_hw || !flat_boxes || !nms_boxes || !nms_scores || !raw_scores || !cat_ids)) return D2B_EINVAL;
  if (!rot && (misaligned16(flat_boxes) || misaligned16(nms_boxes))) return D2B_EINVAL;
  D2B_CUDA(cudaMemsetAsync(nonfinite, 0, sizeof(int), (cudaStream_t)stream));
  if (N == 0 || T == 0) return D2B_OK;
  const auto kernel = rot ? rpn_prepare_kernel<RotBox> : rpn_prepare_kernel<XyxyBox>;
  kernel<<<N, kThreads, 0, (cudaStream_t)stream>>>(P, (int)T, image_hw, min_box_size, (flags & D2B_SELECT_NO_OFFSETS) ? 0 : 1,
                                                   (flags & D2B_SELECT_SEG_PER_IMAGE) ? 1 : 0, flat_boxes, nms_boxes,
                                                   nms_scores, raw_scores, (long long*)cat_ids, nonfinite);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_frcnn_prepare(const float* boxes, const float* scores, const int* row_start, int N, int num_classes, int kreg,
                              const float* image_hw, float score_thresh, int cap, int flags, float* cand_boxes,
                              float* nms_boxes, float* nms_scores, float* raw_scores, int64_t* cand_flat, int64_t* cat_ids,
                              int64_t* n_cand, int64_t* row_map, void* stream) {
  const bool rot = (flags & D2B_SELECT_ROTATED) != 0;
  if (bad_flags(flags, D2B_SELECT_ROTATED | D2B_SELECT_SEG_PER_IMAGE) || N < 0 || N > D2B_MAX_IMAGES || num_classes <= 0 ||
      (kreg != 1 && kreg != num_classes) || cap < 0 || !row_start)
    return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  FrcnnImages I = {};
  I.N = N;
  for (int i = 0; i <= N; ++i) {
    I.row_start[i] = row_start[i];
    if (i ? row_start[i] < row_start[i - 1] : row_start[0] < 0) return D2B_EINVAL;  // a row before boxes[0]
  }
  if (!image_hw || !n_cand) return D2B_EINVAL;
  if (row_start[N] > row_start[0] && (!boxes || !scores || !row_map)) return D2B_EINVAL;
  if (cap > 0 && (!cand_boxes || !nms_boxes || !nms_scores || !raw_scores || !cand_flat || !cat_ids)) return D2B_EINVAL;
  if (!rot && (misaligned16(cand_boxes) || misaligned16(nms_boxes))) return D2B_EINVAL;
  const auto kernel = rot ? frcnn_prepare_kernel<RotBox> : frcnn_prepare_kernel<XyxyBox>;
  kernel<<<N, kThreads, 0, (cudaStream_t)stream>>>(I, boxes, scores, num_classes, kreg, image_hw, score_thresh, cap,
                                                   (flags & D2B_SELECT_SEG_PER_IMAGE) ? 1 : 0, cand_boxes, nms_boxes,
                                                   nms_scores, raw_scores, (long long*)cand_flat, (long long*)cat_ids,
                                                   (long long*)n_cand, (long long*)row_map);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_dense_prepare(const d2b_dense_levels* lv, int N, int num_classes, const float* weights, float scale_clamp,
                              int flags, float* flat_boxes, float* nms_boxes, float* nms_scores, float* raw_scores,
                              int64_t* classes, int64_t* cat_ids, void* stream) {
  const bool linear = (flags & D2B_SELECT_LINEAR) != 0;
  if (bad_flags(flags, D2B_SELECT_LINEAR) || !lv || lv->num_levels < 1 || lv->num_levels > D2B_MAX_LEVELS || N < 0 ||
      num_classes <= 0 || (!weights && !linear))
    return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  DenseLevels P = {};
  P.L = lv->num_levels;
  long long T = 0;
  for (int l = 0; l < P.L; ++l) {
    if (lv->R[l] < 0 || lv->k[l] < 0) return D2B_EINVAL;
    if (lv->k[l] > 0 && (!lv->anchors[l] || !lv->deltas[l] || !lv->topk_idx[l] || !lv->topk_scores[l])) return D2B_EINVAL;
    if (misaligned16(lv->anchors[l]) || misaligned16(lv->deltas[l])) return D2B_EINVAL;
    P.anchors[l] = lv->anchors[l];
    P.deltas[l] = lv->deltas[l];
    P.topk_idx[l] = lv->topk_idx[l];
    P.topk_scores[l] = lv->topk_scores[l];
    P.R[l] = lv->R[l];
    P.k[l] = lv->k[l];
    P.t0[l] = (int)T;
    T += lv->k[l];
  }
  if (T > INT_MAX) return D2B_EINVAL;
  P.t0[P.L] = (int)T;
  if (T == 0) return D2B_OK;
  if (!flat_boxes || !nms_boxes || !nms_scores || !raw_scores || !classes || !cat_ids) return D2B_EINVAL;
  if (misaligned16(flat_boxes) || misaligned16(nms_boxes)) return D2B_EINVAL;
  const float unused[4] = {1.f, 1.f, 1.f, 1.f};
  const float* w = linear ? unused : weights;
  const auto kernel = linear ? dense_prepare_kernel<true> : dense_prepare_kernel<false>;
  kernel<<<N, kThreads, 0, (cudaStream_t)stream>>>(P, (int)T, num_classes, w[0], w[1], w[2], w[3], scale_clamp, flat_boxes,
                                                   nms_boxes, nms_scores, raw_scores, (long long*)classes,
                                                   (long long*)cat_ids);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// ================================================================================================ mask targets + loss
// Mask-head training target and loss in one pass (SURVEY.md 8f-4):
//   BitMasks.crop_and_resize (detectron2/structures/masks.py:193-224): RoIAlign(S x S, scale 1, sampling_ratio 0, aligned)
//   of the proposal's ground-truth bitmask, thresholded at 0.5
//   + the per-class gather and binary_cross_entropy_with_logits of mask_rcnn_loss (modeling/roi_heads/mask_head.py:60-112).
// The reference first materialises one H x W byte mask PER PROPOSAL (BitMasks indexing, K x H x W bytes), converts it to
// fp32, pools it, thresholds, gathers the class channel of the logits and reduces.  Here a CTA per proposal samples the
// ground-truth mask it is matched to (mask_index) straight from the [G,H,W] byte tensor, one thread per output bin with the
// reference's accumulation order (torchvision roi_align: sum over iy, ix of w1 v1 + w2 v2 + w3 v3 + w4 v4, then / count),
// writes the 0/1 target (kept for the backward and the accuracy statistics) and the proposal's loss sum.
namespace {

struct Tap1 {
  int lo, hi;
  float wl, wh;
};

__device__ __forceinline__ Tap1 make_tap1(float v, int size) {  // torchvision roi_align bilinear_interpolate
  Tap1 t;
  if (v < -1.0f || v > (float)size) {
    t.lo = t.hi = 0;
    t.wl = t.wh = 0.f;
    return t;
  }
  v = fmaxf(v, 0.f);
  int lo = (int)v, hi;
  if (lo >= size - 1) {
    hi = lo = size - 1;
    v = (float)lo;
  } else {
    hi = lo + 1;
  }
  const float l = v - (float)lo;
  t.lo = lo;
  t.hi = hi;
  t.wh = l;
  t.wl = 1.f - l;
  return t;
}

// The target of each bin comes from a policy: BitmaskTarget pools the ground-truth bitmask (the RoIAlign above),
// PolygonTarget rasterizes the matched instance's polygons into shared memory first (polygon_raster.cuh).  begin() is called
// by every thread of the CTA; the returned Roi answers one bin.
struct BitmaskTarget {
  const unsigned char* __restrict__ gt;
  int G, H, W;
  const float* __restrict__ boxes;
  const long long* __restrict__ mask_index;
  struct Smem {};
  struct Roi {
    const unsigned char* __restrict__ m;
    int H, W, S, gh, gw;
    bool have_mask;
    float sw, sh, bin_w, bin_h, count;
    __device__ __forceinline__ bool operator()(int bin) const {
      const int ph = bin / S, pw = bin - ph * S;
      float v = 0.f;
      if (have_mask) {
        for (int iy = 0; iy < gh; ++iy) {
          const Tap1 ty = make_tap1(sh + (float)ph * bin_h + ((float)iy + .5f) * bin_h / (float)gh, H);
          for (int ix = 0; ix < gw; ++ix) {
            const Tap1 tx = make_tap1(sw + (float)pw * bin_w + ((float)ix + .5f) * bin_w / (float)gw, W);
            const float v1 = m[(size_t)ty.lo * W + tx.lo] ? 1.f : 0.f, v2 = m[(size_t)ty.lo * W + tx.hi] ? 1.f : 0.f;
            const float v3 = m[(size_t)ty.hi * W + tx.lo] ? 1.f : 0.f, v4 = m[(size_t)ty.hi * W + tx.hi] ? 1.f : 0.f;
            v += (ty.wl * tx.wl) * v1 + (ty.wl * tx.wh) * v2 + (ty.wh * tx.wl) * v3 + (ty.wh * tx.wh) * v4;
          }
        }
        v /= count;
      }
      return v >= 0.5f;
    }
  };
  __device__ __forceinline__ Roi begin(int k, int S, Smem&) const {
    Roi r;
    const float* b = boxes + (size_t)k * 4;
    // aligned = True, spatial_scale = 1: box - 0.5, no minimum size
    r.sw = b[0] * 1.0f - 0.5f;
    r.sh = b[1] * 1.0f - 0.5f;
    const float ew = b[2] * 1.0f - 0.5f, eh = b[3] * 1.0f - 0.5f;
    const float rw = ew - r.sw, rh = eh - r.sh;
    r.bin_h = rh / (float)S;
    r.bin_w = rw / (float)S;
    r.gh = max((int)ceilf(rh / (float)S), 0);
    r.gw = max((int)ceilf(rw / (float)S), 0);
    r.count = (float)max(r.gh * r.gw, 1);
    const long long mi = mask_index ? mask_index[k] : k;
    r.have_mask = mi >= 0 && mi < G;
    r.m = gt + (size_t)(r.have_mask ? mi : 0) * H * W;
    r.H = H;
    r.W = W;
    r.S = S;
    return r;
  }
};

struct PolygonTarget {
  PolyBatch pb;
  const float* __restrict__ boxes;
  const long long* __restrict__ mask_index;
  using Smem = PolyTileSmem;
  struct Roi {
    const PolyTileSmem* sm;
    int S;
    __device__ __forceinline__ bool operator()(int bin) const {
      const int r = bin / S;
      return poly_mask_bit(*sm, r, bin - r * S);
    }
  };
  __device__ __forceinline__ Roi begin(int k, int S, Smem& sm) const {
    PolyTransform tf;
    const bool box_ok = poly_box_transform(boxes + (size_t)k * 4, S, tf);
    poly_raster_instance(pb, !box_ok ? -1 : mask_index ? mask_index[k] : k, tf, S, S, 0, S, 0, S, sm);
    return Roi{&sm, S};
  }
};

template <class Target>
__global__ void __launch_bounds__(256) mask_loss_fwd_kernel(const float* __restrict__ logits, int C, int S, Target target,
                                                            const long long* __restrict__ classes,
                                                            float* __restrict__ loss_per_roi,
                                                            unsigned char* __restrict__ targets) {
  __shared__ float s_red[8];
  __shared__ typename Target::Smem s_target;
  const int k = blockIdx.x, tid = threadIdx.x;
  const typename Target::Roi roi = target.begin(k, S, s_target);
  const long long cls = classes ? classes[k] : 0;
  const bool cls_ok = cls >= 0 && cls < C;
  const float* __restrict__ lg = logits + ((size_t)k * C + (cls_ok ? cls : 0)) * S * S;
  float acc_loss = 0.f;
  for (int bin = tid; bin < S * S; bin += 256) {
    const bool tb = roi(bin);
    const float t = tb ? 1.f : 0.f;
    targets[(size_t)k * S * S + bin] = (unsigned char)tb;
    if (cls_ok) {
      const float x = lg[bin];
      // binary_cross_entropy_with_logits: (1 - t) x + max(-x, 0) + log(exp(-max) + exp(-x - max)),  max = max(-x, 0)
      const float mxv = fmaxf(-x, 0.f);
      acc_loss += (1.f - t) * x + mxv + logf(expf(-mxv) + expf(-x - mxv));
    }
  }
  for (int o = 16; o; o >>= 1) acc_loss += __shfl_xor_sync(0xffffffffu, acc_loss, o);
  if ((tid & 31) == 0) s_red[tid >> 5] = acc_loss;
  __syncthreads();
  if (tid == 0) {
    float s = 0.f;
    for (int i = 0; i < 8; ++i) s += s_red[i];
    loss_per_roi[k] = s;
  }
}

// grad_logits[k, c, :] = (c == class_k) ? (sigmoid(x) - t) * grad_scale[k] : 0      grid (K, C)
__global__ void __launch_bounds__(256) mask_loss_bwd_kernel(const float* __restrict__ logits, int C, int S,
                                                            const unsigned char* __restrict__ targets,
                                                            const long long* __restrict__ classes,
                                                            const float* __restrict__ grad_scale,
                                                            float* __restrict__ grad_logits) {
  const int k = blockIdx.x, c = blockIdx.y;
  const long long cls = classes ? classes[k] : 0;
  const size_t base = ((size_t)k * C + c) * S * S;
  const float scale = grad_scale[k];  // d loss / d loss_per_roi[k]
  for (int bin = threadIdx.x; bin < S * S; bin += 256) {
    float gval = 0.f;
    if (c == cls) {
      const float x = logits[base + bin];
      const float t = targets[(size_t)k * S * S + bin] ? 1.f : 0.f;
      gval = (1.f / (1.f + expf(-x)) - t) * scale;
    }
    grad_logits[base + bin] = gval;
  }
}

}  // namespace

D2B_API int d2b_mask_loss_forward(const float* logits, int K, int C, int S, const uint8_t* gt_masks, int G, int H, int W,
                                  const float* boxes, const int64_t* mask_index, const int64_t* classes,
                                  float* loss_per_roi, uint8_t* targets, void* stream) {
  if (K < 0 || C <= 0 || S <= 0 || G < 0 || H <= 0 || W <= 0) return D2B_EINVAL;
  if (K == 0) return D2B_OK;
  if (!logits || !gt_masks || !boxes || !loss_per_roi || !targets) return D2B_EINVAL;
  mask_loss_fwd_kernel<<<K, 256, 0, (cudaStream_t)stream>>>(
      logits, C, S, BitmaskTarget{gt_masks, G, H, W, boxes, (const long long*)mask_index}, (const long long*)classes,
      loss_per_roi, targets);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_mask_loss_polygons_forward(const float* logits, int K, int C, int S, const double* coords, int V,
                                           const int* poly_start, int P, const int* inst_start, int G, const float* boxes,
                                           const int64_t* mask_index, const int64_t* classes, float* loss_per_roi,
                                           uint8_t* targets, void* stream) {
  if (K < 0 || C < 1 || S < 1 || S > D2B_POLYGON_MAX_S || V < 0 || P < 0 || G < 0) return D2B_EINVAL;
  if (K == 0) return D2B_OK;
  if (!logits || !boxes || !loss_per_roi || !targets || (G > 0 && !inst_start) || (P > 0 && !poly_start) ||
      (V > 0 && !coords))
    return D2B_EINVAL;
  mask_loss_fwd_kernel<<<K, 256, 0, (cudaStream_t)stream>>>(
      logits, C, S, PolygonTarget{PolyBatch{coords, V, poly_start, P, inst_start, G}, boxes, (const long long*)mask_index},
      (const long long*)classes, loss_per_roi, targets);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_mask_loss_backward(const float* logits, int K, int C, int S, const uint8_t* targets, const int64_t* classes,
                                   const float* grad_scale, float* grad_logits, void* stream) {
  if (K < 0 || C <= 0 || S <= 0 || C > 65535) return D2B_EINVAL;
  if (K == 0) return D2B_OK;
  if (!logits || !targets || !grad_scale || !grad_logits) return D2B_EINVAL;
  dim3 grid(K, C);
  mask_loss_bwd_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(logits, C, S, targets, (const long long*)classes, grad_scale,
                                                               grad_logits);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
