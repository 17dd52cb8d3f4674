// Box types of the bit-exact box kernels (postproc.cu, match.cu, losses.cu): layout, the reference's clip, the batched-NMS
// coordinate offsets, the IoU, Box2BoxTransform[Rotated].get_deltas and the apply_deltas decodes, each written once.
// Every operation keeps the reference's fp32 expression order, so this header is only included from files compiled with
// -fmad=false (build.py), where every operation rounds like the reference's separate torch ops.
//   XyxyBox  Boxes (x1, y1, x2, y2): clip = clamp to the image; torchvision's offsets idx * (max coordinate + 1) on all four;
//            pairwise_iou (structures/boxes.py:312-358); Box2BoxTransform.get_deltas.
//   RotBox   RotatedBoxes (cx, cy, w, h, angle_deg): RotatedBoxes.clip (structures/rotated_boxes.py:248-303); the offsets of
//            batched_nms_rotated (layers/nms.py:137-146), idx * (max - min + 1), on the centre only; the rotated IoU of
//            nms.cu (rotated_iou.cuh); Box2BoxTransformRotated.get_deltas.
#pragma once

#include "rotated_iou.cuh"

namespace {

// torch.min / torch.max propagate NaN; fminf / fmaxf would drop it
__device__ __forceinline__ float nan_min(float a, float b) { return (a != a || b != b) ? a + b : fminf(a, b); }
__device__ __forceinline__ float nan_max(float a, float b) { return (a != a || b != b) ? a + b : fmaxf(a, b); }

struct BoxWeights {
  float w[5];  // RotBox: w[4] = wa * pi / 180 rounded to fp32, the scalar torch multiplies by
};

struct XyxyBox {
  static constexpr int D = 4;
  static constexpr bool kRotated = false;
  float v[4];
  __device__ __forceinline__ void clip(float ih, float iw) {  // clamp(min=0, max=w / h)
    v[0] = fminf(fmaxf(v[0], 0.f), iw);
    v[1] = fminf(fmaxf(v[1], 0.f), ih);
    v[2] = fminf(fmaxf(v[2], 0.f), iw);
    v[3] = fminf(fmaxf(v[3], 0.f), ih);
  }
  // the nonempty test's width / height; the width is also what get_deltas' assertion reads of the source box
  static __device__ __forceinline__ float width(const float* b) { return b[2] - b[0]; }
  static __device__ __forceinline__ float height(const float* b) { return b[3] - b[1]; }
  __device__ __forceinline__ float hi() const { return fmaxf(fmaxf(v[0], v[1]), fmaxf(v[2], v[3])); }  // boxes.max()
  __device__ __forceinline__ float lo() const { return 0.f; }                                          // not part of the range
  static __device__ __forceinline__ float scale(bool any, float mx, float) { return (any ? mx : 0.f) + 1.0f; }
  __device__ __forceinline__ void shift(float off) {
    v[0] += off;
    v[1] += off;
    v[2] += off;
    v[3] += off;
  }
  // pairwise_iou(boxes1 = gt, boxes2 = prediction): the same fp32 operations in the same order
  static __device__ __forceinline__ float iou(const float* __restrict__ g, const float* __restrict__ a) {
    const float area1 = (g[2] - g[0]) * (g[3] - g[1]);
    const float area2 = (a[2] - a[0]) * (a[3] - a[1]);
    float w = nan_min(g[2], a[2]) - nan_max(g[0], a[0]);
    float h = nan_min(g[3], a[3]) - nan_max(g[1], a[1]);
    w = w < 0.f ? 0.f : w;  // clamp_(min=0): NaN stays NaN
    h = h < 0.f ? 0.f : h;
    const float inter = w * h;
    return inter > 0.f ? inter / (area1 + area2 - inter) : 0.f;
  }
  // Box2BoxTransform.get_deltas (box_regression.py:43-76), op for op
  static __device__ __forceinline__ void get_deltas(const float* s, const float* t, const BoxWeights& w, float* d) {
    const float sw = s[2] - s[0], sh = s[3] - s[1];
    const float scx = s[0] + 0.5f * sw, scy = s[1] + 0.5f * sh;
    const float tw = t[2] - t[0], th = t[3] - t[1];
    const float tcx = t[0] + 0.5f * tw, tcy = t[1] + 0.5f * th;
    d[0] = w.w[0] * (tcx - scx) / sw;
    d[1] = w.w[1] * (tcy - scy) / sh;
    d[2] = w.w[2] * logf(tw / sw);
    d[3] = w.w[3] * logf(th / sh);
  }
};

struct RotBox {
  static constexpr int D = 5;
  static constexpr bool kRotated = true;
  float v[5];
  // (a + 180) % 360 - 180 with torch's float remainder (the result takes the divisor's sign)
  static __device__ __forceinline__ float wrap_angle(float a) {
    float m = fmodf(a + 180.f, 360.f);
    if (m < 0.f) m += 360.f;
    return m - 180.f;
  }
  __device__ __forceinline__ void clip(float ih, float iw) {
    v[4] = wrap_angle(v[4]);  // normalize_angles
    if (fabsf(v[4]) <= 1.0f) {  // clip_angle_threshold: only near-horizontal boxes are clipped, as xyxy boxes
      const float x1 = fminf(fmaxf(v[0] - v[2] / 2.f, 0.f), iw), y1 = fminf(fmaxf(v[1] - v[3] / 2.f, 0.f), ih);
      const float x2 = fminf(fmaxf(v[0] + v[2] / 2.f, 0.f), iw), y2 = fminf(fmaxf(v[1] + v[3] / 2.f, 0.f), ih);
      v[0] = (x1 + x2) / 2.f;
      v[1] = (y1 + y2) / 2.f;
      v[2] = fminf(v[2], x2 - x1);  // widths and heights never grow through rounding
      v[3] = fminf(v[3], y2 - y1);
    }
  }
  static __device__ __forceinline__ float width(const float* b) { return b[2]; }
  static __device__ __forceinline__ float height(const float* b) { return b[3]; }
  __device__ __forceinline__ float hi() const { return fmaxf(v[0], v[1]) + fmaxf(v[2], v[3]) / 2; }
  __device__ __forceinline__ float lo() const { return fminf(v[0], v[1]) - fmaxf(v[2], v[3]) / 2; }
  static __device__ __forceinline__ float scale(bool any, float mx, float mn) { return (any ? mx - mn : 0.f) + 1.0f; }
  __device__ __forceinline__ void shift(float off) {
    v[0] += off;
    v[1] += off;
  }
  // box_iou_rotated(boxes1 = gt, boxes2 = prediction)[g, a]
  static __device__ __forceinline__ float iou(const float* __restrict__ g, const float* __restrict__ a) {
    return rotated_iou(g, a);
  }
  // Box2BoxTransformRotated.get_deltas (box_regression.py:145-180), op for op
  static __device__ __forceinline__ void get_deltas(const float* s, const float* t, const BoxWeights& w, float* d) {
    d[0] = w.w[0] * (t[0] - s[0]) / s[2];
    d[1] = w.w[1] * (t[1] - s[1]) / s[3];
    d[2] = w.w[2] * logf(t[2] / s[2]);
    d[3] = w.w[3] * logf(t[3] / s[3]);
    d[4] = wrap_angle(t[4] - s[4]) * w.w[4];
  }
};

template <class Box>
__device__ __forceinline__ Box load_box(const float* __restrict__ p) {  // scalar loads: rows of the inputs need no alignment
  Box b;
#pragma unroll
  for (int q = 0; q < Box::D; ++q) b.v[q] = p[q];
  return b;
}

template <class Box>
__device__ __forceinline__ Box load_box_aligned(const float* __restrict__ p) {  // xyxy buffers are 16-byte aligned
  if constexpr (Box::D == 4) {
    const float4 q = *reinterpret_cast<const float4*>(p);
    return Box{{q.x, q.y, q.z, q.w}};
  } else {
    return load_box<Box>(p);
  }
}

template <class Box>
__device__ __forceinline__ void store_box(float* __restrict__ p, const Box& b) {  // xyxy buffers are 16-byte aligned
  if constexpr (Box::D == 4) {
    *reinterpret_cast<float4*>(p) = make_float4(b.v[0], b.v[1], b.v[2], b.v[3]);
  } else {
#pragma unroll
    for (int q = 0; q < Box::D; ++q) p[q] = b.v[q];
  }
}

template <class Box>
__device__ __forceinline__ Box zero_box() {
  Box b;
#pragma unroll
  for (int q = 0; q < Box::D; ++q) b.v[q] = 0.f;
  return b;
}

// Box2BoxTransform.apply_deltas (box_regression.py:78-116) for one xyxy box, op for op: the RetinaNet inference decode
// (postproc.cu) and the GIoU box-regression loss (losses.cu).
struct DecodedBox {
  float x1, y1, x2, y2;
  // what the backward needs: the anchor's width / height, exp(dw) / exp(dh), and whether dw / dh passed the clamp
  // (torch.clamp(max=) passes the gradient at equality, zero strictly above)
  float widths, heights, ew, eh;
  bool pass_w, pass_h;
};

__device__ __forceinline__ DecodedBox apply_deltas(float4 an, float4 d, float wx, float wy, float ww, float wh,
                                                   float scale_clamp) {
  DecodedBox b;
  b.widths = an.z - an.x;
  b.heights = an.w - an.y;
  const float ctr_x = an.x + 0.5f * b.widths, ctr_y = an.y + 0.5f * b.heights;
  const float dx = d.x / wx, dy = d.y / wy;
  float dw = d.z / ww, dh = d.w / wh;
  b.pass_w = !(dw > scale_clamp);
  b.pass_h = !(dh > scale_clamp);
  dw = dw > scale_clamp ? scale_clamp : dw;  // torch.clamp(max=): NaN stays NaN
  dh = dh > scale_clamp ? scale_clamp : dh;
  const float pcx = dx * b.widths + ctr_x, pcy = dy * b.heights + ctr_y;
  b.ew = expf(dw);
  b.eh = expf(dh);
  const float pw = b.ew * b.widths, ph = b.eh * b.heights;
  b.x1 = pcx - 0.5f * pw;
  b.y1 = pcy - 0.5f * ph;
  b.x2 = pcx + 0.5f * pw;
  b.y2 = pcy + 0.5f * ph;
  return b;
}

// Box2BoxTransformLinear.apply_deltas (box_regression.py:275-307) with normalize_by_size=True, op for op: relu(deltas)
// times the anchor's stride (width, height), then the centre minus (l, t) and plus (r, b).  The FCOS inference decode
// (postproc.cu) and the FCOS GIoU loss (losses.cu).
struct LinearBox {
  float x1, y1, x2, y2;
  float sw, sh;  // the stride, what the backward multiplies by
};

// F.relu = clamp_min(0): NaN stays NaN
__device__ __forceinline__ float relu_nan(float v) { return v != v ? v : (v > 0.f ? v : 0.f); }

__device__ __forceinline__ LinearBox apply_deltas_linear(float4 an, float4 d) {
  LinearBox b;
  const float ctr_x = 0.5f * (an.x + an.z), ctr_y = 0.5f * (an.y + an.w);
  b.sw = an.z - an.x;
  b.sh = an.w - an.y;
  b.x1 = ctr_x - relu_nan(d.x) * b.sw;
  b.y1 = ctr_y - relu_nan(d.y) * b.sh;
  b.x2 = ctr_x + relu_nan(d.z) * b.sw;
  b.y2 = ctr_y + relu_nan(d.w) * b.sh;
  return b;
}

}  // namespace
