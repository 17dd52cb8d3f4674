// Box2BoxTransform.apply_deltas (detectron2/modeling/box_regression.py:78-116) for one xyxy box, op for op.  Shared by the
// RetinaNet inference decode (postproc.cu) and the GIoU box-regression loss (losses.cu); both files are compiled with
// -fmad=false so that every operation rounds like the reference's separate torch ops.
#pragma once

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
// times the anchor's stride (width, height), then the centre minus (l, t) and plus (r, b).  Shared by the FCOS inference
// decode (postproc.cu) and the FCOS GIoU loss (losses.cu).
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
