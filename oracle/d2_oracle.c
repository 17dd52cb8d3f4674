/*
 * d2_oracle.c -- CPU restatement of the detectron2 per-image detection ops.
 *
 * THIS IS TEST INFRASTRUCTURE, NOT PRODUCT CODE.  Only tests/, the smoke check in
 * __graft_entry__.py and bench.py's cpu_baseline / --impl reference leg may load
 * this library.  The product path (detectron2_b200/) never links or calls it.
 *
 * Every function restates, in plain scalar C, the algorithm of the reference
 * (paths relative to /root/reference/), citing the file:line it follows.
 * Parity status: PINNED.  tests/test_oracle_pins.py checks this file against
 *   - the reference's own golden tables (tests/layers/test_roi_align.py:28-41,
 *     test_roi_align_rotated.py:57-69, test_deformable.py:38-46,
 *     tests/structures/test_rotated_boxes.py:46-147,247-369),
 *   - the reference CPU csrc compiled in place (oracle/_ref, see build.py),
 *   - torchvision CPU ops (the reference's backend for roi_align/nms/deform_conv2d,
 *     detectron2/layers/roi_align.py:3,58  nms.py:5-22  deform_conv.py:9,55),
 *   - the committed fixtures in tests/golden/ generated from those.
 *
 * Build: gcc -O2 -ffp-contract=off -fPIC -shared (see oracle/build.py).  FP contraction
 * is disabled so float expressions round exactly like the reference's x86-64 CPU build
 * (no FMA), which is what the bit-exact ops (rotated IoU, NMS) are compared against.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_API __attribute__((visibility("default")))

/* ------------------------------------------------------------------------------------------
 * RoIAlign (axis-aligned).  Reference: torchvision roi_align, reached from
 * detectron2/layers/roi_align.py:58-65.  Arithmetic follows torchvision/ops/roi_align.py
 * (_roi_align / _bilinear_interpolate, the transcription of the tv kernel) and the in-repo
 * sibling ROIAlignRotated_cpu.cpp:27-129 (same Caffe2 lineage).
 * ---------------------------------------------------------------------------------------- */

typedef struct {
  int p1, p2, p3, p4; /* flat h*W+w positions of the four taps */
  float w1, w2, w3, w4;
} orc_tap;

/* ROIAlignRotated_cpu.cpp:63-122 / tv _bilinear_interpolate: out-of-range test, clamp, taps */
static int orc_bilinear_taps(int H, int W, float y, float x, orc_tap* t) {
  if (y < -1.0f || y > (float)H || x < -1.0f || x > (float)W) {
    t->p1 = t->p2 = t->p3 = t->p4 = 0;
    t->w1 = t->w2 = t->w3 = t->w4 = 0.f;
    return 0;
  }
  if (y < 0.f) y = 0.f;
  if (x < 0.f) x = 0.f;
  int yl = (int)y, xl = (int)x, yh, xh;
  if (yl >= H - 1) { yh = yl = H - 1; y = (float)yl; } else { yh = yl + 1; }
  if (xl >= W - 1) { xh = xl = W - 1; x = (float)xl; } else { xh = xl + 1; }
  float ly = y - (float)yl, lx = x - (float)xl;
  float hy = 1.f - ly, hx = 1.f - lx;
  t->p1 = yl * W + xl; t->p2 = yl * W + xh; t->p3 = yh * W + xl; t->p4 = yh * W + xh;
  t->w1 = hy * hx; t->w2 = hy * lx; t->w3 = ly * hx; t->w4 = ly * lx;
  return 1;
}

typedef struct {
  int b;           /* batch index */
  float start_h, start_w, bin_h, bin_w;
  int gh, gw;      /* sampling grid */
  float count;
  /* rotated only */
  float ctr_h, ctr_w, cos_t, sin_t;
} orc_roi_geom;

/* tv _roi_align: roi_start = coord*scale - offset; !aligned -> clamp size to >= 1 */
static void orc_geom_aligned(const float* roi, float scale, int PH, int PW, int sampling_ratio,
                             int aligned, orc_roi_geom* g) {
  float off = aligned ? 0.5f : 0.0f;
  g->b = (int)roi[0];
  float sw = roi[1] * scale - off, sh = roi[2] * scale - off;
  float ew = roi[3] * scale - off, eh = roi[4] * scale - off;
  float rw = ew - sw, rh = eh - sh;
  if (!aligned) { if (rw < 1.f) rw = 1.f; if (rh < 1.f) rh = 1.f; }
  g->start_h = sh; g->start_w = sw;
  g->bin_h = rh / (float)PH; g->bin_w = rw / (float)PW;
  g->gh = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(rh / (float)PH);
  g->gw = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(rw / (float)PW);
  int c = g->gh * g->gw; if (c < 1) c = 1;
  g->count = (float)c;
  g->ctr_h = g->ctr_w = 0.f; g->cos_t = 1.f; g->sin_t = 0.f;
}

/* ROIAlignRotated_cpu.cpp:225-263: centre*scale-0.5, size*scale, theta = a*pi/180 */
static void orc_geom_rotated(const float* roi, float scale, int PH, int PW, int sampling_ratio,
                             orc_roi_geom* g) {
  g->b = (int)roi[0];
  g->ctr_w = roi[1] * scale - 0.5f;
  g->ctr_h = roi[2] * scale - 0.5f;
  float rw = roi[3] * scale, rh = roi[4] * scale;
  float theta = (float)((double)roi[5] * M_PI / 180.0);
  g->cos_t = cosf(theta); g->sin_t = sinf(theta);
  g->bin_h = rh / (float)PH; g->bin_w = rw / (float)PW;
  g->gh = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(rh / (float)PH);
  g->gw = sampling_ratio > 0 ? sampling_ratio : (int)ceilf(rw / (float)PW);
  int c = g->gh * g->gw; if (c < 1) c = 1;
  g->count = (float)c;
  g->start_h = (float)(-(double)rh / 2.0); g->start_w = (float)(-(double)rw / 2.0);
}

static void orc_sample_xy(const orc_roi_geom* g, int rotated, int ph, int pw, int iy, int ix,
                          float* y, float* x) {
  float yy = g->start_h + (float)ph * g->bin_h + ((float)iy + .5f) * g->bin_h / (float)g->gh;
  float xx = g->start_w + (float)pw * g->bin_w + ((float)ix + .5f) * g->bin_w / (float)g->gw;
  if (rotated) { /* ROIAlignRotated_cpu.cpp:61-62 */
    *y = yy * g->cos_t - xx * g->sin_t + g->ctr_h;
    *x = yy * g->sin_t + xx * g->cos_t + g->ctr_w;
  } else { *y = yy; *x = xx; }
}

static void orc_roi_fwd(const float* in, int N, int C, int H, int W, const float* rois, int K,
                        int roi_cols, float scale, int PH, int PW, int sr, int aligned,
                        int rotated, float* out) {
  (void)N;
  for (int k = 0; k < K; ++k) {
    orc_roi_geom g;
    if (rotated) orc_geom_rotated(rois + (size_t)k * roi_cols, scale, PH, PW, sr, &g);
    else orc_geom_aligned(rois + (size_t)k * roi_cols, scale, PH, PW, sr, aligned, &g);
    size_t ntap = (size_t)PH * PW * (g.gh > 0 ? g.gh : 0) * (g.gw > 0 ? g.gw : 0);
    orc_tap* taps = (orc_tap*)malloc(sizeof(orc_tap) * (ntap ? ntap : 1));
    size_t ti = 0; /* ROIAlignRotated_cpu.cpp:46-128: taps shared by all channels */
    for (int ph = 0; ph < PH; ++ph) for (int pw = 0; pw < PW; ++pw)
      for (int iy = 0; iy < g.gh; ++iy) for (int ix = 0; ix < g.gw; ++ix) {
        float y, x; orc_sample_xy(&g, rotated, ph, pw, iy, ix, &y, &x);
        orc_bilinear_taps(H, W, y, x, &taps[ti++]);
      }
    for (int c = 0; c < C; ++c) { /* :279-307 */
      const float* src = in + ((size_t)g.b * C + c) * H * W;
      float* dst = out + ((size_t)k * C + c) * PH * PW;
      ti = 0;
      for (int p = 0; p < PH * PW; ++p) {
        float acc = 0.f;
        for (int s = 0; s < g.gh * g.gw; ++s) {
          const orc_tap* t = &taps[ti++];
          acc += t->w1 * src[t->p1] + t->w2 * src[t->p2] + t->w3 * src[t->p3] + t->w4 * src[t->p4];
        }
        dst[p] = acc / g.count;
      }
    }
    free(taps);
  }
}

/* ROIAlignRotated_cpu.cpp:312-416 (bwd) / tv _roi_align_backward: scatter g*w/count */
static void orc_roi_bwd(const float* gout, const float* rois, int K, int roi_cols, float scale,
                        int PH, int PW, int N, int C, int H, int W, int sr, int aligned,
                        int rotated, float* gin) {
  memset(gin, 0, sizeof(float) * (size_t)N * C * H * W);
  for (int k = 0; k < K; ++k) {
    orc_roi_geom g;
    if (rotated) orc_geom_rotated(rois + (size_t)k * roi_cols, scale, PH, PW, sr, &g);
    else orc_geom_aligned(rois + (size_t)k * roi_cols, scale, PH, PW, sr, aligned, &g);
    float count = (float)(g.gh * g.gw); /* bwd uses the raw product (:372) */
    for (int c = 0; c < C; ++c) {
      float* dst = gin + ((size_t)g.b * C + c) * H * W;
      const float* go = gout + ((size_t)k * C + c) * PH * PW;
      for (int ph = 0; ph < PH; ++ph) for (int pw = 0; pw < PW; ++pw) {
        float gv = go[ph * PW + pw];
        for (int iy = 0; iy < g.gh; ++iy) for (int ix = 0; ix < g.gw; ++ix) {
          float y, x; orc_sample_xy(&g, rotated, ph, pw, iy, ix, &y, &x);
          orc_tap t;
          if (!orc_bilinear_taps(H, W, y, x, &t)) continue;
          dst[t.p1] += gv * t.w1 / count; dst[t.p2] += gv * t.w2 / count;
          dst[t.p3] += gv * t.w3 / count; dst[t.p4] += gv * t.w4 / count;
        }
      }
    }
  }
}

ORC_API void orc_roi_align_forward(const float* in, int N, int C, int H, int W, const float* rois,
                                   int K, float scale, int PH, int PW, int sr, int aligned,
                                   float* out) {
  orc_roi_fwd(in, N, C, H, W, rois, K, 5, scale, PH, PW, sr, aligned, 0, out);
}
ORC_API void orc_roi_align_backward(const float* gout, const float* rois, int K, float scale,
                                    int PH, int PW, int N, int C, int H, int W, int sr,
                                    int aligned, float* gin) {
  orc_roi_bwd(gout, rois, K, 5, scale, PH, PW, N, C, H, W, sr, aligned, 0, gin);
}
ORC_API void orc_roi_align_rotated_forward(const float* in, int N, int C, int H, int W,
                                           const float* rois, int K, float scale, int PH, int PW,
                                           int sr, float* out) {
  orc_roi_fwd(in, N, C, H, W, rois, K, 6, scale, PH, PW, sr, 1, 1, out);
}
ORC_API void orc_roi_align_rotated_backward(const float* gout, const float* rois, int K,
                                            float scale, int PH, int PW, int N, int C, int H,
                                            int W, int sr, float* gin) {
  orc_roi_bwd(gout, rois, K, 6, scale, PH, PW, N, C, H, W, sr, 1, 1, gin);
}

/* ------------------------------------------------------------------------------------------
 * Axis-aligned NMS.  Reference: torchvision::nms (CPU kernel), reached through
 * detectron2/layers/nms.py:11-22.  Algorithm per SURVEY A.7 and black-box probes: stable
 * descending score order, area=(x2-x1)*(y2-y1), inter=max(0,.)*max(0,.),
 * suppress iff inter/(a_i+a_j-inter) > thr (strict; float ovr vs double thr).
 * ---------------------------------------------------------------------------------------- */
typedef struct { float s; int64_t i; } orc_si;
/* torch.sort(descending=True, stable=True): NaN (either sign) above every number, -0 == +0, then lower index first.
 * A total order for any input, as qsort requires. */
static int orc_cmp_desc(const void* a, const void* b) {
  const orc_si *x = (const orc_si*)a, *y = (const orc_si*)b;
  const int xn = isnan(x->s), yn = isnan(y->s);
  if (xn != yn) return xn ? -1 : 1;
  if (!xn) {
    if (x->s > y->s) return -1;
    if (x->s < y->s) return 1;
  }
  return (x->i > y->i) - (x->i < y->i); /* stable: lower index first on ties */
}
static int64_t* orc_order_desc(const float* scores, int64_t M) {
  orc_si* a = (orc_si*)malloc(sizeof(orc_si) * (size_t)(M ? M : 1));
  for (int64_t i = 0; i < M; ++i) { a[i].s = scores[i]; a[i].i = i; }
  qsort(a, (size_t)M, sizeof(orc_si), orc_cmp_desc);
  int64_t* o = (int64_t*)malloc(sizeof(int64_t) * (size_t)(M ? M : 1));
  for (int64_t i = 0; i < M; ++i) o[i] = a[i].i;
  free(a);
  return o;
}

ORC_API int64_t orc_nms(const float* boxes, const float* scores, int64_t M, double thr,
                        int64_t* keep) {
  int64_t* order = orc_order_desc(scores, M);
  uint8_t* sup = (uint8_t*)calloc((size_t)(M ? M : 1), 1);
  float* area = (float*)malloc(sizeof(float) * (size_t)(M ? M : 1));
  for (int64_t i = 0; i < M; ++i)
    area[i] = (boxes[4 * i + 2] - boxes[4 * i]) * (boxes[4 * i + 3] - boxes[4 * i + 1]);
  int64_t nk = 0;
  for (int64_t _i = 0; _i < M; ++_i) {
    int64_t i = order[_i];
    if (sup[i]) continue;
    keep[nk++] = i;
    float ix1 = boxes[4 * i], iy1 = boxes[4 * i + 1], ix2 = boxes[4 * i + 2], iy2 = boxes[4 * i + 3];
    for (int64_t _j = _i + 1; _j < M; ++_j) {
      int64_t j = order[_j];
      if (sup[j]) continue;
      float xx1 = fmaxf(ix1, boxes[4 * j]), yy1 = fmaxf(iy1, boxes[4 * j + 1]);
      float xx2 = fminf(ix2, boxes[4 * j + 2]), yy2 = fminf(iy2, boxes[4 * j + 3]);
      float w = fmaxf(0.f, xx2 - xx1), h = fmaxf(0.f, yy2 - yy1);
      float inter = w * h;
      float ovr = inter / (area[i] + area[j] - inter);
      if ((double)ovr > thr) sup[j] = 1;
    }
  }
  free(order); free(sup); free(area);
  return nk;
}

/* ------------------------------------------------------------------------------------------
 * Rotated-box IoU.  Reference: detectron2/layers/csrc/box_iou_rotated/box_iou_rotated_utils.h
 * (CPU branch of convex_hull_graham, :228-262).  float/double promotions follow the C++
 * expression types exactly (double literals promote, results narrow on assignment).
 * ---------------------------------------------------------------------------------------- */
typedef struct { float x, y; } orc_pt;

static float orc_cross(orc_pt a, orc_pt b) { return a.x * b.y - b.x * a.y; } /* :53-56 */
static float orc_dot(orc_pt a, orc_pt b) { return a.x * b.x + a.y * b.y; }   /* :47-49 */

static void orc_vertices(float xc, float yc, float w, float h, float a, orc_pt* p) { /* :58-76 */
  double theta = (double)a * 0.01745329251;
  float c2 = (float)cos(theta) * 0.5f, s2 = (float)sin(theta) * 0.5f;
  p[0].x = xc + s2 * h + c2 * w; p[0].y = yc + c2 * h - s2 * w;
  p[1].x = xc - s2 * h + c2 * w; p[1].y = yc - c2 * h - s2 * w;
  p[2].x = 2 * xc - p[0].x; p[2].y = 2 * yc - p[0].y;
  p[3].x = 2 * xc - p[1].x; p[3].y = 2 * yc - p[1].y;
}

static int orc_intersections(const orc_pt* p1, const orc_pt* p2, orc_pt* out) { /* :78-164 */
  orc_pt v1[4], v2[4];
  for (int i = 0; i < 4; ++i) {
    v1[i].x = p1[(i + 1) % 4].x - p1[i].x; v1[i].y = p1[(i + 1) % 4].y - p1[i].y;
    v2[i].x = p2[(i + 1) % 4].x - p2[i].x; v2[i].y = p2[(i + 1) % 4].y - p2[i].y;
  }
  const double EPS = 1e-5;
  int num = 0;
  for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) {
    float det = orc_cross(v2[j], v1[i]);
    if (fabs((double)det) <= 1e-14) continue;
    orc_pt v12 = { p2[j].x - p1[i].x, p2[j].y - p1[i].y };
    float t1 = orc_cross(v2[j], v12) / det;
    float t2 = orc_cross(v1[i], v12) / det;
    if ((double)t1 > -EPS && (double)t1 < (double)1.0f + EPS && (double)t2 > -EPS &&
        (double)t2 < (double)1.0f + EPS) {
      out[num].x = p1[i].x + v1[i].x * t1; out[num].y = p1[i].y + v1[i].y * t1; ++num;
    }
  }
  for (int pass = 0; pass < 2; ++pass) { /* :121-161: vertices of one rect inside the other */
    const orc_pt* pa = pass == 0 ? p1 : p2; /* points tested */
    const orc_pt* pb = pass == 0 ? p2 : p1; /* rectangle */
    const orc_pt* vb = pass == 0 ? v2 : v1;
    orc_pt AB = vb[0], DA = vb[3];
    float ABdotAB = orc_dot(AB, AB), ADdotAD = orc_dot(DA, DA);
    for (int i = 0; i < 4; ++i) {
      orc_pt AP = { pa[i].x - pb[0].x, pa[i].y - pb[0].y };
      float APdotAB = orc_dot(AP, AB);
      float APdotAD = -orc_dot(AP, DA);
      if (((double)APdotAB > -EPS) && ((double)APdotAD > -EPS) &&
          ((double)APdotAB < (double)ABdotAB + EPS) && ((double)APdotAD < (double)ADdotAD + EPS))
        out[num++] = pa[i];
    }
  }
  return num;
}

static int orc_hull(const orc_pt* p, int n, orc_pt* q) { /* :166-320, shift_to_zero = true */
  int t = 0;
  for (int i = 1; i < n; ++i)
    if (p[i].y < p[t].y || (p[i].y == p[t].y && p[i].x < p[t].x)) t = i;
  orc_pt start = p[t];
  for (int i = 0; i < n; ++i) { q[i].x = p[i].x - start.x; q[i].y = p[i].y - start.y; }
  orc_pt tmp = q[0]; q[0] = q[t]; q[t] = tmp;
  float dist[24];
  for (int i = 0; i < n; ++i) dist[i] = orc_dot(q[i], q[i]);
  for (int i = 1; i < n - 1; ++i) for (int j = i + 1; j < n; ++j) { /* :242-255 */
    float cp = orc_cross(q[i], q[j]);
    if (((double)cp < -1e-6) || (fabs((double)cp) < 1e-6 && dist[i] > dist[j])) {
      orc_pt qt = q[i]; q[i] = q[j]; q[j] = qt;
      float dt = dist[i]; dist[i] = dist[j]; dist[j] = dt;
    }
  }
  for (int i = 0; i < n; ++i) dist[i] = orc_dot(q[i], q[i]); /* CPU branch :257-260 */
  int k;
  for (k = 1; k < n; ++k) if ((double)dist[k] > 1e-8) break;
  if (k == n) { q[0] = p[t]; return 1; }
  q[1] = q[k];
  int m = 2;
  for (int i = k + 1; i < n; ++i) {
    while (m > 1) {
      orc_pt q1 = { q[i].x - q[m - 2].x, q[i].y - q[m - 2].y };
      orc_pt q2 = { q[m - 1].x - q[m - 2].x, q[m - 1].y - q[m - 2].y };
      if (q1.x * q2.y >= q2.x * q1.y) m--; else break; /* :294-298 */
    }
    q[m++] = q[i];
  }
  return m;
}

static float orc_single_iou(const float* b1, const float* b2) { /* :363-390 */
  double sx = (double)(b1[0] + b2[0]) / 2.0, sy = (double)(b1[1] + b2[1]) / 2.0;
  float x1 = (float)((double)b1[0] - sx), y1 = (float)((double)b1[1] - sy);
  float x2 = (float)((double)b2[0] - sx), y2 = (float)((double)b2[1] - sy);
  float area1 = b1[2] * b1[3], area2 = b2[2] * b2[3];
  if ((double)area1 < 1e-14 || (double)area2 < 1e-14) return 0.f;
  orc_pt p1[4], p2[4], ip[24], op[24];
  orc_vertices(x1, y1, b1[2], b1[3], b1[4], p1);
  orc_vertices(x2, y2, b2[2], b2[3], b2[4], p2);
  int num = orc_intersections(p1, p2, ip);
  float inter;
  if (num <= 2) inter = 0.f;
  else {
    int m = orc_hull(ip, num, op);
    if (m <= 2) inter = 0.f;
    else { /* polygon_area :322-334 */
      float area = 0.f;
      for (int i = 1; i < m - 1; ++i) {
        orc_pt a = { op[i].x - op[0].x, op[i].y - op[0].y };
        orc_pt b = { op[i + 1].x - op[0].x, op[i + 1].y - op[0].y };
        area += fabsf(orc_cross(a, b));
      }
      inter = (float)((double)area / 2.0);
    }
  }
  return inter / (area1 + area2 - inter);
}

/* box_iou_rotated_cpu.cpp:7-37 */
ORC_API void orc_box_iou_rotated(const float* b1, int64_t N, const float* b2, int64_t M, float* out) {
  for (int64_t i = 0; i < N; ++i) for (int64_t j = 0; j < M; ++j)
    out[i * M + j] = orc_single_iou(b1 + 5 * i, b2 + 5 * j);
}

/* nms_rotated_cpu.cpp:7-60 (note `>=`, unlike the axis-aligned strict `>`) */
ORC_API int64_t orc_nms_rotated(const float* dets, const float* scores, int64_t M, double thr,
                                int64_t* keep) {
  int64_t* order = orc_order_desc(scores, M);
  uint8_t* sup = (uint8_t*)calloc((size_t)(M ? M : 1), 1);
  int64_t nk = 0;
  for (int64_t _i = 0; _i < M; ++_i) {
    int64_t i = order[_i];
    if (sup[i]) continue;
    keep[nk++] = i;
    for (int64_t _j = _i + 1; _j < M; ++_j) {
      int64_t j = order[_j];
      if (sup[j]) continue;
      float ovr = orc_single_iou(dets + 5 * i, dets + 5 * j);
      if ((double)ovr >= thr) sup[j] = 1;
    }
  }
  free(order); free(sup);
  return nk;
}

/* ------------------------------------------------------------------------------------------
 * Deformable convolution v1/v2.  Reference: detectron2/layers/csrc/deformable/
 * deform_conv_cuda_kernel.cu (im2col :216-288, bilinear :96-130, col2im :291-363,
 * col2im_coord :366-452, modulated :785-1066) and host loops deform_conv_cuda.cu
 * (:382-431 fwd GEMM, :549-619 bwd input, :756-812 bwd weight, :927-972, :1087-1215).
 * Written as a direct (column-free) evaluation: columns[] values are computed on the fly.
 * mask == NULL -> DCNv1; bias == NULL -> no bias.
 * ---------------------------------------------------------------------------------------- */
typedef struct {
  int N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, G, DG, Ho, Wo;
} orc_dc;

static float orc_dc_bilinear(const float* im, int H, int W, float h, float w) { /* :96-130 */
  int hl = (int)floorf(h), wl = (int)floorf(w), hh_ = hl + 1, wh = wl + 1;
  float lh = h - (float)hl, lw = w - (float)wl, hh = 1.f - lh, hw = 1.f - lw;
  float v1 = (hl >= 0 && wl >= 0) ? im[hl * W + wl] : 0.f;
  float v2 = (hl >= 0 && wh <= W - 1) ? im[hl * W + wh] : 0.f;
  float v3 = (hh_ <= H - 1 && wl >= 0) ? im[hh_ * W + wl] : 0.f;
  float v4 = (hh_ <= H - 1 && wh <= W - 1) ? im[hh_ * W + wh] : 0.f;
  return hh * hw * v1 + hh * lw * v2 + lh * hw * v3 + lh * lw * v4;
}

/* :163-214 get_coordinate_weight: d(bilinear)/dh (dir 0) or /dw (dir 1) */
static float orc_dc_coord_w(const float* im, int H, int W, float h, float w, int dir) {
  if (h <= -1 || h >= H || w <= -1 || w >= W) return 0.f;
  int hl = (int)floorf(h), wl = (int)floorf(w), hh = hl + 1, wh = wl + 1;
  float r = 0.f;
  if (dir == 0) {
    if (hl >= 0 && wl >= 0) r += -1 * ((float)wl + 1 - w) * im[hl * W + wl];
    if (hl >= 0 && wh <= W - 1) r += -1 * (w - (float)wl) * im[hl * W + wh];
    if (hh <= H - 1 && wl >= 0) r += ((float)wl + 1 - w) * im[hh * W + wl];
    if (hh <= H - 1 && wh <= W - 1) r += (w - (float)wl) * im[hh * W + wh];
  } else {
    if (hl >= 0 && wl >= 0) r += -1 * ((float)hl + 1 - h) * im[hl * W + wl];
    if (hl >= 0 && wh <= W - 1) r += ((float)hl + 1 - h) * im[hl * W + wh];
    if (hh <= H - 1 && wl >= 0) r += -1 * (h - (float)hl) * im[hh * W + wl];
    if (hh <= H - 1 && wh <= W - 1) r += (h - (float)hl) * im[hh * W + wh];
  }
  return r;
}

static void orc_dc_pos(const orc_dc* d, const float* offset, int b, int dg, int i, int j, int ho,
                       int wo, float* h, float* w) { /* :263-272 */
  int kp = i * d->kw + j;
  size_t base = ((size_t)(b * d->DG + dg) * 2 * d->kh * d->kw) * d->Ho * d->Wo;
  float oh = offset[base + ((size_t)(2 * kp) * d->Ho + ho) * d->Wo + wo];
  float ow = offset[base + ((size_t)(2 * kp + 1) * d->Ho + ho) * d->Wo + wo];
  *h = (float)(ho * d->sh - d->ph + i * d->dh) + oh;
  *w = (float)(wo * d->sw - d->pw + j * d->dw) + ow;
}
static float orc_dc_mask(const orc_dc* d, const float* mask, int b, int dg, int kp, int ho, int wo) {
  if (!mask) return 1.f;
  return mask[(((size_t)(b * d->DG + dg) * d->kh * d->kw + kp) * d->Ho + ho) * d->Wo + wo];
}

ORC_API void orc_deform_conv_forward(const float* x, const float* offset, const float* mask,
                                     const float* weight, const float* bias, int N, int Cin, int H,
                                     int W, int Cout, int kh, int kw, int sh, int sw, int ph, int pw,
                                     int dh, int dw, int G, int DG, float* out) {
  orc_dc d = { N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, G, DG,
               (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1 };
  int cpg = Cin / G, opg = Cout / G, cpdg = Cin / DG, K = cpg * kh * kw;
  float* col = (float*)malloc(sizeof(float) * (size_t)Cin * kh * kw);
  for (int b = 0; b < N; ++b) for (int ho = 0; ho < d.Ho; ++ho) for (int wo = 0; wo < d.Wo; ++wo) {
    for (int c = 0; c < Cin; ++c) { /* one column of columns[] (:238-287, :862) */
      int dg = c / cpdg;
      const float* im = x + ((size_t)b * Cin + c) * H * W;
      for (int i = 0; i < kh; ++i) for (int j = 0; j < kw; ++j) {
        float h, w; orc_dc_pos(&d, offset, b, dg, i, j, ho, wo, &h, &w);
        float v = 0.f;
        if (h > -1 && w > -1 && h < H && w < W) v = orc_dc_bilinear(im, H, W, h, w);
        col[(c * kh + i) * kw + j] = v * orc_dc_mask(&d, mask, b, dg, i * kw + j, ho, wo);
      }
    }
    for (int g = 0; g < G; ++g) for (int m = 0; m < opg; ++m) { /* deform_conv_cuda.cu:409-414 */
      const float* wr = weight + (size_t)(g * opg + m) * K;
      const float* cr = col + (size_t)g * K;
      double acc = 0.0; /* accumulate in double: the oracle is the low-noise side of the 1e-4 check */
      for (int k = 0; k < K; ++k) acc += (double)wr[k] * (double)cr[k];
      if (bias) acc += (double)bias[g * opg + m];
      out[(((size_t)b * Cout + g * opg + m) * d.Ho + ho) * d.Wo + wo] = (float)acc;
    }
  }
  free(col);
}

/* grads are accumulated in double and written (not added) to the outputs; pass NULL to skip */
ORC_API void orc_deform_conv_backward(const float* x, const float* offset, const float* mask,
                                      const float* weight, const float* gout, int N, int Cin, int H,
                                      int W, int Cout, int kh, int kw, int sh, int sw, int ph,
                                      int pw, int dh, int dw, int G, int DG, int with_bias,
                                      float* gx, float* goff, float* gmask, float* gw, float* gb) {
  orc_dc d = { N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, G, DG,
               (H + 2 * ph - (dh * (kh - 1) + 1)) / sh + 1, (W + 2 * pw - (dw * (kw - 1) + 1)) / sw + 1 };
  int cpg = Cin / G, opg = Cout / G, cpdg = Cin / DG, K = cpg * kh * kw, KK = kh * kw;
  size_t nx = (size_t)N * Cin * H * W, noff = (size_t)N * DG * 2 * KK * d.Ho * d.Wo;
  size_t nm = (size_t)N * DG * KK * d.Ho * d.Wo, nw = (size_t)Cout * K;
  double* dgx = (double*)calloc(nx, sizeof(double));
  double* dgo = (double*)calloc(noff, sizeof(double));
  double* dgm = (double*)calloc(nm ? nm : 1, sizeof(double));
  double* dgw = (double*)calloc(nw, sizeof(double));
  double* dgb = (double*)calloc((size_t)Cout, sizeof(double));
  for (int b = 0; b < N; ++b) for (int ho = 0; ho < d.Ho; ++ho) for (int wo = 0; wo < d.Wo; ++wo) {
    for (int c = 0; c < Cin; ++c) {
      int dg = c / cpdg, g = c / cpg, cl = c % cpg;
      const float* im = x + ((size_t)b * Cin + c) * H * W;
      double* gim = dgx + ((size_t)b * Cin + c) * H * W;
      for (int i = 0; i < kh; ++i) for (int j = 0; j < kw; ++j) {
        int kp = i * kw + j, krow = (cl * kh + i) * kw + j;
        /* grad_columns = W_g^T . grad_out_g (deform_conv_cuda.cu:566-572) */
        double gcol = 0.0;
        for (int m = 0; m < opg; ++m)
          gcol += (double)weight[(size_t)(g * opg + m) * K + krow] *
                  (double)gout[(((size_t)b * Cout + g * opg + m) * d.Ho + ho) * d.Wo + wo];
        float h, w; orc_dc_pos(&d, offset, b, dg, i, j, ho, wo, &h, &w);
        float mk = orc_dc_mask(&d, mask, b, dg, kp, ho, wo);
        int inside = (h > -1 && w > -1 && h < H && w < W);
        float val = inside ? orc_dc_bilinear(im, H, W, h, w) : 0.f;
        /* grad_weight += grad_out . columns^T (deform_conv_cuda.cu:790-799) */
        for (int m = 0; m < opg; ++m)
          dgw[(size_t)(g * opg + m) * K + krow] +=
              (double)gout[(((size_t)b * Cout + g * opg + m) * d.Ho + ho) * d.Wo + wo] *
              (double)(val * mk);
        if (!inside) continue;
        /* grad_mask (:1031-1038,1053-1064) */
        if (mask)
          dgm[(((size_t)(b * DG + dg) * KK + kp) * d.Ho + ho) * d.Wo + wo] += gcol * (double)val;
        /* grad_offset (:390-451, modulated :1048) */
        size_t ob = ((size_t)(b * DG + dg) * 2 * KK) * d.Ho * d.Wo;
        dgo[ob + ((size_t)(2 * kp) * d.Ho + ho) * d.Wo + wo] +=
            gcol * (double)mk * (double)orc_dc_coord_w(im, H, W, h, w, 0);
        dgo[ob + ((size_t)(2 * kp + 1) * d.Ho + ho) * d.Wo + wo] +=
            gcol * (double)mk * (double)orc_dc_coord_w(im, H, W, h, w, 1);
        /* grad_input: scatter to the in-range taps with the forward weights (:313-362) */
        int hl = (int)floorf(h), wl = (int)floorf(w);
        float lh = h - (float)hl, lw = w - (float)wl;
        double gm = gcol * (double)mk;
        if (hl >= 0 && wl >= 0) gim[hl * W + wl] += gm * (double)((1.f - lh) * (1.f - lw));
        if (hl >= 0 && wl + 1 <= W - 1) gim[hl * W + wl + 1] += gm * (double)((1.f - lh) * lw);
        if (hl + 1 <= H - 1 && wl >= 0) gim[(hl + 1) * W + wl] += gm * (double)(lh * (1.f - lw));
        if (hl + 1 <= H - 1 && wl + 1 <= W - 1) gim[(hl + 1) * W + wl + 1] += gm * (double)(lh * lw);
      }
    }
    if (with_bias) /* deform_conv_cuda.cu:1197-1203 */
      for (int m = 0; m < Cout; ++m)
        dgb[m] += (double)gout[(((size_t)b * Cout + m) * d.Ho + ho) * d.Wo + wo];
  }
  if (gx) for (size_t i = 0; i < nx; ++i) gx[i] = (float)dgx[i];
  if (goff) for (size_t i = 0; i < noff; ++i) goff[i] = (float)dgo[i];
  if (gmask && mask) for (size_t i = 0; i < nm; ++i) gmask[i] = (float)dgm[i];
  if (gw) for (size_t i = 0; i < nw; ++i) gw[i] = (float)dgw[i];
  if (gb && with_bias) for (int i = 0; i < Cout; ++i) gb[i] = (float)dgb[i];
  free(dgx); free(dgo); free(dgm); free(dgw); free(dgb);
}

/* ------------------------------------------------------------------------------------------
 * paste_masks_in_image.  Reference: detectron2/layers/mask_ops.py:17-69 (_do_paste_mask) and
 * :74-147, with F.grid_sample(bilinear, zeros padding, align_corners=False) semantics:
 * gx = (px+0.5-x0)/(x1-x0)*2-1 (:53-54), unnormalise ((g+1)*M-1)/2, corners nw/ne/sw/se with
 * weights (se-ix)*(se-iy)..., out-of-range taps contribute 0.  threshold >= 0 -> (v >= thr)
 * as 0/1 bytes; threshold < 0 -> (uint8)(v*255) (:137-141).  soft (optional) gets the float v.
 * ---------------------------------------------------------------------------------------- */
ORC_API void orc_paste_masks(const float* masks, const float* boxes, int N, int M, int H, int W,
                             float threshold, uint8_t* out, float* soft) {
  for (int n = 0; n < N; ++n) {
    const float* mk = masks + (size_t)n * M * M;
    float x0 = boxes[4 * n], y0 = boxes[4 * n + 1], x1 = boxes[4 * n + 2], y1 = boxes[4 * n + 3];
    for (int py = 0; py < H; ++py) {
      float gy = ((float)py + 0.5f - y0) / (y1 - y0) * 2.f - 1.f;
      float iy = ((gy + 1.f) * (float)M - 1.f) / 2.f;
      for (int px = 0; px < W; ++px) {
        float gx = ((float)px + 0.5f - x0) / (x1 - x0) * 2.f - 1.f;
        float ix = ((gx + 1.f) * (float)M - 1.f) / 2.f;
        float fx = floorf(ix), fy = floorf(iy);
        float v = 0.f;
        /* NaN/inf coordinates (degenerate boxes) fail every in-range test -> 0 */
        if (ix == ix && iy == iy && fabsf(ix) < 1e9f && fabsf(iy) < 1e9f) {
          int xw = (int)fx, yn = (int)fy, xe = xw + 1, ys = yn + 1;
          float tnw = ((float)xe - ix) * ((float)ys - iy), tne = (ix - (float)xw) * ((float)ys - iy);
          float tsw = ((float)xe - ix) * (iy - (float)yn), tse = (ix - (float)xw) * (iy - (float)yn);
          if (yn >= 0 && yn < M && xw >= 0 && xw < M) v += mk[yn * M + xw] * tnw;
          if (yn >= 0 && yn < M && xe >= 0 && xe < M) v += mk[yn * M + xe] * tne;
          if (ys >= 0 && ys < M && xw >= 0 && xw < M) v += mk[ys * M + xw] * tsw;
          if (ys >= 0 && ys < M && xe >= 0 && xe < M) v += mk[ys * M + xe] * tse;
        }
        size_t o = ((size_t)n * H + py) * W + px;
        if (soft) soft[o] = v;
        if (threshold >= 0.f) out[o] = (v >= threshold) ? 1 : 0;
        else out[o] = (uint8_t)(v * 255.f);
      }
    }
  }
}
