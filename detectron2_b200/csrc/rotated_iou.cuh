// Rotated-box IoU device function shared by nms.cu (rotated NMS, d2b_box_iou_rotated) and match.cu (anchor / proposal
// matching).  Include it only from translation units compiled with -fmad=false: the parity target rounds every float
// expression separately (see DESIGN.md "bit-exactness").
#pragma once

namespace {

// ------------------------------------------------------------------------------------------------
// rotated IoU, after box_iou_rotated_utils.h (CPU branch).  float / double promotions follow the reference's
// C++ expression types exactly; see oracle/d2_oracle.c for the line-by-line citations.
// ------------------------------------------------------------------------------------------------
struct P2 {
  float x, y;
};
__device__ __forceinline__ float crs(P2 a, P2 b) { return a.x * b.y - b.x * a.y; }
__device__ __forceinline__ float dt(P2 a, P2 b) { return a.x * b.x + a.y * b.y; }
__device__ __forceinline__ P2 sub(P2 a, P2 b) { return P2{a.x - b.x, a.y - b.y}; }

__device__ __forceinline__ void rot_vertices(float xc, float yc, float w, float h, float a, P2* p) {
  double theta = (double)a * 0.01745329251;
  float c2 = (float)cos(theta) * 0.5f, s2 = (float)sin(theta) * 0.5f;
  p[0].x = xc + s2 * h + c2 * w;
  p[0].y = yc + c2 * h - s2 * w;
  p[1].x = xc - s2 * h + c2 * w;
  p[1].y = yc - c2 * h - s2 * w;
  p[2].x = 2 * xc - p[0].x;
  p[2].y = 2 * yc - p[0].y;
  p[3].x = 2 * xc - p[1].x;
  p[3].y = 2 * yc - p[1].y;
}

__device__ float rotated_iou(const float* __restrict__ b1, const float* __restrict__ b2) {
  const double sx = (double)(b1[0] + b2[0]) / 2.0, sy = (double)(b1[1] + b2[1]) / 2.0;
  const float x1 = (float)((double)b1[0] - sx), y1 = (float)((double)b1[1] - sy);
  const float x2 = (float)((double)b2[0] - sx), y2 = (float)((double)b2[1] - sy);
  const float area1 = b1[2] * b1[3], area2 = b2[2] * b2[3];
  if ((double)area1 < 1e-14 || (double)area2 < 1e-14) return 0.f;

  P2 p1[4], p2[4], v1[4], v2[4];
  rot_vertices(x1, y1, b1[2], b1[3], b1[4], p1);
  rot_vertices(x2, y2, b2[2], b2[3], b2[4], p2);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    v1[i] = sub(p1[(i + 1) & 3], p1[i]);
    v2[i] = sub(p2[(i + 1) & 3], p2[i]);
  }
  P2 ip[24];
  int num = 0;
  const double EPS = 1e-5;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      float det = crs(v2[j], v1[i]);
      if (fabs((double)det) <= 1e-14) continue;
      P2 v12 = sub(p2[j], p1[i]);
      float t1 = crs(v2[j], v12) / det;
      float t2 = crs(v1[i], v12) / det;
      if ((double)t1 > -EPS && (double)t1 < (double)1.0f + EPS && (double)t2 > -EPS &&
          (double)t2 < (double)1.0f + EPS) {
        ip[num].x = p1[i].x + v1[i].x * t1;
        ip[num].y = p1[i].y + v1[i].y * t1;
        ++num;
      }
    }
  }
  {  // vertices of rect1 inside rect2
    const P2 AB = v2[0], DA = v2[3];
    const float ABdotAB = dt(AB, AB), ADdotAD = dt(DA, DA);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      P2 AP = sub(p1[i], p2[0]);
      float APdotAB = dt(AP, AB), APdotAD = -dt(AP, DA);
      if (((double)APdotAB > -EPS) && ((double)APdotAD > -EPS) && ((double)APdotAB < (double)ABdotAB + EPS) &&
          ((double)APdotAD < (double)ADdotAD + EPS))
        ip[num++] = p1[i];
    }
  }
  {  // vertices of rect2 inside rect1
    const P2 AB = v1[0], DA = v1[3];
    const float ABdotAB = dt(AB, AB), ADdotAD = dt(DA, DA);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      P2 AP = sub(p2[i], p1[0]);
      float APdotAB = dt(AP, AB), APdotAD = -dt(AP, DA);
      if (((double)APdotAB > -EPS) && ((double)APdotAD > -EPS) && ((double)APdotAB < (double)ABdotAB + EPS) &&
          ((double)APdotAD < (double)ADdotAD + EPS))
        ip[num++] = p2[i];
    }
  }
  float inter = 0.f;
  if (num > 2) {
    // Graham scan, shift_to_zero variant
    int t = 0;
    for (int i = 1; i < num; ++i)
      if (ip[i].y < ip[t].y || (ip[i].y == ip[t].y && ip[i].x < ip[t].x)) t = i;
    const P2 start = ip[t];
    P2 q[24];
    float dist[24];
    for (int i = 0; i < num; ++i) q[i] = sub(ip[i], start);
    {
      P2 tmp = q[0];
      q[0] = q[t];
      q[t] = tmp;
    }
    for (int i = 0; i < num; ++i) dist[i] = dt(q[i], q[i]);
    for (int i = 1; i < num - 1; ++i)
      for (int j = i + 1; j < num; ++j) {
        float cp = crs(q[i], q[j]);
        if (((double)cp < -1e-6) || (fabs((double)cp) < 1e-6 && dist[i] > dist[j])) {
          P2 qt = q[i];
          q[i] = q[j];
          q[j] = qt;
          float d = dist[i];
          dist[i] = dist[j];
          dist[j] = d;
        }
      }
    // the CPU reference recomputes dist after the sort; after the swaps above dist[] already travels with q[],
    // and dot(q,q) is a pure function of q, so the recomputed values are identical.
    int k;
    for (k = 1; k < num; ++k)
      if ((double)dist[k] > 1e-8) break;
    int m;
    if (k == num) {
      m = 1;
    } else {
      q[1] = q[k];
      m = 2;
      for (int i = k + 1; i < num; ++i) {
        while (m > 1) {
          P2 q1 = sub(q[i], q[m - 2]), q2 = sub(q[m - 1], q[m - 2]);
          if (q1.x * q2.y >= q2.x * q1.y) m--;
          else break;
        }
        q[m++] = q[i];
      }
    }
    if (m > 2) {
      float area = 0.f;
      for (int i = 1; i < m - 1; ++i) area += fabsf(crs(sub(q[i], q[0]), sub(q[i + 1], q[0])));
      inter = (float)((double)area / 2.0);
    }
  }
  return inter / (area1 + area2 - inter);
}

}  // namespace
