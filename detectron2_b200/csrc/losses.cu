// Box-branch training losses: RPN / RRPN and RetinaNet (dense, per anchor) and Fast R-CNN (per proposal), forward and
// backward, for all images of the batch at once and without a host synchronisation.
//
//   d2b_dense_loss_forward / _backward   RPN.losses (proposal_generator/rpn.py:366-429) and RetinaNet.losses
//       (meta_arch/retinanet.py:160-210): the sigmoid focal loss (fvcore; gamma = 0 and alpha < 0 is the RPN's
//       binary_cross_entropy_with_logits) over the valid rows of the per-level logits, and the smooth-L1 loss of
//       _dense_box_regression_loss (modeling/box_regression.py:310-369) over the positive rows, with the targets of
//       Box2BoxTransform[Rotated].get_deltas computed on the fly.  One launch: classification CTAs stream the logits
//       (16-byte vectors, the row label re-read only when the row changes), regression CTAs own one anchor row per
//       thread; a second single-CTA launch adds the per-CTA partials in a fixed order.
//       With D2B_LOSS_LINEAR_GIOU they are FCOS.losses + compute_ctrness_targets (meta_arch/fcos.py:193-251): the same
//       kernel with kFcos -- GIoU of Box2BoxTransformLinear's decode and, on the positive rows, the centerness BCE as a
//       third sum.
//   d2b_frcnn_loss_forward / _backward   FastRCNNOutputLayers.losses / box_reg_loss (roi_heads/fast_rcnn.py:307-352,
//       424-463) and _log_classification_stats (:88-115): one warp per proposal row -- max, log-sum-exp, argmax, the class
//       gather of the deltas, the targets and smooth-L1 -- then the same fixed-order finish.
//
// Reductions are deterministic (per-CTA partials, no float atomics): loss and gradients are bitwise reproducible.
// Compiled with -fmad=false so that the targets round like the reference's separate torch ops.
#include <climits>
#include <cmath>

#include "boxes.cuh"
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kItems = 4;  // 16-byte vectors per thread in one classification CTA

template <class T> struct alignas(16) Vec {
  static constexpr int N = 16 / sizeof(T);
  T v[N];
};

// fvcore smooth_l1_loss: |d| for beta < 1e-5, else 0.5 d^2 / beta inside |d| < beta and |d| - 0.5 beta outside.
// g = d loss / d d, through torch's abs backward: sign(d), which is 0 at 0 and for NaN.
__device__ __forceinline__ float smooth_l1(float diff, float beta, float& g) {
  const float n = fabsf(diff);
  const float sgn = diff > 0.f ? 1.f : (diff < 0.f ? -1.f : 0.f);
  if (beta < 1e-5f) {
    g = sgn;
    return n;
  }
  if (n < beta) {
    g = n / beta * sgn;
    return 0.5f * (n * n) / beta;
  }
  g = sgn;
  return n - 0.5f * beta;
}

// torch.max / torch.min of two tensors: NaN propagates; the backward splits the gradient in half at a tie
__device__ __forceinline__ float tmax(float a, float b) { return a != a ? a : (b != b ? b : (a > b ? a : b)); }
__device__ __forceinline__ float tmin(float a, float b) { return a != a ? a : (b != b ? b : (a < b ? a : b)); }
__device__ __forceinline__ float share_max(float a, float b) { return a > b ? 1.f : (a == b ? 0.5f : 0.f); }
__device__ __forceinline__ float share_min(float a, float b) { return a < b ? 1.f : (a == b ? 0.5f : 0.f); }

// fvcore giou_loss (eps = 1e-7) of the predicted box p against q, both (x1, y1, x2, y2); g = d loss / d p as torch's
// autograd forms it.  `ordered` is fvcore's assertion x2 >= x1 and y2 >= y1 on both boxes.
__device__ __forceinline__ float giou_loss(const float (&p)[4], const float* q, float (&g)[4], bool& ordered) {
  const float eps = 1e-7f;
  ordered = p[2] >= p[0] && p[3] >= p[1] && q[2] >= q[0] && q[3] >= q[1];
  const float xk1 = tmax(p[0], q[0]), yk1 = tmax(p[1], q[1]), xk2 = tmin(p[2], q[2]), yk2 = tmin(p[3], q[3]);
  const bool inter = (yk2 > yk1) && (xk2 > xk1);
  const float iw = xk2 - xk1, ih = yk2 - yk1;
  const float I = inter ? iw * ih : 0.f;
  const float pw = p[2] - p[0], ph = p[3] - p[1];
  const float U = pw * ph + (q[2] - q[0]) * (q[3] - q[1]) - I;
  const float iou = I / (U + eps);
  const float xc1 = tmin(p[0], q[0]), yc1 = tmin(p[1], q[1]), xc2 = tmax(p[2], q[2]), yc2 = tmax(p[3], q[3]);
  const float cw = xc2 - xc1, ch = yc2 - yc1;
  const float C = cw * ch;
  const float loss = 1.f - (iou - (C - U) / (C + eps));
  // loss = 1 - I / (U + eps) + (C - U) / (C + eps) with U = area_p + area_q - I
  const float dU = I / ((U + eps) * (U + eps)) - 1.f / (C + eps);
  const float dI = -1.f / (U + eps) - dU;
  const float dC = (U + eps) / ((C + eps) * (C + eps));
  g[0] = -dU * ph;
  g[2] = dU * ph;
  g[1] = -dU * pw;
  g[3] = dU * pw;
  if (inter) {
    g[0] += -dI * ih * share_max(p[0], q[0]);
    g[1] += -dI * iw * share_max(p[1], q[1]);
    g[2] += dI * ih * share_min(p[2], q[2]);
    g[3] += dI * iw * share_min(p[3], q[3]);
  }
  g[0] += -dC * ch * share_min(p[0], q[0]);
  g[1] += -dC * cw * share_min(p[1], q[1]);
  g[2] += dC * ch * share_max(p[2], q[2]);
  g[3] += dC * cw * share_max(p[3], q[3]);
  return loss;
}

// GIoU regression of one row: the deltas decoded on the anchor / proposal (apply_deltas), the loss against the GT box,
// and g = d loss / d deltas through the decode and torch.clamp(max=scale_clamp).
__device__ __forceinline__ float giou_row(const float* an, const float (&d)[4], const float* gt, const BoxWeights& w,
                                         float scale_clamp, float (&g)[4], bool& ordered) {
  const DecodedBox b = apply_deltas(make_float4(an[0], an[1], an[2], an[3]), make_float4(d[0], d[1], d[2], d[3]), w.w[0],
                                    w.w[1], w.w[2], w.w[3], scale_clamp);
  const float p[4] = {b.x1, b.y1, b.x2, b.y2};
  float gp[4];
  const float loss = giou_loss(p, gt, gp, ordered);
  const float gcx = gp[0] + gp[2], gcy = gp[1] + gp[3];
  const float gpw = 0.5f * gp[2] - 0.5f * gp[0], gph = 0.5f * gp[3] - 0.5f * gp[1];
  g[0] = gcx * b.widths / w.w[0];
  g[1] = gcy * b.heights / w.w[1];
  g[2] = b.pass_w ? gpw * b.widths * b.ew / w.w[2] : 0.f;
  g[3] = b.pass_h ? gph * b.heights * b.eh / w.w[3] : 0.f;
  return loss;
}

// FCOS GIoU regression of one row: the deltas decoded by Box2BoxTransformLinear.apply_deltas on the anchor point, the loss
// against the GT box, and g = d loss / d deltas through the decode and the relu (threshold_backward: 0 where delta <= 0).
__device__ __forceinline__ float giou_row_linear(const float* an, const float (&d)[4], const float* gt, float (&g)[4],
                                                bool& ordered) {
  const LinearBox b = apply_deltas_linear(make_float4(an[0], an[1], an[2], an[3]), make_float4(d[0], d[1], d[2], d[3]));
  const float p[4] = {b.x1, b.y1, b.x2, b.y2};
  float gp[4];
  const float loss = giou_loss(p, gt, gp, ordered);
  g[0] = d[0] <= 0.f ? 0.f : -gp[0] * b.sw;
  g[1] = d[1] <= 0.f ? 0.f : -gp[1] * b.sh;
  g[2] = d[2] <= 0.f ? 0.f : gp[2] * b.sw;
  g[3] = d[3] <= 0.f ? 0.f : gp[3] * b.sh;
  return loss;
}

// FCOS.compute_ctrness_targets (meta_arch/fcos.py:240-251) of one row: Box2BoxTransformLinear.get_deltas (l, t, r, b
// divided by the stride, box_regression.py:243-273), then sqrt((min(l, r) / max(l, r)) * (min(t, b) / max(t, b))).
__device__ __forceinline__ float ctrness_target(const float* an, const float* gt) {
  const float cx = 0.5f * (an[0] + an[2]), cy = 0.5f * (an[1] + an[3]);
  const float sw = an[2] - an[0], sh = an[3] - an[1];
  const float l = (cx - gt[0]) / sw, t = (cy - gt[1]) / sh, r = (gt[2] - cx) / sw, b = (gt[3] - cy) / sh;
  return sqrtf((tmin(l, r) / tmax(l, r)) * (tmin(t, b) / tmax(t, b)));
}

// fvcore sigmoid_focal_loss of one element; g = d loss / d x.  ce = binary_cross_entropy_with_logits as torch writes it,
// (1 - t) x - log_sigmoid(x) with log_sigmoid(x) = min(x, 0) - log1p(exp(-|x|)).  gamma = 0 is taken analytically
// (g = sigmoid(x) - t, where autograd of (1 - p_t) ** 0 would give 0 * inf at saturation).
__device__ __forceinline__ float focal(float x, float t, float gamma, float alpha, float& g) {
  const float ce = (1.f - t) * x - (fminf(x, 0.f) - log1pf(expf(-fabsf(x))));
  const float p = 1.f / (1.f + expf(-x));
  float loss;
  if (gamma == 0.f) {
    loss = ce;
    g = p - t;
  } else {
    const float q = 1.f - (p * t + (1.f - p) * (1.f - t));  // 1 - p_t
    const float m = gamma == 2.f ? q * q : powf(q, gamma);
    loss = ce * m;
    // binary targets: d/dx [ce (1 - p_t)^gamma] = -+ q^gamma (q + gamma (1 - q) ce), minus for t = 1
    const float d = m * (q + gamma * (1.f - q) * ce);
    g = t > 0.5f ? -d : d;
  }
  if (alpha >= 0.f) {
    const float at = alpha * t + (1.f - alpha) * (1.f - t);
    loss = at * loss;
    g = at * g;
  }
  return loss;
}

// ---- per-CTA partials and the fixed-order finish ------------------------------------------------------------------
struct Partial {
  float sum[3];      // classification, regression, FCOS centerness
  int status;
  long long cnt[4];  // dense: num_pos, num_neg; Fast R-CNN: num_fg, num_accurate, fg_num_accurate, num_false_negative
};

struct BlockRed {
  float f[3][kWarps];
  long long c[4][kWarps];
  int s[kWarps];
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ long long warp_sum(long long v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Sums of the CTA in a fixed order (lanes by butterfly, then warps 0..7), written by thread 0 to `out`.
__device__ __forceinline__ void block_partial(float s0, float s1, float s2, const long long (&c)[4], int status,
                                              BlockRed& red, Partial* __restrict__ out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  s0 = warp_sum(s0);
  s1 = warp_sum(s1);
  s2 = warp_sum(s2);
  long long w[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) w[i] = warp_sum(c[i]);
  status = __reduce_or_sync(0xffffffffu, (unsigned)status);
  if (lane == 0) {
    red.f[0][warp] = s0;
    red.f[1][warp] = s1;
    red.f[2][warp] = s2;
#pragma unroll
    for (int i = 0; i < 4; ++i) red.c[i][warp] = w[i];
    red.s[warp] = status;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    Partial p = {};
    for (int k = 0; k < kWarps; ++k) {
      p.sum[0] += red.f[0][k];
      p.sum[1] += red.f[1][k];
      p.sum[2] += red.f[2][k];
#pragma unroll
      for (int i = 0; i < 4; ++i) p.cnt[i] += red.c[i][k];
      p.status |= red.s[k];
    }
    *out = p;
  }
}

// Adds the partials in a fixed order; writes sums[0, nsums), counts[0, ncounts) and status.
__global__ void __launch_bounds__(kThreads) finish_kernel(const Partial* __restrict__ part, int nparts, int nsums,
                                                          int ncounts, float* __restrict__ sums,
                                                          int64_t* __restrict__ counts, int* __restrict__ status) {
  __shared__ double s_f[3][kThreads];
  __shared__ long long s_c[4][kThreads];
  __shared__ int s_s[kThreads];
  const int tid = threadIdx.x;
  double f0 = 0.0, f1 = 0.0, f2 = 0.0;
  long long c[4] = {0, 0, 0, 0};
  int st = 0;
  for (int i = tid; i < nparts; i += kThreads) {
    const Partial p = part[i];
    f0 += (double)p.sum[0];
    f1 += (double)p.sum[1];
    f2 += (double)p.sum[2];
#pragma unroll
    for (int k = 0; k < 4; ++k) c[k] += p.cnt[k];
    st |= p.status;
  }
  s_f[0][tid] = f0;
  s_f[1][tid] = f1;
  s_f[2][tid] = f2;
#pragma unroll
  for (int k = 0; k < 4; ++k) s_c[k][tid] = c[k];
  s_s[tid] = st;
  __syncthreads();
  for (int o = kThreads / 2; o; o >>= 1) {
    if (tid < o) {
      s_f[0][tid] += s_f[0][tid + o];
      s_f[1][tid] += s_f[1][tid + o];
      s_f[2][tid] += s_f[2][tid + o];
#pragma unroll
      for (int k = 0; k < 4; ++k) s_c[k][tid] += s_c[k][tid + o];
      s_s[tid] |= s_s[tid + o];
    }
    __syncthreads();
  }
  if (tid == 0) {
    for (int k = 0; k < nsums; ++k) sums[k] = (float)s_f[k][0];
    for (int k = 0; k < ncounts; ++k) counts[k] = s_c[k][0];
    *status = s_s[0];
  }
}

// ---- dense (RPN / RetinaNet) ---------------------------------------------------------------------------------------
struct DenseLevels {
  int L;
  const void* logits[D2B_MAX_LEVELS];
  const void* deltas[D2B_MAX_LEVELS];
  void* grad_logits[D2B_MAX_LEVELS];
  void* grad_deltas[D2B_MAX_LEVELS];
  const void* ctr[D2B_MAX_LEVELS];        // FCOS centerness logits [N, R_l]
  void* grad_ctr[D2B_MAX_LEVELS];
  int R[D2B_MAX_LEVELS];
  int a0[D2B_MAX_LEVELS + 1];             // first anchor of each level
  long long blk0[D2B_MAX_LEVELS + 1];     // first classification CTA of each level
};

// RPN labels: int8 {-1, 0, 1} with one logit per anchor; RetinaNet: int64 classes {-1, 0..K-1, K = background}.
struct LabelsI8 {
  using T = int8_t;
  static __device__ __forceinline__ float target(long long l, int) { return l == 1 ? 1.f : 0.f; }
  static __device__ __forceinline__ bool pos(long long l, int) { return l == 1; }
  static __device__ __forceinline__ bool neg(long long l, int) { return l == 0; }
  static __device__ __forceinline__ bool in_range(long long l, int) { return l >= -1 && l <= 1; }
};
struct LabelsI64 {
  using T = long long;
  static __device__ __forceinline__ float target(long long l, int c) { return l == c ? 1.f : 0.f; }
  static __device__ __forceinline__ bool pos(long long l, int K) { return l >= 0 && l < K; }
  static __device__ __forceinline__ bool neg(long long l, int K) { return l == K; }
  static __device__ __forceinline__ bool in_range(long long l, int K) { return l >= -1 && l <= K; }  // F.one_hot's range
};

struct DenseArgs {
  int N, K, Rtot;
  long long cls_blocks;
  const float* anchors;   // [Rtot, D]
  const float* gt_boxes;  // [N, Rtot, D]
  const void* labels;     // [N, Rtot]
  float gamma, alpha, beta;
  int giou;               // regression loss: 0 smooth-L1 on the get_deltas targets, 1 GIoU of the decoded boxes
  float scale_clamp;
  BoxWeights w;
  const float* grad_cls;  // backward: d loss / d classification sum (device scalar)
  const float* grad_reg;
  const float* grad_ctr;  // FCOS
  Partial* part;          // forward
};

// kFcos: FCOS.losses -- the regression is the GIoU of Box2BoxTransformLinear's decode, and the positive rows add the
// centerness term, binary_cross_entropy_with_logits against ctrness_target (the third sum; gradient sigmoid(x) - t).
template <int DT, class Box, class Lab, bool kBackward, bool kFcos = false>
__global__ void __launch_bounds__(kThreads) dense_loss_kernel(const DenseLevels P, const DenseArgs A) {
  using E = Elem<DT>;
  using T = typename E::T;
  using V = Vec<T>;
  constexpr int D = Box::D;
  __shared__ BlockRed red;
  const int tid = threadIdx.x;
  const long long b = blockIdx.x;
  const typename Lab::T* __restrict__ labels = (const typename Lab::T*)A.labels;
  float s_cls = 0.f, s_reg = 0.f, s_ctr = 0.f;
  long long cnt[4] = {0, 0, 0, 0};
  int status = 0;
  if (b < A.cls_blocks) {
    int l = 0;
    while (l + 1 < P.L && b >= P.blk0[l + 1]) ++l;
    const int Rl = P.R[l];
    const long long El = (long long)A.N * Rl * A.K;
    const long long e_begin = (b - P.blk0[l]) * (long long)(kThreads * kItems * V::N);
    const T* __restrict__ x = (const T*)P.logits[l];
    T* __restrict__ gx = kBackward ? (T*)P.grad_logits[l] : nullptr;
    const float gs = kBackward ? *A.grad_cls : 0.f;
#pragma unroll 1
    for (int it = 0; it < kItems; ++it) {
      const long long e0 = e_begin + ((long long)it * kThreads + tid) * V::N;
      if (e0 >= El) break;
      const bool full = e0 + V::N <= El;
      V in, out;
      if (full) {
        in = *reinterpret_cast<const V*>(x + e0);
      } else {
#pragma unroll
        for (int j = 0; j < V::N; ++j) in.v[j] = e0 + j < El ? x[e0 + j] : E::st(0.f);
      }
      long long row = e0 / A.K;
      int c = (int)(e0 - row * A.K);
      auto row_label = [&](long long rw) {
        const long long n = rw / Rl;
        return (long long)labels[n * A.Rtot + P.a0[l] + (rw - n * Rl)];
      };
      long long lab = row_label(row);
#pragma unroll
      for (int j = 0; j < V::N; ++j) {
        float g = 0.f;
        if (lab >= 0 && (full || e0 + j < El)) {  // ignored rows are never read: a NaN there does not reach the loss
          const float loss = focal(E::ld(in.v[j]), Lab::target(lab, c), A.gamma, A.alpha, g);
          s_cls += loss;
        }
        if (kBackward) out.v[j] = E::st(g * gs);
        if (++c == A.K && j + 1 < V::N) {
          c = 0;
          ++row;
          if (e0 + j + 1 < El) lab = row_label(row);
        }
      }
      if (kBackward) {
        if (full) {
          *reinterpret_cast<V*>(gx + e0) = out;
        } else {
          for (int j = 0; e0 + j < El; ++j) gx[e0 + j] = out.v[j];
        }
      }
    }
  } else {
    const long long row = (b - A.cls_blocks) * kThreads + tid;
    if (row < (long long)A.N * A.Rtot) {
      const int n = (int)(row / A.Rtot), a = (int)(row - (long long)n * A.Rtot);
      int l = 0;
      while (l + 1 < P.L && a >= P.a0[l + 1]) ++l;
      const int r = a - P.a0[l];
      const long long lab = labels[row];
      const float* an = A.anchors + (size_t)a * D;
      // get_deltas' assertion covers every anchor (smooth-L1 only: the GIoU branch decodes, it has no targets)
      if (!A.giou && n == 0 && !(Box::width(an) > 0.f)) status |= D2B_LOSS_STATUS_INVALID_BOX;
      if (!Lab::in_range(lab, A.K)) status |= D2B_LOSS_STATUS_INVALID_CLASS;
      const bool pos = Lab::pos(lab, A.K);
      cnt[0] = pos ? 1 : 0;
      cnt[1] = Lab::neg(lab, A.K) ? 1 : 0;
      const size_t o = ((size_t)n * P.R[l] + r) * D;
      const T* __restrict__ dl = (const T*)P.deltas[l] + o;
      float g[D];
#pragma unroll
      for (int q = 0; q < D; ++q) g[q] = 0.f;
      if constexpr (kFcos) {
        float gc = 0.f;
        const size_t oc = (size_t)n * P.R[l] + r;
        if (pos) {
          const float* gt = A.gt_boxes + (size_t)row * 4;
          const float dv[4] = {E::ld(dl[0]), E::ld(dl[1]), E::ld(dl[2]), E::ld(dl[3])};
          bool ordered;
          s_reg += giou_row_linear(an, dv, gt, g, ordered);
          if (!ordered) status |= D2B_LOSS_STATUS_INVALID_BOX_ORDER;
          s_ctr += focal(E::ld(((const T*)P.ctr[l])[oc]), ctrness_target(an, gt), 0.f, -1.f, gc);
        }
        if (kBackward) ((T*)P.grad_ctr[l])[oc] = E::st(gc * *A.grad_ctr);
      } else if (pos) {
        if constexpr (D == 4) {
          if (A.giou) {
            const float dv[4] = {E::ld(dl[0]), E::ld(dl[1]), E::ld(dl[2]), E::ld(dl[3])};
            bool ordered;
            s_reg += giou_row(an, dv, A.gt_boxes + (size_t)row * D, A.w, A.scale_clamp, g, ordered);
            if (!ordered) status |= D2B_LOSS_STATUS_INVALID_BOX_ORDER;
          }
        }
        if (!A.giou) {
          float t[D];
          Box::get_deltas(an, A.gt_boxes + (size_t)row * D, A.w, t);
#pragma unroll
          for (int q = 0; q < D; ++q) s_reg += smooth_l1(E::ld(dl[q]) - t[q], A.beta, g[q]);
        }
      }
      if (kBackward) {
        const float gs = *A.grad_reg;
        T* __restrict__ gd = (T*)P.grad_deltas[l] + o;
#pragma unroll
        for (int q = 0; q < D; ++q) gd[q] = E::st(g[q] * gs);
      }
    }
  }
  if (!kBackward) block_partial(s_cls, s_reg, s_ctr, cnt, status, red, A.part + b);
}

// ---- Fast R-CNN ----------------------------------------------------------------------------------------------------
struct FrcnnArgs {
  int R, K, kreg;           // scores [R, K+1], deltas [R, kreg * D]
  const void* scores;
  const void* deltas;
  const float* proposals;   // [R, D]
  const float* gt_boxes;    // [R, D]
  const long long* gt_classes;
  float beta;
  int giou;
  float scale_clamp;
  BoxWeights w;
  const float* grad_cls;
  const float* grad_reg;
  void* grad_scores;
  void* grad_deltas;
  Partial* part;
};

// torch.argmax on CUDA: a NaN beats every number (the first NaN wins), ties go to the smaller index
__device__ __forceinline__ bool argmax_better(float a, int ia, float b, int ib) {
  const bool an = a != a, bn = b != b;
  if (an || bn) return an && (!bn || ia < ib);
  return a > b || (a == b && ia < ib);
}

template <int DT, class Box, bool kBackward>
__global__ void __launch_bounds__(kThreads) frcnn_loss_kernel(const FrcnnArgs A) {
  using E = Elem<DT>;
  using T = typename E::T;
  constexpr int D = Box::D;
  __shared__ BlockRed red;
  const int lane = threadIdx.x & 31;
  const int r = blockIdx.x * kWarps + (threadIdx.x >> 5);
  float s_cls = 0.f, s_reg = 0.f;
  long long cnt[4] = {0, 0, 0, 0};
  int status = 0;
  if (r < A.R) {
    const int K1 = A.K + 1;
    const T* __restrict__ sr = (const T*)A.scores + (size_t)r * K1;
    const long long c = A.gt_classes[r];
    const bool cls_ok = c >= 0 && c <= A.K;
    float best = -INFINITY, mx = -INFINITY;
    int bi = INT_MAX;
    bool nan = false;
    for (int j = lane; j < K1; j += 32) {
      const float v = E::ld(sr[j]);
      if (bi == INT_MAX || argmax_better(v, j, best, bi)) {
        best = v;
        bi = j;
      }
      nan |= v != v;
      mx = fmaxf(mx, v);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const float ob = __shfl_xor_sync(0xffffffffu, best, o);
      const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (oi != INT_MAX && (bi == INT_MAX || argmax_better(ob, oi, best, bi))) {
        best = ob;
        bi = oi;
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    nan = __any_sync(0xffffffffu, nan);
    const float m = nan ? NAN : mx;
    float se = 0.f;
    for (int j = lane; j < K1; j += 32) se += expf(E::ld(sr[j]) - m);
    se = warp_sum(se);
    const bool fg = c >= 0 && c < A.K;
    if (lane == 0) {
      if (!cls_ok) status |= D2B_LOSS_STATUS_INVALID_CLASS;
      else s_cls = logf(se) - (E::ld(sr[c]) - m);  // cross_entropy = -log_softmax[c]
      cnt[0] = fg ? 1 : 0;
      cnt[1] = bi == c ? 1 : 0;
      cnt[2] = fg && bi == c ? 1 : 0;
      cnt[3] = fg && bi == A.K ? 1 : 0;
    }
    if (kBackward) {
      const float gs = *A.grad_cls;
      T* __restrict__ gr = (T*)A.grad_scores + (size_t)r * K1;
      const float lse = logf(se);
      for (int j = lane; j < K1; j += 32) {
        const float p = expf(E::ld(sr[j]) - m - lse);
        gr[j] = E::st(cls_ok ? (p - (j == c ? 1.f : 0.f)) * gs : 0.f);
      }
    }
    // box regression on the foreground rows, class-specific deltas gathered at the GT class
    const int col = A.kreg == 1 ? 0 : (int)(fg ? c : 0) * D;
    const T* __restrict__ dr = (const T*)A.deltas + (size_t)r * A.kreg * D;
    float g = 0.f;
    if constexpr (D == 4) {
      if (A.giou && fg && lane < D) {  // every lane of the four decodes the row and keeps its own coordinate's gradient
        const float dv[4] = {E::ld(dr[col]), E::ld(dr[col + 1]), E::ld(dr[col + 2]), E::ld(dr[col + 3])};
        float gg[4];
        bool ordered;
        const float loss = giou_row(A.proposals + (size_t)r * D, dv, A.gt_boxes + (size_t)r * D, A.w, A.scale_clamp, gg,
                                    ordered);
        g = lane == 0 ? gg[0] : (lane == 1 ? gg[1] : (lane == 2 ? gg[2] : gg[3]));
        if (lane == 0) {
          s_reg = loss;
          if (!ordered) status |= D2B_LOSS_STATUS_INVALID_BOX_ORDER;
        }
      }
    }
    if (!A.giou && fg && lane < D) {
      const float* pr = A.proposals + (size_t)r * D;
      if (lane == 0 && !(Box::width(pr) > 0.f)) status |= D2B_LOSS_STATUS_INVALID_BOX;
      float t[D];
      Box::get_deltas(pr, A.gt_boxes + (size_t)r * D, A.w, t);
      float tq = t[0];
#pragma unroll
      for (int q = 1; q < D; ++q) tq = lane == q ? t[q] : tq;
      s_reg = smooth_l1(E::ld(dr[col + lane]) - tq, A.beta, g);
    }
    if (kBackward) {
      const float gs = *A.grad_reg;
      T* __restrict__ gd = (T*)A.grad_deltas + (size_t)r * A.kreg * D;
      for (int j = lane; j < A.kreg * D; j += 32) gd[j] = E::st(0.f);
      __syncwarp();
      if (fg && lane < D) gd[col + lane] = E::st(g * gs);
    }
  }
  if (!kBackward) block_partial(s_cls, s_reg, 0.f, cnt, status, red, A.part + blockIdx.x);
}

// ---- host side -----------------------------------------------------------------------------------------------------
constexpr int vec_elems(int dtype) { return dtype == D2B_F32 ? 4 : 8; }

bool valid_dtype(int dtype) { return dtype == D2B_F32 || dtype == D2B_F16 || dtype == D2B_BF16; }

bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// GIoU is defined on axis-aligned boxes only, as in the reference
bool loss_type_ok(int loss_type, int box_dim) {
  return loss_type == D2B_LOSS_SMOOTH_L1 || (loss_type == D2B_LOSS_GIOU && box_dim == 4);
}

BoxWeights box_weights(const float* weights, int D) {
  BoxWeights w = {};
  for (int q = 0; q < D; ++q) w.w[q] = weights[q];
  if (D == 5) w.w[4] = (float)((double)weights[4] * 3.141592653589793 / 180.0);  // wa * math.pi / 180.0
  return w;
}

// Checks the level table and fills P; returns the number of classification CTAs, or -1.
long long dense_levels(const d2b_dense_loss_levels* lv, int N, int K, int dtype, bool backward, DenseLevels& P) {
  if (!lv || lv->num_levels < 1 || lv->num_levels > D2B_MAX_LEVELS) return -1;
  P = {};
  P.L = lv->num_levels;
  long long a = 0, blk = 0;
  const long long chunk = (long long)kThreads * kItems * vec_elems(dtype);
  for (int l = 0; l < P.L; ++l) {
    const int Rl = lv->R[l];
    if (Rl < 0) return -1;
    const bool some = (long long)N * Rl > 0;
    if (some && (!lv->logits[l] || !lv->deltas[l] || !aligned16(lv->logits[l]))) return -1;
    if (some && backward && (!lv->grad_logits[l] || !lv->grad_deltas[l] || !aligned16(lv->grad_logits[l]))) return -1;
    P.logits[l] = lv->logits[l];
    P.deltas[l] = lv->deltas[l];
    P.grad_logits[l] = lv->grad_logits[l];
    P.grad_deltas[l] = lv->grad_deltas[l];
    P.R[l] = Rl;
    P.a0[l] = (int)a;
    P.blk0[l] = blk;
    a += Rl;
    blk += ((long long)N * Rl * K + chunk - 1) / chunk;
    if (a > INT_MAX) return -1;
  }
  P.a0[P.L] = (int)a;
  P.blk0[P.L] = blk;
  return blk;
}

long long dense_reg_blocks(int N, int Rtot) { return ((long long)N * Rtot + kThreads - 1) / kThreads; }

template <int DT, class Box, class Lab, bool kBackward, bool kFcos = false>
void launch_dense(long long blocks, const DenseLevels& P, const DenseArgs& A, cudaStream_t st) {
  dense_loss_kernel<DT, Box, Lab, kBackward, kFcos><<<(unsigned)blocks, kThreads, 0, st>>>(P, A);
}

template <bool kBackward>
int dense_dispatch(long long blocks, int dtype, int D, int label_kind, int loss_type, const DenseLevels& P,
                   const DenseArgs& A, cudaStream_t st) {
#define D2B_DENSE_CASE(DT)                                                                                              \
  if (dtype == DT) {                                                                                                    \
    if (loss_type == D2B_LOSS_LINEAR_GIOU) launch_dense<DT, XyxyBox, LabelsI64, kBackward, true>(blocks, P, A, st);     \
    else if (D == 4 && label_kind == D2B_LABELS_I8) launch_dense<DT, XyxyBox, LabelsI8, kBackward>(blocks, P, A, st);   \
    else if (D == 4 && label_kind == D2B_LABELS_I64) launch_dense<DT, XyxyBox, LabelsI64, kBackward>(blocks, P, A, st); \
    else if (D == 5 && label_kind == D2B_LABELS_I8) launch_dense<DT, RotBox, LabelsI8, kBackward>(blocks, P, A, st);    \
    else if (D == 5 && label_kind == D2B_LABELS_I64) launch_dense<DT, RotBox, LabelsI64, kBackward>(blocks, P, A, st);  \
  }
  D2B_DENSE_CASE(D2B_F32)
  D2B_DENSE_CASE(D2B_F16)
  D2B_DENSE_CASE(D2B_BF16)
#undef D2B_DENSE_CASE
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// Shared argument rules of the dense forward and backward; fills P and A.
int dense_setup(const d2b_dense_loss_levels* lv, int N, int K, int box_dim, int dtype, const float* anchors,
                const float* gt_boxes, const void* labels, int label_kind, float gamma, float alpha, float beta,
                int loss_type, float scale_clamp, const float* weights, bool backward, DenseLevels& P, DenseArgs& A,
                long long& blocks) {
  const bool linear = loss_type == D2B_LOSS_LINEAR_GIOU;  // FCOS: no Box2BoxTransform weights, a centerness per level
  if (N < 0 || K <= 0 || (box_dim != 4 && box_dim != 5) || !valid_dtype(dtype) || (!weights && !linear))
    return D2B_EINVAL;
  if (label_kind != D2B_LABELS_I8 && label_kind != D2B_LABELS_I64) return D2B_EINVAL;
  if (label_kind == D2B_LABELS_I8 && K != 1) return D2B_EINVAL;
  if (!(gamma >= 0.f) || !(beta >= 0.f) || alpha != alpha) return D2B_EINVAL;
  if (linear ? box_dim != 4 || label_kind != D2B_LABELS_I64 : !loss_type_ok(loss_type, box_dim)) return D2B_EINVAL;
  const long long cls_blocks = dense_levels(lv, N, K, dtype, backward, P);
  if (cls_blocks < 0) return D2B_EINVAL;
  for (int l = 0; l < P.L; ++l) {
    if (!linear && (lv->ctr[l] || lv->grad_ctr[l])) return D2B_EINVAL;
    if (linear && (long long)N * P.R[l] > 0 && (!lv->ctr[l] || (backward && !lv->grad_ctr[l]))) return D2B_EINVAL;
    P.ctr[l] = lv->ctr[l];
    P.grad_ctr[l] = lv->grad_ctr[l];
  }
  const int Rtot = P.a0[P.L];
  if ((long long)N * Rtot > 0 && (!anchors || !gt_boxes || !labels)) return D2B_EINVAL;
  blocks = cls_blocks + dense_reg_blocks(N, Rtot);
  if (blocks > INT_MAX) return D2B_EINVAL;
  A = {};
  A.N = N;
  A.K = K;
  A.Rtot = Rtot;
  A.cls_blocks = cls_blocks;
  A.anchors = anchors;
  A.gt_boxes = gt_boxes;
  A.labels = labels;
  A.gamma = gamma;
  A.alpha = alpha;
  A.beta = beta;
  A.giou = loss_type == D2B_LOSS_GIOU || linear;  // decoded boxes, no get_deltas targets: no width assertion
  A.scale_clamp = scale_clamp;
  if (!linear) A.w = box_weights(weights, box_dim);
  return D2B_OK;
}

int frcnn_setup(int R, int K, int kreg, int box_dim, int dtype, const void* scores, const void* deltas,
                const float* proposals, const float* gt_boxes, const int64_t* gt_classes, float beta, int loss_type,
                float scale_clamp, const float* weights, FrcnnArgs& A) {
  if (R < 0 || K <= 0 || (kreg != 1 && kreg != K) || (box_dim != 4 && box_dim != 5) || !valid_dtype(dtype) || !weights)
    return D2B_EINVAL;
  if (!(beta >= 0.f) || (long long)kreg * box_dim > INT_MAX / 2 || !loss_type_ok(loss_type, box_dim)) return D2B_EINVAL;
  if (R > 0 && (!scores || !deltas || !proposals || !gt_boxes || !gt_classes)) return D2B_EINVAL;
  A = {};
  A.R = R;
  A.K = K;
  A.kreg = kreg;
  A.scores = scores;
  A.deltas = deltas;
  A.proposals = proposals;
  A.gt_boxes = gt_boxes;
  A.gt_classes = (const long long*)gt_classes;
  A.beta = beta;
  A.giou = loss_type == D2B_LOSS_GIOU;
  A.scale_clamp = scale_clamp;
  A.w = box_weights(weights, box_dim);
  return D2B_OK;
}

template <bool kBackward>
int frcnn_dispatch(int dtype, int D, const FrcnnArgs& A, cudaStream_t st) {
  const unsigned blocks = (unsigned)d2b_cdiv(A.R, kWarps);
#define D2B_FRCNN_CASE(DT)                                                                                          \
  if (dtype == DT) {                                                                                                \
    if (D == 4) frcnn_loss_kernel<DT, XyxyBox, kBackward><<<blocks, kThreads, 0, st>>>(A);                         \
    else frcnn_loss_kernel<DT, RotBox, kBackward><<<blocks, kThreads, 0, st>>>(A);                                 \
  }
  D2B_FRCNN_CASE(D2B_F32)
  D2B_FRCNN_CASE(D2B_F16)
  D2B_FRCNN_CASE(D2B_BF16)
#undef D2B_FRCNN_CASE
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

}  // namespace

D2B_API size_t d2b_dense_loss_workspace_bytes(const d2b_dense_loss_levels* lv, int N, int K, int dtype) {
  DenseLevels P;
  if (N < 0 || K <= 0 || !valid_dtype(dtype)) return 0;
  const long long cls_blocks = dense_levels(lv, N, K, dtype, false, P);
  if (cls_blocks < 0) return 0;
  return (size_t)(cls_blocks + dense_reg_blocks(N, P.a0[P.L])) * sizeof(Partial);
}

D2B_API int d2b_dense_loss_forward(const d2b_dense_loss_levels* lv, int N, int K, int box_dim, int dtype,
                                   const float* anchors, const float* gt_boxes, const void* labels, int label_kind,
                                   float gamma, float alpha, float beta, int loss_type, float scale_clamp,
                                   const float* weights, float* sums, int64_t* counts, int* status, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  DenseLevels P;
  DenseArgs A;
  long long blocks = 0;
  const int rc = dense_setup(lv, N, K, box_dim, dtype, anchors, gt_boxes, labels, label_kind, gamma, alpha, beta,
                             loss_type, scale_clamp, weights, false, P, A, blocks);
  if (rc) return rc;
  if (!sums || !counts || !status) return D2B_EINVAL;
  if (blocks > 0 && (!workspace || !aligned16(workspace))) return D2B_EINVAL;
  if (workspace_bytes < (size_t)blocks * sizeof(Partial)) return D2B_EWORKSPACE;
  const cudaStream_t st = (cudaStream_t)stream;
  A.part = (Partial*)workspace;
  if (blocks > 0) {
    const int e = dense_dispatch<false>(blocks, dtype, box_dim, label_kind, loss_type, P, A, st);
    if (e) return e;
  }
  finish_kernel<<<1, kThreads, 0, st>>>(A.part, (int)blocks, 3, 2, sums, counts, status);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_dense_loss_backward(const d2b_dense_loss_levels* lv, int N, int K, int box_dim, int dtype,
                                    const float* anchors, const float* gt_boxes, const void* labels, int label_kind,
                                    float gamma, float alpha, float beta, int loss_type, float scale_clamp,
                                    const float* weights, const float* grad_sums, void* stream) {
  DenseLevels P;
  DenseArgs A;
  long long blocks = 0;
  const int rc = dense_setup(lv, N, K, box_dim, dtype, anchors, gt_boxes, labels, label_kind, gamma, alpha, beta,
                             loss_type, scale_clamp, weights, true, P, A, blocks);
  if (rc) return rc;
  if (!grad_sums) return D2B_EINVAL;
  if (blocks == 0) return D2B_OK;
  A.grad_cls = grad_sums;
  A.grad_reg = grad_sums + 1;
  A.grad_ctr = grad_sums + 2;
  return dense_dispatch<true>(blocks, dtype, box_dim, label_kind, loss_type, P, A, (cudaStream_t)stream);
}

D2B_API size_t d2b_frcnn_loss_workspace_bytes(int R) {
  return R <= 0 ? 0 : (size_t)d2b_cdiv(R, kWarps) * sizeof(Partial);
}

D2B_API int d2b_frcnn_loss_forward(const void* scores, const void* deltas, int R, int K, int kreg, int box_dim, int dtype,
                                   const float* proposals, const float* gt_boxes, const int64_t* gt_classes, float beta,
                                   int loss_type, float scale_clamp, const float* weights, float* sums, int64_t* counts,
                                   int* status, void* workspace, size_t workspace_bytes, void* stream) {
  FrcnnArgs A;
  const int rc = frcnn_setup(R, K, kreg, box_dim, dtype, scores, deltas, proposals, gt_boxes, gt_classes, beta, loss_type,
                             scale_clamp, weights, A);
  if (rc) return rc;
  if (!sums || !counts || !status) return D2B_EINVAL;
  if (R > 0 && (!workspace || !aligned16(workspace))) return D2B_EINVAL;
  if (workspace_bytes < d2b_frcnn_loss_workspace_bytes(R)) return D2B_EWORKSPACE;
  const cudaStream_t st = (cudaStream_t)stream;
  A.part = (Partial*)workspace;
  if (R > 0) {
    const int e = frcnn_dispatch<false>(dtype, box_dim, A, st);
    if (e) return e;
  }
  finish_kernel<<<1, kThreads, 0, st>>>(A.part, d2b_cdiv(R, kWarps), 2, 4, sums, counts, status);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_frcnn_loss_backward(const void* scores, const void* deltas, int R, int K, int kreg, int box_dim,
                                    int dtype, const float* proposals, const float* gt_boxes, const int64_t* gt_classes,
                                    float beta, int loss_type, float scale_clamp, const float* weights,
                                    const float* grad_sums, void* grad_scores, void* grad_deltas, void* stream) {
  FrcnnArgs A;
  const int rc = frcnn_setup(R, K, kreg, box_dim, dtype, scores, deltas, proposals, gt_boxes, gt_classes, beta, loss_type,
                             scale_clamp, weights, A);
  if (rc) return rc;
  if (R == 0) return D2B_OK;
  if (!grad_sums || !grad_scores || !grad_deltas) return D2B_EINVAL;
  A.grad_cls = grad_sums;
  A.grad_reg = grad_sums + 1;
  A.grad_scores = grad_scores;
  A.grad_deltas = grad_deltas;
  return frcnn_dispatch<true>(dtype, box_dim, A, (cudaStream_t)stream);
}
