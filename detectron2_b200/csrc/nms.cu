// NMS (axis-aligned + rotated) and pairwise rotated-box IoU for sm_90a.
//
// Replaces torchvision::nms as reached from detectron2/layers/nms.py:5-22, and
// detectron2/layers/csrc/{nms_rotated/nms_rotated_cuda.cu, box_iou_rotated/box_iou_rotated_cuda.cu}.
// This file is compiled with -fmad=false: every float expression rounds like the reference's CPU build
// (x86-64, no FMA), which is the bit-exact parity target (see DESIGN.md "bit-exactness").
//
// Pipeline of d2b_nms (all on the caller's stream, no host round trip -- the reference copies the N x N/64 bitmask
// to the host and scans it there, nms_rotated_cuda.cu:114-137).  One memset + THREE launches, no library sort:
//   1. nms_rank_kernel: the position of every box in the stable descending score order AND in the category-major order
//      (descending scores inside a category) by counting -- what two stable radix sorts would give -- together with the
//      segment bounds, the boxes gathered into that order and the coordinate range of the batched-NMS offset trick;
//   2. nms_mask_kernel: IoU bitmask, 64x64 tiles inside the categories only, stored in word planes maskT[w][row] so that
//      both the tile writes and the scan's reads are coalesced; memory = planes(max category size) x M words;
//   3. nms_scan_kernel: greedy scan, one CTA per category segment in parallel: per 64-box block one thread resolves the
//      intra-block chain (branch-free) from the diagonal word, then 16 warps OR the kept rows into the `removed` words
//      (rows prefetched one block ahead in ping-pong registers); kept boxes are flagged at their global score rank and
//      the last CTA to finish compacts the flags into kept original indices (0-padded) + the device-side count.
#include "common.cuh"

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

// box_iou_rotated_cuda.cu:14-63 equivalent: one thread per (i,j) pair, j fastest for coalesced output.
__global__ void __launch_bounds__(128) box_iou_rotated_kernel(const float* __restrict__ b1, long long N,
                                                              const float* __restrict__ b2, long long M,
                                                              float* __restrict__ out) {
  __shared__ float sb2[128 * 5];
  const long long j0 = (long long)blockIdx.x * 128;
  const int nj = (int)min((long long)128, M - j0);
  for (int t = threadIdx.x; t < nj * 5; t += 128) sb2[t] = b2[j0 * 5 + t];
  __syncthreads();
  if ((int)threadIdx.x >= nj) return;
  for (long long i = blockIdx.y; i < N; i += gridDim.y) {
    float a[5];
#pragma unroll
    for (int c = 0; c < 5; ++c) a[c] = b1[i * 5 + c];
    out[i * M + j0 + threadIdx.x] = rotated_iou(a, sb2 + threadIdx.x * 5);
  }
}

// ------------------------------------------------------------------------------------------------
// NMS
// ------------------------------------------------------------------------------------------------
// Control block at the start of the workspace; zeroed together with keepflag[] by ONE memset per call.
struct NmsCtrl {
  int nseg;          // number of category segments found
  unsigned ticket;   // CTAs of the scan kernel that have finished
  unsigned mx;       // ordered-uint encoding of the largest coordinate (batched-NMS offset trick)
  unsigned mn_neg;   // ... of the negated smallest coordinate (rotated variant)
  int error;         // a category held more boxes than the caller's bound
  int pad[3];
};

// monotone float <-> uint map (atomicMax on floats of either sign); 0 encodes "smaller than everything"
__device__ __forceinline__ unsigned enc_f(float f) {
  const unsigned b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float dec_f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}
// canonical value for the ordered encoding: -0.0 becomes +0.0 and every NaN the one positive NaN, which enc_f places above
// +inf.  This is the score order of torch.sort(descending=True, stable=True): NaN first, +-0 equal.
__device__ __forceinline__ float canon_f(float f) { return f != f ? __uint_as_float(0x7fc00000u) : (f == 0.f ? 0.f : f); }
// 64-bit key of box i in the stable descending score order (ascending key == score order; distinct for distinct i)
__device__ __forceinline__ unsigned long long score_key(float s, int i) {
  return ((unsigned long long)(~enc_f(canon_f(s))) << 32) | (unsigned)i;
}
// max / min that return NaN when either operand is NaN, like torch.max / torch.min (fmaxf / fminf drop the NaN)
__device__ __forceinline__ float max_nan(float a, float b) { return (a > b || a != a) ? a : b; }
__device__ __forceinline__ float min_nan(float a, float b) { return (a < b || a != a) ? a : b; }

// ---- kernel 1: order by counting.  One warp per TWO boxes; the scores / categories of all boxes stream through shared
// memory once per CTA.  For box i, with k_i = score_key(s_i, i):
//   grank = #{j : k_j < k_i}                                           position in the stable descending score order
//   pos   = #{j : c_j < c_i} + #{j : c_j == c_i and k_j < k_i}         position in the category-major order
// which is what two stable radix sorts would produce -- but in one launch, with the segment bounds of every position and
// the segment list as by-products.  The keys are distinct, so grank and pos are permutations of [0, M) whatever the scores
// (NaN, +-0): the scan indexes with them.  O(M^2 / 32) warp steps: 3 us at M = 8819, ~3 ms at M = 100 000.
constexpr int kRankTile = 1792;
constexpr int kRankWarps = 8;
constexpr int kRankHist = 4096;  // category ids in [-1, kRankHist) take the histogram path

template <bool ROT>
__global__ void __launch_bounds__(kRankWarps * 32) nms_rank_kernel(const float* __restrict__ boxes,
                                                                   const float* __restrict__ scores,
                                                                   const int64_t* __restrict__ idxs, int M, int max_segment,
                                                                   int use_range, int one_segment, NmsCtrl* __restrict__ ctrl,
                                                                   int* __restrict__ grank_of_pos, int* __restrict__ orig_of_grank,
                                                                   int* __restrict__ seg_hi_of_pos, float* __restrict__ clsf_of_pos,
                                                                   float* __restrict__ sorted_boxes, int* __restrict__ seg_start,
                                                                   int* __restrict__ seg_end, unsigned char* __restrict__ keepflag) {
  // tile of the streamed boxes: {64-bit order key, category} (int64 on the generic path, int32 on the histogram path)
  __shared__ unsigned long long s_key[kRankTile];
  __shared__ long long s_cls[kRankTile];
  __shared__ int s_hist[kRankHist + 2];  // [c + 1] = number of boxes of category c, then exclusive prefix = #{smaller category}
  __shared__ int s_wtot[kRankWarps];
  __shared__ float s_mx[kRankWarps], s_mn[kRankWarps];
  constexpr int D = ROT ? 5 : 4;
  constexpr int kT = kRankWarps * 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int i0 = (blockIdx.x * kRankWarps + warp) * 2, i1 = i0 + 1;
  const bool ok0 = i0 < M, ok1 = i1 < M;
  const float sa = ok0 ? scores[i0] : 0.f, sb = ok1 ? scores[i1] : 0.f;
  // category ids set the coordinate offsets; segment ids group the boxes for the mask and the scan.  They are the same
  // unless one_segment puts every non-ignored box into segment 0.
  auto seg = [one_segment](long long c) { return (one_segment && c >= 0) ? 0LL : c; };
  const long long ida = (ok0 && idxs) ? idxs[i0] : 0, idb = (ok1 && idxs) ? idxs[i1] : 0;
  const long long ca = seg(ida), cb = seg(idb);
  const unsigned long long ka = score_key(sa, i0), kb = score_key(sb, i1);
  int ga = 0, gb = 0, sma = 0, smb = 0, bea = 0, beb = 0, na = 0, nb = 0;  // grank, smaller-class, before-in-class, class size
  // ---- category histogram (every CTA builds its own: M small loads from L2): when all ids fit, the O(M^2) loop below only
  //      has to count "before me in the score order" and "... and of my category" -- two compares per pair.
  for (int c = tid; c < kRankHist + 2; c += kT) s_hist[c] = 0;
  __syncthreads();
  int small = 1;
  if (idxs) {
    for (int j = tid; j < M; j += kT) {
      const long long c = seg(idxs[j]);
      if (c < -1 || c >= kRankHist) small = 0;
      else atomicAdd(&s_hist[(int)c + 1], 1);
    }
  } else if (tid == 0) {
    s_hist[1] = M;
  }
  small = __syncthreads_and(small);
  if (small) {
    // exclusive prefix over the bins: strip per thread + scan of the strip totals
    constexpr int kStrip = (kRankHist + 2 + kT - 1) / kT;
    const int c0 = tid * kStrip;
    int loc[kStrip], sum = 0;
#pragma unroll
    for (int e = 0; e < kStrip; ++e) {
      loc[e] = (c0 + e < kRankHist + 2) ? s_hist[c0 + e] : 0;
      sum += loc[e];
    }
    int inc = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) s_wtot[warp] = inc;
    __syncthreads();
    int base = inc - sum;
    for (int w = 0; w < warp; ++w) base += s_wtot[w];
    // s_hist[c + 1] <- #{boxes of a smaller category}; the count itself is recovered as the difference to the next bin
    __syncthreads();
#pragma unroll
    for (int e = 0; e < kStrip; ++e)
      if (c0 + e < kRankHist + 2) {
        s_hist[c0 + e] = base;
        base += loc[e];
      }
    __syncthreads();
    const int ca32 = (int)ca, cb32 = (int)cb;
    int* s_c32 = reinterpret_cast<int*>(s_cls);
    for (int t0 = 0; t0 < M; t0 += kRankTile) {
      const int tn = min(kRankTile, M - t0);
      __syncthreads();
      for (int j = tid; j < tn; j += kT) {
        s_key[j] = score_key(scores[t0 + j], t0 + j);
        s_c32[j] = idxs ? (int)seg(idxs[t0 + j]) : 0;
      }
      __syncthreads();
      for (int jl = lane; jl < tn; jl += 32) {
        const unsigned long long kj = s_key[jl];
        const int c = s_c32[jl];
        const bool fa = kj < ka, fb = kj < kb;
        ga += fa;
        gb += fb;
        bea += fa && (c == ca32);
        beb += fb && (c == cb32);
      }
    }
  } else {
    for (int t0 = 0; t0 < M; t0 += kRankTile) {
      const int tn = min(kRankTile, M - t0);
      __syncthreads();
      for (int j = tid; j < tn; j += kT) {
        s_key[j] = score_key(scores[t0 + j], t0 + j);
        s_cls[j] = idxs ? seg(idxs[t0 + j]) : 0;
      }
      __syncthreads();
      for (int jl = lane; jl < tn; jl += 32) {
        const unsigned long long kj = s_key[jl];
        const long long c = s_cls[jl];
        const bool fa = kj < ka, fb = kj < kb;
        ga += fa;
        gb += fb;
        sma += c < ca;
        smb += c < cb;
        na += c == ca;
        nb += c == cb;
        bea += (c == ca) && fa;
        beb += (c == cb) && fb;
      }
    }
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    ga += __shfl_xor_sync(0xffffffffu, ga, o);
    gb += __shfl_xor_sync(0xffffffffu, gb, o);
    sma += __shfl_xor_sync(0xffffffffu, sma, o);
    smb += __shfl_xor_sync(0xffffffffu, smb, o);
    na += __shfl_xor_sync(0xffffffffu, na, o);
    nb += __shfl_xor_sync(0xffffffffu, nb, o);
    bea += __shfl_xor_sync(0xffffffffu, bea, o);
    beb += __shfl_xor_sync(0xffffffffu, beb, o);
  }
  if (small) {  // category start / size from the prefix table
    if (ok0) { sma = s_hist[(int)ca + 1]; na = s_hist[(int)ca + 2] - sma; }
    if (ok1) { smb = s_hist[(int)cb + 1]; nb = s_hist[(int)cb + 2] - smb; }
  }
  float mx = -INFINITY, mn = INFINITY;
#pragma unroll
  for (int e = 0; e < 2; ++e) {
    const int i = e ? i1 : i0;
    if (!(e ? ok1 : ok0)) continue;
    const int g = e ? gb : ga, sm = e ? smb : sma, be = e ? beb : bea, n = e ? nb : na;
    const long long c = e ? cb : ca;
    const int pos = sm + be;
    float b[D];
#pragma unroll
    for (int q = 0; q < D; ++q) b[q] = boxes[(size_t)i * D + q];
    const bool ignored = c < 0;  // negative category: the box takes part in nothing and is never kept
    if (!ignored) {  // NaN-propagating like the reference's torch reductions: one NaN coordinate makes every offset NaN
      if (ROT) {  // detectron2/layers/nms.py:137-143
        const float half = max_nan(b[2], b[3]) / 2;
        mx = max_nan(mx, max_nan(b[0], b[1]) + half);
        mn = min_nan(mn, min_nan(b[0], b[1]) - half);
      } else {  // torchvision _batched_nms_coordinate_trick: boxes.max()
        mx = max_nan(mx, max_nan(max_nan(b[0], b[1]), max_nan(b[2], b[3])));
      }
    }
    if (lane == 0) {
      grank_of_pos[pos] = g;
      orig_of_grank[g] = i;
      seg_hi_of_pos[pos] = (ignored || n == 1) ? pos : sm + n;  // empty column range: the mask kernel skips the row
      clsf_of_pos[pos] = (float)(e ? idb : ida);
#pragma unroll
      for (int q = 0; q < D; ++q) sorted_boxes[(size_t)pos * D + q] = b[q];
      if (ignored) {
      } else if (n == 1) {  // alone in its category: kept, nothing to scan
        keepflag[g] = 1;
      } else if (be == 0) {  // first box of its category: publish the segment
        const int slot = atomicAdd(&ctrl->nseg, 1);
        seg_start[slot] = sm;
        seg_end[slot] = sm + n;
        if (n > max_segment) ctrl->error = 1;
      }
    }
  }
  if (use_range) {  // one atomic per CTA
    if (lane == 0) {
      s_mx[warp] = mx;
      s_mn[warp] = mn;
    }
    __syncthreads();
    if (tid == 0) {
      for (int q = 1; q < kRankWarps; ++q) {
        mx = max_nan(mx, s_mx[q]);
        mn = min_nan(mn, s_mn[q]);
      }
      // the canonical NaN encodes above +inf, so a NaN wins the atomicMax and decodes back to NaN
      if (mx != -INFINITY) atomicMax(&ctrl->mx, enc_f(canon_f(mx)));
      if (ROT && mn != INFINITY) atomicMax(&ctrl->mn_neg, enc_f(canon_f(-mn)));
    }
  }
}

// ---- kernel 2: IoU bitmask, one CTA per 64 x 64 tile (row block x word plane; tiles no row reaches exit at once).  A row only
// meets the later boxes of its own category: columns (row, seg_hi[row]).  Word w of row r (64 columns starting at block (r/64)+w) lives
// at maskT[w * M + r] (word-plane-major: the CTA's writes and the scan's reads are both coalesced); `wcap` planes, sized
// from the caller's bound on the category size -- not from M.
// Thread layout: kSub threads per row, each testing 64/kSub columns, partial words OR-ed with warp shuffles.  The rotated
// IoU is ~50x the work of the axis-aligned one, so it gets 8 threads per row (512-thread CTAs), the cheap one gets 4.
template <bool ROT, int kSub>
__global__ void __launch_bounds__(64 * kSub) nms_mask_kernel(const float* __restrict__ sb, const int* __restrict__ seg_hi_of_pos,
                                                             const float* __restrict__ clsf_of_pos,
                                                             const NmsCtrl* __restrict__ ctrl, int apply_offsets, int M,
                                                             int wcap, double thr, unsigned long long* __restrict__ maskT) {
  // grid (row blocks, word planes): CTA (rb, w) owns the 64 x 64 tile of rows [64 rb, +64) against columns [64 (rb + w), +64)
  constexpr int D = ROT ? 5 : 4;
  constexpr int kCols = 64 / kSub;
  __shared__ float cbox[64 * D];
  __shared__ int s_hi;
  const int rb = blockIdx.x, r0 = rb * 64;
  const int cb = rb + (int)blockIdx.y, c0 = cb * 64;
  if (c0 >= M) return;
  const int lrow = threadIdx.x / kSub, sub = threadIdx.x % kSub;
  const int row = r0 + lrow;
  const bool row_ok = row < M;
  const int my_hi = row_ok ? seg_hi_of_pos[row] : 0;
  if (threadIdx.x == 0) s_hi = 0;
  __syncthreads();
  if (sub == 0 && row_ok && my_hi > c0) atomicMax(&s_hi, my_hi);
  __syncthreads();
  if (s_hi == 0) return;  // no row of this block reaches the column block (block-uniform): nothing to write
  // batched-NMS coordinate offsets, fp32 like the reference: axis-aligned box + idx*(max+1); rotated centre + idx*(max-min+1)
  float scale = 0.f;
  if (apply_offsets) scale = ROT ? (dec_f(ctrl->mx) - (-dec_f(ctrl->mn_neg)) + 1.0f) : (dec_f(ctrl->mx) + 1.0f);
  float a[D];
#pragma unroll
  for (int c = 0; c < D; ++c) a[c] = sb[(size_t)(row_ok ? row : M - 1) * D + c];
  if (apply_offsets) {
    const float off = clsf_of_pos[row_ok ? row : M - 1] * scale;
    a[0] += off;
    a[1] += off;
    if (!ROT) {
      a[2] += off;
      a[3] += off;
    }
  }
  const int nc = min(64, M - c0);
  for (int t = threadIdx.x; t < nc * D; t += 64 * kSub) {
    const int j = t / D, q = t - j * D;
    float v = sb[(size_t)c0 * D + t];
    if (apply_offsets && (ROT ? q < 2 : true)) v += clsf_of_pos[c0 + j] * scale;
    cbox[t] = v;
  }
  __syncthreads();
  // rows whose category ends before this block have an empty column range and write nothing, but every lane takes part in
  // the shuffles below
  const bool active = row_ok && c0 < my_hi;
  unsigned long long bits = 0ull;
  const int jbeg = max(sub * kCols, row + 1 - c0), jend = active ? min(min(nc, (sub + 1) * kCols), my_hi - c0) : 0;
  if (ROT) {
    for (int j = jbeg; j < jend; ++j) {
      const float iou = rotated_iou(a, cbox + j * 5);
      if ((double)iou >= thr) bits |= 1ull << j;  // nms_rotated_cpu.cpp:54
    }
  } else {
    const float area_a = (a[2] - a[0]) * (a[3] - a[1]);
    for (int j = jbeg; j < jend; ++j) {
      const float* b = cbox + j * 4;
      const float xx1 = fmaxf(a[0], b[0]), yy1 = fmaxf(a[1], b[1]);
      const float xx2 = fminf(a[2], b[2]), yy2 = fminf(a[3], b[3]);
      const float w = fmaxf(0.f, xx2 - xx1), h = fmaxf(0.f, yy2 - yy1);
      const float inter = w * h;
      const float area_b = (b[2] - b[0]) * (b[3] - b[1]);
      const float ovr = inter / (area_a + area_b - inter);
      if ((double)ovr > thr) bits |= 1ull << j;  // torchvision nms: strict
    }
  }
#pragma unroll
  for (int o = 1; o < kSub; o <<= 1) bits |= __shfl_xor_sync(0xffffffffu, bits, o);  // the kSub lanes of a row are adjacent
  if (active && sub == 0) maskT[(size_t)blockIdx.y * M + row] = bits;
}

constexpr int kScanThreads = 512;
constexpr int kScanWarps = kScanThreads / 32;
constexpr int kMaxColsPerWarp = 10;  // register-prefetched column words per warp (covers segments <= 64*16*10 = 10240)

// Exclusive prefix sum of one int per thread over the CTA (shuffle scan inside the warps, one barrier); `total` receives
// the sum over the CTA.  warp_tot: 32 ints of shared memory.  blockDim.x <= 1024, multiple of 32.
__device__ __forceinline__ int block_excl_scan(int v, int* __restrict__ warp_tot, int& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  const int wt = lane < nwarps ? warp_tot[lane] : 0;
  int winc = wt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, winc, o);
    if (lane >= o) winc += t;
  }
  total = __shfl_sync(0xffffffffu, winc, 31);
  const int wbase = __shfl_sync(0xffffffffu, winc, warp) - __shfl_sync(0xffffffffu, wt, warp);
  return wbase + inc - v;
}

// ---- kernel 3: greedy scan over the bitmask, one CTA per category segment (plain NMS = one segment), then -- in the CTA
// that finishes last -- compaction of the kept boxes in global score order.
// dynamic smem: removed[] (uint64), one word per 64-box block of the segment.  Per block b: (B) warp 0 resolves the greedy
// selection inside the block from removed[b] and the diagonal word of each row in a few parallel rounds; (C) the warps OR the
// kept rows into the `removed` words of the later blocks.  Everything the next block needs from global memory (its diagonal words, its rows of the later
// columns) is requested one full iteration ahead and parked in registers, so the serial chain never waits on L2.
__global__ void __launch_bounds__(kScanThreads, 1) nms_scan_kernel(const unsigned long long* __restrict__ maskT,
                                                                   const int* __restrict__ grank_of_pos,
                                                                   const int* __restrict__ orig_of_grank,
                                                                   const int* __restrict__ seg_start,
                                                                   const int* __restrict__ seg_end, NmsCtrl* __restrict__ ctrl,
                                                                   int M, int wcap, unsigned char* __restrict__ keepflag,
                                                                   long long* __restrict__ keep, long long* __restrict__ num_keep) {
  extern __shared__ unsigned long long removed[];
  __shared__ __align__(16) unsigned long long s_diag[2][64];
  __shared__ unsigned long long s_kept;
  __shared__ int warp_tot[32];
  __shared__ unsigned s_last;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nseg = ctrl->nseg;
  for (int seg = blockIdx.x; seg < nseg; seg += gridDim.x) {
    const int p0 = seg_start[seg], p1 = seg_end[seg];
    const int b0 = p0 >> 6, nb = ((p1 - 1) >> 6) + 1;  // blocks [b0, nb) of the global tiling touch this segment
    // n <= ms boxes from row (p0 & 63) <= 63 span nb - b0 <= (63 + ms + 63) / 64 = wcap blocks; word planes w - b and
    // removed[] slots then stay below wcap.  A longer span is a segment over the caller's bound (error already flagged).
    if (nb - b0 > wcap) continue;
    __syncthreads();                                     // previous segment done with removed[] / s_diag
    for (int i = b0 + tid; i < nb; i += kScanThreads) removed[i - b0] = 0ull;

    // rows 2*lane, 2*lane+1 of block b, column blocks w = b + 1 + warp + kScanWarps*c (stored as word plane w - b)
    auto fetch = [&](int b, ulonglong2 (&dst)[kMaxColsPerWarp]) {
      const int r = b * 64 + 2 * lane;
#pragma unroll
      for (int c = 0; c < kMaxColsPerWarp; ++c) {
        const int w = b + 1 + warp + kScanWarps * c;
        dst[c] = make_ulonglong2(0ull, 0ull);
        if (b < nb && w < nb) {
          const unsigned long long* p = maskT + (size_t)(w - b) * M + r;
          // rows outside [p0, p1) of a boundary block belong to other segments: their words are never set in `kept`
          if (r + 1 < M) {
            if ((M & 1) == 0) dst[c] = *reinterpret_cast<const ulonglong2*>(p);  // 16 B aligned when M is even
            else dst[c] = make_ulonglong2(p[0], p[1]);
          } else if (r < M) {
            dst[c].x = p[0];
          }
        }
      }
    };
    auto diag_word = [&](int b) -> unsigned long long {
      const int r = b * 64 + tid;
      return (b < nb && tid < 64 && r >= p0 && r < p1) ? maskT[r] : 0ull;  // word plane 0
    };
    ulonglong2 bufA[kMaxColsPerWarp], bufB[kMaxColsPerWarp];
    fetch(b0, bufA);
    if (tid < 64) s_diag[b0 & 1][tid] = diag_word(b0);
    unsigned long long dnext = diag_word(b0 + 1);
    __syncthreads();

    // one block of 64 boxes; `cur` holds its rows (requested one iteration ago), `nxt` receives the next block's rows.
    // The two register buffers ping-pong (no copies: a copy would be a use and would expose the load latency).
    auto process = [&](int b, ulonglong2 (&cur)[kMaxColsPerWarp], ulonglong2 (&nxt)[kMaxColsPerWarp]) {
      const int lo = max(p0 - b * 64, 0), hi = min(p1 - b * 64, 64);  // rows [lo, hi) of this block belong to the segment
      const unsigned long long vmask =
          (hi >= 64 ? ~0ull : ((1ull << hi) - 1ull)) & ~((1ull << lo) - 1ull);
      // ---- step B: greedy selection inside the block, by warp 0 in parallel ROUNDS instead of a 64-step serial chain.
      //      U = rows still undecided.  A row of U that no other row of U suppresses is kept (every earlier row that could
      //      still suppress it is undecided too, and would show up in T); its own suppressions leave U.  The lowest row of U
      //      always qualifies (the diagonal words only hold later columns), so a round decides at least one row -- in practice
      //      most of them: the number of rounds is the longest suppression chain inside the block (a handful), each round two
      //      warp-wide OR reductions.  Same result as the sequential greedy scan.
      if (warp == 0) {
        const ulonglong2 dd = reinterpret_cast<const ulonglong2*>(s_diag[b & 1])[lane];  // rows 2*lane, 2*lane + 1
        unsigned long long U = vmask & ~removed[b - b0], K = 0ull;
        while (U) {
          const bool u0 = (U >> (2 * lane)) & 1ull, u1 = (U >> (2 * lane + 1)) & 1ull;
          unsigned long long t = (u0 ? dd.x : 0ull) | (u1 ? dd.y : 0ull);
          t = ((unsigned long long)__reduce_or_sync(0xffffffffu, (unsigned)(t >> 32)) << 32) |
              __reduce_or_sync(0xffffffffu, (unsigned)t);
          const unsigned long long Kr = U & ~t;
          K |= Kr;
          const bool k0b = (Kr >> (2 * lane)) & 1ull, k1b = (Kr >> (2 * lane + 1)) & 1ull;
          unsigned long long rm = (k0b ? dd.x : 0ull) | (k1b ? dd.y : 0ull);
          rm = ((unsigned long long)__reduce_or_sync(0xffffffffu, (unsigned)(rm >> 32)) << 32) |
               __reduce_or_sync(0xffffffffu, (unsigned)rm);
          U &= ~Kr & ~rm;
        }
        if (lane == 0) s_kept = K;
      }
      __syncthreads();
      const unsigned long long kept = s_kept;
      // requests for block b+1 / b+2 go out now and are consumed one iteration later
      fetch(b + 1, nxt);
      if (tid < 64) s_diag[(b + 1) & 1][tid] = dnext;
      dnext = diag_word(b + 2);
      // ---- publish the kept boxes of this block at their score rank
      if (tid < 64 && ((kept >> tid) & 1ull)) keepflag[grank_of_pos[b * 64 + tid]] = 1;
      // ---- step C: OR kept rows into later column words
      const unsigned long long k0 = (kept >> (2 * lane)) & 1ull ? ~0ull : 0ull;
      const unsigned long long k1 = (kept >> (2 * lane + 1)) & 1ull ? ~0ull : 0ull;
#pragma unroll
      for (int c = 0; c < kMaxColsPerWarp; ++c) {
        const int w = b + 1 + warp + kScanWarps * c;
        if (w < nb) {  // warp-uniform
          unsigned long long v = (cur[c].x & k0) | (cur[c].y & k1);
          unsigned lo32 = __reduce_or_sync(0xffffffffu, (unsigned)v);
          unsigned hi32 = __reduce_or_sync(0xffffffffu, (unsigned)(v >> 32));
          if (lane == 0) removed[w - b0] |= ((unsigned long long)hi32 << 32) | lo32;
        }
      }
      // columns beyond the register-prefetched window (very large segments): plain loads
      for (int w = b + 1 + warp + kScanWarps * kMaxColsPerWarp; w < nb; w += kScanWarps) {
        const int r = b * 64 + 2 * lane;
        unsigned long long v = 0ull;
        if (r < M) v |= maskT[(size_t)(w - b) * M + r] & k0;
        if (r + 1 < M) v |= maskT[(size_t)(w - b) * M + r + 1] & k1;
        unsigned lo32 = __reduce_or_sync(0xffffffffu, (unsigned)v);
        unsigned hi32 = __reduce_or_sync(0xffffffffu, (unsigned)(v >> 32));
        if (lane == 0) removed[w - b0] |= ((unsigned long long)hi32 << 32) | lo32;
      }
      __syncthreads();  // removed[], s_diag[(b+1)&1] visible; s_kept consumed
    };
    for (int b = b0; b < nb; b += 2) {
      process(b, bufA, bufB);
      if (b + 1 < nb) process(b + 1, bufB, bufA);
    }
  }
  // ---- the last CTA to get here compacts the flags in score order: keep[] = kept original indices, 0-padded to M
  __threadfence();
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(&ctrl->ticket, 1u) == gridDim.x - 1 ? 1u : 0u;
  __syncthreads();
  if (!s_last) return;
  __threadfence();
  const volatile unsigned char* kf = keepflag;
  const int per = (M + kScanThreads - 1) / kScanThreads;
  const int r0 = min(M, tid * per), r1 = min(M, r0 + per);
  int cnt = 0;
  for (int r = r0; r < r1; ++r) cnt += kf[r] ? 1 : 0;
  int total;
  int idx = block_excl_scan(cnt, warp_tot, total);
  for (int r = r0; r < r1; ++r)
    if (kf[r]) keep[idx++] = (long long)orig_of_grank[r];
  for (int r = total + tid; r < M; r += kScanThreads) keep[r] = 0;  // deterministic padding
  if (tid == 0) *num_keep = ctrl->error ? -1LL : (long long)total;
}

struct NmsWorkspace {
  NmsCtrl* ctrl;
  unsigned char* keepflag;
  int* grank_of_pos;
  int* orig_of_grank;
  int* seg_hi_of_pos;
  float* clsf_of_pos;
  int* seg_start;
  int* seg_end;
  float* sorted_boxes;
  unsigned long long* maskT;
  size_t zero_bytes;  // ctrl + keepflag are contiguous: one memset
  int wcap;
  size_t total;
};

size_t align_up(size_t v) { return (v + 255) & ~(size_t)255; }

NmsWorkspace carve(void* base, int64_t M, int rotated, int64_t max_segment) {
  NmsWorkspace w;
  size_t off = 0;
  char* p = (char*)base;
  auto take = [&](size_t bytes) {
    void* r = p ? p + off : nullptr;
    off += align_up(bytes);
    return r;
  };
  const size_t m = (size_t)(M > 0 ? M : 1);
  const size_t ms = (size_t)((max_segment <= 0 || max_segment > M) ? m : max_segment);
  w.wcap = (int)((ms + 62) / 64 + 1);  // word planes: a row meets at most ms - 1 later boxes, starting anywhere in its block
  w.ctrl = (NmsCtrl*)take(256);
  w.keepflag = (unsigned char*)take(m);
  w.zero_bytes = off;
  w.grank_of_pos = (int*)take(m * 4);
  w.orig_of_grank = (int*)take(m * 4);
  w.seg_hi_of_pos = (int*)take(m * 4);
  w.clsf_of_pos = (float*)take(m * 4);
  w.seg_start = (int*)take(m * 4);
  w.seg_end = (int*)take(m * 4);
  w.sorted_boxes = (float*)take(m * (rotated ? 5 : 4) * 4);
  w.maskT = (unsigned long long*)take((size_t)w.wcap * m * 8);
  w.total = off;
  return w;
}

}  // namespace

D2B_API size_t d2b_nms_workspace_bytes(int64_t M, int flags, int64_t max_segment) {
  return carve(nullptr, M, (flags & D2B_NMS_ROTATED) ? 1 : 0, max_segment).total;
}

D2B_API int d2b_nms(const float* boxes, const float* scores, const int64_t* idxs, int64_t M, double iou_threshold,
                    int flags, int64_t max_segment, int64_t* keep, int64_t* num_keep, void* workspace,
                    size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int rotated = (flags & D2B_NMS_ROTATED) ? 1 : 0;
  const bool no_offset = (flags & D2B_NMS_NO_OFFSET) != 0;  // idxs only segment the boxes; coordinates are used as given
  if (!num_keep || M < 0) return D2B_EINVAL;
  if (M == 0) {
    D2B_CUDA(cudaMemsetAsync(num_keep, 0, sizeof(int64_t), stream));
    return D2B_OK;
  }
  if (!boxes || !scores || !keep || !workspace) return D2B_EINVAL;
  if (M > (1 << 30)) return D2B_EUNSUPPORTED;
  if (max_segment <= 0 || max_segment > M) max_segment = M;
  NmsWorkspace w = carve(workspace, M, rotated, max_segment);
  if (workspace_bytes < w.total) return D2B_EWORKSPACE;
  const int m = (int)M, nb = (m + 63) / 64;
  const size_t smem = (size_t)w.wcap * sizeof(unsigned long long);  // removed[]: one word per block of a segment
  if (smem > 200 * 1024 || w.wcap > 65535) return D2B_EUNSUPPORTED;
  D2B_CUDA(cudaMemsetAsync(w.ctrl, 0, w.zero_bytes, stream));
  const int apply_offsets = (idxs && !no_offset) ? 1 : 0;
  // The reference runs ONE nms over the offset boxes, so two boxes of different categories meet with IoU 0 (or NaN when an
  // offset is NaN).  A threshold that IoU 0 passes (rotated iou >= thr, axis-aligned iou > thr) therefore suppresses
  // across categories: all non-ignored boxes then form one segment, still with their categories' offsets.
  const int one_segment = (apply_offsets && (rotated ? iou_threshold <= 0.0 : iou_threshold < 0.0)) ? 1 : 0;
  // 1. positions in the score order and in the category-major order, segments, coordinate range
  const int rank_grid = d2b_cdiv(m, 2 * kRankWarps);
  if (rotated)
    nms_rank_kernel<true><<<rank_grid, kRankWarps * 32, 0, stream>>>(boxes, scores, idxs, m, (int)max_segment, apply_offsets,
                                                                     one_segment, w.ctrl, w.grank_of_pos, w.orig_of_grank, w.seg_hi_of_pos,
                                                                     w.clsf_of_pos, w.sorted_boxes, w.seg_start, w.seg_end, w.keepflag);
  else
    nms_rank_kernel<false><<<rank_grid, kRankWarps * 32, 0, stream>>>(boxes, scores, idxs, m, (int)max_segment, apply_offsets,
                                                                      one_segment, w.ctrl, w.grank_of_pos, w.orig_of_grank, w.seg_hi_of_pos,
                                                                      w.clsf_of_pos, w.sorted_boxes, w.seg_start, w.seg_end, w.keepflag);
  D2B_CHECK_LAUNCH();
  // 2. IoU bitmask inside the categories (coordinate offsets of the reference's batched-NMS trick applied in fp32)
  if (rotated)
    nms_mask_kernel<true, 8><<<dim3(nb, w.wcap), 512, 0, stream>>>(w.sorted_boxes, w.seg_hi_of_pos, w.clsf_of_pos, w.ctrl, apply_offsets, m,
                                                     w.wcap, iou_threshold, w.maskT);
  else
    nms_mask_kernel<false, 4><<<dim3(nb, w.wcap), 256, 0, stream>>>(w.sorted_boxes, w.seg_hi_of_pos, w.clsf_of_pos, w.ctrl, apply_offsets, m,
                                                      w.wcap, iou_threshold, w.maskT);
  D2B_CHECK_LAUNCH();
  // 3. per-segment greedy scans in parallel + compaction in global score order by the last CTA
  D2B_ALLOW_BIG_SMEM(nms_scan_kernel);
  const int scan_grid = idxs ? (m < 2 * d2b_num_sms() ? m : 2 * d2b_num_sms()) : 1;
  nms_scan_kernel<<<scan_grid, kScanThreads, smem, stream>>>(w.maskT, w.grank_of_pos, w.orig_of_grank, w.seg_start, w.seg_end,
                                                             w.ctrl, m, w.wcap, w.keepflag, (long long*)keep, (long long*)num_keep);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_box_iou_rotated(const float* boxes1, int64_t N, const float* boxes2, int64_t M, float* ious,
                                void* stream) {
  if (N == 0 || M == 0) return D2B_OK;
  if (!boxes1 || !boxes2 || !ious || N < 0 || M < 0) return D2B_EINVAL;
  long long gx = (M + 127) / 128;
  if (gx > 2147483647LL) return D2B_EUNSUPPORTED;
  long long gy = N < 65535 ? N : 65535;
  // keep the grid a few waves deep; rows beyond gridDim.y are covered by the stride loop
  dim3 grid((unsigned)gx, (unsigned)gy);
  box_iou_rotated_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(boxes1, N, boxes2, M, ious);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
