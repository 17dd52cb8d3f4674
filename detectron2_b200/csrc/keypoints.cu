// Keypoint R-CNN head: heatmap-to-keypoint decoding (inference) and the fused keypoint loss (training).
//
// d2b_keypoints_from_heatmaps replaces the per-detection loop of heatmaps_to_keypoints
// (detectron2/structures/keypoints.py:164-235): per ROI a ceil(h) x ceil(w) bicubic resize of the K maps, the spatial
// argmax, and the softmax score of the argmax normalised over the S x S map.  The reference materialises every resized map
// and syncs with the host once per detection (int(heights_ceil[i])); here the bicubic map is evaluated on the fly and never
// stored, and the work is split into fixed pixel tiles so that a full-image box does not serialise on one CTA:
//   keypoints_prep_kernel     one CTA: tiles per ROI -> inclusive prefix (device), argmax keys zeroed
//   keypoints_argmax_kernel   persistent CTAs over the (tile, keypoint) items: the S x S map staged in shared memory, the
//                             tile's pixels evaluated with PyTorch's upsample_bicubic2d arithmetic, one 64-bit atomicMax
//                             of (order-preserving value bits << 32 | ~pixel index) per warp
//   keypoints_finish_kernel   one warp per (ROI, keypoint): the value at the winning pixel, the exp-sum over the S x S map,
//                             the coordinates
// Argmax rule (torch.argmax / max on CUDA): the largest value, ties to the smallest linear index; any NaN beats every
// number, the first NaN wins.  -0.0 and +0.0 are equal (the key is built from v + 0.0f); the reported logit is re-evaluated
// at the winning pixel, so it is bitwise the map value there.
//
// d2b_keypoint_loss_forward / _backward replace keypoint_rcnn_loss (modeling/roi_heads/keypoint_head.py:40-96): the
// per-image Keypoints.to_heatmap (_keypoints_to_heatmap, structures/keypoints.py:105-161), the nonzero() host sync, the
// gather of the valid logit rows and F.cross_entropy, as one CTA per (proposal, keypoint) row.
//
// This file is compiled with -fmad=false: every fused multiply-add below is written as __fmaf_rn where PyTorch's own
// build of upsample_bicubic2d_out_frame<float, float> contracts, everything else rounds each operation on its own as the
// reference's separate kernels do.  The contraction pattern (source index, both cubic-convolution polynomials, and the
// four-tap sums, whose first FMA adds x0 * c0 to the rounded x1 * c1) is the one the sm_90 SASS of that kernel in
// libtorch_cuda.so shows; on an H100 it reproduced PyTorch's CUDA bicubic output bit for bit over every pixel tested,
// where each other candidate pattern missed some.
#include <climits>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kPixPerThread = 16;
constexpr long long kTile = (long long)kThreads * kPixPerThread;  // output pixels per work item
constexpr int kArgmaxBlocksPerSm = 4;
constexpr double kMaxPixels = 4294967296.0;  // 2^32: the packed key holds a 32-bit pixel index

// ---- ROI geometry: heatmaps_to_keypoints lines 183-195 -------------------------------------------------------------
struct RoiGeom {
  float x1, y1, cw, ch;   // offsets and width / height corrections
  float wo_f, ho_f;       // ceil(w), ceil(h)
  unsigned wo, ho;        // the same as integers (valid only when ok)
  unsigned long long npix;
  bool ok;                // finite and at most 2^32 output pixels
};

__device__ __forceinline__ float clamp_min1(float v) { return v < 1.f ? 1.f : v; }  // torch.clamp(min=1): NaN stays NaN

__device__ __forceinline__ RoiGeom roi_geom(const float* __restrict__ roi) {
  RoiGeom g;
  g.x1 = roi[0];
  g.y1 = roi[1];
  const float w = clamp_min1(__fsub_rn(roi[2], roi[0]));
  const float h = clamp_min1(__fsub_rn(roi[3], roi[1]));
  g.wo_f = ceilf(w);
  g.ho_f = ceilf(h);
  g.cw = __fdiv_rn(w, g.wo_f);
  g.ch = __fdiv_rn(h, g.ho_f);
  g.ok = isfinite(g.wo_f) && isfinite(g.ho_f) && (double)g.wo_f * (double)g.ho_f <= kMaxPixels;
  g.wo = g.ok ? (unsigned)g.wo_f : 0u;
  g.ho = g.ok ? (unsigned)g.ho_f : 0u;
  g.npix = (unsigned long long)g.wo * g.ho;
  return g;
}

// ---- PyTorch's upsample_bicubic2d (align_corners=False) at one output pixel ------------------------------------------
// area_pixel_compute_source_index(scale, d, false, cubic=true) = scale * (d + 0.5) - 0.5, no clamp at 0.
__device__ __forceinline__ float src_index(float scale, unsigned d) {
  return __fmaf_rn(scale, __fadd_rn((float)d, 0.5f), -0.5f);
}

// cubic_interp1d(x0, x1, x2, x3, t) with A = -0.75 (UpSample.h get_cubic_upsample_coefficients):
//   c0 = ((A (t+1) - 5A) (t+1) + 8A) (t+1) - 4A,  c1 = ((A+2) t - (A+3)) t t + 1,  c2 = c1(1 - t),  c3 = c0(2 - t)
struct Cubic {
  float c0, c1, c2, c3;
};

__device__ __forceinline__ float conv1(float x) {  // ((A + 2) * x - (A + 3)) * x * x + 1
  return __fmaf_rn(__fmul_rn(__fmaf_rn(1.25f, x, -2.25f), x), x, 1.f);
}

__device__ __forceinline__ float conv2(float x) {  // ((A * x - 5 * A) * x + 8 * A) * x - 4 * A
  return __fmaf_rn(__fmaf_rn(__fmaf_rn(-0.75f, x, 3.75f), x, -6.f), x, 3.f);
}

__device__ __forceinline__ Cubic cubic_coeffs(float t) {
  Cubic c;
  c.c0 = conv2(__fadd_rn(t, 1.f));
  c.c1 = conv1(t);
  const float t2 = __fsub_rn(1.f, t);
  c.c2 = conv1(t2);
  c.c3 = conv2(__fadd_rn(t2, 1.f));
  return c;
}

__device__ __forceinline__ float interp(const Cubic& c, float x0, float x1, float x2, float x3) {
  // x0 * c0 + x1 * c1 + x2 * c2 + x3 * c3, left to right; PyTorch's build fuses x0 * c0 into the first add (x1 * c1 is
  // rounded on its own), then x2 * c2 and x3 * c3 into the next two
  return __fmaf_rn(x3, c.c3, __fmaf_rn(x2, c.c2, __fmaf_rn(x0, c.c0, __fmul_rn(x1, c.c1))));
}

struct Axis {
  int i[4];  // clamped source indices in-1 .. in+2
  Cubic c;
};

__device__ __forceinline__ Axis make_axis(float scale, unsigned d, int S) {
  const float real = src_index(scale, d);
  const int in = (int)floorf(real);
  Axis a;
  a.c = cubic_coeffs(__fsub_rn(real, (float)in));
#pragma unroll
  for (int k = 0; k < 4; ++k) a.i[k] = min(max(in - 1 + k, 0), S - 1);  // upsample_get_value_bounded
  return a;
}

// One output pixel of the (Ho, Wo) bicubic resize of the S x S map `m` (shared or global memory).  When the sizes are
// equal PyTorch copies the input (the kernel's special case), which differs from the arithmetic only for non-finite values.
__device__ __forceinline__ float bicubic_pixel(const float* m, int S, bool copy, float sx, float sy, unsigned ox,
                                               unsigned oy) {
  if (copy) return m[(size_t)oy * S + ox];
  const Axis ax = make_axis(sx, ox, S), ay = make_axis(sy, oy, S);
  float r[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const float* row = m + (size_t)ay.i[k] * S;
    r[k] = interp(ax.c, row[ax.i[0]], row[ax.i[1]], row[ax.i[2]], row[ax.i[3]]);
  }
  return interp(ay.c, r[0], r[1], r[2], r[3]);
}

// Order-preserving key: larger value -> larger key; NaN above +inf; ties -> the smaller index (stored complemented).
__device__ __forceinline__ unsigned long long argmax_key(float v, unsigned idx) {
  const unsigned u = __float_as_uint(__fadd_rn(v, 0.f));  // -0.0 -> +0.0
  const unsigned ord = (v != v) ? 0xFFFFFFFFu : ((u & 0x80000000u) ? ~u : (u | 0x80000000u));
  return ((unsigned long long)ord << 32) | (unsigned long long)(~idx);
}

struct MapScale {
  float sx, sy;
  bool copy;
};

__device__ __forceinline__ MapScale map_scale(const RoiGeom& g, int S) {
  MapScale s;
  s.sx = __fdiv_rn((float)S, g.wo_f);  // area_pixel_compute_scale: (float)input_size / output_size
  s.sy = __fdiv_rn((float)S, g.ho_f);
  s.copy = g.wo == (unsigned)S && g.ho == (unsigned)S;
  return s;
}

__global__ void __launch_bounds__(1024) keypoints_prep_kernel(const float* __restrict__ rois, int R, int K,
                                                              long long* __restrict__ tiles_end,
                                                              unsigned long long* __restrict__ keys) {
  __shared__ long long s_scan[1024];
  const int tid = threadIdx.x;
  const long long nkeys = (long long)R * K;
  for (long long i = tid; i < nkeys; i += 1024) keys[i] = 0ull;  // below every real key
  const int chunk = d2b_cdiv(R, 1024);
  const int r0 = min(tid * chunk, R), r1 = min(r0 + chunk, R);
  long long local = 0;
  for (int r = r0; r < r1; ++r) {
    const RoiGeom g = roi_geom(rois + (size_t)r * 4);
    local += (long long)((g.npix + kTile - 1) / kTile);
  }
  s_scan[tid] = local;
  __syncthreads();
  for (int off = 1; off < 1024; off <<= 1) {  // Hillis-Steele inclusive scan of the per-thread tile counts
    const long long v = tid >= off ? s_scan[tid - off] : 0;
    __syncthreads();
    s_scan[tid] += v;
    __syncthreads();
  }
  long long run = s_scan[tid] - local;
  for (int r = r0; r < r1; ++r) {
    const RoiGeom g = roi_geom(rois + (size_t)r * 4);
    run += (long long)((g.npix + kTile - 1) / kTile);
    tiles_end[r] = run;
  }
}

__global__ void __launch_bounds__(kThreads, kArgmaxBlocksPerSm) keypoints_argmax_kernel(
    const float* __restrict__ maps, const float* __restrict__ rois, int R, int K, int S,
    const long long* __restrict__ tiles_end, unsigned long long* __restrict__ keys) {
  extern __shared__ float s_map[];
  const int tid = threadIdx.x;
  const long long items = tiles_end[R - 1] * K;
  const int ss = S * S;
  for (long long item = blockIdx.x; item < items; item += gridDim.x) {
    const long long t = item / K;
    const int k = (int)(item - t * K);
    int lo = 0, hi = R - 1;  // first ROI whose tiles end after t
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (tiles_end[mid] > t) hi = mid; else lo = mid + 1;
    }
    const int r = lo;
    const long long tile = t - (r ? tiles_end[r - 1] : 0);
    const RoiGeom g = roi_geom(rois + (size_t)r * 4);
    const MapScale sc = map_scale(g, S);
    const float* __restrict__ src = maps + ((size_t)r * K + k) * ss;
    __syncthreads();  // the previous item is done with s_map
    for (int i = tid; i < ss; i += kThreads) s_map[i] = src[i];
    __syncthreads();
    const unsigned long long p0 = (unsigned long long)tile * kTile;
    unsigned long long best = 0ull;
#pragma unroll 4
    for (int j = 0; j < kPixPerThread; ++j) {
      const unsigned long long p = p0 + (unsigned long long)j * kThreads + tid;
      if (p < g.npix) {
        const unsigned idx = (unsigned)p;
        const unsigned oy = idx / g.wo, ox = idx - oy * g.wo;
        const float v = bicubic_pixel(s_map, S, sc.copy, sc.sx, sc.sy, ox, oy);
        const unsigned long long key = argmax_key(v, idx);
        best = key > best ? key : best;
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      best = other > best ? other : best;
    }
    if ((tid & 31) == 0 && best) atomicMax(keys + (size_t)r * K + k, best);
  }
}

__global__ void __launch_bounds__(kThreads) keypoints_finish_kernel(const float* __restrict__ maps,
                                                                   const float* __restrict__ rois, int R, int K, int S,
                                                                   const unsigned long long* __restrict__ keys,
                                                                   float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long rk = (long long)blockIdx.x * (kThreads / 32) + (threadIdx.x >> 5);
  if (rk >= (long long)R * K) return;
  const int r = (int)(rk / K);
  const RoiGeom g = roi_geom(rois + (size_t)r * 4);
  const unsigned long long key = keys[rk];
  float4* o = reinterpret_cast<float4*>(out) + rk;
  if (!g.ok || key == 0ull) {  // non-finite box, or more than 2^32 output pixels: a NaN row
    if (lane == 0) *o = make_float4(NAN, NAN, NAN, NAN);
    return;
  }
  const int ss = S * S;
  const float* __restrict__ m = maps + (size_t)rk * ss;
  const unsigned idx = ~(unsigned)key;
  const unsigned oy = idx / g.wo, ox = idx - oy * g.wo;
  const MapScale sc = map_scale(g, S);
  const float logit = bicubic_pixel(m, S, sc.copy, sc.sx, sc.sy, ox, oy);  // == the map's max (NaN if it holds one)
  float sum = 0.f;
  for (int i = lane; i < ss; i += 32) sum += expf(__fsub_rn(m[i], logit));
#pragma unroll
  for (int off = 16; off; off >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, off);
  if (lane == 0) {
    // score = exp(roi_map[pos] - max) / sum_{S x S} exp(maps - max); the numerator is exp(0) = 1 for a finite max
    const float score = __fdiv_rn(expf(__fsub_rn(logit, logit)), sum);
    const float x = __fadd_rn(__fmul_rn(__fadd_rn((float)ox, 0.5f), g.cw), g.x1);
    const float y = __fadd_rn(__fmul_rn(__fadd_rn((float)oy, 0.5f), g.ch), g.y1);
    *o = make_float4(x, y, logit, score);
  }
}

// ---- keypoint loss ------------------------------------------------------------------------------------------------
// One coordinate of _keypoints_to_heatmap: floor((c - lo) * (S / (hi - lo))), where torch evaluates S / t as
// t.reciprocal() * S; c == hi maps to S - 1.  Returns -1 when the cell is outside [0, S).  A NaN f (a NaN coordinate, or
// 0 * inf at c == lo of a subnormal-width box) is outside too: the reference's floor().long() gives INT64_MIN for it on
// CUDA, so the keypoint is not valid.
__device__ __forceinline__ int heatmap_cell(float c, float lo, float hi, int S) {
  if (c == hi) return S - 1;
  const float scale = __fmul_rn(__frcp_rn(__fsub_rn(hi, lo)), (float)S);
  const float f = floorf(__fmul_rn(__fsub_rn(c, lo), scale));
  return (f >= 0.f && f < (float)S) ? (int)f : -1;
}

__device__ __forceinline__ float block_reduce(float v, bool is_max, float* s_red) {
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = is_max ? fmaxf(v, w) : v + w;
  }
  __syncthreads();  // s_red may still be read by a previous reduction
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  v = s_red[0];
#pragma unroll
  for (int i = 1; i < kThreads / 32; ++i) v = is_max ? fmaxf(v, s_red[i]) : v + s_red[i];
  return v;
}

// Row max and exp-sum of one S*S logit row (log-sum-exp = m + log(sum)).  A NaN logit makes both NaN (fmaxf drops NaN,
// so it is carried separately), as log_softmax on CUDA.
template <int DT>
__device__ __forceinline__ void row_lse(const typename Elem<DT>::T* __restrict__ row, int n, float* s_red, float& m,
                                        float& sum) {
  float mx = -INFINITY;
  bool nan = false;
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const float x = Elem<DT>::ld(row + i);
    nan |= x != x;
    mx = fmaxf(mx, x);
  }
  nan = __syncthreads_or(nan);
  m = nan ? NAN : block_reduce(mx, true, s_red);
  float s = 0.f;
  for (int i = threadIdx.x; i < n; i += kThreads) s += expf(__fsub_rn(Elem<DT>::ld(row + i), m));
  sum = block_reduce(s, false, s_red);
}

template <int DT>
__global__ void __launch_bounds__(kThreads) keypoint_loss_fwd_kernel(const typename Elem<DT>::T* __restrict__ logits,
                                                                     int K, int S, const float* __restrict__ kps,
                                                                     const float* __restrict__ boxes,
                                                                     long long* __restrict__ target,
                                                                     uint8_t* __restrict__ valid, float* __restrict__ loss,
                                                                     unsigned long long* __restrict__ num_valid) {
  __shared__ float s_red[kThreads / 32];
  const long long row = blockIdx.x;
  const long long n = row / K;
  const float* b = boxes + n * 4;
  const float* kp = kps + row * 3;
  const int cx = heatmap_cell(kp[0], b[0], b[2], S), cy = heatmap_cell(kp[1], b[1], b[3], S);
  const bool ok = cx >= 0 && cy >= 0 && kp[2] > 0.f;
  const int lin = ok ? cy * S + cx : 0;
  if (threadIdx.x == 0) {
    target[row] = lin;
    valid[row] = ok ? 1 : 0;
    if (ok) atomicAdd(num_valid, 1ull);
  }
  if (!logits) return;  // targets only
  if (!ok) {
    if (threadIdx.x == 0) loss[row] = 0.f;
    return;
  }
  const int ss = S * S;
  const typename Elem<DT>::T* lr = logits + (size_t)row * ss;
  float m, sum;
  row_lse<DT>(lr, ss, s_red, m, sum);
  // cross_entropy = -log_softmax[t] = log(sum) - (x_t - m)
  if (threadIdx.x == 0) loss[row] = __fsub_rn(logf(sum), __fsub_rn(Elem<DT>::ld(lr + lin), m));
}

template <int DT>
__global__ void __launch_bounds__(kThreads) keypoint_loss_bwd_kernel(const typename Elem<DT>::T* __restrict__ logits, int S,
                                                                     const long long* __restrict__ target,
                                                                     const uint8_t* __restrict__ valid,
                                                                     const float* __restrict__ grad_scale,
                                                                     typename Elem<DT>::T* __restrict__ grad) {
  __shared__ float s_red[kThreads / 32];
  const long long row = blockIdx.x;
  const int ss = S * S;
  typename Elem<DT>::T* gr = grad + (size_t)row * ss;
  if (!valid[row]) {
    for (int i = threadIdx.x; i < ss; i += kThreads) gr[i] = Elem<DT>::st(0.f);
    return;
  }
  const typename Elem<DT>::T* lr = logits + (size_t)row * ss;
  float m, sum;
  row_lse<DT>(lr, ss, s_red, m, sum);
  const long long t = target[row];
  const float gs = grad_scale[row];
  for (int i = threadIdx.x; i < ss; i += kThreads) {
    const float p = __fdiv_rn(expf(__fsub_rn(Elem<DT>::ld(lr + i), m)), sum);
    gr[i] = Elem<DT>::st(__fmul_rn(__fsub_rn(p, i == t ? 1.f : 0.f), gs));
  }
}

bool map_fits(int S) { return S > 0 && S <= D2B_KEYPOINTS_MAX_S; }

}  // namespace

D2B_API size_t d2b_keypoints_workspace_bytes(int R, int K) {
  if (R <= 0 || K <= 0) return 0;
  return (size_t)R * K * sizeof(unsigned long long) + (size_t)R * sizeof(long long);
}

D2B_API int d2b_keypoints_from_heatmaps(const float* maps, int R, int K, int S, const float* rois, float* out,
                                        void* workspace, size_t workspace_bytes, void* stream) {
  if (R < 0 || K <= 0 || !map_fits(S)) return D2B_EINVAL;
  if (R == 0) return D2B_OK;
  if (!maps || !rois || !out || !workspace) return D2B_EINVAL;
  if (workspace_bytes < d2b_keypoints_workspace_bytes(R, K)) return D2B_EWORKSPACE;
  if ((uintptr_t)workspace % 8 || (uintptr_t)out % 16) return D2B_EINVAL;
  unsigned long long* keys = (unsigned long long*)workspace;
  long long* tiles_end = (long long*)(keys + (size_t)R * K);
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)S * S * sizeof(float);
  if (smem > 48 * 1024) D2B_ALLOW_BIG_SMEM(keypoints_argmax_kernel);
  keypoints_prep_kernel<<<1, 1024, 0, st>>>(rois, R, K, tiles_end, keys);
  D2B_CHECK_LAUNCH();
  keypoints_argmax_kernel<<<d2b_num_sms() * kArgmaxBlocksPerSm, kThreads, smem, st>>>(maps, rois, R, K, S, tiles_end, keys);
  D2B_CHECK_LAUNCH();
  const long long warps = (long long)R * K;
  keypoints_finish_kernel<<<d2b_cdiv(warps, kThreads / 32), kThreads, 0, st>>>(maps, rois, R, K, S, keys, out);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_keypoint_loss_forward(const void* logits, int dtype, int N, int K, int S, const float* keypoints,
                                      const float* boxes, int64_t* target, uint8_t* valid, float* loss_per_kp,
                                      int64_t* num_valid, void* stream) {
  if (N < 0 || K <= 0 || S <= 0 || (long long)S * S > INT_MAX || (long long)N * K > INT_MAX) return D2B_EINVAL;
  if (dtype != D2B_F32 && dtype != D2B_F16 && dtype != D2B_BF16) return D2B_EINVAL;
  if (!num_valid) return D2B_EINVAL;
  if (!logits != !loss_per_kp) return D2B_EINVAL;
  if (N > 0 && (!keypoints || !boxes || !target || !valid)) return D2B_EINVAL;
  const cudaStream_t st = (cudaStream_t)stream;
  D2B_CUDA(cudaMemsetAsync(num_valid, 0, sizeof(int64_t), st));
  if (N == 0) return D2B_OK;
  const int rows = N * K;
  unsigned long long* nv = (unsigned long long*)num_valid;
  long long* tg = (long long*)target;
  if (dtype == D2B_F32)
    keypoint_loss_fwd_kernel<D2B_F32><<<rows, kThreads, 0, st>>>((const float*)logits, K, S, keypoints, boxes, tg, valid,
                                                                  loss_per_kp, nv);
  else if (dtype == D2B_F16)
    keypoint_loss_fwd_kernel<D2B_F16><<<rows, kThreads, 0, st>>>((const __half*)logits, K, S, keypoints, boxes, tg, valid,
                                                                  loss_per_kp, nv);
  else
    keypoint_loss_fwd_kernel<D2B_BF16><<<rows, kThreads, 0, st>>>((const __nv_bfloat16*)logits, K, S, keypoints, boxes, tg,
                                                                   valid, loss_per_kp, nv);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_keypoint_loss_backward(const void* logits, int dtype, int N, int K, int S, const int64_t* target,
                                       const uint8_t* valid, const float* grad_scale, void* grad_logits, void* stream) {
  if (N < 0 || K <= 0 || S <= 0 || (long long)S * S > INT_MAX || (long long)N * K > INT_MAX) return D2B_EINVAL;
  if (dtype != D2B_F32 && dtype != D2B_F16 && dtype != D2B_BF16) return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  if (!logits || !target || !valid || !grad_scale || !grad_logits) return D2B_EINVAL;
  const cudaStream_t st = (cudaStream_t)stream;
  const int rows = N * K;
  const long long* tg = (const long long*)target;
  if (dtype == D2B_F32)
    keypoint_loss_bwd_kernel<D2B_F32><<<rows, kThreads, 0, st>>>((const float*)logits, S, tg, valid, grad_scale,
                                                                  (float*)grad_logits);
  else if (dtype == D2B_F16)
    keypoint_loss_bwd_kernel<D2B_F16><<<rows, kThreads, 0, st>>>((const __half*)logits, S, tg, valid, grad_scale,
                                                                  (__half*)grad_logits);
  else
    keypoint_loss_bwd_kernel<D2B_BF16><<<rows, kThreads, 0, st>>>((const __nv_bfloat16*)logits, S, tg, valid, grad_scale,
                                                                   (__nv_bfloat16*)grad_logits);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
