// Semantic segmentation loss: bilinear upsampling fused into the pixel cross-entropy, forward and backward.
// Restates SemSegFPNHead.losses (modeling/meta_arch/semantic_seg.py:255-267), the cross-entropy losses of the DeepLab heads
// and DeepLabCE (projects/DeepLab/deeplab/loss.py) without the [N, C, H, W] upsampled map, its log_softmax copy, or the
// float atomics of PyTorch's upsample_bilinear2d_backward.
//
//   sem_seg_fwd_kernel    one thread per output pixel (all images, kChunk pixels per CTA): the C upsampled values from the
//                         low-res footprint (read through L1 / L2), an online logsumexp, loss = lse - v[target]; writes lse,
//                         the per-pixel loss (top-k selection only) and per-CTA partials (sum, valid count, status)
//   topk_hist_kernel      x4 (top-k selection only): the radix select of the k-th largest per-pixel loss, 8 bits per launch
//                         over an order-preserving uint32 image of the fp32 values; integer histogram atomics only
//   topk_sum_kernel       per-CTA partials of the values above the threshold t and of the pixels tied at t
//   finish_kernel         one CTA: the partials added in a fixed order (double), + (k - #{v > t}) * t; the tie prefix
//   topk_mark_kernel      selected[p]: the k largest, ties at t taken in ascending flat index
//   sem_seg_bwd_kernel    owner computes: one CTA per (image, T x T tile of low-res pixels, channel chunk) evaluates
//                         g(p) * (softmax_c(p) - [t(p) = c]) once for every output pixel whose taps reach the tile (shared
//                         memory), then every low-res logit gathers its taps' weighted terms in a fixed order and is
//                         written once in the logits' dtype
// No float atomics: the loss, the counts and the gradient are bitwise reproducible.
//
// This file is compiled with -fmad=false: the upsampled values are PyTorch's CUDA upsample_bilinear2d arithmetic with the
// fused multiply-adds where its sm_90 build contracts (bilinear.cuh), so every value equals F.interpolate's bit for bit.
#include <algorithm>
#include <climits>
#include <cmath>

#include "bilinear.cuh"
#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kPixPerThread = 4;
constexpr int kChunk = kThreads * kPixPerThread;  // output pixels per CTA of the per-pixel launches
constexpr int kFinishThreads = 1024;
constexpr int kBins = 256;
constexpr int kLevels = 4;  // 8 bits per radix level
constexpr int kBwdThreads = 512;
constexpr size_t kBwdSmemTarget = 100 * 1024;  // two backward CTAs per SM where the stride allows it
constexpr size_t kAlign = 256;

inline size_t align_up(size_t v) { return (v + kAlign - 1) / kAlign * kAlign; }

enum Mode { kMean = 0, kAll = 1, kSelect = 2 };  // mean over valid pixels; top-k 1.0; top-k with a selection

// the taps of output row / column d; stride 1 is PyTorch's same-size copy
__device__ __forceinline__ Tap loss_tap(float scale, int stride, int d, int in_size) {
  if (stride == 1) {
    Tap t;
    t.i0 = t.i1 = d;
    t.l0 = 1.f, t.l1 = 0.f;
    return t;
  }
  return make_tap(scale, d, in_size);
}

// one upsampled value of channel plane s, fp32 (predictions.float() first)
template <int DT>
__device__ __forceinline__ float upsampled(const typename Elem<DT>::T* __restrict__ s, int Wp, const Tap& ty, const Tap& tx,
                                           bool copy) {
  if (copy) return Elem<DT>::ld(s + (size_t)ty.i0 * Wp + tx.i0);
  const size_t r0 = (size_t)ty.i0 * Wp, r1 = (size_t)ty.i1 * Wp;
  const float a = Elem<DT>::ld(s + r0 + tx.i0), b = Elem<DT>::ld(s + r0 + tx.i1);
  const float d = Elem<DT>::ld(s + r1 + tx.i0), e = Elem<DT>::ld(s + r1 + tx.i1);
  const float top = __fmaf_rn(tx.l0, a, __fmul_rn(tx.l1, b));
  const float bot = __fmaf_rn(tx.l0, d, __fmul_rn(tx.l1, e));
  return __fmaf_rn(ty.l0, top, __fmul_rn(ty.l1, bot));
}

// Order-preserving image of an fp32 value: every NaN above +inf (torch.topk's order), -0.0 and +0.0 one value.
__device__ __forceinline__ uint32_t order_key(float v) {
  if (v != v) return 0xffffffffu;
  if (v == 0.f) v = 0.f;
  const uint32_t u = __float_as_uint(v);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

__device__ __forceinline__ float key_value(uint32_t k) {
  if (k == 0xffffffffu) return __uint_as_float(0x7fc00000u);
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k);
}

template <class T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// CTA sum in a fixed order (warp butterflies, then the warp totals in warp order); the result is valid in thread 0.
template <class T, int kT>
__device__ __forceinline__ T block_sum(T v, T* s_red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) s_red[threadIdx.x >> 5] = v;
  __syncthreads();
  T t = T(0);
  if (threadIdx.x == 0)
    for (int k = 0; k < kT / 32; ++k) t += s_red[k];
  return t;
}

struct FwdArgs {
  const void* logits;
  const int64_t* targets;
  const float* weights;
  long long ignore;
  int N, C, Hp, Wp, H, W, stride, P, mode;
  float scale;
  float* lse;
  float* pix;       // [P] per-pixel loss * weight (kSelect)
  float* part_sum;  // [nb]
  int* part_cnt;    // [nb]
  int* part_stat;   // [nb]
  unsigned* hist;   // [kLevels, kBins] (kSelect): cleared here for the radix launches
};

template <int DT>
__global__ void __launch_bounds__(kThreads) sem_seg_fwd_kernel(const __grid_constant__ FwdArgs a) {
  __shared__ float s_f[kThreads / 32];
  __shared__ int s_i[kThreads / 32];
  using T = typename Elem<DT>::T;
  const T* __restrict__ logits = static_cast<const T*>(a.logits);
  if (a.hist && blockIdx.x == 0)
    for (int k = threadIdx.x; k < kLevels * kBins; k += kThreads) a.hist[k] = 0u;
  const int HW = a.H * a.W, C = a.C;
  const size_t plane = (size_t)a.Hp * a.Wp;
  const bool copy = a.stride == 1;
  float acc = 0.f;
  int cnt = 0, bad = 0;
  const int base = blockIdx.x * kChunk;
  for (int j = 0; j < kPixPerThread; ++j) {
    const int p = base + j * kThreads + threadIdx.x;
    if (p >= a.P) break;
    const long long t = a.targets[p];
    float loss = 0.f, lse = 0.f;
    bool valid = false;
    if (t != a.ignore) {
      if (t < 0 || t >= C) {
        bad = 1;
      } else {
        const int n = p / HW, q = p - n * HW, oy = q / a.W, ox = q - oy * a.W;
        const Tap ty = loss_tap(a.scale, a.stride, oy, a.Hp), tx = loss_tap(a.scale, a.stride, ox, a.Wp);
        const T* __restrict__ src = logits + (size_t)n * C * plane;
        float m = -INFINITY, s = 0.f, vt = 0.f;
        bool nan = false;
        for (int c = 0; c < C; ++c) {  // online logsumexp: one exp per channel
          const float v = upsampled<DT>(src + c * plane, a.Wp, ty, tx, copy);
          if (c == (int)t) vt = v;
          nan |= v != v;  // flagged apart from s: the first finite max resets s, whatever came before it
          if (v > m) {
            s = __fadd_rn(m == -INFINITY ? 0.f : __fmul_rn(s, __expf(__fsub_rn(m, v))), 1.f);
            m = v;
          } else if (v != -INFINITY) {
            s = __fadd_rn(s, __expf(__fsub_rn(v, m)));
          }
        }
        // log_softmax's max - log(sum exp(v - max)) is NaN when a channel is NaN, or +inf (inf - inf); so is the loss and
        // the backward's every exp(v - lse) of the pixel
        lse = nan || m == INFINITY ? __int_as_float(0x7fc00000) : __fadd_rn(m, __logf(s));
        loss = __fsub_rn(lse, vt);
        valid = true;
      }
    }
    a.lse[p] = lse;
    cnt += valid;
    if (a.mode == kMean) {
      if (valid) acc = __fadd_rn(acc, loss);
    } else {
      const float v = a.weights ? __fmul_rn(loss, a.weights[p]) : loss;  // criterion(...) * weights
      if (a.mode == kAll)
        acc = __fadd_rn(acc, v);
      else
        a.pix[p] = v;
    }
  }
  const float bs = block_sum<float, kThreads>(acc, s_f);
  __syncthreads();
  const int bc = block_sum<int, kThreads>(cnt, s_i);
  const int bb = __syncthreads_or(bad);
  if (threadIdx.x == 0) {
    a.part_sum[blockIdx.x] = bs;
    a.part_cnt[blockIdx.x] = bc;
    a.part_stat[blockIdx.x] = bb ? D2B_SEMSEG_STATUS_BAD_LABEL : 0;
  }
}

// ---- top-k selection --------------------------------------------------------------------------------------------------
struct SelState {
  uint32_t prefix;  // the key bits chosen so far (after kLevels levels: the k-th largest key t)
  long long above;  // values whose key is above the prefix's bucket (after kLevels levels: #{key > t})
  long long rem;    // k - above: the rank still to find inside the bucket (after kLevels levels: the ties taken at t)
};

// Walk the histograms of levels [0, levels): warp 0 finds each level's bucket of the k-th largest key, in a fixed order.
// Called by every thread (contains a barrier).  1 <= k <= P.
__device__ void select_state(const unsigned* __restrict__ hist, int levels, long long k, SelState* out) {
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    uint32_t prefix = 0;
    long long above = 0, rem = k;
    for (int L = 0; L < levels; ++L) {
      const unsigned* h = hist + L * kBins + lane * 8;
      unsigned v[8];
      long long mine = 0;
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = h[i], mine += v[i];
      long long inc = mine;  // suffix sum over the lanes >= lane (higher bins)
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const long long t = __shfl_down_sync(0xffffffffu, inc, o);
        if (lane + o < 32) inc += t;
      }
      long long run = inc - mine;  // keys in the buckets above this lane's
      int found = -1;
      long long found_above = 0;
#pragma unroll
      for (int i = 7; i >= 0; --i) {
        if (found < 0 && run < rem && run + v[i] >= rem) found = lane * 8 + i, found_above = run;
        run += v[i];
      }
      const unsigned ball = __ballot_sync(0xffffffffu, found >= 0);
      const int src = ball ? __ffs(ball) - 1 : 0;
      const int bin = __shfl_sync(0xffffffffu, found, src);
      const long long fa = __shfl_sync(0xffffffffu, found_above, src);
      prefix = (prefix << 8) | (uint32_t)(bin < 0 ? 0 : bin);
      above += fa;
      rem -= fa;
    }
    if (lane == 0) *out = SelState{prefix, above, rem};
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) topk_hist_kernel(const float* __restrict__ pix, int P, long long k,
                                                              unsigned* __restrict__ hist, int level) {
  __shared__ unsigned s_h[kBins];
  __shared__ SelState s_st;
  for (int i = threadIdx.x; i < kBins; i += kThreads) s_h[i] = 0u;
  select_state(hist, level, k, &s_st);
  const uint32_t prefix = s_st.prefix;
  const int shift = 24 - 8 * level;
  const int base = blockIdx.x * kChunk;
  for (int j = 0; j < kPixPerThread; ++j) {
    const int p = base + j * kThreads + threadIdx.x;
    if (p >= P) break;
    const uint32_t key = order_key(pix[p]);
    if (level == 0 || (key >> (shift + 8)) == prefix) atomicAdd(&s_h[(key >> shift) & (kBins - 1)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < kBins; i += kThreads)
    if (s_h[i]) atomicAdd(hist + level * kBins + i, s_h[i]);  // integer: the order does not matter
}

__global__ void __launch_bounds__(kThreads) topk_sum_kernel(const float* __restrict__ pix, int P, long long k,
                                                             const unsigned* __restrict__ hist, float* __restrict__ part_sum,
                                                             int* __restrict__ part_ties) {
  __shared__ float s_f[kThreads / 32];
  __shared__ int s_i[kThreads / 32];
  __shared__ SelState s_st;
  select_state(hist, kLevels, k, &s_st);
  const uint32_t t = s_st.prefix;
  float acc = 0.f;
  int ties = 0;
  const int base = blockIdx.x * kChunk;
  for (int j = 0; j < kPixPerThread; ++j) {
    const int p = base + j * kThreads + threadIdx.x;
    if (p >= P) break;
    const float v = pix[p];
    const uint32_t key = order_key(v);
    if (key > t)
      acc = __fadd_rn(acc, v);
    else if (key == t)
      ++ties;
  }
  const float bs = block_sum<float, kThreads>(acc, s_f);
  __syncthreads();
  const int bt = block_sum<int, kThreads>(ties, s_i);
  if (threadIdx.x == 0) part_sum[blockIdx.x] = bs, part_ties[blockIdx.x] = bt;
}

struct FinArgs {
  const float* part_sum;   // main partials (kMean / kAll) or the above-threshold partials (kSelect)
  const int* part_cnt;
  const int* part_stat;
  const int* part_ties;    // kSelect
  int* tie_base;           // kSelect: exclusive prefix of part_ties
  const unsigned* hist;
  long long k;
  int nb, mode;
  float* loss_sum;
  int64_t* count;
  int* status;
};

__global__ void __launch_bounds__(kFinishThreads) finish_kernel(const __grid_constant__ FinArgs a) {
  __shared__ double s_d[kFinishThreads];
  __shared__ long long s_c[kFinishThreads];
  __shared__ int s_s[kFinishThreads];
  __shared__ int s_tot[32];
  __shared__ SelState s_st;
  const int tid = threadIdx.x;
  const bool sums = a.mode != kSelect || a.k > 0;
  double f = 0.0;
  long long c = 0;
  int st = 0;
  for (int i = tid; i < a.nb; i += kFinishThreads) {
    if (sums) f += (double)a.part_sum[i];
    c += a.part_cnt[i];
    st |= a.part_stat[i];
  }
  s_d[tid] = f, s_c[tid] = c, s_s[tid] = st;
  __syncthreads();
  for (int o = kFinishThreads / 2; o; o >>= 1) {
    if (tid < o) s_d[tid] += s_d[tid + o], s_c[tid] += s_c[tid + o], s_s[tid] |= s_s[tid + o];
    __syncthreads();
  }
  if (a.mode == kSelect && a.k > 0) {
    select_state(a.hist, kLevels, a.k, &s_st);
    int run = 0;
    for (int i0 = 0; i0 < a.nb; i0 += kFinishThreads) {  // tie prefix over the CTAs, in CTA order
      const int i = i0 + tid;
      int total;
      const int before = block_exclusive_scan(i < a.nb ? a.part_ties[i] : 0, s_tot, total);
      if (i < a.nb) a.tie_base[i] = run + before;
      run += total;
      __syncthreads();
    }
  }
  if (tid == 0) {
    double total = s_d[0];
    if (a.mode == kSelect && a.k > 0 && s_st.rem > 0) total += (double)s_st.rem * (double)key_value(s_st.prefix);
    *a.loss_sum = (float)total;
    *a.count = s_c[0];
    *a.status = s_s[0];
  }
}

__global__ void __launch_bounds__(kThreads) topk_mark_kernel(const float* __restrict__ pix, int P, long long k,
                                                              const unsigned* __restrict__ hist,
                                                              const int* __restrict__ tie_base,
                                                              uint8_t* __restrict__ selected) {
  __shared__ int s_tot[32];
  __shared__ SelState s_st;
  const int base = blockIdx.x * kChunk;
  if (k == 0) {
    for (int j = 0; j < kPixPerThread; ++j) {
      const int p = base + j * kThreads + threadIdx.x;
      if (p < P) selected[p] = 0;
    }
    return;
  }
  select_state(hist, kLevels, k, &s_st);
  const uint32_t t = s_st.prefix;
  const long long rem = s_st.rem;
  long long taken = tie_base[blockIdx.x];
  for (int j = 0; j < kPixPerThread; ++j) {  // pixel order: j-major, then thread: ascending flat index
    const int p = base + j * kThreads + threadIdx.x;
    const uint32_t key = p < P ? order_key(pix[p]) : 0u;
    const int tie = p < P && key == t;
    int total;
    const int before = block_exclusive_scan(tie, s_tot, total);
    if (p < P) selected[p] = (key > t || (tie && taken + before < rem)) ? 1 : 0;
    taken += total;
    __syncthreads();
  }
}

// ---- backward ---------------------------------------------------------------------------------------------------------
struct BwdArgs {
  const void* logits;
  const int64_t* targets;
  const float* weights;
  const uint8_t* selected;
  const float* lse;
  const float* grad_sum;
  void* grad;
  long long ignore;
  int N, C, Hp, Wp, H, W, stride;
  float scale;
  int T, tiles_x, CC, nchunks, RBY, RBX;  // tile side, tiles per row, channels per CTA, channel chunks, region bounds
};

// first d in [0, n) with pred(d) true (pred monotone false -> true); n when none
template <class F>
__device__ __forceinline__ int first_true(int n, F pred) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (pred(mid))
      hi = mid;
    else
      lo = mid + 1;
  }
  return lo;
}

template <int DT>
__global__ void __launch_bounds__(kBwdThreads) sem_seg_bwd_kernel(const __grid_constant__ BwdArgs a) {
  extern __shared__ float smem[];
  using T = typename Elem<DT>::T;
  const int chunk = blockIdx.x % a.nchunks, tile = blockIdx.x / a.nchunks, n = blockIdx.y;
  const int ty0 = (tile / a.tiles_x) * a.T, tx0 = (tile % a.tiles_x) * a.T;
  const int ty1 = min(ty0 + a.T, a.Hp), tx1 = min(tx0 + a.T, a.Wp);
  const int c0 = chunk * a.CC, cc = min(a.CC, a.C - c0);
  const int H = a.H, W = a.W, Hp = a.Hp, Wp = a.Wp, stride = a.stride;
  const float scale = a.scale;
  const bool copy = stride == 1;
  // the output rows whose taps reach rows [ty0, ty1): i1 >= ty0 and i0 < ty1 (both monotone in the output row)
  const int oy_lo = first_true(H, [&](int d) { return loss_tap(scale, stride, d, Hp).i1 >= ty0; });
  const int oy_hi = first_true(H, [&](int d) { return loss_tap(scale, stride, d, Hp).i0 >= ty1; });
  const int ox_lo = first_true(W, [&](int d) { return loss_tap(scale, stride, d, Wp).i1 >= tx0; });
  const int ox_hi = first_true(W, [&](int d) { return loss_tap(scale, stride, d, Wp).i0 >= tx1; });
  const int RY = min(oy_hi - oy_lo, a.RBY), RX = min(ox_hi - ox_lo, a.RBX), RQ = RY * RX;
  const int RBQ = a.RBY * a.RBX;
  float* D = smem;                       // [cc, RY, RX] g(p) * (softmax_c(p) - [t(p) = c])
  float* sL = D + (size_t)a.CC * RBQ;    // [RQ] lse
  float* sG = sL + RBQ;                  // [RQ] g(p)
  int* sT = reinterpret_cast<int*>(sG + RBQ);  // [RQ] target, -1: no gradient
  int* ry0 = sT + RBQ;
  int* ry1 = ry0 + a.RBY;
  float* rl0 = reinterpret_cast<float*>(ry1 + a.RBY);
  float* rl1 = rl0 + a.RBY;
  int* cx0 = reinterpret_cast<int*>(rl1 + a.RBY);
  int* cx1 = cx0 + a.RBX;
  float* cl0 = reinterpret_cast<float*>(cx1 + a.RBX);
  float* cl1 = cl0 + a.RBX;
  int* yr = reinterpret_cast<int*>(cl1 + a.RBX);  // [2 T] per tile row: its output rows [yr[2i], yr[2i+1]) (region-local)
  int* xr = yr + 2 * a.T;
  const int tid = threadIdx.x;
  for (int i = tid; i < RY; i += kBwdThreads) {
    const Tap t = loss_tap(scale, stride, oy_lo + i, Hp);
    ry0[i] = t.i0, ry1[i] = t.i1, rl0[i] = t.l0, rl1[i] = t.l1;
  }
  for (int i = tid; i < RX; i += kBwdThreads) {
    const Tap t = loss_tap(scale, stride, ox_lo + i, Wp);
    cx0[i] = t.i0, cx1[i] = t.i1, cl0[i] = t.l0, cl1[i] = t.l1;
  }
  for (int i = tid; i < ty1 - ty0; i += kBwdThreads) {
    const int y = ty0 + i;
    const int lo = first_true(H, [&](int d) { return loss_tap(scale, stride, d, Hp).i1 >= y; });
    const int hi = first_true(H, [&](int d) { return loss_tap(scale, stride, d, Hp).i0 >= y + 1; });
    yr[2 * i] = max(lo - oy_lo, 0), yr[2 * i + 1] = min(hi - oy_lo, RY);
  }
  for (int i = tid; i < tx1 - tx0; i += kBwdThreads) {
    const int x = tx0 + i;
    const int lo = first_true(W, [&](int d) { return loss_tap(scale, stride, d, Wp).i1 >= x; });
    const int hi = first_true(W, [&](int d) { return loss_tap(scale, stride, d, Wp).i0 >= x + 1; });
    xr[2 * i] = max(lo - ox_lo, 0), xr[2 * i + 1] = min(hi - ox_lo, RX);
  }
  const float gs = *a.grad_sum;
  for (int q = tid; q < RQ; q += kBwdThreads) {  // g(p): d loss / d loss_p
    const int qy = q / RX;
    const size_t p = ((size_t)n * H + oy_lo + qy) * W + ox_lo + (q - qy * RX);
    const long long t = a.targets[p];
    int tt = -1;
    float g = 0.f, l = 0.f;
    if (t != a.ignore && t >= 0 && t < a.C && (!a.selected || a.selected[p])) {
      tt = (int)t;
      g = a.weights ? __fmul_rn(gs, a.weights[p]) : gs;
      l = a.lse[p];
    }
    sT[q] = tt, sG[q] = g, sL[q] = l;
  }
  __syncthreads();
  const size_t plane = (size_t)Hp * Wp;
  const T* __restrict__ src = static_cast<const T*>(a.logits) + ((size_t)n * a.C + c0) * plane;
  for (int idx = tid; idx < cc * RQ; idx += kBwdThreads) {
    const int c = idx / RQ, q = idx - c * RQ;
    const int tt = sT[q];
    float d = 0.f;
    if (tt >= 0) {
      const int qy = q / RX, qx = q - qy * RX;
      Tap ty, tx;
      ty.i0 = ry0[qy], ty.i1 = ry1[qy], ty.l0 = rl0[qy], ty.l1 = rl1[qy];
      tx.i0 = cx0[qx], tx.i1 = cx1[qx], tx.l0 = cl0[qx], tx.l1 = cl1[qx];
      const float v = upsampled<DT>(src + c * plane, Wp, ty, tx, copy);
      const float pr = __expf(__fsub_rn(v, sL[q]));
      d = __fmul_rn(sG[q], c0 + c == tt ? __fsub_rn(pr, 1.f) : pr);
    }
    D[idx] = d;
  }
  __syncthreads();
  const int TY = ty1 - ty0, TX = tx1 - tx0, TQ = TY * TX;
  T* __restrict__ grad = static_cast<T*>(a.grad) + ((size_t)n * a.C + c0) * plane;
  for (int idx = tid; idx < cc * TQ; idx += kBwdThreads) {
    const int c = idx / TQ, r = idx - c * TQ, iy = r / TX, ix = r - iy * TX;
    const int y = ty0 + iy, x = tx0 + ix;
    const float* Dc = D + c * RQ;
    float acc = 0.f;
    for (int qy = yr[2 * iy]; qy < yr[2 * iy + 1]; ++qy) {  // output rows, then columns, ascending
      const float wy = __fadd_rn(ry0[qy] == y ? rl0[qy] : 0.f, ry1[qy] == y ? rl1[qy] : 0.f);
      float row = 0.f;
      for (int qx = xr[2 * ix]; qx < xr[2 * ix + 1]; ++qx) {
        const float wx = __fadd_rn(cx0[qx] == x ? cl0[qx] : 0.f, cx1[qx] == x ? cl1[qx] : 0.f);
        row = __fmaf_rn(wx, Dc[qy * RX + qx], row);
      }
      acc = __fmaf_rn(wy, row, acc);
    }
    grad[(size_t)c * plane + (size_t)y * Wp + x] = Elem<DT>::st(acc);
  }
}

// ---- host ---------------------------------------------------------------------------------------------------------
bool shape_ok(int N, int C, int Hp, int Wp, int stride, int dtype) {
  if (N < 0 || N > 65535 || C < 1 || Hp < 1 || Wp < 1 || stride < 1 || stride > D2B_SEMSEG_MAX_STRIDE) return false;
  if (dtype != D2B_F32 && dtype != D2B_F16 && dtype != D2B_BF16) return false;
  const long long H = (long long)Hp * stride, W = (long long)Wp * stride;
  return (long long)N * H * W <= INT_MAX - kChunk && (long long)C * Hp * Wp <= INT_MAX;
}

// rule 1 of the forward; sets the mode and k
bool fwd_args_ok(int N, int C, int Hp, int Wp, int stride, int dtype, int reduction, double top_k, bool has_weights,
                 int& mode, long long& k) {
  if (!shape_ok(N, C, Hp, Wp, stride, dtype)) return false;
  const long long P = (long long)N * Hp * stride * Wp * stride;
  if (reduction == D2B_SEMSEG_MEAN) {
    if (has_weights) return false;
    mode = kMean, k = 0;
    return true;
  }
  if (reduction != D2B_SEMSEG_TOP_K || !(top_k >= 0.0 && top_k <= 1.0)) return false;
  k = (long long)(top_k * (double)P);  // int(top_k_percent_pixels * numel) in Python
  mode = top_k == 1.0 ? kAll : kSelect;
  return true;
}

struct Layout {
  size_t part_sum, part_cnt, part_stat, hist, pix, part_sum2, part_ties, tie_base, total;
};

Layout fwd_layout(long long P, int mode) {
  const size_t nb = (size_t)d2b_cdiv(P, kChunk);
  Layout L{};
  size_t off = 0;
  L.part_sum = off, off = align_up(off + nb * 4);
  L.part_cnt = off, off = align_up(off + nb * 4);
  L.part_stat = off, off = align_up(off + nb * 4);
  if (mode == kSelect) {
    L.hist = off, off = align_up(off + kLevels * kBins * 4);
    L.pix = off, off = align_up(off + (size_t)P * 4);
    L.part_sum2 = off, off = align_up(off + nb * 4);
    L.part_ties = off, off = align_up(off + nb * 4);
    L.tie_base = off, off = align_up(off + nb * 4);
  }
  L.total = off < kAlign ? kAlign : off;
  return L;
}

// backward tiling: T x T low-res pixels per CTA, the output region of a tile bounded by (T + 1) * stride + 2 per axis
struct BwdPlan {
  int T, RBY, RBX, CC;
  size_t smem;
};

size_t bwd_smem(int T, int RBY, int RBX, int CC) {
  const size_t rbq = (size_t)RBY * RBX;
  return (size_t)CC * rbq * 4 + rbq * 12 + (size_t)(RBY + RBX) * 16 + (size_t)T * 16;
}

BwdPlan bwd_plan(int C, int Hp, int Wp, int stride) {
  BwdPlan b;
  b.T = std::max(2, 32 / stride);
  b.RBY = (int)std::min<long long>((long long)(b.T + 1) * stride + 2, (long long)Hp * stride);
  b.RBX = (int)std::min<long long>((long long)(b.T + 1) * stride + 2, (long long)Wp * stride);
  const size_t fixed = bwd_smem(b.T, b.RBY, b.RBX, 0), per = (size_t)b.RBY * b.RBX * 4;
  b.CC = kBwdSmemTarget > fixed + per ? (int)((kBwdSmemTarget - fixed) / per) : 1;
  b.CC = std::max(1, std::min(b.CC, C));
  b.smem = bwd_smem(b.T, b.RBY, b.RBX, b.CC);
  return b;
}

template <int DT>
int launch_bwd(const BwdArgs& a, const BwdPlan& b, long long ctas, cudaStream_t st) {
  D2B_ALLOW_BIG_SMEM(sem_seg_bwd_kernel<DT>);
  sem_seg_bwd_kernel<DT><<<dim3((unsigned)ctas, a.N), kBwdThreads, b.smem, st>>>(a);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

}  // namespace

D2B_API size_t d2b_sem_seg_loss_workspace_bytes(int N, int C, int Hp, int Wp, int stride, int dtype, int reduction,
                                                double top_k_percent_pixels) {
  int mode = 0;
  long long k = 0;
  if (!fwd_args_ok(N, C, Hp, Wp, stride, dtype, reduction, top_k_percent_pixels, false, mode, k)) return 0;
  return fwd_layout((long long)N * Hp * stride * Wp * stride, mode).total;
}

D2B_API int d2b_sem_seg_loss_forward(const void* logits, int dtype, int N, int C, int Hp, int Wp, int stride,
                                     const int64_t* targets, int64_t ignore_value, int reduction,
                                     double top_k_percent_pixels, const float* weights, float* lse, uint8_t* selected,
                                     float* loss_sum, int64_t* count, int* status, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  int mode = 0;
  long long k = 0;
  if (!fwd_args_ok(N, C, Hp, Wp, stride, dtype, reduction, top_k_percent_pixels, weights != nullptr, mode, k))
    return D2B_EINVAL;
  if (!loss_sum || !count || !status) return D2B_EINVAL;
  if (N > 0 && (!logits || !targets || !lse)) return D2B_EINVAL;
  if (mode == kSelect && !selected) return D2B_EINVAL;
  if (!workspace || (uintptr_t)workspace % kAlign) return D2B_EINVAL;
  const long long P = (long long)N * Hp * stride * Wp * stride;
  const Layout L = fwd_layout(P, mode);
  if (workspace_bytes < L.total) return D2B_EWORKSPACE;
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const int nb = d2b_cdiv(P, kChunk);
  const cudaStream_t st = (cudaStream_t)stream;
  float* part_sum = (float*)(ws + L.part_sum);
  int* part_cnt = (int*)(ws + L.part_cnt);
  int* part_stat = (int*)(ws + L.part_stat);
  unsigned* hist = mode == kSelect ? (unsigned*)(ws + L.hist) : nullptr;
  float* pix = mode == kSelect ? (float*)(ws + L.pix) : nullptr;
  if (nb > 0) {
    FwdArgs a;
    a.logits = logits, a.targets = targets, a.weights = weights, a.ignore = ignore_value;
    a.N = N, a.C = C, a.Hp = Hp, a.Wp = Wp, a.H = Hp * stride, a.W = Wp * stride, a.stride = stride, a.P = (int)P;
    a.mode = mode, a.scale = (float)(1.0 / stride);  // PyTorch's scale from a scale factor, not input / output size
    a.lse = lse, a.pix = pix, a.part_sum = part_sum, a.part_cnt = part_cnt, a.part_stat = part_stat, a.hist = hist;
    if (dtype == D2B_F32)
      sem_seg_fwd_kernel<D2B_F32><<<nb, kThreads, 0, st>>>(a);
    else if (dtype == D2B_F16)
      sem_seg_fwd_kernel<D2B_F16><<<nb, kThreads, 0, st>>>(a);
    else
      sem_seg_fwd_kernel<D2B_BF16><<<nb, kThreads, 0, st>>>(a);
    D2B_CHECK_LAUNCH();
  }
  FinArgs f;
  f.part_sum = part_sum, f.part_cnt = part_cnt, f.part_stat = part_stat, f.part_ties = nullptr, f.tie_base = nullptr;
  f.hist = hist, f.k = k, f.nb = nb, f.mode = mode, f.loss_sum = loss_sum, f.count = count, f.status = status;
  if (mode == kSelect && k > 0) {
    for (int level = 0; level < kLevels; ++level) {
      topk_hist_kernel<<<nb, kThreads, 0, st>>>(pix, (int)P, k, hist, level);
      D2B_CHECK_LAUNCH();
    }
    float* part_sum2 = (float*)(ws + L.part_sum2);
    int* part_ties = (int*)(ws + L.part_ties);
    topk_sum_kernel<<<nb, kThreads, 0, st>>>(pix, (int)P, k, hist, part_sum2, part_ties);
    D2B_CHECK_LAUNCH();
    f.part_sum = part_sum2, f.part_ties = part_ties, f.tie_base = (int*)(ws + L.tie_base);
  }
  finish_kernel<<<1, kFinishThreads, 0, st>>>(f);
  D2B_CHECK_LAUNCH();
  if (mode == kSelect && nb > 0) {
    topk_mark_kernel<<<nb, kThreads, 0, st>>>(pix, (int)P, k, hist, f.tie_base, selected);
    D2B_CHECK_LAUNCH();
  }
  return D2B_OK;
}

D2B_API int d2b_sem_seg_loss_backward(const void* logits, int dtype, int N, int C, int Hp, int Wp, int stride,
                                      const int64_t* targets, int64_t ignore_value, const float* weights,
                                      const uint8_t* selected, const float* lse, const float* grad_sum,
                                      void* grad_logits, void* stream) {
  if (!shape_ok(N, C, Hp, Wp, stride, dtype)) return D2B_EINVAL;
  if (N == 0) return D2B_OK;
  if (!logits || !targets || !lse || !grad_sum || !grad_logits) return D2B_EINVAL;
  const BwdPlan b = bwd_plan(C, Hp, Wp, stride);
  BwdArgs a;
  a.logits = logits, a.targets = targets, a.weights = weights, a.selected = selected, a.lse = lse;
  a.grad_sum = grad_sum, a.grad = grad_logits, a.ignore = ignore_value;
  a.N = N, a.C = C, a.Hp = Hp, a.Wp = Wp, a.H = Hp * stride, a.W = Wp * stride, a.stride = stride;
  a.scale = (float)(1.0 / stride);
  a.T = b.T, a.tiles_x = d2b_cdiv(Wp, b.T), a.CC = b.CC, a.nchunks = d2b_cdiv(C, b.CC), a.RBY = b.RBY, a.RBX = b.RBX;
  const long long ctas = (long long)d2b_cdiv(Hp, b.T) * a.tiles_x * a.nchunks;
  if (ctas > INT_MAX) return D2B_EINVAL;
  const cudaStream_t st = (cudaStream_t)stream;
  if (dtype == D2B_F32) return launch_bwd<D2B_F32>(a, b, ctas, st);
  if (dtype == D2B_F16) return launch_bwd<D2B_F16>(a, b, ctas, st);
  return launch_bwd<D2B_BF16>(a, b, ctas, st);
}
