// RoIAlign / ROIAlignRotated forward + backward for sm_90a.
//
// Semantics follow torchvision roi_align (detectron2/layers/roi_align.py:58-65; arithmetic as in
// torchvision/ops/roi_align.py::_roi_align) and detectron2/layers/csrc/ROIAlignRotated/ROIAlignRotated_cuda.cu:143-323.
//
// Design (differs from the reference's one-thread-per-output grid-stride loop):
//   * axis-aligned forward on channels-last storage: roi_align_nhwc_kernel -- lane = 4 channels, a warp reads a tap pixel's
//     128 channels as one 512-byte request with warp-uniform tap index / weight, 8 loads in flight; used in place for
//     torch.channels_last inputs, or after nchw_to_nhwc_kernel (one launch for a whole pyramid) when that pays;
//   * axis-aligned forward (NCHW) AND backward: roi_align_v3_kernel<BWD> -- per-RoI separable tap lists built once per CTA,
//     every warp stages (forward) or accumulates (backward) the RoI's pixel footprint of 4 channel planes in its private
//     shared-memory slice, lane == bin, no CTA barrier in the channel loop; the FPN level of a RoI is picked in-kernel so
//     that a whole multi-level ROIPooler call is one launch;
//   * rotated forward: one CTA per (RoI, channel slab) with a 2-D tap table in shared memory (the sample grid of a
//     rotated RoI is not a product grid), threads mapped to (channel, bin);
//   * rotated backward: thread per (channel, bin), red.global.add per tap;
//   * the rotated kernels (both layouts) pick the FPN level of a RoI in-kernel as well, from its w*h: a multi-level
//     ROIPooler(pooler_type="ROIAlignRotated") call is one launch per direction.
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;

#define D2B_DISPATCH_DTYPE(dt, ...)                  \
  do {                                               \
    if ((dt) == D2B_F32) {                           \
      constexpr int DT = D2B_F32;                    \
      __VA_ARGS__;                                   \
    } else if ((dt) == D2B_F16) {                    \
      constexpr int DT = D2B_F16;                    \
      __VA_ARGS__;                                   \
    } else {                                         \
      constexpr int DT = D2B_BF16;                   \
      __VA_ARGS__;                                   \
    }                                                \
  } while (0)
static inline bool dtype_ok(int dt) { return dt == D2B_F32 || dt == D2B_F16 || dt == D2B_BF16; }

struct RoiGeom {
  int b;
  float start_h, start_w, bin_h, bin_w;
  int gh, gw;
  float inv_count;  // 1 / max(gh*gw,1)
  float count_raw;  // gh*gw (backward divides by the raw product)
  float ctr_h, ctr_w, cos_t, sin_t;
};

// Feature pyramid passed by value to the kernels (single-level ops use num_levels == 1).
struct Pyr {
  int num_levels;
  const float* feat[D2B_MAX_LEVELS];
  float* grad[D2B_MAX_LEVELS];
  int H[D2B_MAX_LEVELS], W[D2B_MAX_LEVELS];
  float scale[D2B_MAX_LEVELS];
  int min_level, max_level, canonical_level;
  float canonical_box_size;
  const float* level_rois;  // [K,5] boxes the FPN level is computed from; null = the sampling rois themselves
};

// FPN level of a box: detectron2/modeling/poolers.py:54-62 (assign_boxes_to_levels), fp32 like torch:
//   floor(canonical_level + log2(sqrt(area) / canonical_box_size + 1e-8)), clamped to [min_level, max_level]
// `roi` is a pooler row: (b, x1, y1, x2, y2) with area (x2-x1)(y2-y1), or with ROT (b, cx, cy, w, h, angle) with area w*h
// (RotatedBoxes.area, structures/rotated_boxes.py:236-245).
template <bool ROT = false>
__device__ __forceinline__ int pick_level(const Pyr& P, const float* __restrict__ roi) {
  if (P.num_levels == 1) return 0;
  const float area = ROT ? roi[3] * roi[4] : (roi[3] - roi[1]) * (roi[4] - roi[2]);
  const float size = sqrtf(area);
  float lvl = floorf((float)P.canonical_level + log2f(size / P.canonical_box_size + 1e-8f));
  // A NaN level (negative or NaN area: malformed box) survives torch.clamp as NaN and matches no level in the reference's loop
  // (poolers.py:245-263): the RoI's output stays zero and it receives no gradient.  -1 tells the kernels exactly that.
  if (!(lvl == lvl)) return -1;
  lvl = fminf(fmaxf(lvl, (float)P.min_level), (float)P.max_level);
  return (int)lvl - P.min_level;
}

template <bool ROT>
__device__ __forceinline__ RoiGeom load_geom(const float* __restrict__ roi, float scale, int PH, int PW, int sr,
                                             int aligned, bool dead = false) {
  RoiGeom g;
  g.b = (int)roi[0];
  float rw, rh;
  if (ROT) {  // ROIAlignRotated_cuda.cu:166-183
    g.ctr_w = roi[1] * scale - 0.5f;
    g.ctr_h = roi[2] * scale - 0.5f;
    rw = roi[3] * scale;
    rh = roi[4] * scale;
    float theta = (float)((double)roi[5] * 3.14159265358979323846 / 180.0);  // ROIAlignRotated_cuda.cu:173
    sincosf(theta, &g.sin_t, &g.cos_t);
    g.start_h = -rh / 2.0f;
    g.start_w = -rw / 2.0f;
  } else {
    float off = aligned ? 0.5f : 0.0f;
    float sw = roi[1] * scale - off, sh = roi[2] * scale - off;
    float ew = roi[3] * scale - off, eh = roi[4] * scale - off;
    rw = ew - sw;
    rh = eh - sh;
    if (!aligned) {
      rw = fmaxf(rw, 1.f);
      rh = fmaxf(rh, 1.f);
    }
    g.start_h = sh;
    g.start_w = sw;
    g.ctr_h = g.ctr_w = 0.f;
    g.cos_t = 1.f;
    g.sin_t = 0.f;
  }
  g.bin_h = rh / (float)PH;
  g.bin_w = rw / (float)PW;
  g.gh = sr > 0 ? sr : (int)ceilf(rh / (float)PH);
  g.gw = sr > 0 ? sr : (int)ceilf(rw / (float)PW);
  if (g.gh < 0) g.gh = 0;
  if (g.gw < 0) g.gw = 0;
  if (dead) g.gh = g.gw = 0;  // RoI without a level: an empty sampling grid gives zero output and no gradient
  int c = g.gh * g.gw;
  g.count_raw = (float)c;
  g.inv_count = 1.0f / (float)(c < 1 ? 1 : c);
  return g;
}

// 1-D tap: low/high index (clamped) and the two weights; valid=0 when the coordinate is outside [-1, size].
struct Tap1 {
  int lo, hi;
  float wl, wh;  // wh = frac, wl = 1-frac ; both 0 when invalid
};

__device__ __forceinline__ Tap1 make_tap1(float v, int size) {
  Tap1 t;
  if (v < -1.0f || v > (float)size) {
    t.lo = t.hi = 0;
    t.wl = t.wh = 0.f;
    return t;
  }
  v = fmaxf(v, 0.f);
  int lo = (int)v;
  int hi;
  if (lo >= size - 1) {
    hi = lo = size - 1;
    v = (float)lo;
  } else {
    hi = lo + 1;
  }
  float l = v - (float)lo;
  t.lo = lo;
  t.hi = hi;
  t.wh = l;
  t.wl = 1.f - l;
  return t;
}

// ------------------------------------------------------------------ rotated forward
struct Tap2 {
  int p1, p2, p3, p4;
  float w1, w2, w3, w4;
};

__device__ __forceinline__ Tap2 make_tap2(float y, float x, int H, int W) {
  Tap2 t;
  if (y < -1.0f || y > (float)H || x < -1.0f || x > (float)W) {
    t.p1 = t.p2 = t.p3 = t.p4 = -1;
    t.w1 = t.w2 = t.w3 = t.w4 = 0.f;
    return t;
  }
  Tap1 ty = make_tap1(y, H), tx = make_tap1(x, W);
  t.p1 = ty.lo * W + tx.lo;
  t.p2 = ty.lo * W + tx.hi;
  t.p3 = ty.hi * W + tx.lo;
  t.p4 = ty.hi * W + tx.hi;
  t.w1 = ty.wl * tx.wl;
  t.w2 = ty.wl * tx.wh;
  t.w3 = ty.wh * tx.wl;
  t.w4 = ty.wh * tx.wh;
  return t;
}

__device__ __forceinline__ void rot_xy(const RoiGeom& g, int ph, int pw, int iy, int ix, float& y, float& x) {
  float yy = g.start_h + (float)ph * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh;
  float xx = g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw;
  y = yy * g.cos_t - xx * g.sin_t + g.ctr_h;  // ROIAlignRotated_cuda.cu:210-212
  x = yy * g.sin_t + xx * g.cos_t + g.ctr_w;
}

// The FPN level of the RoI is picked per CTA (single-level calls: num_levels == 1, level 0); a RoI without a level gets an
// empty sampling grid, i.e. a zero output.
template <int MAXTAP>
__global__ void __launch_bounds__(kThreads) roi_align_rot_fwd_kernel(const Pyr P, const float* __restrict__ rois,
                                                                     int C, int PH, int PW, int sr, int c_per_cta,
                                                                     float* __restrict__ out) {
  __shared__ Tap2 taps[MAXTAP];
  const int k = blockIdx.x;
  const int c0 = blockIdx.y * c_per_cta;
  const int cn = min(c_per_cta, C - c0);
  const int lvl_raw = pick_level<true>(P, rois + (size_t)k * 6);
  const int lvl = max(lvl_raw, 0);
  const float* __restrict__ in = P.feat[lvl];
  const int H = P.H[lvl], W = P.W[lvl];
  const RoiGeom g = load_geom<true>(rois + (size_t)k * 6, P.scale[lvl], PH, PW, sr, 1, lvl_raw < 0);
  const int bins = PH * PW;
  const int spb = g.gh * g.gw;  // samples per bin
  const long long ntap = (long long)bins * spb;
  const bool tab = ntap <= MAXTAP;
  if (tab) {
    for (int i = threadIdx.x; i < (int)ntap; i += kThreads) {
      int bin = i / spb, s = i - bin * spb;
      int ph = bin / PW, pw = bin - ph * PW, iy = s / g.gw, ix = s - iy * g.gw;
      float y, x;
      rot_xy(g, ph, pw, iy, ix, y, x);
      taps[i] = make_tap2(y, x, H, W);
    }
    __syncthreads();
  }
  const int total = cn * bins;
  const float* __restrict__ base = in + ((size_t)g.b * C + c0) * H * W;
  float* __restrict__ obase = out + ((size_t)k * C + c0) * bins;
  for (int idx = threadIdx.x; idx < total; idx += kThreads) {
    int c = idx / bins, bin = idx - c * bins;
    int ph = bin / PW, pw = bin - ph * PW;
    const float* __restrict__ plane = base + (size_t)c * H * W;
    float acc = 0.f;
    for (int s = 0; s < spb; ++s) {
      Tap2 t;
      if (tab) t = taps[bin * spb + s];
      else {
        int iy = s / g.gw, ix = s - iy * g.gw;
        float y, x;
        rot_xy(g, ph, pw, iy, ix, y, x);
        t = make_tap2(y, x, H, W);
      }
      if (t.p1 >= 0)
        acc += t.w1 * __ldg(plane + t.p1) + t.w2 * __ldg(plane + t.p2) + t.w3 * __ldg(plane + t.p3) +
               t.w4 * __ldg(plane + t.p4);
    }
    obase[idx] = acc * g.inv_count;
  }
}

// ------------------------------------------------------------------ rotated backward
// One CTA per (RoI, channel slab).  Threads map to (channel, bin); every sample scatters
// g*w/count to its four taps (ROIAlignRotated_cuda.cu:238-322).
// Lanes of a warp cover neighbouring bins of one channel, so their taps collide on the same pixels:
// red.global.add (no return value) lets the L2 atomic unit merge them.
__global__ void __launch_bounds__(kThreads) roi_align_rot_bwd_kernel(const Pyr P, const float* __restrict__ gout,
                                                                     const float* __restrict__ rois, int C, int PH, int PW,
                                                                     int sr, int c_per_cta) {
  const int k = blockIdx.x;
  const int c0 = blockIdx.y * c_per_cta;
  const int cn = min(c_per_cta, C - c0);
  const int lvl_raw = pick_level<true>(P, rois + (size_t)k * 6);  // rotated pyramids carry no level_rois
  const int lvl = max(lvl_raw, 0);
  float* __restrict__ gin = P.grad[lvl];
  const int H = P.H[lvl], W = P.W[lvl];
  const RoiGeom g = load_geom<true>(rois + (size_t)k * 6, P.scale[lvl], PH, PW, sr, 1, lvl_raw < 0);
  if (g.gh <= 0 || g.gw <= 0) return;
  const int bins = PH * PW;
  const int total = cn * bins;
  float* __restrict__ base = gin + ((size_t)g.b * C + c0) * H * W;
  const float* __restrict__ gbase = gout + ((size_t)k * C + c0) * bins;
  for (int idx = threadIdx.x; idx < total; idx += kThreads) {
    int c = idx / bins, bin = idx - c * bins;
    int ph = bin / PW, pw = bin - ph * PW;
    float* __restrict__ plane = base + (size_t)c * H * W;
    const float gv = gbase[idx];
    for (int iy = 0; iy < g.gh; ++iy)
      for (int ix = 0; ix < g.gw; ++ix) {
        float y, x;
        rot_xy(g, ph, pw, iy, ix, y, x);
        Tap2 t = make_tap2(y, x, H, W);
        if (t.p1 < 0) continue;
        atomicAdd(plane + t.p1, gv * t.w1 / g.count_raw);
        atomicAdd(plane + t.p2, gv * t.w2 / g.count_raw);
        atomicAdd(plane + t.p3, gv * t.w3 / g.count_raw);
        atomicAdd(plane + t.p4, gv * t.w4 / g.count_raw);
      }
  }
}

// ------------------------------------------------------------------ axis-aligned forward (staged, barrier-free)
// One CTA per (RoI, slab of channels); every WARP owns kChW channels at a time and runs on its own:
//   1. [once per CTA] the g_h x g_w bilinear samples of each bin collapse into short (row, weight) x (column, weight)
//      tap lists (the sample grid is a product grid): <= g+1 distinct rows / columns per bin instead of 4*g*g taps.
//      The lists live in shared memory, entry-major ([tap][bin row]) so that lanes of different bins read them
//      without bank conflicts, and are padded to a uniform length with zero-weight taps (no divergence);
//   2. a warp stages the RoI's pixel footprint of its kChW channel planes into its private slice of shared memory
//      with coalesced row reads (many independent loads in flight per lane), __syncwarp()s, then evaluates the bins
//      with lane == bin, reading taps from shared memory, and stores its outputs straight to global memory
//      (lanes = consecutive bins -> coalesced).  There is no CTA-wide barrier in the channel loop, so the 24 resident
//      warps per SM overlap each other's load latency freely.
// RoIs whose footprint exceeds a warp's slice are processed in bands of bin rows.  Very large or sparsely sampled RoIs
// (fixed sampling_ratio on a big box: far fewer taps than footprint pixels) skip the staging and read their taps
// straight from global memory through the same lists; only a tap-list overflow (sampling grid > 31) or a pooled size
// > 16 falls back to computing taps on the fly.
constexpr int kMaxE = 32;   // taps per bin row / column: covers sampling grids up to 31 (clipped, elongated RoIs)
constexpr int kMaxP = 16;   // pooled size supported by the staged path
constexpr int kChW = 4;     // channels per warp
constexpr int kV3Warps = 8;
constexpr int kV3Threads = kV3Warps * 32;
constexpr int kCapPx = 448;   // pixels per channel in a warp's slice:  8 warps * 4 ch * 448 px * 4 B = 56 KB per CTA
constexpr int kRowoffCap = 1536;  // largest whole-RoI footprint (pixels) with a precomputed offset table

struct CTap {
  int idx;
  float w;
};

__device__ __forceinline__ void add_tap(CTap* list, int stride, int& n, int idx, float w, int& overflow) {
  if (w == 0.f) return;
  for (int e = 0; e < n; ++e)
    if (list[e * stride].idx == idx) {
      list[e * stride].w += w;
      return;
    }
  if (n >= kMaxE) {
    overflow = 1;
    return;
  }
  list[n * stride].idx = idx;
  list[n * stride].w = w;
  ++n;
}

// BWD = false: out[k,c,bin] = pooled value.   BWD = true: the transpose -- gout[k,c,bin] is scattered with the same tap
// weights into the level's gradient map; a warp accumulates the footprint of its kChW channels in its shared-memory
// slice (shared-memory atomics between the bins of one RoI) and flushes every touched pixel with ONE red.global.add,
// instead of the reference's 4*g*g global atomics per output element (ROIAlignRotated_cuda.cu:311-318).
template <bool BWD>
__global__ void __launch_bounds__(kV3Threads, 3) roi_align_v3_kernel(const Pyr P, const float* __restrict__ rois, int C,
                                                                     int PH, int PW, int sr, int aligned,
                                                                     int groups_per_cta, const float* __restrict__ gout,
                                                                     float* __restrict__ out) {
  extern __shared__ __align__(16) float stage_all[];  // [warp][kCapPx][kChW]: the kChW channels of a pixel are one 16-byte word
  __shared__ CTap ytab[kMaxE * kMaxP];  // [tap][ph]
  __shared__ CTap xtab[kMaxE * kMaxP];  // [tap][pw]   (idx relative to the footprint's first column)
  __shared__ int rowoff[kRowoffCap];    // global offset (y*W + x) of every footprint pixel, row-major
  __shared__ int yn[kMaxP], xn[kMaxP], ylo[kMaxP], yhi[kMaxP];
  __shared__ int band_ph0[kMaxP + 1], band_yb[kMaxP], band_npx[kMaxP];
  __shared__ int s_overflow, s_tapov, s_xmin, s_xmax, s_nbands, s_direct, s_nyu, s_nxu, s_ymin, s_ymax;

  const int k = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int lvl_raw = pick_level(P, (P.level_rois ? P.level_rois : rois) + (size_t)k * 5);
  const int lvl = max(lvl_raw, 0);
  const float* __restrict__ in = BWD ? nullptr : P.feat[lvl];
  float* __restrict__ gin = BWD ? P.grad[lvl] : nullptr;
  const int H = P.H[lvl], W = P.W[lvl];
  const RoiGeom g = load_geom<false>(rois + (size_t)k * 5, P.scale[lvl], PH, PW, sr, aligned, lvl_raw < 0);
  const int bins = PH * PW;
  const int ngroup = d2b_cdiv(C, kChW);
  const int g_begin = blockIdx.y * groups_per_cta, g_end = min(ngroup, g_begin + groups_per_cta);

  if (tid == 0) {
    s_overflow = (PH > kMaxP || PW > kMaxP) ? 1 : 0;  // written here only; tap-list overflow goes to s_tapov (atomic)
    s_tapov = 0;
    s_xmin = 1 << 30;
    s_xmax = -1;
  }
  __syncthreads();
  if (!s_overflow) {
    if (tid < PH) {
      CTap* list = ytab + tid;
      int n = 0, ov = 0, lo = 1 << 30, hi = -1;
      for (int iy = 0; iy < g.gh; ++iy) {
        Tap1 t = make_tap1(g.start_h + (float)tid * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
        add_tap(list, kMaxP, n, t.lo, t.wl, ov);
        add_tap(list, kMaxP, n, t.hi, t.wh, ov);
      }
      for (int e = 0; e < n; ++e) {
        lo = min(lo, list[e * kMaxP].idx);
        hi = max(hi, list[e * kMaxP].idx);
      }
      yn[tid] = n;
      ylo[tid] = lo;
      yhi[tid] = hi;
      if (ov) atomicOr(&s_tapov, 1);
    } else if (tid >= 32 && tid < 32 + PW) {
      const int pw = tid - 32;
      CTap* list = xtab + pw;
      int n = 0, ov = 0;
      for (int ix = 0; ix < g.gw; ++ix) {
        Tap1 t = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
        add_tap(list, kMaxP, n, t.lo, t.wl, ov);
        add_tap(list, kMaxP, n, t.hi, t.wh, ov);
      }
      for (int e = 0; e < n; ++e) {
        atomicMin(&s_xmin, list[e * kMaxP].idx);
        atomicMax(&s_xmax, list[e * kMaxP].idx);
      }
      xn[pw] = n;
      if (ov) atomicOr(&s_tapov, 1);
    }
  }
  __syncthreads();
  const int xmin = s_xmin, fw = s_xmax - s_xmin + 1;
  if (tid == 0) {  // uniform list lengths, band schedule
    const int overflow = s_overflow | s_tapov;
    int direct = overflow, nb = 0, nyu = 0, nxu = 0, ymin = 1 << 30, ymax = -1;
    if (!direct) {
      for (int ph = 0; ph < PH; ++ph) {
        nyu = max(nyu, yn[ph]);
        if (yn[ph] > 0) {
          ymin = min(ymin, ylo[ph]);
          ymax = max(ymax, yhi[ph]);
        }
      }
      for (int pw = 0; pw < PW; ++pw) nxu = max(nxu, xn[pw]);
    }
    if (!direct && fw > 0 && ymax >= ymin) {
      if ((long long)(ymax - ymin + 1) * fw > kRowoffCap) direct = 1;
      int ph0 = 0;
      while (ph0 < PH && !direct) {
        int yb = 1 << 30, ye = -1, ph1 = ph0;
        while (ph1 < PH) {
          int nyb = yb, nye = ye;
          if (yn[ph1] > 0) {
            nyb = min(yb, ylo[ph1]);
            nye = max(ye, yhi[ph1]);
          }
          if (nye >= nyb && (nye - nyb + 1) * fw > kCapPx) {
            if (ph1 == ph0) direct = 1;  // a single bin row does not fit
            break;
          }
          yb = nyb;
          ye = nye;
          ++ph1;
        }
        band_ph0[nb] = ph0;
        band_yb[nb] = (ye >= yb) ? yb : ymin;
        band_npx[nb] = (ye >= yb) ? (ye - yb + 1) * fw : 0;
        ++nb;
        ph0 = ph1;
      }
    } else if (!direct) {  // no valid sample at all: every output is 0
      band_ph0[0] = 0;
      band_yb[0] = 0;
      band_npx[0] = 0;
      nb = 1;
      nyu = nxu = 0;
      ymin = 0;
      ymax = -1;
    }
    band_ph0[nb] = PH;
    s_nbands = nb;
    // mode 0: staged footprint; 1: tap lists + loads straight from global (footprint too large for a warp's slice, or
    // sparsely sampled: fewer distinct taps than half the footprint pixels); 2: tap lists overflowed -> taps on the fly
    int mode = overflow ? 2 : (direct ? 1 : 0);
    if (mode == 0 && fw > 0 && ymax >= ymin) {
      int sy = 0, sx = 0;
      for (int ph = 0; ph < PH; ++ph) sy += yn[ph];
      for (int pw = 0; pw < PW; ++pw) sx += xn[pw];
      if (2LL * sy * sx < (long long)(ymax - ymin + 1) * fw) mode = 1;
    }
    direct = mode;
    s_direct = direct;
    s_nyu = nyu;
    s_nxu = nxu;
    s_ymin = ymin;
    s_ymax = ymax;
  }
  __syncthreads();
  const int mode = s_direct;
  const bool direct = mode == 2;
  const int nbands = s_nbands, nyu = s_nyu, nxu = s_nxu, ymin = s_ymin;
  if (mode != 2) {
    // pad the lists to the uniform lengths with zero-weight taps on a valid row / column; make columns relative
    if (tid < PH) {
      const int n = yn[tid];
      const int fill = n > 0 ? ytab[tid].idx : 0;  // rows are clamped into the band at use
      for (int e = n; e < nyu; ++e) ytab[e * kMaxP + tid] = CTap{fill, 0.f};
    } else if (tid >= 32 && tid < 32 + PW) {
      const int pw = tid - 32, n = xn[pw];
      for (int e = 0; e < n; ++e) xtab[e * kMaxP + pw].idx -= xmin;
      for (int e = n; e < ((nxu + 3) & ~3); ++e) xtab[e * kMaxP + pw] = CTap{0, 0.f};  // gather path reads 4 at a time
    }
    if (mode == 0 && fw > 0 && s_ymax >= ymin) {
      const int npx_all = (s_ymax - ymin + 1) * fw;  // <= kRowoffCap by construction
      for (int i = tid; i < npx_all; i += kV3Threads) {
        const int y = i / fw, x = i - y * fw;
        rowoff[i] = (ymin + y) * W + xmin + x;
      }
    }
  }
  __syncthreads();

  float* __restrict__ st = stage_all + (size_t)warp * kChW * kCapPx;
  for (int grp = g_begin + warp; grp < g_end; grp += kV3Warps) {
    const int c0 = grp * kChW;
    const int cn = min(kChW, C - c0);
    const float* __restrict__ base = BWD ? nullptr : in + ((size_t)g.b * C + c0) * H * W;
    float* __restrict__ gbase = BWD ? gin + ((size_t)g.b * C + c0) * H * W : nullptr;
    float* __restrict__ obase = BWD ? nullptr : out + ((size_t)k * C + c0) * bins;
    const float* __restrict__ gobase = BWD ? gout + ((size_t)k * C + c0) * bins : nullptr;
    if (direct && BWD) {  // rare: taps on the fly, global atomics per sample
      for (int idx = lane; idx < cn * bins; idx += 32) {
        const int c = idx / bins, bin = idx - c * bins;
        const int ph = bin / PW, pw = bin - ph * PW;
        float* __restrict__ plane = gbase + (size_t)c * H * W;
        const float gv = gobase[idx] * g.inv_count;
        for (int iy = 0; iy < g.gh; ++iy) {
          Tap1 ty = make_tap1(g.start_h + (float)ph * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
          for (int ix = 0; ix < g.gw; ++ix) {
            Tap1 tx = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
            atomicAdd(plane + ty.lo * W + tx.lo, gv * ty.wl * tx.wl);
            atomicAdd(plane + ty.lo * W + tx.hi, gv * ty.wl * tx.wh);
            atomicAdd(plane + ty.hi * W + tx.lo, gv * ty.wh * tx.wl);
            atomicAdd(plane + ty.hi * W + tx.hi, gv * ty.wh * tx.wh);
          }
        }
      }
      continue;
    }
    if (direct) {  // rare: taps on the fly, straight from global memory (one warp: its kChW channels)
      for (int idx = lane; idx < cn * bins; idx += 32) {
        const int c = idx / bins, bin = idx - c * bins;
        const int ph = bin / PW, pw = bin - ph * PW;
        const float* __restrict__ plane = base + (size_t)c * H * W;
        float acc = 0.f;
        for (int iy = 0; iy < g.gh; ++iy) {
          Tap1 ty = make_tap1(g.start_h + (float)ph * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
          const float* __restrict__ r0 = plane + (size_t)ty.lo * W;
          const float* __restrict__ r1 = plane + (size_t)ty.hi * W;
          for (int ix = 0; ix < g.gw; ++ix) {
            Tap1 tx = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
            acc += (ty.wl * tx.wl) * __ldg(r0 + tx.lo) + (ty.wl * tx.wh) * __ldg(r0 + tx.hi) +
                   (ty.wh * tx.wl) * __ldg(r1 + tx.lo) + (ty.wh * tx.wh) * __ldg(r1 + tx.hi);
          }
        }
        obase[idx] = acc * g.inv_count;
      }
      continue;
    }
    // channel planes of this warp (a ragged last group re-reads its last valid plane into unused slices)
    const float* __restrict__ pl[kChW];
    float* __restrict__ gpl[kChW];
#pragma unroll
    for (int q = 0; q < kChW; ++q) {
      pl[q] = BWD ? nullptr : base + (size_t)min(q, cn - 1) * H * W;
      gpl[q] = BWD ? gbase + (size_t)min(q, cn - 1) * H * W : nullptr;
    }

    if (BWD && mode == 1) {  // tap lists, one global atomic per (tap, channel)
      for (int b0 = 0; b0 < bins; b0 += 32) {
        const int bin = b0 + lane;
        if (bin >= bins) continue;
        const int ph = bin / PW, pw = bin - (bin / PW) * PW;
        float gv[kChW];
#pragma unroll
        for (int q = 0; q < kChW; ++q) gv[q] = q < cn ? gobase[q * bins + bin] * g.inv_count : 0.f;
        for (int ey = 0; ey < nyu; ++ey) {
          const CTap ty = ytab[ey * kMaxP + ph];
          if (ty.w == 0.f) continue;
          const int rbase = ty.idx * W + xmin;
          for (int ex = 0; ex < nxu; ++ex) {
            const CTap tx = xtab[ex * kMaxP + pw];
            const float wgt = ty.w * tx.w;
            if (wgt == 0.f) continue;
#pragma unroll
            for (int q = 0; q < kChW; ++q)
              if (q < cn) atomicAdd(gpl[q] + rbase + tx.idx, wgt * gv[q]);
          }
        }
      }
      continue;
    }
    if (BWD) {  // staged: accumulate the footprint in the warp's slice, flush each touched pixel once
      for (int band = 0; band < nbands; ++band) {
        const int ph0 = band_ph0[band], ph1 = band_ph0[band + 1];
        const int yb = band_yb[band], npx = band_npx[band];
        const int ylast = yb + (fw > 0 ? npx / fw : 0) - 1;
        const int* __restrict__ ro = rowoff + (yb - ymin) * fw;
        __syncwarp();
        for (int i = lane; i < npx; i += 32) {
#pragma unroll
          for (int q = 0; q < kChW; ++q) st[i * kChW + q] = 0.f;
        }
        __syncwarp();
        const int nbin = (ph1 - ph0) * PW;
        for (int b0 = 0; b0 < nbin; b0 += 32) {
          const int bin = b0 + lane;
          if (bin >= nbin) continue;
          const int dph = bin / PW;
          const int ph = ph0 + dph, pw = bin - dph * PW;
          float gv[kChW];
#pragma unroll
          for (int q = 0; q < kChW; ++q) gv[q] = q < cn ? gobase[q * bins + ph * PW + pw] * g.inv_count : 0.f;
          for (int ey = 0; ey < nyu; ++ey) {
            const CTap ty = ytab[ey * kMaxP + ph];
            if (ty.w == 0.f) continue;
            float* __restrict__ srow = st + (min(max(ty.idx, yb), ylast) - yb) * fw * kChW;
            for (int ex = 0; ex < nxu; ++ex) {
              const CTap tx = xtab[ex * kMaxP + pw];
              const float wgt = ty.w * tx.w;
              if (wgt == 0.f) continue;
#pragma unroll
              for (int q = 0; q < kChW; ++q) atomicAdd(srow + tx.idx * kChW + q, wgt * gv[q]);
            }
          }
        }
        __syncwarp();
        for (int i = lane; i < npx; i += 32) {
          const int off = ro[i];
#pragma unroll
          for (int q = 0; q < kChW; ++q) {
            const float v = st[i * kChW + q];
            if (q < cn && v != 0.f) atomicAdd(gpl[q] + off, v);
          }
        }
      }
      continue;
    }

    if (mode == 1) {  // tap lists, data straight from global / L2 (large or sparsely sampled RoIs)
      for (int b0 = 0; b0 < bins; b0 += 32) {
        const int bin = b0 + lane;
        const bool live = bin < bins;
        const int bb = live ? bin : 0;
        const int ph = bb / PW, pw = bb - (bb / PW) * PW;
        float acc[kChW];
#pragma unroll
        for (int q = 0; q < kChW; ++q) acc[q] = 0.f;
        for (int ey = 0; ey < nyu; ++ey) {
          const CTap ty = ytab[ey * kMaxP + ph];
          const int rbase = ty.idx * W + xmin;
          float r[kChW];
#pragma unroll
          for (int q = 0; q < kChW; ++q) r[q] = 0.f;
          for (int ex = 0; ex < nxu; ex += 4) {  // 4 taps x kChW channels = 16 independent loads in flight (lists padded)
            CTap tx[4];
            float v[4][kChW];
#pragma unroll
            for (int e = 0; e < 4; ++e) tx[e] = xtab[(ex + e) * kMaxP + pw];
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
              for (int q = 0; q < kChW; ++q) v[e][q] = __ldg(pl[q] + rbase + tx[e].idx);
#pragma unroll
            for (int e = 0; e < 4; ++e)
#pragma unroll
              for (int q = 0; q < kChW; ++q) r[q] = fmaf(tx[e].w, v[e][q], r[q]);
          }
#pragma unroll
          for (int q = 0; q < kChW; ++q) acc[q] = fmaf(ty.w, r[q], acc[q]);
        }
        if (live) {
#pragma unroll
          for (int q = 0; q < kChW; ++q)
            if (q < cn) obase[q * bins + bin] = acc[q] * g.inv_count;
        }
      }
      continue;
    }

    for (int band = 0; band < nbands; ++band) {
      const int ph0 = band_ph0[band], ph1 = band_ph0[band + 1];
      const int yb = band_yb[band], npx = band_npx[band];
      const int ylast = yb + (fw > 0 ? npx / fw : 0) - 1;
      const int* __restrict__ ro = rowoff + (yb - ymin) * fw;
      __syncwarp();  // the previous band's / group's reads of `st` are complete
      // ---- stage: 2 pixel strides x kChW channels = 8 independent loads in flight per lane
      for (int pix = lane; pix < npx; pix += 64) {
        const bool two = pix + 32 < npx;
        const int o0 = ro[pix], o1 = two ? ro[pix + 32] : o0;
        float a[kChW], b[kChW];
#pragma unroll
        for (int q = 0; q < kChW; ++q) {
          a[q] = __ldg(pl[q] + o0);
          b[q] = __ldg(pl[q] + o1);
        }
        static_assert(kChW == 4, "one float4 per pixel");
        *reinterpret_cast<float4*>(st + pix * kChW) = make_float4(a[0], a[1], a[2], a[3]);
        if (two) *reinterpret_cast<float4*>(st + (pix + 32) * kChW) = make_float4(b[0], b[1], b[2], b[3]);
      }
      __syncwarp();
      // ---- compute: lane == bin
      const int nbin = (ph1 - ph0) * PW;
      for (int b0 = 0; b0 < nbin; b0 += 32) {
        const int bin = b0 + lane;
        const bool live = bin < nbin;
        const int bb = live ? bin : 0;
        const int dph = bb / PW;
        const int ph = ph0 + dph, pw = bb - dph * PW;
        float acc[kChW];
#pragma unroll
        for (int q = 0; q < kChW; ++q) acc[q] = 0.f;
        for (int ey = 0; ey < nyu; ++ey) {
          const CTap ty = ytab[ey * kMaxP + ph];
          const float* __restrict__ srow = st + (min(max(ty.idx, yb), ylast) - yb) * fw * kChW;  // pad taps (w = 0) stay in-band
          float r[kChW];
#pragma unroll
          for (int q = 0; q < kChW; ++q) r[q] = 0.f;
          for (int ex = 0; ex < nxu; ++ex) {
            const CTap tx = xtab[ex * kMaxP + pw];
            const float4 dv = *reinterpret_cast<const float4*>(srow + tx.idx * kChW);  // 4 channels of the tap pixel
            r[0] = fmaf(tx.w, dv.x, r[0]);
            r[1] = fmaf(tx.w, dv.y, r[1]);
            r[2] = fmaf(tx.w, dv.z, r[2]);
            r[3] = fmaf(tx.w, dv.w, r[3]);
          }
#pragma unroll
          for (int q = 0; q < kChW; ++q) acc[q] = fmaf(ty.w, r[q], acc[q]);
        }
        if (live) {
#pragma unroll
          for (int q = 0; q < kChW; ++q)
            if (q < cn) obase[q * bins + ph * PW + pw] = acc[q] * g.inv_count;
        }
      }
    }
  }
}

static int launch_fwd(const Pyr& P, const float* rois, int K, int C, int PH, int PW, int sr, int aligned, float* out,
                      cudaStream_t stream, const float* gout = nullptr) {
  const size_t smem = sizeof(float) * (size_t)kV3Warps * kChW * kCapPx;
  if (gout) D2B_ALLOW_BIG_SMEM(roi_align_v3_kernel<true>);
  else D2B_ALLOW_BIG_SMEM(roi_align_v3_kernel<false>);
  const int ngroup = d2b_cdiv(C, kChW);
  int groups_per_cta = ngroup;  // split the channel groups until the grid is several waves deep
  while (groups_per_cta > kV3Warps && (long long)K * d2b_cdiv(ngroup, groups_per_cta) < 24LL * d2b_num_sms())
    groups_per_cta = (groups_per_cta + 1) / 2;
  dim3 grid(K, d2b_cdiv(ngroup, groups_per_cta));
  if (gout) roi_align_v3_kernel<true><<<grid, kV3Threads, smem, stream>>>(P, rois, C, PH, PW, sr, aligned, groups_per_cta, gout, nullptr);
  else roi_align_v3_kernel<false><<<grid, kV3Threads, smem, stream>>>(P, rois, C, PH, PW, sr, aligned, groups_per_cta, nullptr, out);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// channels per CTA: enough CTAs to fill the SMs a few times over without shrinking the per-CTA tap reuse.
int pick_c_per_cta(int K, int C) {
  int cpc = C;
  while (cpc > 16 && (long long)K * d2b_cdiv(C, cpc) < 4LL * d2b_num_sms()) cpc = (cpc + 1) / 2;
  return cpc;
}

// ------------------------------------------------------------------ channels-last (NHWC) forward
// With the channels innermost the roles flip: lane == 4 channels (one 16-byte word), so a warp reads the 128
// channels of a tap pixel as one coalesced 512-byte LDG.128 and the tap index / weight are warp-uniform (no per-lane
// address arithmetic, no shared-memory staging of the footprint: L1 is the staging buffer, the 7 or 8 warps of a CTA
// walk neighbouring bins of the same RoI at the same time).  One warp owns one bin at a time; the [bin] x [channel]
// results are transposed through shared memory so that the NCHW-shaped output is written in contiguous runs.
constexpr int kNhwcCh = 128;    // channels per CTA
constexpr int kNhwcChunk = 64;  // bins per output chunk (shared-memory transpose tile: 128 ch x chunk)
constexpr int kNhwcThreads = 224;  // 7 warps: the 49 bins of a 7x7 output (and 7-multiples of a 14x14 chunk) split evenly

// Pairs of fp32 lanes: d.xy = w * v.xy + c.xy (two fused multiply-adds, each rounded once)
struct F2 {
  float x, y;
};
__device__ __forceinline__ F2 f2_pack(float a, float b) { return F2{a, b}; }
__device__ __forceinline__ void f2_unpack(F2 p, float& a, float& b) {
  a = p.x;
  b = p.y;
}
__device__ __forceinline__ F2 f2_fma(F2 w, F2 v, F2 c) { return F2{__fmaf_rn(w.x, v.x, c.x), __fmaf_rn(w.y, v.y, c.y)}; }

// One bin: XC x-taps (byte offsets / weights held in registers) times RY rows per step = XC * RY independent 512-byte loads in
// flight per warp.  Table entries hold BYTE offsets premultiplied for the NHWC layout (row: y*W*C*4, column: x*C*4) and the
// lists are padded to multiples of XC / RY with zero-weight taps on a valid pixel, so the loop carries no predicates: per tap
// one address add, one LDG.128 and two packed FMAs (+ two per row for the y weight).
template <int XC, int RY>
__device__ __forceinline__ void nhwc_bin(const char* __restrict__ base, const CTap* __restrict__ yt0,
                                         const CTap* __restrict__ xt0, int ny, int nx, float4& acc) {
  F2 a01 = f2_pack(acc.x, acc.y), a23 = f2_pack(acc.z, acc.w);
  for (int x0 = 0; x0 < nx; x0 += XC) {
    unsigned xo[XC];
    F2 xw[XC];
#pragma unroll
    for (int e = 0; e < XC; ++e) {
      const CTap t = xt0[(x0 + e) * kMaxP];
      xo[e] = (unsigned)t.idx;
      xw[e] = f2_pack(t.w, t.w);
    }
    for (int ey = 0; ey < ny; ey += RY) {
      const char* __restrict__ rowp[RY];
      F2 wy[RY];
#pragma unroll
      for (int j = 0; j < RY; ++j) {
        const CTap t = yt0[(ey + j) * kMaxP];
        rowp[j] = base + (size_t)(unsigned)t.idx;
        wy[j] = f2_pack(t.w, t.w);
      }
      float4 v[RY][XC];
#pragma unroll
      for (int j = 0; j < RY; ++j)
#pragma unroll
        for (int e = 0; e < XC; ++e) v[j][e] = __ldg(reinterpret_cast<const float4*>(rowp[j] + xo[e]));
#pragma unroll
      for (int j = 0; j < RY; ++j) {
        F2 r01 = f2_pack(0.f, 0.f), r23 = r01;
#pragma unroll
        for (int e = 0; e < XC; ++e) {
          r01 = f2_fma(xw[e], f2_pack(v[j][e].x, v[j][e].y), r01);
          r23 = f2_fma(xw[e], f2_pack(v[j][e].z, v[j][e].w), r23);
        }
        a01 = f2_fma(wy[j], r01, a01);
        a23 = f2_fma(wy[j], r23, a23);
      }
    }
  }
  f2_unpack(a01, acc.x, acc.y);
  f2_unpack(a23, acc.z, acc.w);
}

// Column-shared form of the bin loop (the fast path).  A warp owns a UNIT = 7 consecutive bins of one bin row and walks the
// footprint columns of those bins ONCE, left to right: a column is "owned" by the first bin that touches it and feeds that
// bin (weight wa) and, when the next bin's sample window reaches it too, the next bin (weight wb); two rotating accumulators
// (current bin, next bin) are enough because no column may touch three bins (checked when the table is built; such RoIs --
// bins narrower than a pixel -- take the per-bin loop above).  Per owned column the warp loads the RY tap rows of its bin row
// (RY * XC independent 512-byte requests in flight), collapses them with the row weights and adds the result to the two
// accumulators: RY loads per column instead of RY per (bin, column) pair -- the per-bin loop re-reads the columns that
// neighbouring bins share and pads every bin's lists to whole chunks, 930 k against 453 k requests for the 1 024 RoIs of the
// bench.  Entries: {byte offset of the column, wa, wb, last-column-of-its-bin flag}; every bin has at least one entry.
constexpr int kColCap = 192;  // column entries per RoI (footprint width + pooled width + chunk padding)

__device__ __forceinline__ void nhwc_emit(float* __restrict__ o, int chunk_pad, F2 c01, F2 c23, float inv, bool first) {
  float a, b, c, d;
  f2_unpack(c01, a, b);
  f2_unpack(c23, c, d);
  // later row chunks of a tall bin row accumulate (the cells of a unit belong to one warp); predicated reads, one code path
  o[0] = fmaf(a, inv, first ? 0.f : o[0]);
  o[32 * chunk_pad] = fmaf(b, inv, first ? 0.f : o[32 * chunk_pad]);
  o[64 * chunk_pad] = fmaf(c, inv, first ? 0.f : o[64 * chunk_pad]);
  o[96 * chunk_pad] = fmaf(d, inv, first ? 0.f : o[96 * chunk_pad]);
}

template <int RY, int XC>
__device__ __forceinline__ void nhwc_unit(const char* __restrict__ base, const CTap* __restrict__ yt0, int ny, int nch,
                                          const float4* __restrict__ colE, int cb, int ce, int skip, float* __restrict__ o,
                                          int chunk_pad, float inv) {
  for (int ch = 0; ch < nch; ++ch) {
    unsigned ro[RY];
    float wy[RY];
#pragma unroll
    for (int j = 0; j < RY; ++j) {
      const int e = ch * RY + j;
      const CTap t = yt0[(e < ny ? e : 0) * kMaxP];
      ro[j] = (unsigned)t.idx;
      wy[j] = e < ny ? t.w : 0.f;
    }
    const F2 z = f2_pack(0.f, 0.f);
    F2 c01 = z, c23 = z, n01 = z, n23 = z;
    int b = -skip;  // bin of the unit the current accumulator belongs to (-1: the carry-in bin left of the unit)
    for (int s = cb; s < ce; s += XC) {
      float4 en[XC];
      float4 v[XC][RY];
#pragma unroll
      for (int x = 0; x < XC; ++x) {
        en[x] = colE[s + x];  // entries past ce exist (next bins or table padding): valid offsets, weights masked below
        const char* __restrict__ cp = base + (size_t)(unsigned)__float_as_int(en[x].x);
#pragma unroll
        for (int j = 0; j < RY; ++j) v[x][j] = __ldg(reinterpret_cast<const float4*>(cp + ro[j]));
      }
#pragma unroll
      for (int x = 0; x < XC; ++x) {
        const bool live = XC == 1 || s + x < ce;  // warp-uniform
        F2 t01 = z, t23 = z;
#pragma unroll
        for (int j = 0; j < RY; ++j) {
          const F2 w = f2_pack(wy[j], wy[j]);
          t01 = f2_fma(w, f2_pack(v[x][j].x, v[x][j].y), t01);
          t23 = f2_fma(w, f2_pack(v[x][j].z, v[x][j].w), t23);
        }
        const float wa = live ? en[x].y : 0.f, wb = live ? en[x].z : 0.f;
        const F2 a2 = f2_pack(wa, wa), b2 = f2_pack(wb, wb);
        c01 = f2_fma(a2, t01, c01);
        c23 = f2_fma(a2, t23, c23);
        n01 = f2_fma(b2, t01, n01);
        n23 = f2_fma(b2, t23, n23);
        if (live && __float_as_int(en[x].w) != 0) {  // last owned column of its bin: the bin is complete
          if (b >= 0) nhwc_emit(o + b, chunk_pad, c01, c23, inv, ch == 0);
          c01 = n01;
          c23 = n23;
          n01 = z;
          n23 = z;
          ++b;
        }
      }
    }
  }
}

// 4 CTAs x 7 warps per SM at 72 registers: measured faster than 3 CTAs at 80 (95 vs 97 us on the box-head call)
template <int ODT>
__global__ void __launch_bounds__(kNhwcThreads, 4) roi_align_nhwc_kernel(const Pyr P, const float* __restrict__ rois, int C, int PH,
                                                             int PW, int sr, int aligned, int chunk, int chunk_pad,
                                                             void* __restrict__ out_v) {
  extern __shared__ __align__(16) float otile[];  // [4 (channel of the quad)][32 (lane)][chunk_pad]
  __shared__ CTap ytab[kMaxE * kMaxP];            // [tap][ph]
  __shared__ CTap xtab[kMaxE * kMaxP];            // [tap][pw]
  __shared__ int yn[kMaxP], xn[kMaxP];
  __shared__ int ynr[kMaxP], xnr[kMaxP];   // list lengths before padding (the column-shared path uses the lists as built)
  __shared__ float4 colE[kColCap];         // owned-column entries, bin after bin
  __shared__ int cbeg[kMaxP + 1];          // first entry of every bin
  __shared__ int s_overflow, s_tapov, s_colok, s_nymax;
  __shared__ RoiGeom sg;  // read from shared memory where needed: keeps the tap loop's register budget small

  const int k = blockIdx.x;
  const int c0 = blockIdx.y * kNhwcCh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int lvl_raw = pick_level(P, (P.level_rois ? P.level_rois : rois) + (size_t)k * 5);
  const int lvl = max(lvl_raw, 0);
  const int H = P.H[lvl], W = P.W[lvl];
  const int bins = PH * PW;
  const int C4 = C >> 2;
  const int ncta = min(kNhwcCh, C - c0);  // channels of this CTA
  const bool lane_live = lane * 4 < ncta;
  // a dead lane (ragged last slab) re-reads the slab's first quad and is never stored
  if (tid == 0) {
    s_overflow = (PH > kMaxP || PW > kMaxP) ? 1 : 0;  // written here only; tap-list overflow goes to s_tapov (atomic)
    s_tapov = 0;
    s_colok = 0;
    s_nymax = 0;
    sg = load_geom<false>(rois + (size_t)k * 5, P.scale[lvl], PH, PW, sr, aligned, lvl_raw < 0);
  }
  __syncthreads();
  const float4* __restrict__ base =
      reinterpret_cast<const float4*>(P.feat[lvl]) + (size_t)sg.b * H * W * C4 + (c0 >> 2) + (lane_live ? lane : 0);
  const char* __restrict__ base_b = reinterpret_cast<const char*>(base);
  if (!s_overflow) {
    if (tid < PH) {
      const RoiGeom g = sg;
      CTap* list = ytab + tid;
      int n = 0, ov = 0;
      for (int iy = 0; iy < g.gh; ++iy) {
        Tap1 t = make_tap1(g.start_h + (float)tid * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
        add_tap(list, kMaxP, n, t.lo, t.wl, ov);
        add_tap(list, kMaxP, n, t.hi, t.wh, ov);
      }
      for (int e = 0; e < n; ++e) list[e * kMaxP].idx *= W * C4 * 16;  // row offset in bytes
      ynr[tid] = n;
      atomicMax(&s_nymax, n);
      if (n > 0)  // pad to a whole number of row pairs: zero-weight taps on a valid row
        for (; n & 1; ++n) list[n * kMaxP] = CTap{list[0].idx, 0.f};
      yn[tid] = n;
      if (ov) atomicOr(&s_tapov, 1);
    } else if (warp == 1) {  // the whole warp: lanes >= PW only take part in the shuffles
      const int pw = lane;
      const bool act = pw < PW;
      const RoiGeom g = sg;
      CTap* list = xtab + pw;
      int n = 0, ov = 0;
      if (act) {
        for (int ix = 0; ix < g.gw; ++ix) {
          Tap1 t = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
          add_tap(list, kMaxP, n, t.lo, t.wl, ov);
          add_tap(list, kMaxP, n, t.hi, t.wh, ov);
        }
        for (int e = 0; e < n; ++e) list[e * kMaxP].idx *= C4 * 16;  // column offset in bytes
        xnr[pw] = n;
        if (ov) atomicOr(&s_tapov, 1);
      }
      __syncwarp();
      // ---- owned-column entries of the column-shared path (nhwc_unit): a column belongs to the first bin that touches it
      const int n1 = act && pw >= 1 ? xnr[pw - 1] : 0, n2 = act && pw >= 2 ? xnr[pw - 2] : 0;
      const int n3 = act && pw + 1 < PW ? xnr[pw + 1] : 0;
      int own = 0, bad = ov;
      unsigned ownmask = 0;  // lists hold <= kMaxE = 32 entries
      for (int e = 0; e < n; ++e) {
        const int c = list[e * kMaxP].idx;
        bool in1 = false, in2 = false;
        for (int q = 0; q < n1; ++q) in1 |= xtab[q * kMaxP + pw - 1].idx == c;
        for (int q = 0; q < n2; ++q) in2 |= xtab[q * kMaxP + pw - 2].idx == c;
        if (in1 && in2) bad = 1;  // three bins on one column: bins narrower than a pixel
        if (!in1) {
          ++own;
          ownmask |= 1u << e;
        }
      }
      const int cnt = act ? max(own, 1) : 0;  // a bin without an owned column still gets one (zero-weight) entry
      int incl = cnt;
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, incl, d);
        if (lane >= d) incl += t;
      }
      const int beg = incl - cnt;
      const int total = __shfl_sync(0xffffffffu, incl, 31);
      if (total + 4 > kColCap) bad = 1;
      // worth it only when neighbouring bins really share columns / the per-bin lists carry padding: the column walk keeps
      // fewer loads in flight than the per-bin loop (measured: fixed sampling_ratio on large boxes is faster per bin)
      int padded = act ? (n == 0 ? 0 : (n <= 4 ? 4 : (n + 7) & ~7)) : 0;
#pragma unroll
      for (int d = 16; d; d >>= 1) padded += __shfl_xor_sync(0xffffffffu, padded, d);
      if (total * 5 > padded * 4) bad = 1;
      bad = __any_sync(0xffffffffu, bad);
      if (!bad) {
        if (act) {
          cbeg[pw] = beg;
          int i = beg;
          for (int e = 0; e < n; ++e)
            if (ownmask >> e & 1u) {
              const CTap t = list[e * kMaxP];
              float wb = 0.f;
              for (int q = 0; q < n3; ++q)
                if (xtab[q * kMaxP + pw + 1].idx == t.idx) wb = xtab[q * kMaxP + pw + 1].w;
              ++i;
              colE[i - 1] = make_float4(__int_as_float(t.idx), t.w, wb, __int_as_float(i == beg + own ? 1 : 0));
            }
          if (own == 0) colE[beg] = make_float4(__int_as_float(0), 0.f, 0.f, __int_as_float(1));
        }
        if (lane < 4) colE[total + lane] = make_float4(__int_as_float(0), 0.f, 0.f, __int_as_float(0));
        if (lane == 0) {
          cbeg[PW] = total;
          s_colok = 1;
        }
      }
      __syncwarp();
      if (act) {
        if (n > 0)  // pad to a multiple of the x-tap chunk (4, or 8 for long lists): zero-weight taps on a valid column
          for (const int m = n <= 4 ? 3 : 7; n & m; ++n) list[n * kMaxP] = CTap{list[0].idx, 0.f};
        xn[pw] = n;
      }
    }
  }
  __syncthreads();
  const bool onfly = (s_overflow | s_tapov) != 0;

  {
    const int bin0 = blockIdx.z * chunk;  // one output chunk per CTA
    const int nb = min(chunk, bins - bin0);
    // column-shared path: pooled widths that split into units of 7 bins (7x7 box head, 14x14 mask head), chunks of whole units
    const bool shared_cols = !onfly && s_colok && s_nymax <= 6 && PW % 7 == 0 && chunk % 7 == 0;
    if (shared_cols) {
      const float inv_count = sg.inv_count;
      for (int u = warp; u * 7 < nb; u += nwarps) {
        const int fb = bin0 + u * 7;
        const int ph = fb / PW, pw0 = fb - ph * PW;
        const int ny = ynr[ph];
        float* __restrict__ o = otile + lane * chunk_pad + u * 7;
        if (ny == 0) {  // bin row outside the map
#pragma unroll
          for (int b = 0; b < 7; ++b) o[b] = o[b + 32 * chunk_pad] = o[b + 64 * chunk_pad] = o[b + 96 * chunk_pad] = 0.f;
          continue;
        }
        const int skip = pw0 > 0 ? 1 : 0;  // columns owned by the bin left of the unit may reach into its first bin
        const int cb = cbeg[pw0 - skip], ce = cbeg[pw0 + 7];
        const int nch = (ny + 5) / 6, ry = (ny + nch - 1) / nch;  // tap rows in chunks of <= 6
        const CTap* __restrict__ yt0 = ytab + ph;
        switch (ry) {
          case 1: nhwc_unit<1, 4>(base_b, yt0, ny, nch, colE, cb, ce, skip, o, chunk_pad, inv_count); break;
          case 2: nhwc_unit<2, 3>(base_b, yt0, ny, nch, colE, cb, ce, skip, o, chunk_pad, inv_count); break;
          case 3: nhwc_unit<3, 2>(base_b, yt0, ny, nch, colE, cb, ce, skip, o, chunk_pad, inv_count); break;
          case 4: nhwc_unit<4, 1>(base_b, yt0, ny, nch, colE, cb, ce, skip, o, chunk_pad, inv_count); break;
          case 5: nhwc_unit<5, 1>(base_b, yt0, ny, nch, colE, cb, ce, skip, o, chunk_pad, inv_count); break;
          default: nhwc_unit<6, 1>(base_b, yt0, ny, nch, colE, cb, ce, skip, o, chunk_pad, inv_count); break;
        }
      }
    } else
    for (int bl = warp; bl < nb; bl += nwarps) {
      const int bin = bin0 + bl;
      const int ph = bin / PW, pw = bin - ph * PW;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      if (!onfly) {
        const int ny = yn[ph], nx = xn[pw];
        if (nx <= 4) nhwc_bin<4, 2>(base_b, ytab + ph, xtab + pw, ny, nx, acc);
        else nhwc_bin<8, 1>(base_b, ytab + ph, xtab + pw, ny, nx, acc);
      } else {  // rare: sampling grid too large for the tap lists (or pooled size > 16): taps on the fly
        const RoiGeom g = sg;
        for (int iy = 0; iy < g.gh; ++iy) {
          const Tap1 ty = make_tap1(g.start_h + (float)ph * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
          const float4* __restrict__ r0 = base + ty.lo * W * C4;
          const float4* __restrict__ r1 = base + ty.hi * W * C4;
          for (int ix = 0; ix < g.gw; ++ix) {
            const Tap1 tx = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
            const float4 v1 = __ldg(r0 + tx.lo * C4), v2 = __ldg(r0 + tx.hi * C4);
            const float4 v3 = __ldg(r1 + tx.lo * C4), v4 = __ldg(r1 + tx.hi * C4);
            const float w1 = ty.wl * tx.wl, w2 = ty.wl * tx.wh, w3 = ty.wh * tx.wl, w4 = ty.wh * tx.wh;
            acc.x += w1 * v1.x + w2 * v2.x + w3 * v3.x + w4 * v4.x;
            acc.y += w1 * v1.y + w2 * v2.y + w3 * v3.y + w4 * v4.y;
            acc.z += w1 * v1.z + w2 * v2.z + w3 * v3.z + w4 * v4.z;
            acc.w += w1 * v1.w + w2 * v2.w + w3 * v3.w + w4 * v4.w;
          }
        }
      }
      float* __restrict__ o = otile + lane * chunk_pad + bl;  // odd pitch: the 32 lanes hit 32 banks
      const float inv_count = sg.inv_count;
      o[0] = acc.x * inv_count;
      o[32 * chunk_pad] = acc.y * inv_count;
      o[64 * chunk_pad] = acc.z * inv_count;
      o[96 * chunk_pad] = acc.w * inv_count;
    }
    __syncthreads();
    // channel-major write-out: channel c0+cl, bins [bin0, bin0+nb) -- one contiguous run of the output per channel
    typename Elem<ODT>::T* __restrict__ obase = reinterpret_cast<typename Elem<ODT>::T*>(out_v) + ((size_t)k * C + c0) * bins + bin0;
    const unsigned magic = 0xFFFFFFFFu / (unsigned)nb + 1u;  // i / nb == umulhi(i, magic) for i < 2^16 (i < 128 * 64 here)
    for (int i = tid; i < ncta * nb; i += blockDim.x) {
      const int cl = nb == 1 ? i : (int)__umulhi((unsigned)i, magic), bl = i - cl * nb;  // (magic wraps to 0 for nb == 1)
      obase[(size_t)cl * bins + bl] = Elem<ODT>::st(otile[((cl & 3) * 32 + (cl >> 2)) * chunk_pad + bl]);
    }
  }
}

static int launch_fwd_nhwc(const Pyr& P, int N, const float* rois, int K, int C, int PH, int PW, int sr, int aligned,
                           void* out, cudaStream_t stream, int out_dt = D2B_F32) {
  (void)N;
  const int bins = PH * PW;
  const int slabs = d2b_cdiv(C, kNhwcCh);
  // bins of a RoI are split into chunks (grid.z): at least enough for the transpose tile, more when K x slabs alone
  // would leave SMs idle (a mask-head call has 100 RoIs x 196 bins)
  const long long want = d2b_cdiv(8LL * d2b_num_sms(), (long long)K * slabs);
  int nchunks = (int)std::max<long long>(d2b_cdiv(bins, kNhwcChunk), std::min<long long>(want, d2b_cdiv(bins, 8)));
  int chunk = d2b_cdiv(bins, nchunks);
  if (nchunks > 1) chunk = std::min(kNhwcChunk - 1, d2b_cdiv(chunk, 7) * 7);  // whole rounds of the CTA's 7 warps
  nchunks = d2b_cdiv(bins, chunk);
  const int chunk_pad = chunk | 1;
  const size_t smem = sizeof(float) * 128 * (size_t)chunk_pad;
  dim3 grid(K, slabs, nchunks);  // nchunks <= 65535: chunks hold >= 7 bins (nhwc_supported)
  D2B_DISPATCH_DTYPE(out_dt, (roi_align_nhwc_kernel<DT><<<grid, kNhwcThreads, smem, stream>>>(P, rois, C, PH, PW, sr, aligned, chunk,
                                                                                            chunk_pad, out)));
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// ------------------------------------------------------------------ channels-last (NHWC) backward
// The transpose of the forward, formulated per FOOTPRINT PIXEL instead of per sample: the g_h x g_w sample grid of a bin
// is a product grid, so the weight of bin (ph, pw) on pixel (y, x) is Wy[ph][y] * Wx[pw][x] with 1-D tables that are built
// once per RoI (a pixel row is touched by 1-2 bin rows, rarely more).  A warp owns one footprint pixel at a time
// (lane = 4 channels): it sums the <= few contributing bins from the RoI's gradient tile in shared memory and issues ONE
// red.global.add.v4.f32 per pixel -- against 4*g*g scalar atomics per output element in the reference
// (ROIAlignRotated_cuda.cu:311-318 / torchvision roi_align_backward) and one scalar red per pixel and channel in the NCHW
// kernel above.
constexpr int kBwdBand = 64;     // footprint rows per pass
constexpr int kBwdMaxFw = 96;    // footprint columns with a table (FPN-assigned RoIs span < 60); wider RoIs take the per-sample path
constexpr int kBwdThreads = 256;

__device__ __forceinline__ void red_add_v4(float* p, float4 v) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Per-sample scatter (taps on the fly, one red.v4 per tap): pooled sizes > 16 and footprints wider than the column table.
template <int GDT>
__device__ void bwd_nhwc_per_sample(const RoiGeom& g, const typename Elem<GDT>::T* __restrict__ go, float* __restrict__ gimg,
                                    int H, int W, int C, int PH, int PW, bool lane_live, int ph0, int PHl) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int bins = PH * PW;
  for (int bl = warp; bl < PHl * PW; bl += nwarps) {  // the CTA's bin rows [ph0, ph0 + PHl)
    const int ph = ph0 + bl / PW, pw = bl - (ph - ph0) * PW, bin = ph * PW + pw;
    float4 gv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane_live) {
      const typename Elem<GDT>::T* q = go + (size_t)(lane * 4) * bins + bin;
      gv = make_float4(Elem<GDT>::ld(q) * g.inv_count, Elem<GDT>::ld(q + bins) * g.inv_count,
                       Elem<GDT>::ld(q + 2 * bins) * g.inv_count, Elem<GDT>::ld(q + 3 * bins) * g.inv_count);
    }
    for (int iy = 0; iy < g.gh; ++iy) {
      const Tap1 ty = make_tap1(g.start_h + (float)ph * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
      for (int ix = 0; ix < g.gw; ++ix) {
        const Tap1 tx = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
        if (!lane_live) continue;
        const float w1 = ty.wl * tx.wl, w2 = ty.wl * tx.wh, w3 = ty.wh * tx.wl, w4 = ty.wh * tx.wh;
        if (w1 != 0.f) red_add_v4(gimg + ((size_t)ty.lo * W + tx.lo) * C, make_float4(gv.x * w1, gv.y * w1, gv.z * w1, gv.w * w1));
        if (w2 != 0.f) red_add_v4(gimg + ((size_t)ty.lo * W + tx.hi) * C, make_float4(gv.x * w2, gv.y * w2, gv.z * w2, gv.w * w2));
        if (w3 != 0.f) red_add_v4(gimg + ((size_t)ty.hi * W + tx.lo) * C, make_float4(gv.x * w3, gv.y * w3, gv.z * w3, gv.w * w3));
        if (w4 != 0.f) red_add_v4(gimg + ((size_t)ty.hi * W + tx.hi) * C, make_float4(gv.x * w4, gv.y * w4, gv.z * w4, gv.w * w4));
      }
    }
  }
}

template <int GDT>
__global__ void __launch_bounds__(kBwdThreads) roi_align_bwd_nhwc_kernel(const Pyr P, const float* __restrict__ rois, int C,
                                                                       int PH, int PW, int sr, int aligned, int rows_per_cta,
                                                                       const void* __restrict__ gout) {
  extern __shared__ __align__(16) float gs[];  // [bin][128 ch], float4 slots XOR-swizzled with the bin index
  __shared__ float WyT[kBwdBand * kMaxP];      // [row of the band][ph]
  __shared__ float WxT[kBwdMaxFw * kMaxP];     // [column of the footprint][pw]
  __shared__ unsigned char ylo[kBwdBand], yhi[kBwdBand], xlo[kBwdMaxFw], xhi[kBwdMaxFw];  // non-zero bin range per row / column
  // the common case -- at most two bins touch a pixel row / column (bins at least one pixel wide): {bin a, bin b, w a, w b}
  __shared__ float4 colE[kBwdMaxFw], rowE[kBwdBand];
  __shared__ RoiGeom sg;
  __shared__ int s_xmin, s_xmax, s_ymin, s_ymax, s_wide;

  const int k = blockIdx.x;
  const int c0 = blockIdx.y * kNhwcCh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int kWarps = kBwdThreads / 32;
  const int lvl_raw = pick_level(P, (P.level_rois ? P.level_rois : rois) + (size_t)k * 5);
  const int lvl = max(lvl_raw, 0);
  const int H = P.H[lvl], W = P.W[lvl];
  const int bins = PH * PW;
  // bin rows [ph0, ph0 + PHl) of the RoI: a 14x14 mask-head tile (157 KB of shared memory, one CTA per SM) is split over
  // grid.z so that several CTAs share an SM; rows shared by two CTAs' footprints simply receive both contributions
  const int ph0 = blockIdx.z * rows_per_cta, PHl = min(rows_per_cta, PH - ph0), bins_l = PHl * PW;
  const int ncta = min(kNhwcCh, C - c0);
  const bool lane_live = lane * 4 < ncta;
  if (tid == 0) {
    sg = load_geom<false>(rois + (size_t)k * 5, P.scale[lvl], PH, PW, sr, aligned, lvl_raw < 0);
    s_xmin = s_ymin = 1 << 30;
    s_xmax = s_ymax = -1;
    s_wide = 0;
  }
  __syncthreads();
  const RoiGeom g = sg;
  float* __restrict__ gimg = P.grad[lvl] + (size_t)g.b * H * W * C + c0 + lane * 4;
  const typename Elem<GDT>::T* __restrict__ go = reinterpret_cast<const typename Elem<GDT>::T*>(gout) + ((size_t)k * C + c0) * bins;

  if (PH > kMaxP || PW > kMaxP) {  // pooled size beyond the tables: per-sample path
    bwd_nhwc_per_sample<GDT>(g, go, gimg, H, W, C, PH, PW, lane_live, ph0, PHl);
    return;
  }
  // ---- footprint bounds (rows / columns that receive a non-zero weight)
  if (tid < PHl) {
    int lo = 1 << 30, hi = -1;
    for (int iy = 0; iy < g.gh; ++iy) {
      const Tap1 t = make_tap1(g.start_h + (float)(ph0 + tid) * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
      if (t.wl != 0.f) { lo = min(lo, t.lo); hi = max(hi, t.lo); }
      if (t.wh != 0.f) { lo = min(lo, t.hi); hi = max(hi, t.hi); }
    }
    if (hi >= 0) {
      atomicMin(&s_ymin, lo);
      atomicMax(&s_ymax, hi);
    }
  } else if (tid >= 32 && tid < 32 + PW) {
    const int pw = tid - 32;
    int lo = 1 << 30, hi = -1;
    for (int ix = 0; ix < g.gw; ++ix) {
      const Tap1 t = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
      if (t.wl != 0.f) { lo = min(lo, t.lo); hi = max(hi, t.lo); }
      if (t.wh != 0.f) { lo = min(lo, t.hi); hi = max(hi, t.hi); }
    }
    if (hi >= 0) {
      atomicMin(&s_xmin, lo);
      atomicMax(&s_xmax, hi);
    }
  }
  __syncthreads();
  const int xmin = s_xmin, fw = s_xmax - s_xmin + 1, ymin = s_ymin, ymax = s_ymax;
  if (s_xmax < 0 || ymax < 0) return;  // no sample inside the map: zero gradient
  if (fw > kBwdMaxFw) {  // very wide footprint (block-uniform)
    bwd_nhwc_per_sample<GDT>(g, go, gimg, H, W, C, PH, PW, lane_live, ph0, PHl);
    return;
  }
  // ---- column table + gradient tile
  for (int i = tid; i < fw * kMaxP; i += kBwdThreads) WxT[i] = 0.f;
  __syncthreads();
  if (tid >= 32 && tid < 32 + PW) {
    const int pw = tid - 32;
    for (int ix = 0; ix < g.gw; ++ix) {
      const Tap1 t = make_tap1(g.start_w + (float)pw * g.bin_w + ((float)ix + .5f) * g.bin_w / (float)g.gw, W);
      if (t.wl != 0.f) WxT[(t.lo - xmin) * kMaxP + pw] += t.wl;
      if (t.wh != 0.f) WxT[(t.hi - xmin) * kMaxP + pw] += t.wh;
    }
  }
  for (int e = tid; e < ncta * bins_l; e += kBwdThreads) {  // coalesced read of [ch][bin], transposed + swizzled store
    const int c = e / bins_l, bin = e - c * bins_l;             // bin: index inside the CTA's rows
    gs[bin * kNhwcCh + ((((c >> 2) ^ bin) & 31) << 2) + (c & 3)] =
        Elem<GDT>::ld(go + (size_t)c * bins + ph0 * PW + bin) * g.inv_count;
  }
  __syncthreads();
  for (int x = tid; x < fw; x += kBwdThreads) {
    int lo = 255, hi = 0, cnt = 0, ia = 0, ib = 0;
    float wa = 0.f, wb = 0.f;
    for (int pw = 0; pw < PW; ++pw) {
      const float w = WxT[x * kMaxP + pw];
      if (w != 0.f) {
        lo = min(lo, pw);
        hi = max(hi, pw + 1);
        if (cnt == 0) { ia = pw; wa = w; }
        else if (cnt == 1) { ib = pw; wb = w; }
        ++cnt;
      }
    }
    xlo[x] = (unsigned char)lo;
    xhi[x] = (unsigned char)hi;
    colE[x] = make_float4(__int_as_float(ia), __int_as_float(ib), wa, wb);
    if (cnt > 2) atomicOr(&s_wide, 1);
  }
  float* __restrict__ Ts = gs + (size_t)bins_l * kNhwcCh + (size_t)warp * PW * kNhwcCh;  // this warp's row-collapsed gradients
  // ---- bands of footprint rows
  for (int yb = ymin; yb <= ymax; yb += kBwdBand) {
    const int nrow = min(kBwdBand, ymax - yb + 1);
    __syncthreads();  // previous band consumed
    for (int i = tid; i < nrow * kMaxP; i += kBwdThreads) WyT[i] = 0.f;
    __syncthreads();
    if (tid < PHl) {
      for (int iy = 0; iy < g.gh; ++iy) {
        const Tap1 t = make_tap1(g.start_h + (float)(ph0 + tid) * g.bin_h + ((float)iy + .5f) * g.bin_h / (float)g.gh, H);
        if (t.wl != 0.f && t.lo >= yb && t.lo < yb + nrow) WyT[(t.lo - yb) * kMaxP + tid] += t.wl;
        if (t.wh != 0.f && t.hi >= yb && t.hi < yb + nrow) WyT[(t.hi - yb) * kMaxP + tid] += t.wh;
      }
    }
    __syncthreads();
    for (int y = tid; y < nrow; y += kBwdThreads) {
      int lo = 255, hi = 0, cnt = 0, ia = 0, ib = 0;
      float wa = 0.f, wb = 0.f;
      for (int ph = 0; ph < PHl; ++ph) {
        const float w = WyT[y * kMaxP + ph];
        if (w != 0.f) {
          lo = min(lo, ph);
          hi = max(hi, ph + 1);
          if (cnt == 0) { ia = ph; wa = w; }
          else if (cnt == 1) { ib = ph; wb = w; }
          ++cnt;
        }
      }
      ylo[y] = (unsigned char)lo;
      yhi[y] = (unsigned char)hi;
      rowE[y] = make_float4(__int_as_float(ia), __int_as_float(ib), wa, wb);
      if (cnt > 2) atomicOr(&s_wide, 1);
    }
    __syncthreads();
    if (!s_wide) {
      // separable two-step form: a warp owns a footprint row; T[pw] = wy_a g[ph_a][pw] + wy_b g[ph_b][pw] once per row
      // (warp-private shared memory), then every pixel of the row is wx_a T[pw_a] + wx_b T[pw_b]: ~12 instructions / pixel
      for (int yr = warp; yr < nrow; yr += kWarps) {
        const float4 re = rowE[yr];
        if (re.z == 0.f && re.w == 0.f) continue;  // warp-uniform
        const int pa = __float_as_int(re.x), pb = __float_as_int(re.y);
        const F2 wya = f2_pack(re.z, re.z), wyb = f2_pack(re.w, re.w);
        __syncwarp();
        for (int pw = 0; pw < PW; ++pw) {
          const int ba = pa * PW + pw, bb = pb * PW + pw;
          const float4 ga = *reinterpret_cast<const float4*>(gs + ba * kNhwcCh + (((lane ^ ba) & 31) << 2));
          const float4 gb = *reinterpret_cast<const float4*>(gs + bb * kNhwcCh + (((lane ^ bb) & 31) << 2));
          const F2 z = f2_pack(0.f, 0.f);
          const F2 t01 = f2_fma(wyb, f2_pack(gb.x, gb.y), f2_fma(wya, f2_pack(ga.x, ga.y), z));
          const F2 t23 = f2_fma(wyb, f2_pack(gb.z, gb.w), f2_fma(wya, f2_pack(ga.z, ga.w), z));
          float4 tv;
          f2_unpack(t01, tv.x, tv.y);
          f2_unpack(t23, tv.z, tv.w);
          *reinterpret_cast<float4*>(Ts + pw * kNhwcCh + lane * 4) = tv;
        }
        __syncwarp();
        float* __restrict__ grow = gimg + (size_t)(yb + yr) * W * C + (size_t)xmin * C;
        for (int xr = 0; xr < fw; ++xr) {
          const float4 ce = colE[xr];
          if (ce.z == 0.f && ce.w == 0.f) continue;
          const float4 ta = *reinterpret_cast<const float4*>(Ts + __float_as_int(ce.x) * kNhwcCh + lane * 4);
          const float4 tb = *reinterpret_cast<const float4*>(Ts + __float_as_int(ce.y) * kNhwcCh + lane * 4);
          const F2 z = f2_pack(0.f, 0.f), wxa = f2_pack(ce.z, ce.z), wxb = f2_pack(ce.w, ce.w);
          const F2 a01 = f2_fma(wxb, f2_pack(tb.x, tb.y), f2_fma(wxa, f2_pack(ta.x, ta.y), z));
          const F2 a23 = f2_fma(wxb, f2_pack(tb.z, tb.w), f2_fma(wxa, f2_pack(ta.z, ta.w), z));
          float4 acc;
          f2_unpack(a01, acc.x, acc.y);
          f2_unpack(a23, acc.z, acc.w);
          if (lane_live) red_add_v4(grow + (size_t)xr * C, acc);
        }
      }
      continue;
    }
    // general form (bins narrower than a pixel: more than two bins per row / column)
    for (int yr = 0; yr < nrow; ++yr) {
      const int pa = ylo[yr], pb = yhi[yr];
      if (pa >= pb) continue;
      float* __restrict__ grow = gimg + (size_t)(yb + yr) * W * C;
      for (int xr = warp; xr < fw; xr += kWarps) {
        const int qa = xlo[xr], qb = xhi[xr];
        if (qa >= qb) continue;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int ph = pa; ph < pb; ++ph) {
          const float wy = WyT[yr * kMaxP + ph];
          for (int pw = qa; pw < qb; ++pw) {
            const float w = wy * WxT[xr * kMaxP + pw];
            const int bin = ph * PW + pw;
            const float4 gv = *reinterpret_cast<const float4*>(gs + bin * kNhwcCh + (((lane ^ bin) & 31) << 2));
            acc.x = fmaf(w, gv.x, acc.x);
            acc.y = fmaf(w, gv.y, acc.y);
            acc.z = fmaf(w, gv.z, acc.z);
            acc.w = fmaf(w, gv.w, acc.w);
          }
        }
        if (lane_live) red_add_v4(grow + (size_t)(xmin + xr) * C, acc);
      }
    }
  }
}

// gradient tile [rows * PW][128] + per-warp row-collapsed tile [8 warps][PW][128]
static size_t bwd_nhwc_smem(int rows, int PW) {
  return sizeof(float) * kNhwcCh * ((size_t)rows * PW + (size_t)(kBwdThreads / 32) * PW);
}

static int launch_bwd_nhwc(const Pyr& P, int N, const float* rois, int K, int C, int PH, int PW, int sr, int aligned,
                           const void* gout, cudaStream_t stream, int g_dt = D2B_F32) {
  (void)N;
  // bin rows per CTA: all of them, unless that leaves fewer than ~2 CTAs per SM resident (shared memory) AND in the grid
  const int slabs = d2b_cdiv(C, kNhwcCh);
  int rows = PH;
  while (rows > 4 &&
         (bwd_nhwc_smem(rows, PW) > 100 * 1024 || (long long)K * slabs * d2b_cdiv(PH, rows) < 4LL * d2b_num_sms()) &&
         bwd_nhwc_smem(rows, PW) > 56 * 1024)
    rows = (rows + 1) / 2;
  const size_t smem = bwd_nhwc_smem(rows, PW);  // <= 180 KB (nhwc_supported)
  dim3 grid(K, slabs, d2b_cdiv(PH, rows));
  D2B_DISPATCH_DTYPE(g_dt, {
    D2B_ALLOW_BIG_SMEM(roi_align_bwd_nhwc_kernel<DT>);
    roi_align_bwd_nhwc_kernel<DT><<<grid, kBwdThreads, smem, stream>>>(P, rois, C, PH, PW, sr, aligned, rows, gout);
  });
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// ------------------------------------------------------------------ rotated RoIAlign on channels-last storage
// The sample grid of a rotated RoI is not a product grid, so the axis-aligned tables do not apply; what carries over is the
// layout: lane = 4 channels, a warp owns one bin at a time, the taps of a sample (4 pixel offsets + 4 weights, built once
// per CTA into shared memory) are warp-uniform, every tap is one 512-byte LDG.128 (forward) or one red.global.add.v4.f32
// (backward) per warp.  The reference runs one thread per output element with scalar taps and, in the backward, 4*g*g
// scalar atomics per element (ROIAlignRotated_cuda.cu:143-222, :224-323).
constexpr int kRotMaxTap = 1024;  // (bins x samples) entries of the shared tap table; larger grids compute taps on the fly

// The FPN level is picked per CTA (P.feat[l] / P.grad[l] are fp32 [N,H,W,C]); out / gout are [K,C,PH,PW] elements of DT
// (fp32 arithmetic, half precision converted on load / store).
template <bool BWD, int DT>
__global__ void __launch_bounds__(kBwdThreads) roi_align_rot_nhwc_kernel(const Pyr P, const float* __restrict__ rois, int C,
                                                                       int PH, int PW, int sr, const void* __restrict__ gout,
                                                                       void* __restrict__ out) {
  using E = Elem<DT>;
  extern __shared__ __align__(16) float tile[];  // forward: [128 ch][bins | 1] results; backward: [bin][128 ch] swizzled grads
  __shared__ Tap2 taps[kRotMaxTap];
  const int k = blockIdx.x;
  const int c0 = blockIdx.y * kNhwcCh;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  constexpr int kWarps = kBwdThreads / 32;
  const int lvl_raw = pick_level<true>(P, rois + (size_t)k * 6);
  const int lvl = max(lvl_raw, 0);
  const float* __restrict__ in = BWD ? nullptr : P.feat[lvl];
  float* __restrict__ gin = BWD ? P.grad[lvl] : nullptr;
  const int H = P.H[lvl], W = P.W[lvl];
  const RoiGeom g = load_geom<true>(rois + (size_t)k * 6, P.scale[lvl], PH, PW, sr, 1, lvl_raw < 0);
  const int bins = PH * PW;
  const int spb = g.gh * g.gw;
  const int ncta = min(kNhwcCh, C - c0);
  const bool lane_live = lane * 4 < ncta;
  const bool tab = (long long)bins * spb <= kRotMaxTap;
  const int pitch = bins | 1;
  if (tab) {
    for (int i = tid; i < bins * spb; i += kBwdThreads) {
      const int bin = i / spb, sidx = i - bin * spb;
      const int ph = bin / PW, pw = bin - ph * PW, iy = sidx / g.gw, ix = sidx - iy * g.gw;
      float y, x;
      rot_xy(g, ph, pw, iy, ix, y, x);
      taps[i] = make_tap2(y, x, H, W);
    }
  }
  if (BWD) {
    const typename E::T* __restrict__ go = reinterpret_cast<const typename E::T*>(gout) + ((size_t)k * C + c0) * bins;
    for (int e = tid; e < ncta * bins; e += kBwdThreads) {
      const int c = e / bins, bin = e - c * bins;
      tile[bin * kNhwcCh + ((((c >> 2) ^ bin) & 31) << 2) + (c & 3)] = E::ld(go + e) / g.count_raw;
    }
  }
  __syncthreads();
  const size_t img = (size_t)g.b * H * W * C + c0 + (lane_live ? lane * 4 : 0);
  for (int bin = warp; bin < bins; bin += kWarps) {
    const int ph = bin / PW, pw = bin - ph * PW;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 gv = make_float4(0.f, 0.f, 0.f, 0.f);
    if (BWD) gv = *reinterpret_cast<const float4*>(tile + bin * kNhwcCh + (((lane ^ bin) & 31) << 2));
    for (int sidx = 0; sidx < spb; ++sidx) {
      Tap2 t;
      if (tab) t = taps[bin * spb + sidx];
      else {
        const int iy = sidx / g.gw, ix = sidx - iy * g.gw;
        float y, x;
        rot_xy(g, ph, pw, iy, ix, y, x);
        t = make_tap2(y, x, H, W);
      }
      if (t.p1 < 0) continue;  // warp-uniform
      if (BWD) {
        if (lane_live) {
          float* __restrict__ gb = gin + img;
          red_add_v4(gb + (size_t)t.p1 * C, make_float4(gv.x * t.w1, gv.y * t.w1, gv.z * t.w1, gv.w * t.w1));
          red_add_v4(gb + (size_t)t.p2 * C, make_float4(gv.x * t.w2, gv.y * t.w2, gv.z * t.w2, gv.w * t.w2));
          red_add_v4(gb + (size_t)t.p3 * C, make_float4(gv.x * t.w3, gv.y * t.w3, gv.z * t.w3, gv.w * t.w3));
          red_add_v4(gb + (size_t)t.p4 * C, make_float4(gv.x * t.w4, gv.y * t.w4, gv.z * t.w4, gv.w * t.w4));
        }
      } else {
        const float* __restrict__ fb = in + img;
        const float4 v1 = __ldg(reinterpret_cast<const float4*>(fb + (size_t)t.p1 * C));
        const float4 v2 = __ldg(reinterpret_cast<const float4*>(fb + (size_t)t.p2 * C));
        const float4 v3 = __ldg(reinterpret_cast<const float4*>(fb + (size_t)t.p3 * C));
        const float4 v4 = __ldg(reinterpret_cast<const float4*>(fb + (size_t)t.p4 * C));
        acc.x += t.w1 * v1.x + t.w2 * v2.x + t.w3 * v3.x + t.w4 * v4.x;
        acc.y += t.w1 * v1.y + t.w2 * v2.y + t.w3 * v3.y + t.w4 * v4.y;
        acc.z += t.w1 * v1.z + t.w2 * v2.z + t.w3 * v3.z + t.w4 * v4.z;
        acc.w += t.w1 * v1.w + t.w2 * v2.w + t.w3 * v3.w + t.w4 * v4.w;
      }
    }
    if (!BWD) {
      float* __restrict__ o = tile + lane * pitch + bin;  // odd pitch: the 32 lanes hit 32 banks
      o[0] = acc.x * g.inv_count;
      o[32 * pitch] = acc.y * g.inv_count;
      o[64 * pitch] = acc.z * g.inv_count;
      o[96 * pitch] = acc.w * g.inv_count;
    }
  }
  if (!BWD) {
    __syncthreads();
    typename E::T* __restrict__ obase = reinterpret_cast<typename E::T*>(out) + ((size_t)k * C + c0) * bins;
    for (int i = tid; i < ncta * bins; i += kBwdThreads) {  // channel-major write-out: contiguous runs of the NCHW-shaped output
      const int cl = i / bins, bl = i - cl * bins;
      obase[i] = E::st(tile[((cl & 3) * 32 + (cl >> 2)) * pitch + bl]);
    }
  }
}

// dt: element type of `out` (forward) / `gout` (backward).  Every level's feature map (forward) or gradient map (backward)
// must be 16-byte aligned -- checked by pooler_args.
template <bool BWD>
static size_t rot_nhwc_smem(int PH, int PW) {
  return sizeof(float) * 128 * (size_t)(BWD ? PH * PW : ((PH * PW) | 1));
}

// The shape limits of every channels-last kernel (D2B_OK or D2B_EUNSUPPORTED), stated once: pooler_args and
// d2b_roi_pooler_nhwc_supported both ask this.  Host-only, no CUDA call.
static int nhwc_supported(int num_levels, const int* H, const int* W, int C, int PH, int PW, int flags) {
  if (C % 4 != 0) return D2B_EUNSUPPORTED;  // lane = 4 channels
  for (int l = 0; l < num_levels; ++l)
    if ((long long)H[l] * W[l] * (C / 4) >= (1LL << 28)) return D2B_EUNSUPPORTED;  // 32-bit byte offsets inside an image
  const long long bins = (long long)PH * PW;
  if (flags & D2B_ROI_ROTATED) {
    // [128 ch][bins] fp32 tile in shared memory; the forward's pitch is bins | 1, and the backward is held to the same bound
    if (sizeof(float) * 128 * (bins | 1) > 150 * 1024) return D2B_EUNSUPPORTED;
  } else if (flags & D2B_ROI_BACKWARD) {
    // launch_bwd_nhwc halves the bin rows per CTA at least this far, and further only while the tile stays above 56 KB:
    // its tile exceeds 180 KB exactly when this one does, whatever K
    int rows = PH;
    while (rows > 4 && bwd_nhwc_smem(rows, PW) > 100 * 1024) rows = (rows + 1) / 2;
    if (bwd_nhwc_smem(rows, PW) > 180 * 1024) return D2B_EUNSUPPORTED;
  } else {
    if ((bins + 6) / 7 > 65535) return D2B_EUNSUPPORTED;  // launch_fwd_nhwc's output chunks hold >= 7 bins: grid.z
  }
  return D2B_OK;
}

template <bool BWD>
static int launch_rot_nhwc(const Pyr& P, const float* rois, int K, int C, int PH, int PW, int sr, const void* gout, void* out,
                           cudaStream_t stream, int dt = D2B_F32) {
  const size_t smem = rot_nhwc_smem<BWD>(PH, PW);
  dim3 grid(K, d2b_cdiv(C, kNhwcCh));
  D2B_DISPATCH_DTYPE(dt, {
    D2B_ALLOW_BIG_SMEM((roi_align_rot_nhwc_kernel<BWD, DT>));
    roi_align_rot_nhwc_kernel<BWD, DT><<<grid, kBwdThreads, smem, stream>>>(P, rois, C, PH, PW, sr, gout, out);
  });
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// NCHW -> NHWC of every pyramid level in one launch: 32 channels x 64 pixels per CTA through a padded tile.
struct XposeLevels {
  int num_levels;
  const void* src[D2B_MAX_LEVELS];
  void* dst[D2B_MAX_LEVELS];
  int HW[D2B_MAX_LEVELS];
  int tile_begin[D2B_MAX_LEVELS + 1];
};

template <int SDT>
__global__ void __launch_bounds__(256) nchw_to_nhwc_kernel(const XposeLevels L, int C) {
  __shared__ float tile[32][65];
  int l = 0;
  while (l + 1 < L.num_levels && (int)blockIdx.x >= L.tile_begin[l + 1]) ++l;
  const int HW = L.HW[l];
  const int hw0 = ((int)blockIdx.x - L.tile_begin[l]) * 64;
  const int c0 = blockIdx.y * 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  // source elements of type SDT: for half-precision inputs the layout change doubles as the up-cast
  const typename Elem<SDT>::T* __restrict__ src =
      reinterpret_cast<const typename Elem<SDT>::T*>(L.src[l]) + (size_t)blockIdx.z * C * HW;
  float* __restrict__ dst = reinterpret_cast<float*>(L.dst[l]) + (size_t)blockIdx.z * HW * C;
#pragma unroll
  for (int r = warp; r < 32; r += 8) {  // read: lanes along the pixels of one channel plane
    const int c = c0 + r;
    const int hwa = hw0 + lane, hwb = hw0 + 32 + lane;
    const typename Elem<SDT>::T* __restrict__ p = src + (size_t)min(c, C - 1) * HW;
    tile[r][lane] = hwa < HW ? Elem<SDT>::ld(p + hwa) : 0.f;
    tile[r][lane + 32] = hwb < HW ? Elem<SDT>::ld(p + hwb) : 0.f;
  }
  __syncthreads();
  // write: 8 lanes x float4 = the 32 channels of one pixel (128 B), 4 pixels per warp instruction; tile pitch 65 and
  // (quad, pixel) -> lane mapping make the 32 lanes hit 32 different banks
  const int cq = tid & 7;
  const int c = c0 + cq * 4;
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int hwl = (tid >> 3) + half * 32;
    const int hw = hw0 + hwl;
    if (hw < HW && c < C) {
      const float4 v = make_float4(tile[cq * 4 + 0][hwl], tile[cq * 4 + 1][hwl], tile[cq * 4 + 2][hwl], tile[cq * 4 + 3][hwl]);
      *reinterpret_cast<float4*>(dst + (size_t)hw * C + c) = v;
    }
  }
}

// the inverse (gradients accumulated channels-last go back to the reference's NCHW): same tiling, roles swapped
template <int DDT>
__global__ void __launch_bounds__(256) nhwc_to_nchw_kernel(const XposeLevels L, int C) {
  __shared__ float tile[32][65];
  int l = 0;
  while (l + 1 < L.num_levels && (int)blockIdx.x >= L.tile_begin[l + 1]) ++l;
  const int HW = L.HW[l];
  const int hw0 = ((int)blockIdx.x - L.tile_begin[l]) * 64;
  const int c0 = blockIdx.y * 32;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* __restrict__ src = reinterpret_cast<const float*>(L.src[l]) + (size_t)blockIdx.z * HW * C;
  // destination elements of type DDT: for half-precision gradients the layout change doubles as the down-cast
  typename Elem<DDT>::T* __restrict__ dst = reinterpret_cast<typename Elem<DDT>::T*>(L.dst[l]) + (size_t)blockIdx.z * C * HW;
  const int cq = tid & 7;
  const int c = c0 + cq * 4;
#pragma unroll
  for (int half = 0; half < 2; ++half) {  // read: 8 lanes x float4 = 32 channels of one pixel
    const int hwl = (tid >> 3) + half * 32;
    const int hw = hw0 + hwl;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (hw < HW && c < C) v = __ldg(reinterpret_cast<const float4*>(src + (size_t)hw * C + c));
    tile[cq * 4 + 0][hwl] = v.x;
    tile[cq * 4 + 1][hwl] = v.y;
    tile[cq * 4 + 2][hwl] = v.z;
    tile[cq * 4 + 3][hwl] = v.w;
  }
  __syncthreads();
#pragma unroll
  for (int r = warp; r < 32; r += 8) {  // write: lanes along the pixels of one channel plane
    const int cc = c0 + r;
    if (cc >= C) continue;
    typename Elem<DDT>::T* __restrict__ p = dst + (size_t)cc * HW;
    const int hwa = hw0 + lane, hwb = hw0 + 32 + lane;
    if (hwa < HW) p[hwa] = Elem<DDT>::st(tile[r][lane]);
    if (hwb < HW) p[hwb] = Elem<DDT>::st(tile[r][lane + 32]);
  }
}

}  // namespace

static bool make_pyr(const d2b_pyramid* pyr, Pyr& P) {
  if (!pyr || pyr->num_levels < 1 || pyr->num_levels > D2B_MAX_LEVELS) return false;
  P = Pyr{};
  P.num_levels = pyr->num_levels;
  for (int l = 0; l < pyr->num_levels; ++l) {
    if (pyr->H[l] <= 0 || pyr->W[l] <= 0) return false;
    P.feat[l] = pyr->feat[l];
    P.grad[l] = pyr->grad[l];
    P.H[l] = pyr->H[l];
    P.W[l] = pyr->W[l];
    P.scale[l] = pyr->scale[l];
  }
  P.min_level = pyr->min_level;
  P.max_level = pyr->max_level;
  P.canonical_level = pyr->canonical_level;
  P.canonical_box_size = pyr->canonical_box_size;
  P.level_rois = pyr->level_rois;
  if (P.num_levels > 1 && P.max_level - P.min_level + 1 != P.num_levels) return false;
  return true;
}

// Every backward zero-fills the gradient maps of all levels with one launch before it accumulates into them.
static int zero_grads(const Pyr& P, int N, int C, cudaStream_t stream) {
  void* zp[D2B_MAX_LEVELS];
  size_t zb[D2B_MAX_LEVELS];
  for (int l = 0; l < P.num_levels; ++l) {
    zp[l] = P.grad[l];
    zb[l] = sizeof(float) * (size_t)N * C * P.H[l] * P.W[l];
  }
  return d2b_zero_buffers(zp, zb, P.num_levels, stream);
}

// The argument rule of d2b_roi_pooler_forward / _backward, stated once (include/d2b200.h): every D2B_EINVAL condition comes
// before any D2B_EUNSUPPORTED one, and the entry points launch nothing until it has passed.  `data` is the forward's out or
// the backward's grad_out, `dtype` its element type.  On D2B_OK, P holds the pyramid and `idle` says that the call has
// nothing to write.
static int pooler_args(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int PH, int PW, int flags,
                       const void* data, int dtype, bool bwd, Pyr& P, bool& idle) {
  idle = true;
  if (!bwd && (K == 0 || C == 0)) return D2B_OK;  // nothing to compute: before any other check
  const bool nhwc = flags & D2B_ROI_NHWC;
  if ((flags & ~(D2B_ROI_ROTATED | D2B_ROI_NHWC)) || !make_pyr(pyr, P) || ((flags & D2B_ROI_ROTATED) && P.level_rois))
    return D2B_EINVAL;
  if (N < 0 || C < 0 || K < 0 || (N == 0 && K > 0)) return D2B_EINVAL;  // N == 0, K > 0: RoIs of images that do not exist
  if (!dtype_ok(dtype) || (!nhwc && dtype != D2B_F32)) return D2B_EINVAL;  // the NCHW kernels read and write fp32 only
  if (N == 0 || C == 0) return D2B_OK;                                     // a backward with no gradient element to write
  for (int l = 0; l < P.num_levels; ++l) {
    const void* map = bwd ? static_cast<const void*>(P.grad[l]) : P.feat[l];
    if (!map || (nhwc && (reinterpret_cast<uintptr_t>(map) & 15) != 0)) return D2B_EINVAL;
  }
  if (K > 0 && (!rois || !data || PH < 1 || PW < 1)) return D2B_EINVAL;
  idle = false;
  return nhwc && K > 0 ? nhwc_supported(P.num_levels, P.H, P.W, C, PH, PW, flags | (bwd ? D2B_ROI_BACKWARD : 0)) : D2B_OK;
}

D2B_API int d2b_roi_pooler_nhwc_supported(const d2b_pyramid* pyr, int C, int pooled_h, int pooled_w, int flags) {
  if (!pyr || pyr->num_levels < 1 || pyr->num_levels > D2B_MAX_LEVELS || C < 0 || pooled_h <= 0 || pooled_w <= 0)
    return D2B_EINVAL;
  return nhwc_supported(pyr->num_levels, pyr->H, pyr->W, C, pooled_h, pooled_w, flags);
}

D2B_API int d2b_roi_pooler_forward(const d2b_pyramid* pyr, int N, int C, const float* rois, int K, int pooled_h,
                                   int pooled_w, int sampling_ratio, int aligned, int flags, void* out, int out_dtype,
                                   void* stream) {
  Pyr P;
  bool idle;
  if (int rc = pooler_args(pyr, N, C, rois, K, pooled_h, pooled_w, flags, out, out_dtype, false, P, idle)) return rc;
  if (idle) return D2B_OK;
  const cudaStream_t s = (cudaStream_t)stream;
  switch (flags) {
    case 0:
      return launch_fwd(P, rois, K, C, pooled_h, pooled_w, sampling_ratio, aligned, static_cast<float*>(out), s);
    case D2B_ROI_NHWC:
      return launch_fwd_nhwc(P, N, rois, K, C, pooled_h, pooled_w, sampling_ratio, aligned, out, s, out_dtype);
    case D2B_ROI_ROTATED | D2B_ROI_NHWC:
      return launch_rot_nhwc<false>(P, rois, K, C, pooled_h, pooled_w, sampling_ratio, nullptr, out, s, out_dtype);
  }
  const int cpc = pick_c_per_cta(K, C);  // D2B_ROI_ROTATED
  dim3 grid(K, d2b_cdiv(C, cpc));
  roi_align_rot_fwd_kernel<1024><<<grid, kThreads, 0, s>>>(P, rois, C, pooled_h, pooled_w, sampling_ratio, cpc,
                                                           static_cast<float*>(out));
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_roi_pooler_backward(const d2b_pyramid* pyr, int N, int C, const void* grad_out, int grad_dtype,
                                    const float* rois, int K, int pooled_h, int pooled_w, int sampling_ratio, int aligned,
                                    int flags, void* stream) {
  Pyr P;
  bool idle;
  if (int rc = pooler_args(pyr, N, C, rois, K, pooled_h, pooled_w, flags, grad_out, grad_dtype, true, P, idle)) return rc;
  if (idle) return D2B_OK;
  const cudaStream_t s = (cudaStream_t)stream;
  const int rc = zero_grads(P, N, C, s);
  if (rc || K == 0) return rc;
  switch (flags) {
    case 0:
      return launch_fwd(P, rois, K, C, pooled_h, pooled_w, sampling_ratio, aligned, nullptr, s,
                        static_cast<const float*>(grad_out));
    case D2B_ROI_NHWC:
      return launch_bwd_nhwc(P, N, rois, K, C, pooled_h, pooled_w, sampling_ratio, aligned, grad_out, s, grad_dtype);
    case D2B_ROI_ROTATED | D2B_ROI_NHWC:
      return launch_rot_nhwc<true>(P, rois, K, C, pooled_h, pooled_w, sampling_ratio, grad_out, nullptr, s, grad_dtype);
  }
  const int cpc = pick_c_per_cta(K, C);  // D2B_ROI_ROTATED
  dim3 grid(K, d2b_cdiv(C, cpc));
  roi_align_rot_bwd_kernel<<<grid, kThreads, 0, s>>>(P, static_cast<const float*>(grad_out), rois, C, pooled_h, pooled_w,
                                                     sampling_ratio, cpc);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_pyramid_nchw_to_nhwc(const d2b_pyramid* pyr, int N, int C, float* const* dst, int src_dtype, void* stream) {
  if (!pyr || !dst || pyr->num_levels < 1 || pyr->num_levels > D2B_MAX_LEVELS || N < 0 || C < 0 || !dtype_ok(src_dtype))
    return D2B_EINVAL;
  if (N == 0 || C == 0) return D2B_OK;
  if (C % 4 != 0) return D2B_EUNSUPPORTED;
  XposeLevels L = {};
  L.num_levels = pyr->num_levels;
  int tiles = 0;
  for (int l = 0; l < pyr->num_levels; ++l) {
    if (!pyr->feat[l] || !dst[l] || pyr->H[l] <= 0 || pyr->W[l] <= 0) return D2B_EINVAL;
    if ((reinterpret_cast<uintptr_t>(dst[l]) & 15) != 0) return D2B_EINVAL;
    L.src[l] = pyr->feat[l];
    L.dst[l] = dst[l];
    L.HW[l] = pyr->H[l] * pyr->W[l];
    L.tile_begin[l] = tiles;
    tiles += d2b_cdiv(L.HW[l], 64);
  }
  L.tile_begin[pyr->num_levels] = tiles;
  if (N > 65535 || d2b_cdiv(C, 32) > 65535) return D2B_EUNSUPPORTED;
  dim3 grid(tiles, d2b_cdiv(C, 32), N);
  D2B_DISPATCH_DTYPE(src_dtype, (nchw_to_nhwc_kernel<DT><<<grid, 256, 0, (cudaStream_t)stream>>>(L, C)));
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API int d2b_pyramid_nhwc_to_nchw(const d2b_pyramid* pyr, int N, int C, void* const* dst, int dst_dtype, void* stream) {
  if (!pyr || !dst || pyr->num_levels < 1 || pyr->num_levels > D2B_MAX_LEVELS || N < 0 || C < 0 || !dtype_ok(dst_dtype))
    return D2B_EINVAL;
  if (N == 0 || C == 0) return D2B_OK;
  if (C % 4 != 0) return D2B_EUNSUPPORTED;
  XposeLevels L = {};
  L.num_levels = pyr->num_levels;
  int tiles = 0;
  for (int l = 0; l < pyr->num_levels; ++l) {
    if (!pyr->feat[l] || !dst[l] || pyr->H[l] <= 0 || pyr->W[l] <= 0) return D2B_EINVAL;
    if ((reinterpret_cast<uintptr_t>(pyr->feat[l]) & 15) != 0) return D2B_EINVAL;
    L.src[l] = pyr->feat[l];
    L.dst[l] = dst[l];
    L.HW[l] = pyr->H[l] * pyr->W[l];
    L.tile_begin[l] = tiles;
    tiles += d2b_cdiv(L.HW[l], 64);
  }
  L.tile_begin[pyr->num_levels] = tiles;
  if (N > 65535 || d2b_cdiv(C, 32) > 65535) return D2B_EUNSUPPORTED;
  dim3 grid(tiles, d2b_cdiv(C, 32), N);
  D2B_DISPATCH_DTYPE(dst_dtype, (nhwc_to_nchw_kernel<DT><<<grid, 256, 0, (cudaStream_t)stream>>>(L, C)));
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
