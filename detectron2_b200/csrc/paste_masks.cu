// paste_masks_in_image for sm_90a -- one fused kernel instead of the reference's
// meshgrid + grid_sample + compare + copy chain (detectron2/layers/mask_ops.py:17-69,74-147).
//
// HBM-bound byte kernel: the output (N*H*W bytes) dominates.  Most of every plane cannot see its mask and is written
// as the constant "outside" value with 128-bit stores; only the box's (conservative) rectangle is evaluated, from
// per-column / per-row sample coordinates tabulated in shared memory next to the 28x28 soft mask.  CTAs are handed to
// the masks in proportion to their work (paste_assign), because box areas differ by two orders of magnitude.
//
// Arithmetic mirrors the reference expression order (no FMA contraction: this file is compiled with -fmad=false):
//   g  = ((p + 0.5 - b0) / (b1 - b0)) * 2 - 1          (mask_ops.py:53-54)
//   i  = ((g + 1) * M - 1) / 2                           (grid_sample, align_corners=False)
//   v  = nw*w_nw + ne*w_ne + sw*w_sw + se*w_se           (zeros padding)
#include <algorithm>

#include "common.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kPix = 16;       // output bytes per thread
constexpr int kMaxM = 64;      // largest mask side staged in smem (28 in every shipped config)
constexpr int kMaxGridY = 65535;  // masks per launch of a (CTAs per mask, N) grid; larger N is launched in slices

__device__ __forceinline__ float sample_coord(float p, float b0, float b1, float M) {
  float g = (p + 0.5f - b0) / (b1 - b0) * 2.f - 1.f;
  return ((g + 1.f) * M - 1.f) / 2.f;
}

// exact value of one output pixel from its sample coordinates (reference expression order, see file header)
__device__ __forceinline__ uint32_t paste_value(const float* __restrict__ smask, int M, float fM, float ix, float iy,
                                                float threshold) {
  float v = 0.f;
  // in-range test written so that NaN / inf (degenerate boxes) fall through to 0
  if (ix > -1.f && ix < fM && iy > -1.f && iy < fM) {
    const float fx = floorf(ix), fy = floorf(iy);
    const int xw = (int)fx, yn = (int)fy, xe = xw + 1, ys = yn + 1;
    const float wx1 = ix - fx, wx0 = (float)xe - ix, wy1 = iy - fy, wy0 = (float)ys - iy;
    const bool okw = xw >= 0, oke = xe < M, okn = yn >= 0, oks = ys < M;
    if (okn && okw) v += smask[yn * M + xw] * (wx0 * wy0);
    if (okn && oke) v += smask[yn * M + xe] * (wx1 * wy0);
    if (oks && okw) v += smask[ys * M + xw] * (wx0 * wy1);
    if (oks && oke) v += smask[ys * M + xe] * (wx1 * wy1);
  }
  return threshold >= 0.f ? (v >= threshold ? 1u : 0u) : (uint32_t)(uint8_t)(v * 255.f);
}

__device__ __forceinline__ uint32_t paste_pixel(const float* __restrict__ smask, int M, float fM, int px, int py,
                                                float x0, float y0, float x1, float y1, float threshold) {
  return paste_value(smask, M, fM, sample_coord((float)px, x0, x1, fM), sample_coord((float)py, y0, y1, fM), threshold);
}

// Conservative support of the pasted mask: outside [cx0,cx1] x [ry0,ry1] every sample point lies >= 1.5 px beyond the
// mask's (-1, M) support, far more than fp32 rounding can move it, so the value there is exactly that of v = 0.
// Degenerate / non-finite boxes disable the shortcut (everything is evaluated exactly).
struct PasteRect {
  int cx0, cx1, ry0, ry1;
};

__device__ __forceinline__ PasteRect paste_rect(float x0, float y0, float x1, float y1, float fM, int H, int W) {
  PasteRect r = {0, W - 1, 0, H - 1};
  const float bw = x1 - x0, bh = y1 - y0;
  if (W >= 2 * kPix && bw > 0.f && bh > 0.f && bw < 1e8f && bh < 1e8f && fabsf(x0) < 1e8f && fabsf(y0) < 1e8f) {
    const float fx0 = floorf(x0 - bw / fM) - 2.f, fx1 = ceilf(x1 + bw / fM) + 2.f;
    const float fy0 = floorf(y0 - bh / fM) - 2.f, fy1 = ceilf(y1 + bh / fM) + 2.f;
    r.cx0 = (int)fmaxf(fx0, 0.f);
    r.cx1 = (int)fminf(fx1, (float)(W - 1));
    r.ry0 = (int)fmaxf(fy0, 0.f);
    r.ry1 = (int)fminf(fy1, (float)(H - 1));
  }
  return r;
}

// CTAs of a balanced launch (1-D grid): every mask gets one CTA plus a share of the remaining ones proportional to its
// estimated instruction count (zero-fill of the plane + exact evaluation of its rectangle) -- with a fixed number of CTAs
// per mask the few large boxes of an image finish long after everything else.  Integer arithmetic: every CTA derives the
// same boundaries.  Returns this CTA's mask, its index among the mask's CTAs and their count.
__device__ __forceinline__ void paste_assign(const float* __restrict__ boxes, int N, int M, int H, int W, int& n,
                                             int& local, int& count) {
  __shared__ unsigned long long s_wsum[kThreads / 32];
  __shared__ int s_asg[3];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int per = (N + kThreads - 1) / kThreads;  // masks per thread (contiguous strip)
  const int m0 = min(N, tid * per), m1 = min(N, m0 + per);
  const unsigned long long fill = (unsigned long long)((long long)H * W / kPix) * 24ull;
  unsigned long long mine = 0;
  for (int m = m0; m < m1; ++m) {
    const PasteRect r = paste_rect(boxes[4 * m], boxes[4 * m + 1], boxes[4 * m + 2], boxes[4 * m + 3], (float)M, H, W);
    unsigned long long c = fill;
    if (r.cx1 >= r.cx0 && r.ry1 >= r.ry0) c += (unsigned long long)(r.ry1 - r.ry0 + 1) * (unsigned long long)(r.cx1 - r.cx0 + 32) * 44ull;
    mine += (c >> 8) + 1ull;
  }
  unsigned long long inc = mine;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_wsum[warp] = inc;
  __syncthreads();
  unsigned long long wbase = 0, total = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const unsigned long long t = s_wsum[w];
    if (w < warp) wbase += t;
    total += t;
  }
  unsigned long long prefix = wbase + inc - mine;  // cost of all masks before this thread's strip
  const unsigned long long spare = (unsigned long long)((int)gridDim.x - N);
  const unsigned f = blockIdx.x;
  for (int m = m0; m < m1; ++m) {
    const PasteRect r = paste_rect(boxes[4 * m], boxes[4 * m + 1], boxes[4 * m + 2], boxes[4 * m + 3], (float)M, H, W);
    unsigned long long c = fill;
    if (r.cx1 >= r.cx0 && r.ry1 >= r.ry0) c += (unsigned long long)(r.ry1 - r.ry0 + 1) * (unsigned long long)(r.cx1 - r.cx0 + 32) * 44ull;
    c = (c >> 8) + 1ull;
    const unsigned b0 = (unsigned)m + (unsigned)(spare * prefix / total);
    const unsigned b1 = (unsigned)(m + 1) + (unsigned)(spare * (prefix + c) / total);
    if (f >= b0 && f < b1) {
      s_asg[0] = m;
      s_asg[1] = (int)(f - b0);
      s_asg[2] = (int)(b1 - b0);
    }
    prefix += c;
  }
  __syncthreads();
  n = s_asg[0];
  local = s_asg[1];
  count = s_asg[2];
}

// grid: 1-D balanced launch (paste_assign) or (CTAs per mask, N).  Two phases per mask:
//   1. every 16-byte chunk of the output plane that cannot see the mask (conservative rectangle test) is written as
//      one 128-bit store of the "outside" value -- this is ~90% of the bytes and runs at store bandwidth;
//   2. the rows/columns of the conservative rectangle, widened to whole 16-byte chunks, are evaluated exactly.  The sample
//      coordinates are separable (ix depends on the column only, iy on the row only) and each costs two IEEE divisions,
//      so TAB = true tabulates them once per CTA in shared memory (the same expressions: bit-identical values); a warp
//      then owns a row of the rectangle, a lane 4 neighbouring pixels (one 32-bit store).  TAB = false (image too large
//      for the tables) evaluates one pixel per lane from scratch.
template <bool TAB>
__global__ void __launch_bounds__(kThreads) paste_masks_kernel(const float* __restrict__ masks,
                                                               const float* __restrict__ boxes, int M, int H, int W,
                                                               float threshold, uint8_t* __restrict__ out, int N,
                                                               int balanced) {
  __shared__ float smask[kMaxM * kMaxM];
  int n = blockIdx.y, cta_local = blockIdx.x, cta_count = gridDim.x;  // uniform launch: grid (CTAs per mask, N)
  if (balanced) paste_assign(boxes, N, M, H, W, n, cta_local, cta_count);
  const float* __restrict__ mk = masks + (size_t)n * M * M;
  for (int i = threadIdx.x; i < M * M; i += kThreads) smask[i] = mk[i];
  const float x0 = boxes[4 * n], y0 = boxes[4 * n + 1], x1 = boxes[4 * n + 2], y1 = boxes[4 * n + 3];
  __syncthreads();
  const float fM = (float)M;
  const PasteRect rect = paste_rect(x0, y0, x1, y1, fM, H, W);
  const int cx0 = rect.cx0, cx1 = rect.cx1, ry0 = rect.ry0, ry1 = rect.ry1;
  const bool empty = cx1 < cx0 || ry1 < ry0;  // rectangle entirely off the image
  const uint32_t zbyte = threshold >= 0.f ? ((0.f >= threshold) ? 1u : 0u) : 0u;
  const uint32_t zword = zbyte * 0x01010101u;
  const long long plane = (long long)H * W;
  uint8_t* __restrict__ obase = out + (size_t)n * plane;
  // obase may be misaligned w.r.t. 16 B when H*W is not a multiple of 16: chunk c covers [head + 16c, head + 16c + 16)
  const int head = (int)((16 - ((uintptr_t)obase & 15)) & 15);
  const long long stride = (long long)cta_count * kThreads;
  const long long gtid = (long long)cta_local * kThreads + threadIdx.x;

  // ---- phase 1: chunks that cannot see the mask.  (py, px) of a thread's chunk advance incrementally: one 32-bit
  //      division per thread instead of one 64-bit division per chunk -- this loop is instruction-bound, not HBM-bound.
  {
    const unsigned uW = (unsigned)W;
    const unsigned long long first = (unsigned long long)head + (unsigned long long)gtid * kPix;
    unsigned py = (unsigned)(first / uW), px = (unsigned)(first - (unsigned long long)py * uW);
    const unsigned long long step_bytes = (unsigned long long)stride * kPix;
    const unsigned dpy = (unsigned)(step_bytes / uW), dpx = (unsigned)(step_bytes - (unsigned long long)dpy * uW);
    const uint4 zz = make_uint4(zword, zword, zword, zword);
    const long long last_full = (plane - head) / kPix;  // chunks [0, last_full) lie completely inside the plane
    uint8_t* __restrict__ dst = obase + first;
    for (long long chunk = gtid; chunk < last_full; chunk += stride, dst += step_bytes) {
      bool active = false;
      if (!empty) {
        const int ipy = (int)py, ipx = (int)px, pxe = ipx + kPix - 1;
        if (pxe < W) {
          active = (ipy >= ry0 && ipy <= ry1 && pxe >= cx0 && ipx <= cx1);
        } else {  // chunk wraps into the next row
          active = (ipy >= ry0 && ipy <= ry1 && ipx <= cx1) || (ipy + 1 >= ry0 && ipy + 1 <= ry1 && pxe - W >= cx0);
        }
      }
      if (!active) *reinterpret_cast<uint4*>(dst) = zz;
      px += dpx;
      py += dpy;
      if (px >= uW) {
        px -= uW;
        ++py;
      }
    }
  }
  // ---- phase 2a (TAB): coordinate tables, then one warp per rectangle row, 4 pixels per lane
  if (TAB && !empty) {
    extern __shared__ float tabs[];
    float* __restrict__ ixs = tabs;      // [W]            sample x of every column
    float* __restrict__ iys = tabs + W;  // [nrows + 2]    sample y of rows ry0-1 .. ry1+1 (a widened range may wrap a row)
    const int rbase = ry0 - 1;
    const int nrows = ry1 - ry0 + 1;
    // columns a widened row range can touch: the rectangle +- 15, plus the far edge when the range wraps into a neighbour row
    const int c_lo = max(cx0 - (kPix - 1), 0), c_hi = min(cx1 + (kPix - 1), W - 1);
    for (int i = c_lo + threadIdx.x; i <= c_hi; i += kThreads) ixs[i] = sample_coord((float)i, x0, x1, fM);
    if (threadIdx.x < 2 * kPix) {
      const int i = threadIdx.x < kPix ? threadIdx.x : W - 2 * kPix + threadIdx.x;  // [0,16) and [W-16,W)
      ixs[i] = sample_coord((float)i, x0, x1, fM);
    }
    for (int i = threadIdx.x; i < nrows + 2; i += kThreads) iys[i] = sample_coord((float)(rbase + i), y0, y1, fM);
    __syncthreads();
    const int body_end = head + (int)((plane - head) / kPix) * kPix;  // bytes past it belong to phase 2b
    const int lane = threadIdx.x & 31;
    const int warps = cta_count * (kThreads / 32);
    for (int dr = cta_local * (kThreads / 32) + (threadIdx.x >> 5); dr < nrows; dr += warps) {
      const int r = ry0 + dr;
      const int lo = r * W + cx0, hi = r * W + cx1;  // inclusive flat range of this row
      const int A = lo < head ? head : ((lo - head) & ~(kPix - 1)) + head;
      int B = hi < head ? head : (((hi - head) >> 4) + 1) * kPix + head;
      if (B > body_end) B = body_end;
      for (int b4 = A + 4 * lane; b4 < B; b4 += 128) {  // (obase + A) is 16-byte aligned, B - A a multiple of 16
        uint32_t word = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          int py = r, px = b4 + q - r * W;
          if (px < 0) {
            px += W;
            --py;
          } else if (px >= W) {
            px -= W;
            ++py;
          }
          word |= paste_value(smask, M, fM, ixs[px], iys[py - rbase], threshold) << (8 * q);
        }
        *reinterpret_cast<uint32_t*>(obase + b4) = word;
      }
    }
  }
  // ---- phase 2a (!TAB): the rectangle, row by row, widened to chunk boundaries (one pixel per lane).  32-bit index math;
  //      the byte -> (py, px) mapping needs no division because a widened range spills at most 15 bytes into a neighbour row.
  if (!TAB && !empty) {
    const int RL = (cx1 - cx0 + 1) + 2 * (kPix - 1) + 1;
    const int nrows = ry1 - ry0 + 1;
    const int iplane = (int)plane;  // H*W < 2^31 (checked on the host)
    const unsigned items = (unsigned)nrows * (unsigned)RL;
    for (unsigned it = (unsigned)gtid; it < items; it += (unsigned)stride) {
      const int dr = (int)(it / (unsigned)RL);
      const int t = (int)(it - (unsigned)dr * (unsigned)RL);
      const int r = ry0 + dr;
      const int lo = r * W + cx0, hi = r * W + cx1;  // inclusive flat range of this row
      const int A = lo < head ? 0 : ((lo - head) & ~(kPix - 1)) + head;
      int B = hi < head ? head : (((hi - head) >> 4) + 1) * kPix + head;
      if (B > iplane) B = iplane;
      const int byte = A + t;
      if (byte >= B) continue;
      int py = r, px = byte - r * W;
      while (px < 0) {  // a widened range spills at most 15 bytes: one wrap unless the image is narrower than a chunk
        px += W;
        --py;
      }
      while (px >= W) {
        px -= W;
        ++py;
      }
      obase[byte] = (uint8_t)paste_pixel(smask, M, fM, px, py, x0, y0, x1, y1, threshold);
    }
  }
  // ---- phase 2b: unaligned head and ragged tail bytes (< 32 bytes per mask)
  if (cta_local == 0) {
    const long long tail0 = head + (long long)((plane - head) / kPix) * kPix;
    for (long long byte = threadIdx.x; byte < head && byte < plane; byte += kThreads) {
      const int py = (int)(byte / W), px = (int)(byte - (long long)py * W);
      obase[byte] = (uint8_t)paste_pixel(smask, M, fM, px, py, x0, y0, x1, y1, threshold);
    }
    for (long long byte = tail0 + threadIdx.x; byte < plane; byte += kThreads) {
      if (byte < 0) continue;
      const int py = (int)(byte / W), px = (int)(byte - (long long)py * W);
      obase[byte] = (uint8_t)paste_pixel(smask, M, fM, px, py, x0, y0, x1, y1, threshold);
    }
  }
}

// Bit-packed boolean output: one thread per 32-bit word = 32 pixels of a row (bit b of word w of row y = pixel (y, 32 w + b)),
// rows padded to whole words.  Same rectangle shortcut, same sample_coord / paste_value expressions as the byte kernel, so the
// unpacked result is identical; 13 MB instead of 107 MB for 100 masks on an 800 x 1333 image -- what matters when the masks
// leave the device (the inference post-processing's D2H copy, mask_ops.py:144-147 / postprocessing.py:61-66).
__global__ void __launch_bounds__(kThreads) paste_masks_packed_kernel(const float* __restrict__ masks,
                                                                      const float* __restrict__ boxes, int M, int H, int W,
                                                                      int Ww, float threshold, uint32_t* __restrict__ out) {
  __shared__ float smask[kMaxM * kMaxM];
  const int n = blockIdx.y;
  const float* __restrict__ mk = masks + (size_t)n * M * M;
  for (int i = threadIdx.x; i < M * M; i += kThreads) smask[i] = mk[i];
  const float x0 = boxes[4 * n], y0 = boxes[4 * n + 1], x1 = boxes[4 * n + 2], y1 = boxes[4 * n + 3];
  __syncthreads();
  const float fM = (float)M;
  const PasteRect rect = paste_rect(x0, y0, x1, y1, fM, H, W);
  const bool empty = rect.cx1 < rect.cx0 || rect.ry1 < rect.ry0;
  const uint32_t zbit = (0.f >= threshold) ? 1u : 0u;  // value of a pixel that cannot see the mask
  const long long words = (long long)H * Ww;
  uint32_t* __restrict__ obase = out + (size_t)n * words;
  for (long long idx = (long long)blockIdx.x * kThreads + threadIdx.x; idx < words; idx += (long long)gridDim.x * kThreads) {
    const int y = (int)(idx / Ww), w = (int)(idx - (long long)y * Ww);
    const int px0 = 32 * w;
    const int nvalid = min(32, W - px0);
    const uint32_t valid = nvalid == 32 ? 0xffffffffu : ((1u << nvalid) - 1u);
    uint32_t word;
    if (empty || y < rect.ry0 || y > rect.ry1 || px0 + 31 < rect.cx0 || px0 > rect.cx1) {
      word = zbit ? valid : 0u;
    } else {
      const float iy = sample_coord((float)y, y0, y1, fM);
      word = 0u;
      for (int b = 0; b < nvalid; ++b)
        word |= paste_value(smask, M, fM, sample_coord((float)(px0 + b), x0, x1, fM), iy, threshold) << b;
    }
    obase[idx] = word;
  }
}

}  // namespace

D2B_API int d2b_paste_masks_packed(const float* masks, const float* boxes, int N, int M, int H, int W, float threshold,
                                   uint32_t* out, void* stream) {
  if (N == 0 || H == 0 || W == 0) return D2B_OK;
  if (!masks || !boxes || !out || N < 0 || M <= 0 || H < 0 || W < 0 || !(threshold >= 0.f)) return D2B_EINVAL;
  if (M > kMaxM) return D2B_EUNSUPPORTED;
  const int Ww = d2b_cdiv(W, 32);
  const long long words = (long long)H * Ww;
  if ((long long)H * W >= (1LL << 30)) return D2B_EUNSUPPORTED;
  int gx = (int)std::min<long long>(d2b_cdiv(words, kThreads), std::max<long long>(1, d2b_cdiv(16LL * d2b_num_sms(), N)));
  for (int s = 0; s < N; s += kMaxGridY) {  // grid.y holds at most 65535 masks: one launch per slice
    const int n = std::min(kMaxGridY, N - s);
    paste_masks_packed_kernel<<<dim3(gx, n), kThreads, 0, (cudaStream_t)stream>>>(
        masks + (size_t)s * M * M, boxes + 4 * (size_t)s, M, H, W, Ww, threshold, out + (size_t)s * words);
    D2B_CHECK_LAUNCH();
  }
  return D2B_OK;
}

D2B_API int d2b_paste_masks(const float* masks, const float* boxes, int N, int M, int H, int W, float threshold,
                            uint8_t* out, void* stream) {
  if (N == 0 || H == 0 || W == 0) return D2B_OK;
  if (!masks || !boxes || !out || N < 0 || M <= 0 || H < 0 || W < 0) return D2B_EINVAL;
  if (M > kMaxM) return D2B_EUNSUPPORTED;
  long long plane = (long long)H * W;
  if (plane >= (1LL << 30)) return D2B_EUNSUPPORTED;  // 32-bit pixel indices inside one mask plane
  int chunks = (int)((plane + kPix - 1) / kPix);  // upper bound; chunks past the plane are skipped in-kernel
  const size_t tab_bytes = sizeof(float) * ((size_t)W + (size_t)H + 2);
  const bool tab = W >= 2 * kPix && tab_bytes <= 30 * 1024;  // 16 KB static mask + tables inside the default 48 KB; one-wrap rows
  const int total = 8 * d2b_num_sms();
  if (2 * N <= total) {  // balanced: CTAs handed to the masks in proportion to their work (decided in-kernel from the boxes)
    if (tab) paste_masks_kernel<true><<<total, kThreads, tab_bytes, (cudaStream_t)stream>>>(masks, boxes, M, H, W, threshold, out, N, 1);
    else paste_masks_kernel<false><<<total, kThreads, 0, (cudaStream_t)stream>>>(masks, boxes, M, H, W, threshold, out, N, 1);
  } else {  // many masks: a fixed, small number of CTAs each
    int gx = d2b_cdiv(chunks + 1, kThreads);
    int want = d2b_cdiv(8LL * d2b_num_sms(), N);
    if (gx > want) gx = want < 1 ? 1 : want;
    for (int s = 0; s < N; s += kMaxGridY) {  // grid.y holds at most 65535 masks: one launch per slice
      const int n = std::min(kMaxGridY, N - s);
      const float* mk = masks + (size_t)s * M * M;
      const float* bx = boxes + 4 * (size_t)s;
      uint8_t* o = out + (size_t)s * plane;
      if (tab) paste_masks_kernel<true><<<dim3(gx, n), kThreads, tab_bytes, (cudaStream_t)stream>>>(mk, bx, M, H, W, threshold, o, n, 0);
      else paste_masks_kernel<false><<<dim3(gx, n), kThreads, 0, (cudaStream_t)stream>>>(mk, bx, M, H, W, threshold, o, n, 0);
      D2B_CHECK_LAUNCH();
    }
    return D2B_OK;
  }
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
