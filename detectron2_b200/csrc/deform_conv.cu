// Deformable convolution v1/v2 (DeformConv / ModulatedDeformConv) for sm_90a -- fp32 parity path.
//
// Replaces detectron2/layers/csrc/deformable/{deform_conv_cuda.cu, deform_conv_cuda_kernel.cu}.  The reference
// materialises `columns[Cin*kh*kw, N*Ho*Wo]` in HBM (offset-im2col), then runs per-group addmm_ on it, and its backward
// materialises grad_columns and re-runs im2col (deform_conv_cuda.cu:382-431,549-619,756-812).  Here the gathered
// column tile never leaves the SM: every kernel is an implicit GEMM whose B (or A) operand tile is produced by the
// bilinear gather straight into shared memory.
//
//   forward      out[b, g*opg+m, p]  = sum_{c,kp} W[g*opg+m, c, kp] * col(b, c, kp, p)  (+ bias)
//   bwd data     gcol(b,c,kp,p)      = sum_m W[g*opg+m, c, kp] * gout[b, g*opg+m, p]     -> scattered at once into
//                grad_x (atomics), grad_offset, grad_mask; gcol is never stored
//   bwd weight   gW[g*opg+m, c, kp]  = sum_{b,p} gout[b, g*opg+m, p] * col(b, c, kp, p)  (split over pixel ranges)
//
// Sampling taps (4 positions + 4 weights [+ derivative terms]) depend only on (b, deformable group, kernel point,
// pixel): they are computed once per CTA tile into shared memory and reused by every channel, where the reference
// recomputes them per channel (deform_conv_cuda_kernel.cu:238-287).
//
// The wgmma (bf16 / bf16x3) forward and backward live in deform_conv_tc.cu; this file is the fp32 FFMA path used for
// parity (<= 1e-4 rel) and for shapes the tensor-core kernels do not take, plus the public entry points that pick one.
#include "common.cuh"
#include "deform_conv_tc.cuh"

namespace {

constexpr int BN = 64;  // pixels per tile
constexpr int BM = 64;  // output channels per tile
constexpr int BK = 16;  // input channels per k-step
constexpr int kThreads = 256;

struct Dims {
  int N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, G, DG, Ho, Wo;
  int cpg, opg, cpdg, KK, HoWo;
};

inline bool make_dims(const d2b_dcn_params* p, Dims& d) {
  if (!p) return false;
  d.N = p->N; d.Cin = p->Cin; d.H = p->H; d.W = p->W; d.Cout = p->Cout; d.kh = p->kh; d.kw = p->kw;
  d.sh = p->stride_h; d.sw = p->stride_w; d.ph = p->pad_h; d.pw = p->pad_w; d.dh = p->dil_h; d.dw = p->dil_w;
  d.G = p->groups; d.DG = p->deformable_groups;
  if (d.N < 0 || d.Cin <= 0 || d.H <= 0 || d.W <= 0 || d.Cout <= 0 || d.kh <= 0 || d.kw <= 0 || d.sh <= 0 ||
      d.sw <= 0 || d.ph < 0 || d.pw < 0 || d.dh <= 0 || d.dw <= 0 || d.G <= 0 || d.DG <= 0)
    return false;
  if (d.Cin % d.G || d.Cout % d.G || d.Cin % d.DG) return false;
  d.Ho = (d.H + 2 * d.ph - (d.dh * (d.kh - 1) + 1)) / d.sh + 1;
  d.Wo = (d.W + 2 * d.pw - (d.dw * (d.kw - 1) + 1)) / d.sw + 1;
  if (d.Ho <= 0 || d.Wo <= 0) return false;
  d.cpg = d.Cin / d.G; d.opg = d.Cout / d.G; d.cpdg = d.Cin / d.DG; d.KK = d.kh * d.kw; d.HoWo = d.Ho * d.Wo;
  return true;
}

// taps of BN pixels for one (b, dg, kp): position (or -1) and weight of the four corners, mask value,
// and (backward only) the sampling coordinates.
struct TapTile {
  int pos[4][BN];
  float wgt[4][BN];  // bilinear weights (NOT multiplied by the mask)
  float msk[BN];
  float fh[BN], fw[BN];  // fractional parts lh, lw   (backward)
  int inside[BN];        // sample inside (-1,H)x(-1,W)
};

// deform_conv_cuda_kernel.cu:263-282 (+ :96-130 bilinear with zero padding)
__device__ __forceinline__ void build_taps(TapTile& t, const Dims& d, const float* __restrict__ offset,
                                           const float* __restrict__ mask, int b, int dg, int kp, int p0) {
  for (int n = threadIdx.x; n < BN; n += kThreads) {
    const int p = p0 + n;
    int pos[4] = {-1, -1, -1, -1};
    float w[4] = {0.f, 0.f, 0.f, 0.f};
    float m = 1.f, lh = 0.f, lw = 0.f;
    int inside = 0;
    if (p < d.HoWo) {
      const int ho = p / d.Wo, wo = p - ho * d.Wo;
      const int i = kp / d.kw, j = kp - i * d.kw;
      const size_t obase = ((size_t)(b * d.DG + dg) * 2 * d.KK) * d.HoWo;
      const float oh = offset[obase + (size_t)(2 * kp) * d.HoWo + p];
      const float ow = offset[obase + (size_t)(2 * kp + 1) * d.HoWo + p];
      const float h = (float)(ho * d.sh - d.ph + i * d.dh) + oh;
      const float wv = (float)(wo * d.sw - d.pw + j * d.dw) + ow;
      if (mask) m = mask[((size_t)(b * d.DG + dg) * d.KK + kp) * d.HoWo + p];
      if (h > -1.f && wv > -1.f && h < (float)d.H && wv < (float)d.W) {
        inside = 1;
        const int hl = (int)floorf(h), wl = (int)floorf(wv);
        lh = h - (float)hl;
        lw = wv - (float)wl;
        const float hh = 1.f - lh, hw = 1.f - lw;
        const bool t0 = hl >= 0, t1 = hl + 1 <= d.H - 1, l0 = wl >= 0, l1 = wl + 1 <= d.W - 1;
        if (t0 && l0) { pos[0] = hl * d.W + wl; w[0] = hh * hw; }
        if (t0 && l1) { pos[1] = hl * d.W + wl + 1; w[1] = hh * lw; }
        if (t1 && l0) { pos[2] = (hl + 1) * d.W + wl; w[2] = lh * hw; }
        if (t1 && l1) { pos[3] = (hl + 1) * d.W + wl + 1; w[3] = lh * lw; }
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      t.pos[q][n] = pos[q];
      t.wgt[q][n] = w[q];
    }
    t.msk[n] = m;
    t.fh[n] = lh;
    t.fw[n] = lw;
    t.inside[n] = inside;
  }
}

__device__ __forceinline__ float gather_val(const TapTile& t, const float* __restrict__ plane, int n) {
  float v = 0.f;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    const int pos = t.pos[q][n];
    if (pos >= 0) v += t.wgt[q][n] * __ldg(plane + pos);
  }
  return v;
}

// ------------------------------------------------------------------------------------------------ forward
// grid (pixel tiles, oc tiles, N*G).  256 threads: (ty, tx) = (tid/16, tid%16), each a 4x4 register tile.
__global__ void __launch_bounds__(kThreads) dcn_fwd_kernel(const float* __restrict__ x,
                                                           const float* __restrict__ offset,
                                                           const float* __restrict__ mask,
                                                           const float* __restrict__ weight,
                                                           const float* __restrict__ bias, Dims d,
                                                           float* __restrict__ out) {
  __shared__ TapTile taps;
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  const int p0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
  const int b = blockIdx.z / d.G, g = blockIdx.z - b * d.G;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int K = d.cpg * d.KK;
  float acc[4][4] = {};
  const int cbeg = g * d.cpg, cend = cbeg + d.cpg;
  for (int dg = cbeg / d.cpdg; dg * d.cpdg < cend; ++dg) {
    const int sbeg = max(cbeg, dg * d.cpdg), send = min(cend, (dg + 1) * d.cpdg);
    for (int kp = 0; kp < d.KK; ++kp) {
      __syncthreads();
      build_taps(taps, d, offset, mask, b, dg, kp, p0);
      __syncthreads();
      for (int c0 = sbeg; c0 < send; c0 += BK) {
        // A tile: W[g*opg + m0+m][(c - cbeg)*KK + kp]
        for (int e = tid; e < BK * BM; e += kThreads) {
          const int kk = e / BM, m = e - kk * BM;
          const int c = c0 + kk;
          float v = 0.f;
          if (c < send && m0 + m < d.opg) v = __ldg(weight + (size_t)(g * d.opg + m0 + m) * K + (c - cbeg) * d.KK + kp);
          As[kk][m] = v;
        }
        // B tile: gathered column values (x mask)
        for (int e = tid; e < BK * BN; e += kThreads) {
          const int kk = e / BN, n = e - kk * BN;
          const int c = c0 + kk;
          float v = 0.f;
          if (c < send) v = gather_val(taps, x + ((size_t)b * d.Cin + c) * d.H * d.W, n) * taps.msk[n];
          Bs[kk][n] = v;
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
          float a[4], bb[4];
#pragma unroll
          for (int i = 0; i < 4; ++i) a[i] = As[kk][ty * 4 + i];
#pragma unroll
          for (int j = 0; j < 4; ++j) bb[j] = Bs[kk][tx * 4 + j];
#pragma unroll
          for (int i = 0; i < 4; ++i)
#pragma unroll
            for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
        }
        __syncthreads();
      }
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= d.opg) continue;
    const int oc = g * d.opg + m;
    const float bv = bias ? bias[oc] : 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int p = p0 + tx * 4 + j;
      if (p < d.HoWo) out[((size_t)b * d.Cout + oc) * d.HoWo + p] = acc[i][j] + bv;
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward: data
// grid (pixel tiles, channel-chunk splits, N*G).  For every (dg segment, kp, 16-channel chunk): gcol[16 x 64] = W^T . gout, then the
// scatter epilogue.  Thread mapping in the epilogue: n = tid % 64 (pixel), kk = tid / 64 + 4*i (channel).
__global__ void __launch_bounds__(kThreads) dcn_bwd_data_kernel(const float* __restrict__ x,
                                                                const float* __restrict__ offset,
                                                                const float* __restrict__ mask,
                                                                const float* __restrict__ weight,
                                                                const float* __restrict__ gout, Dims d,
                                                                float* __restrict__ gx, float* __restrict__ goff,
                                                                float* __restrict__ gmask) {
  __shared__ TapTile taps;
  __shared__ float Ws[BK][BK + 1];   // [m chunk][channel]
  __shared__ float Gs[BK][BN + 4];   // [m chunk][pixel]
  __shared__ float red[3][4][BN];    // cross-thread reduction of (goff_h, goff_w, gmask)
  const int p0 = blockIdx.x * BN;
  const int b = blockIdx.z / d.G, g = blockIdx.z - b * d.G;
  const int tid = threadIdx.x, n = tid & 63, kq = tid >> 6;
  const int K = d.cpg * d.KK;
  const int cbeg = g * d.cpg, cend = cbeg + d.cpg;
  const size_t plane = (size_t)d.H * d.W;
  for (int dg = cbeg / d.cpdg; dg * d.cpdg < cend; ++dg) {
    const int sbeg = max(cbeg, dg * d.cpdg), send = min(cend, (dg + 1) * d.cpdg);
    for (int kp = 0; kp < d.KK; ++kp) {
      __syncthreads();
      build_taps(taps, d, offset, mask, b, dg, kp, p0);
      __syncthreads();
      float s_h = 0.f, s_w = 0.f, s_m = 0.f;
      for (int c0 = sbeg + (int)blockIdx.y * BK; c0 < send; c0 += BK * (int)gridDim.y) {  // channel chunks are split over blockIdx.y
        float acc[4] = {0.f, 0.f, 0.f, 0.f};  // gcol for channels kq + 4*i, pixel n
        for (int mm0 = 0; mm0 < d.opg; mm0 += BK) {
          {  // Ws[m][c] : 16 x 16
            const int m = tid >> 4, kk = tid & 15;
            const int c = c0 + kk;
            float v = 0.f;
            if (c < send && mm0 + m < d.opg)
              v = __ldg(weight + (size_t)(g * d.opg + mm0 + m) * K + (c - cbeg) * d.KK + kp);
            Ws[m][kk] = v;
          }
          for (int e = tid; e < BK * BN; e += kThreads) {  // Gs[m][pixel]
            const int m = e / BN, nn = e - m * BN;
            float v = 0.f;
            if (mm0 + m < d.opg && p0 + nn < d.HoWo)
              v = __ldg(gout + ((size_t)b * d.Cout + g * d.opg + mm0 + m) * d.HoWo + p0 + nn);
            Gs[m][nn] = v;
          }
          __syncthreads();
#pragma unroll
          for (int m = 0; m < BK; ++m) {
            const float gv = Gs[m][n];
#pragma unroll
            for (int i = 0; i < 4; ++i) acc[i] = fmaf(Ws[m][kq + 4 * i], gv, acc[i]);
          }
          __syncthreads();
        }
        // scatter epilogue (deform_conv_cuda_kernel.cu:313-362 col2im, :390-451 col2im_coord, :1031-1064 mask)
        if (taps.inside[n]) {
          const float mk = taps.msk[n], lh = taps.fh[n], lw = taps.fw[n];
          const int q0 = taps.pos[0][n], q1 = taps.pos[1][n], q2 = taps.pos[2][n], q3 = taps.pos[3][n];
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const int c = c0 + kq + 4 * i;
            if (c >= send) continue;
            const float gc = acc[i];
            const float gm = gc * mk;
            const float* __restrict__ xp = x + ((size_t)b * d.Cin + c) * plane;
            float* __restrict__ gp = gx ? gx + ((size_t)b * d.Cin + c) * plane : nullptr;
            const float v0 = q0 >= 0 ? __ldg(xp + q0) : 0.f, v1 = q1 >= 0 ? __ldg(xp + q1) : 0.f;
            const float v2 = q2 >= 0 ? __ldg(xp + q2) : 0.f, v3 = q3 >= 0 ? __ldg(xp + q3) : 0.f;
            if (gp) {
              if (q0 >= 0) atomicAdd(gp + q0, gm * taps.wgt[0][n]);
              if (q1 >= 0) atomicAdd(gp + q1, gm * taps.wgt[1][n]);
              if (q2 >= 0) atomicAdd(gp + q2, gm * taps.wgt[2][n]);
              if (q3 >= 0) atomicAdd(gp + q3, gm * taps.wgt[3][n]);
            }
            // d val / d h = -(1-lw) v0 - lw v1 + (1-lw) v2 + lw v3 ;  d val / d w = -(1-lh) v0 + (1-lh) v1 - lh v2 + lh v3
            s_h += gm * ((1.f - lw) * (v2 - v0) + lw * (v3 - v1));
            s_w += gm * ((1.f - lh) * (v1 - v0) + lh * (v3 - v2));
            s_m += gc * (taps.wgt[0][n] * v0 + taps.wgt[1][n] * v1 + taps.wgt[2][n] * v2 + taps.wgt[3][n] * v3);
          }
        }
      }
      // reduce the 4 channel-quarter threads of each pixel, one atomic per (kp, pixel)
      red[0][kq][n] = s_h;
      red[1][kq][n] = s_w;
      red[2][kq][n] = s_m;
      __syncthreads();
      if (tid < 3 * BN) {
        const int which = tid / BN, nn = tid - which * BN;
        const int p = p0 + nn;
        if (p < d.HoWo) {
          const float v = red[which][0][nn] + red[which][1][nn] + red[which][2][nn] + red[which][3][nn];
          if (which < 2) {
            if (goff) atomicAdd(goff + ((size_t)(b * d.DG + dg) * 2 * d.KK + 2 * kp + which) * d.HoWo + p, v);
          } else if (gmask && mask) {
            atomicAdd(gmask + ((size_t)(b * d.DG + dg) * d.KK + kp) * d.HoWo + p, v);
          }
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ backward: weight
// grid (pixel-range splits, oc tiles (BM) x channel tiles (BK), N*G is folded into the pixel loop: blockIdx.z = g).
// acc[m 64][c 16] per kp, reduction over this CTA's (b, pixel) range, flushed with atomics.
__global__ void __launch_bounds__(kThreads) dcn_bwd_weight_kernel(const float* __restrict__ x,
                                                                  const float* __restrict__ offset,
                                                                  const float* __restrict__ mask,
                                                                  const float* __restrict__ gout, Dims d,
                                                                  int tiles_per_cta, int n_ctile,
                                                                  float* __restrict__ gw) {
  __shared__ TapTile taps;
  __shared__ float Gs[BN][BM + 4];  // [pixel][m]
  __shared__ float Cs[BN][BK + 1];  // [pixel][channel]
  const int g = blockIdx.z;
  const int mt = blockIdx.y / n_ctile, ct = blockIdx.y - mt * n_ctile;
  const int m0 = mt * BM;
  const int cbeg = g * d.cpg;
  const int c0 = cbeg + ct * BK;
  const int cend = min(cbeg + d.cpg, c0 + BK);
  const int tid = threadIdx.x, tm = tid >> 2, tc = tid & 3;  // m = tm, channels tc*4 .. tc*4+3
  const int K = d.cpg * d.KK;
  const int ptiles = d2b_cdiv(d.HoWo, BN);
  const int total_tiles = d.N * ptiles;
  const int t_begin = blockIdx.x * tiles_per_cta, t_end = min(total_tiles, t_begin + tiles_per_cta);
  // a 16-channel tile may straddle deformable groups only if cpdg < 16; handle by per-channel dg lookup of the FIRST
  // channel and splitting at the boundary.
  for (int kp = 0; kp < d.KK; ++kp) {
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    for (int t = t_begin; t < t_end; ++t) {
      const int b = t / ptiles, p0 = (t - b * ptiles) * BN;
      for (int cs = c0; cs < cend;) {
        const int dg = cs / d.cpdg;
        const int ce = min(cend, (dg + 1) * d.cpdg);
        __syncthreads();
        build_taps(taps, d, offset, mask, b, dg, kp, p0);
        for (int e = tid; e < BN * BM; e += kThreads) {
          const int nn = e & 63, m = e >> 6;  // pixel fastest -> coalesced gout reads
          float v = 0.f;
          if (m0 + m < d.opg && p0 + nn < d.HoWo)
            v = __ldg(gout + ((size_t)b * d.Cout + g * d.opg + m0 + m) * d.HoWo + p0 + nn);
          Gs[nn][m] = v;
        }
        __syncthreads();
        for (int e = tid; e < BN * BK; e += kThreads) {
          const int nn = e & 63, kk = e >> 6;
          const int c = c0 + kk;
          float v = 0.f;
          if (c >= cs && c < ce) v = gather_val(taps, x + ((size_t)b * d.Cin + c) * d.H * d.W, nn) * taps.msk[nn];
          Cs[nn][kk] = v;
        }
        __syncthreads();
#pragma unroll 8
        for (int nn = 0; nn < BN; ++nn) {
          const float gv = Gs[nn][tm];
#pragma unroll
          for (int i = 0; i < 4; ++i) acc[i] = fmaf(gv, Cs[nn][tc * 4 + i], acc[i]);
        }
        cs = ce;
      }
    }
    if (m0 + tm < d.opg) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const int c = c0 + tc * 4 + i;
        if (c < cend) atomicAdd(gw + (size_t)(g * d.opg + m0 + tm) * K + (c - cbeg) * d.KK + kp, acc[i]);
      }
    }
  }
}

// grad_bias[oc] = sum_{b,p} gout[b,oc,p]   (deform_conv_cuda.cu:1197-1203)
__global__ void __launch_bounds__(256) dcn_bias_grad_kernel(const float* __restrict__ gout, int N, int Cout, int HoWo,
                                                            float* __restrict__ gb) {
  __shared__ float s[8];
  const int oc = blockIdx.x;
  float v = 0.f;
  for (int b = 0; b < N; ++b)
    for (int p = threadIdx.x; p < HoWo; p += 256) v += gout[((size_t)b * Cout + oc) * HoWo + p];
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += s[i];
    gb[oc] = t;
  }
}

// precision: 0 = fp32 FFMA, 1 = bf16x3 on wgmma, 2 = bf16 on wgmma, -1 = auto.  Auto is 1 when the tensor-core kernels take
// the shape in every direction `dirs` names, else 0 -- both are fp32-class, so "auto" never lowers accuracy.  The fused ops
// have no FFMA path and name no direction: their auto is 1.  Saved columns are written by the forward and read by the
// backward, so they name both.  Other values are returned as they are; the calls reject those outside [-1, 2].
enum { kFused = 0, kFwd = 1, kBwd = 2 };
int dcn_precision(const d2b_dcn_params* p, int precision, int dirs) {
  if (precision != -1) return precision;
  const bool fwd = !(dirs & kFwd) || d2b_deform_conv_tc_shape_supported(p, 0);
  const bool bwd = !(dirs & kBwd) || d2b_deform_conv_tc_shape_supported(p, 1);
  return fwd && bwd ? 1 : 0;
}

}  // namespace

D2B_API size_t d2b_deform_conv_forward_workspace_bytes(const d2b_dcn_params* p, int precision, int flags) {
  precision = dcn_precision(p, precision, kFwd);
  return precision ? d2b_deform_conv_tc_fwd_workspace(p, precision, (flags & D2B_DCN_X_NHWC) ? 1 : 0) : 0;
}

// Saved columns (training): the tensor-core forward can keep the sampled columns it builds -- bf16 hi [| lo] tiles in the
// tensor core's operand layout -- and the backward's weight-gradient kernel then streams them back instead of sampling x a
// second time.  0 when the shape / precision has no tensor-core path (pass cols = NULL then).
D2B_API size_t d2b_deform_conv_cols_bytes(const d2b_dcn_params* p, int precision) {
  precision = dcn_precision(p, precision, kFwd | kBwd);
  return precision ? d2b_deform_conv_tc_cols_bytes(p, precision) : 0;
}

D2B_API int d2b_deform_conv_forward(const float* x, const float* offset, const float* mask, const float* weight,
                                    const float* bias, const d2b_dcn_params* p, int precision, int flags, float* out,
                                    void* cols, void* workspace, size_t workspace_bytes, void* stream) {
  Dims d;
  if (!make_dims(p, d)) return D2B_EINVAL;
  if (d.N == 0) return D2B_OK;
  if (!x || !offset || !weight || !out) return D2B_EINVAL;
  if (precision < -1 || precision > 2) return D2B_EINVAL;
  precision = dcn_precision(p, precision, kFwd);
  if (precision != 0)  // no silent precision / path change: an unsupported shape is reported, not rerouted
    return d2b_deform_conv_forward_tc(x, offset, mask, weight, nullptr, bias, 0, p, precision,
                                      (flags & D2B_DCN_X_NHWC) ? 1 : 0, out, cols, workspace, workspace_bytes, stream);
  if (flags & D2B_DCN_X_NHWC) return D2B_EUNSUPPORTED;  // the FFMA parity path reads NCHW planes
  if (cols) return D2B_EINVAL;                          // ... and never materialises columns
  dim3 grid(d2b_cdiv(d.HoWo, BN), d2b_cdiv(d.opg, BM), d.N * d.G);
  dcn_fwd_kernel<<<grid, kThreads, 0, (cudaStream_t)stream>>>(x, offset, mask, weight, bias, d, out);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

D2B_API size_t d2b_deform_conv_backward_workspace_bytes(const d2b_dcn_params* p, int precision, int flags, int need_data,
                                                        int need_weight) {
  precision = dcn_precision(p, precision, kBwd);  // the FFMA path (0) never materialises grad_columns
  return precision ? d2b_deform_conv_tc_bwd_workspace(p, precision, (flags & D2B_DCN_X_NHWC) ? 1 : 0, need_data, need_weight)
                   : 0;
}

D2B_API int d2b_deform_conv_backward(const float* x, const float* offset, const float* mask, const float* weight,
                                     const float* grad_out, const d2b_dcn_params* p, int precision, int flags,
                                     const void* cols, float* grad_x, float* grad_offset, float* grad_mask,
                                     float* grad_weight, float* grad_bias, void* workspace, size_t workspace_bytes,
                                     void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  Dims d;
  if (!make_dims(p, d)) return D2B_EINVAL;
  if (precision < -1 || precision > 2) return D2B_EINVAL;
  precision = dcn_precision(p, precision, kBwd);
  if (d.N > 0 && (!x || !offset || !weight || !grad_out)) return D2B_EINVAL;
  if (cols && precision == 0) return D2B_EINVAL;
  if (grad_bias) {
    if (d.N == 0) {
      D2B_CUDA(cudaMemsetAsync(grad_bias, 0, (size_t)d.Cout * 4, stream));
    } else {
      dcn_bias_grad_kernel<<<d.Cout, 256, 0, stream>>>(grad_out, d.N, d.Cout, d.HoWo, grad_bias);
      D2B_CHECK_LAUNCH();
    }
  }
  if (precision != 0)
    return d2b_deform_conv_backward_tc(x, offset, mask, weight, grad_out, nullptr, nullptr, 0, p, precision,
                                       (flags & D2B_DCN_X_NHWC) ? 1 : 0, cols, grad_x, grad_offset, grad_mask, grad_weight,
                                       workspace, workspace_bytes, stream_);
  if (flags & D2B_DCN_X_NHWC) return D2B_EUNSUPPORTED;
  const size_t nx = (size_t)d.N * d.Cin * d.H * d.W, noff = (size_t)d.N * d.DG * 2 * d.KK * d.HoWo;
  const size_t nm = (size_t)d.N * d.DG * d.KK * d.HoWo, nw = (size_t)d.Cout * d.cpg * d.KK;
  if (grad_x && nx) D2B_CUDA(cudaMemsetAsync(grad_x, 0, nx * 4, stream));
  if (grad_offset && noff) D2B_CUDA(cudaMemsetAsync(grad_offset, 0, noff * 4, stream));
  if (grad_mask && nm) D2B_CUDA(cudaMemsetAsync(grad_mask, 0, nm * 4, stream));
  if (grad_weight) D2B_CUDA(cudaMemsetAsync(grad_weight, 0, nw * 4, stream));
  if (d.N == 0) return D2B_OK;
  if (grad_x || grad_offset || grad_mask) {
    // few pixel tiles (small maps) -> split the channel chunks over blockIdx.y so that the grid still fills the SMs;
    // grad_offset / grad_mask partial sums meet through the atomics the kernel already uses
    const int base_ctas = d2b_cdiv(d.HoWo, BN) * d.N * d.G;
    int csplit = d2b_cdiv(3LL * d2b_num_sms(), base_ctas);
    const int nchunks = d2b_cdiv(d.cpg, BK);
    if (csplit > nchunks) csplit = nchunks;
    if (csplit < 1) csplit = 1;
    dim3 grid(d2b_cdiv(d.HoWo, BN), csplit, d.N * d.G);
    dcn_bwd_data_kernel<<<grid, kThreads, 0, stream>>>(x, offset, mask, weight, grad_out, d, grad_x, grad_offset,
                                                       grad_mask);
    D2B_CHECK_LAUNCH();
  }
  if (grad_weight) {
    const int ptiles = d2b_cdiv(d.HoWo, BN), total = d.N * ptiles;
    const int n_ctile = d2b_cdiv(d.cpg, BK), n_mtile = d2b_cdiv(d.opg, BM);
    // split the pixel reduction so that the grid is a few waves of the SMs
    int per_tile_ctas = n_ctile * n_mtile * d.G;
    int splits = d2b_cdiv(4LL * d2b_num_sms(), per_tile_ctas);
    if (splits > total) splits = total;
    if (splits < 1) splits = 1;
    const int tiles_per_cta = d2b_cdiv(total, splits);
    splits = d2b_cdiv(total, tiles_per_cta);
    dim3 grid(splits, n_mtile * n_ctile, d.G);
    dcn_bwd_weight_kernel<<<grid, kThreads, 0, stream>>>(x, offset, mask, grad_out, d, tiles_per_cta, n_ctile,
                                                         grad_weight);
    D2B_CHECK_LAUNCH();
  }
  return D2B_OK;
}

// ---- conv2 of a DeformBottleneckBlock in one pass (SURVEY.md 8f-3; detectron2/modeling/backbone/resnet.py:305-318):
//   offset_mask [N, 3*DG*kh*kw, Ho, Wo] is the raw output of conv2_offset -- the chunk / cat / sigmoid of :307-311 happen
//   while the sampling taps are built;  y = relu(conv * scale + shift) -- FrozenBatchNorm folded to scale / shift, or
//   scale = NULL and shift = bias -- happens in the accumulator epilogue.  Tensor-core precisions only.
D2B_API int d2b_deform_conv_fused_forward(const float* x, const float* offset_mask, const float* weight, const float* scale,
                                          const float* shift, int relu, const d2b_dcn_params* p, int precision, int flags,
                                          float* out, void* cols, void* workspace, size_t workspace_bytes, void* stream) {
  Dims d;
  if (!make_dims(p, d)) return D2B_EINVAL;
  if (d.N == 0) return D2B_OK;
  if (!x || !offset_mask || !weight || !out || precision == 0 || precision < -1 || precision > 2) return D2B_EINVAL;
  precision = dcn_precision(p, precision, kFused);
  return d2b_deform_conv_forward_tc(x, offset_mask, nullptr, weight, scale, shift, relu, p, precision,
                                    ((flags & D2B_DCN_X_NHWC) ? 1 : 0) | 2, out, cols, workspace, workspace_bytes, stream);
}

// grad_out is the gradient of y; y itself (saved by the caller) gates the ReLU.  grad_offset_mask [N, 3*DG*kh*kw, Ho, Wo].
D2B_API int d2b_deform_conv_fused_backward(const float* x, const float* offset_mask, const float* weight, const float* scale,
                                           int relu, const float* y, const float* grad_out, const d2b_dcn_params* p,
                                           int precision, int flags, const void* cols, float* grad_x,
                                           float* grad_offset_mask, float* grad_weight, void* workspace,
                                           size_t workspace_bytes, void* stream) {
  Dims d;
  if (!make_dims(p, d)) return D2B_EINVAL;
  if (precision == 0 || precision < -1 || precision > 2) return D2B_EINVAL;
  precision = dcn_precision(p, precision, kFused);
  if (d.N > 0 && (!x || !offset_mask || !weight || !grad_out)) return D2B_EINVAL;
  return d2b_deform_conv_backward_tc(x, offset_mask, nullptr, weight, grad_out, scale, y, relu, p, precision,
                                     ((flags & D2B_DCN_X_NHWC) ? 1 : 0) | 2, cols, grad_x, grad_offset_mask, nullptr,
                                     grad_weight, workspace, workspace_bytes, stream);
}
