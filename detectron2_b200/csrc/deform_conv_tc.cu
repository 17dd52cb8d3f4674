// Deformable convolution v1/v2 on the Hopper tensor cores (wgmma), sm_90a: forward, backward-data
// and backward-weight.  Replaces detectron2/layers/csrc/deformable/deform_conv_cuda.cu:272-444 (forward),
// :446-642 / :985-1221 (backward input + offset + mask) and :644-824 (backward filter).
//
// The reference materialises columns[Cin*kh*kw, Ho*Wo] in HBM with a gather kernel and calls cuBLAS per group; its
// backward materialises grad_columns, runs col2im / col2im_coord over them and re-runs im2col for the filter gradient.
// Here no column buffer exists: every kernel is an implicit GEMM on wgmma whose gathered operand is produced (or whose
// result is consumed) on the SM, with the operands that are plain matrices pre-tiled once into the wgmma shared-memory
// image (128-byte swizzle) so that ONE linear TMA copy (cp.async.bulk) brings a whole operand tile.
//
//   K1 forward      D[128 px, oc]   = col[128 px, k'] . W[oc, k']^T        A = gather (K-major), B = weight tiles (TMA)
//   K2 bwd data     gcol[128 px,k'] = gout[128 px, oc] . W[oc, k']          A = gout tiles (TMA), B = W^T tiles (TMA);
//                   epilogue: gcol -> red.global.add.v4 into grad_x (NHWC), grad_offset, grad_mask
//   K3 bwd weight   gW[k', oc]      = col^T[k', px] . gout[px, oc]          A = gather (MN-major), B = gout tiles (TMA)
//
// Layout decisions
//   * x is gathered from channels-last storage [N,H,W,C] fp32: the 64 channels of a tap are 256 contiguous bytes, a
//     half-warp reads them as 16 x LDG.128, a warp keeps 8 such loads in flight per lane.  NCHW inputs are re-laid out once
//     per call by nchw_to_nhwc_kernel (roi_align.cu), and their gradient back by nhwc_to_nchw_kernel; channels_last inputs
//     are used in place.
//   * k' is ordered (kernel point, 64-channel block): one "unit" = 64 k' = one 128-byte swizzle row of bf16, so the
//     bilinear taps of a (pixel, kernel point) are computed once (tap table in shared memory) and reused by all channels.
//   * grouped convolutions with fewer than 64 channels per group are packed into "super-groups" of 64 input channels
//     with block-diagonal (zero-padded) weight tiles: the gather stays 256 bytes per tap and the wasted MMA flops are free.
//   * precision 1 ("bf16x3"): operands are split x = hi + lo (two bf16) and hi*hi + hi*lo + lo*hi is accumulated in fp32 --
//     fp32-class accuracy (<= 1e-4 rel) at a third of the bf16 tensor peak.  precision 2: plain bf16 operands.
//
// Warp roles (640 threads, one CTA per SM): warps 0-15 = four warpgroups that gather / scatter, issue the wgmma of their
// quarter of the 128-row tile (rows 64 * (g & 1), columns (g >> 1) * BN / 2 of warpgroup g; fp32 accumulators in registers)
// and run the epilogue; warp 16 TMA producer (one lane), warp 17 the forward's column saver.  The fifth warpgroup drops to
// kSideRegs registers so that the workers get kWorkerRegs (setmaxnreg).
#include <algorithm>
#include <cstdlib>
#include <type_traits>

#include "common.cuh"
#include "deform_conv_tc.cuh"
#include "tc_common.cuh"

using namespace d2b_tc;

namespace {

// 16 worker warps: the gather / scatter loops are bound by instruction issue and need the warps, not deeper queues; four
// warpgroups also give every quarter of the 128-row accumulator tile its own wgmma issuer.
constexpr int kWorkerWarps = 16;
constexpr int kWorkers = kWorkerWarps * 32;  // 512
constexpr int kThreads = kWorkers + 128;     // + producer / saver warpgroup
// setmaxnreg only moves registers inside the CTA's launch allocation: 640 threads launch with 96 registers each
// (64 K / 640 rounded down to a multiple of 8), so the workers' raise must fit in what the side warpgroup gives back.
constexpr int kLaunchRegs = (65536 / kThreads) & ~7;
constexpr int kWorkerRegs = 112, kSideRegs = 24;
static_assert(kWorkers * kWorkerRegs + (kThreads - kWorkers) * kSideRegs <= kThreads * kLaunchRegs,
              "register budget exceeds the launch allocation");
// what the workers leave of the launch allocation: the side warpgroup of the fused backward (dcn_bwd_fused_kernel), whose
// producer lane does not fit the K3c part of it in kSideRegs
constexpr int kSideRegsMax = ((kThreads * kLaunchRegs - kWorkers * kWorkerRegs) / (kThreads - kWorkers)) & ~7;
static_assert(kSideRegsMax >= kSideRegs, "register budget exceeds the launch allocation");
constexpr int kMaxBN = 128;                  // widest output-channel tile: 64 accumulator columns (32 registers) per warpgroup
constexpr int kRowsPerHalf = 128 / (2 * kWorkerWarps);  // pixel rows of a 128-row tile owned by one half-warp: 4
constexpr int kTile = 16384;                 // [128 rows][128 B]
constexpr int kMaxSmem = 227 * 1024;
constexpr int kGcolPitch = 132;              // floats per pixel row of the drained gcol tile (128 + 4: conflict-free float4)

struct TC {
  int N, Cin, H, W, Cout, kh, kw, sh, sw, ph, pw, dh, dw, G, DG, Ho, Wo, cpg, opg, cpdg, KK, HoWo;
  int pack, SG, cps, ops, cbs, U;  // super-groups: cps input / ops output channels each, cbs 64-channel blocks, U units
  int tiles_img;                   // 128-pixel tiles per image
  int stages_img;                  // 64-pixel stages per image (K3)
  int MC;                          // macro-chunks (pairs of units) per super-group
  int nks;                         // 64-wide K stages over the super-group's output channels (K2)
  // offset / mask addressing: element strides between images, element offset of the mask block relative to `mask`
  // pointer (fused layout: offset and mask logits live in ONE [N, 3*DG*KK, Ho, Wo] tensor, backbone/resnet.py:307-312)
  long long off_bs, mask_bs;
  int mask_sigmoid;                // mask values are logits: sigmoid applied while the taps are built
};

// optional epilogue of the forward (and its transpose in the backward): y = relu(acc * scale[oc] + shift[oc]) --
// the FrozenBatchNorm / bias + ReLU that follow conv2 of a DeformBottleneckBlock (backbone/resnet.py:313-318)
struct Epi {
  const float* scale;  // may be null (1)
  const float* shift;  // may be null (0)
  int relu;
};

// noct: output-channel tiles of a super-group; goct: those of them the launch computes (noct, or 1 when the column-fed K1c
// computes the others); uper: units of the reduction per k-split part (the last part may have fewer); red: k-split partial
// sums meet through red.add
struct K1P { int BN, noct, goct, uper, ksplit, S, tap_bytes, stage_bytes, red; };
struct K2P { int mper, msplit, tap_bytes; };
struct K3P { int BN, noct, sper, nsplit, S, stage_bytes; };

inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

bool make_tc(const d2b_dcn_params* p, TC& d) {
  if (!p) return false;
  d.N = p->N; d.Cin = p->Cin; d.H = p->H; d.W = p->W; d.Cout = p->Cout; d.kh = p->kh; d.kw = p->kw;
  d.sh = p->stride_h; d.sw = p->stride_w; d.ph = p->pad_h; d.pw = p->pad_w; d.dh = p->dil_h; d.dw = p->dil_w;
  d.G = p->groups; d.DG = p->deformable_groups;
  if (d.N < 0 || d.Cin <= 0 || d.H <= 0 || d.W <= 0 || d.Cout <= 0 || d.kh <= 0 || d.kw <= 0 || d.sh <= 0 || d.sw <= 0 ||
      d.ph < 0 || d.pw < 0 || d.dh <= 0 || d.dw <= 0 || d.G <= 0 || d.DG <= 0)
    return false;
  if (d.Cin % d.G || d.Cout % d.G || d.Cin % d.DG) return false;
  d.Ho = (d.H + 2 * d.ph - (d.dh * (d.kh - 1) + 1)) / d.sh + 1;
  d.Wo = (d.W + 2 * d.pw - (d.dw * (d.kw - 1) + 1)) / d.sw + 1;
  if (d.Ho <= 0 || d.Wo <= 0) return false;
  d.cpg = d.Cin / d.G; d.opg = d.Cout / d.G; d.cpdg = d.Cin / d.DG; d.KK = d.kh * d.kw; d.HoWo = d.Ho * d.Wo;
  // ---- shapes the tensor-core kernels take
  if (d.cpg >= 64) {
    if (d.cpg % 64) return false;
    d.pack = 1;
  } else {
    if (d.cpg != 16 && d.cpg != 32) return false;
    d.pack = 64 / d.cpg;
    if (d.G % d.pack) return false;
  }
  if (d.cpdg % 64) return false;  // a 64-channel block never straddles deformable groups
  d.SG = d.G / d.pack; d.cps = d.cpg * d.pack; d.ops = d.opg * d.pack; d.cbs = d.cps / 64; d.U = d.KK * d.cbs;
  if (d.ops % 16) return false;
  if (d.KK > 49) return false;
  if ((long long)d.H * d.W * d.Cin >= (1LL << 29)) return false;  // 32-bit byte offsets inside one image
  if ((long long)d.HoWo * d.Cout >= (1LL << 31) || (long long)d.Cout * d.cpg * d.KK >= (1LL << 31)) return false;
  d.tiles_img = d2b_cdiv(d.HoWo, 128);
  d.stages_img = d2b_cdiv(d.HoWo, 64);
  d.MC = (d.U + 1) / 2;
  d.nks = d.ops / 64;
  if ((long long)d.N * d.tiles_img > 0x7fffffffLL) return false;
  d.off_bs = (long long)d.DG * 2 * d.KK * d.HoWo;
  d.mask_bs = (long long)d.DG * d.KK * d.HoWo;
  d.mask_sigmoid = 0;
  return true;
}

// fused offset+mask tensor: returns the mask pointer inside it and switches the strides / sigmoid on
const float* use_fused_offset_mask(TC& d, const float* offset_mask) {
  d.off_bs = d.mask_bs = (long long)d.DG * 3 * d.KK * d.HoWo;
  d.mask_sigmoid = 1;
  return offset_mask + (size_t)d.DG * 2 * d.KK * d.HoWo;
}

int largest_tile(int n) {  // largest of {kMaxBN,...,16} dividing n
  for (int t = kMaxBN; t >= 16; t >>= 1)
    if (n % t == 0) return t;
  return 0;
}

// Split `work` units of a CTA `base` times replicated over up to `max_split` parts: the number of parts that minimises
// (waves over the device's SMs) x (units per CTA + the CTA's fixed prologue / epilogue cost in units).  One CTA per SM is
// resident, so 153 CTAs cost two full waves.
int best_split(long long base, int work, int max_split, int overhead) {
  int best = 1;
  long long best_cost = -1;
  for (int s = 1; s <= max_split; ++s) {
    const int per = d2b_cdiv(work, s);
    const int parts = d2b_cdiv(work, per);
    const long long cost = (long long)d2b_cdiv(base * parts, d2b_num_sms()) * (per + overhead);
    if (best_cost < 0 || cost < best_cost) {
      best_cost = cost;
      best = parts;
    }
  }
  return best;
}

// kernel points whose taps a range of `units` consecutive units may touch, wherever the range starts inside a kernel point
int k1_tap_points(const TC& d, int units) { return std::min(d.KK, (units + d.cbs - 2) / d.cbs + 1); }

// The reduction is split by units, not by whole kernel points, so that the parts can fill the SMs where a kernel point holds
// many channel blocks (res5: 8 units per kernel point).  A CTA's fixed cost (taps, pipeline fill, the red.add epilogue) is
// counted as one kernel point's units.
// colfed: the gathering K1 runs output-channel tile 0 only and K1c the others (plan_k1c)
bool plan_k1(const TC& d, K1P& k, bool colfed = false) {
  k.BN = largest_tile(d.ops);
  if (k.BN < 16) return false;
  k.noct = d.ops / k.BN;
  k.goct = colfed ? 1 : k.noct;
  const int base = d.N * d.tiles_img * d.SG * k.goct;
  k.ksplit = best_split(base, d.U, d.U, d.cbs);
  k.uper = d2b_cdiv(d.U, k.ksplit);
  k.ksplit = d2b_cdiv(d.U, k.uper);
  k.red = k.ksplit > 1;
  const int ndg = d.DG == 1 ? 1 : std::min(d.DG, d2b_cdiv(d.cps, d.cpdg) + 1);
  k.tap_bytes = ndg * k1_tap_points(d, k.uper) * 128 * 16;
  k.stage_bytes = 2 * kTile + 2 * k.BN * 128;
  k.S = 3;
  while (k.S > 1 && k.S * k.stage_bytes + k.tap_bytes + 1024 + 128 > kMaxSmem) --k.S;
  return k.S >= 2;
}

// K1c: output-channel tiles 1..noct-1 of a column-fed forward, split over units on its own grid.  Both launches write the
// same output: if either splits, both add their partials (k1.red and kc.red are set together).
bool plan_k1c(const TC& d, K1P& k1, K1P& kc) {
  const long long base = (long long)d.N * d.tiles_img * d.SG * (k1.noct - 1);
  if (k1.goct != 1 || k1.noct < 2 || (long long)d.N * d.tiles_img * (k1.noct - 1) > 0x7fffffffLL) return false;
  kc = k1;
  kc.goct = k1.noct - 1;
  kc.ksplit = best_split(base, d.U, d.U, d.cbs);
  kc.uper = d2b_cdiv(d.U, kc.ksplit);
  kc.ksplit = d2b_cdiv(d.U, kc.uper);
  kc.tap_bytes = 0;
  kc.S = 3;
  while (kc.S > 1 && kc.S * kc.stage_bytes + 1024 + 128 > kMaxSmem) --kc.S;
  if (kc.S < 2) return false;
  k1.red = kc.red = k1.ksplit > 1 || kc.ksplit > 1;
  return true;
}

bool plan_k2(const TC& d, K2P& k) {
  if (d.ops % 64) return false;
  const int base = d.N * d.tiles_img * d.SG;
  k.msplit = best_split(base, d.MC, d.MC, 1);
  k.mper = d2b_cdiv(d.MC, k.msplit);
  k.msplit = d2b_cdiv(d.MC, k.mper);
  const int nkp = std::min(d.KK, (2 * k.mper + d.cbs - 1) / d.cbs + 1);
  const int ndg = d.DG == 1 ? 1 : std::min(d.DG, d2b_cdiv(d.cps, d.cpdg) + 1);
  k.tap_bytes = ndg * nkp * 128 * 16;
  return 2 * 4 * kTile + 128 * kGcolPitch * 4 + k.tap_bytes + 1024 + 128 <= kMaxSmem;
}

bool plan_k3(const TC& d, K3P& k) {
  if (d.ops % 64) return false;  // as K2: the backward takes whole 64-channel stages, so BN is 64 or 128
  k.BN = largest_tile(d.ops);
  k.noct = d.ops / k.BN;
  const int units = d.MC * d.SG * k.noct;
  const int total = d.N * d.stages_img;
  k.nsplit = best_split(units, total, std::min(total, 4 * d2b_num_sms()), 3);
  k.sper = d2b_cdiv(total, k.nsplit);
  k.nsplit = d2b_cdiv(total, k.sper);
  k.stage_bytes = 2 * kTile + 2 * k.BN * 128;
  k.S = 3;
  while (k.S > 1 && k.S * k.stage_bytes + 4096 + 1024 + 128 > kMaxSmem) --k.S;
  return k.S >= 2;
}

// ------------------------------------------------------------------------------------------------ call plans
// One plan per direction holds what a host call decides before it launches: the kernels' plans and the byte offset of
// each workspace region.  The size queries return a plan's total and the launchers carve from its offsets, so the two
// cannot disagree.  A plan that does not build means the tensor-core kernels do not take the shape.
struct Carve {  // regions laid out one after the other, each 256-byte aligned; an absent region has 0 bytes
  size_t total = 0;
  size_t add(size_t bytes) {
    const size_t at = total;
    total += align256(bytes);
    return at;
  }
};

struct FwdPlan {
  TC d;
  K1P k1, kc;   // kc: the column-fed launch, when colfed
  bool colfed;  // saved columns over several output-channel tiles: K1 gathers tile 0, K1c computes the others from cols
  int split;    // bf16x3 operands (precision 1)
  size_t wt, x, total;  // workspace: weight tiles, NHWC copy of an NCHW x
  size_t cols_bytes;    // the columns one call saves for the backward
};

bool plan_fwd(const d2b_dcn_params* p, int precision, int x_nhwc, bool cols, FwdPlan& P) {
  if (!make_tc(p, P.d) || !plan_k1(P.d, P.k1)) return false;
  const TC& d = P.d;
  Carve ws;
  P.wt = ws.add((size_t)d.SG * P.k1.noct * d.U * 2 * P.k1.BN * 128);
  P.x = ws.add(x_nhwc ? 0 : sizeof(float) * (size_t)d.N * d.H * d.W * d.Cin);
  P.total = ws.total;
  P.cols_bytes = (size_t)d.N * d.tiles_img * d.SG * d.U * (size_t)(precision == 1 ? 2 : 1) * kTile;
  P.split = precision == 1 ? 1 : 0;
  // With saved columns, x is sampled once per layer rather than once per output-channel tile.
  P.colfed = false;
  K1P k1;
  if (cols && P.k1.noct > 1 && plan_k1(d, k1, true) && plan_k1c(d, k1, P.kc)) {
    P.k1 = k1;
    P.colfed = true;
  }
  return true;
}

struct BwdPlan {
  TC d;
  K2P k2;
  K3P k3;
  int split;  // bf16x3 operands (precision 1)
  // workspace: NHWC copies of an NCHW x and of its gradient, grad_out as pixel-row tiles (K2) and as channel-row tiles (K3),
  // W^T tiles (K2), the weight gradient in the accumulator tiles' layout (gw_bytes)
  size_t x, gx, gt_px, wt, gt_oc, gw, gw_bytes, total;
};

bool plan_bwd(const d2b_dcn_params* p, int precision, int x_nhwc, int need_data, int need_weight, BwdPlan& P) {
  if (!make_tc(p, P.d) || !plan_k2(P.d, P.k2) || !plan_k3(P.d, P.k3)) return false;
  const TC& d = P.d;
  const size_t xbytes = sizeof(float) * (size_t)d.N * d.H * d.W * d.Cin;
  P.gw_bytes = sizeof(float) * (size_t)d.SG * d.MC * 128 * d.ops;
  Carve ws;
  P.x = ws.add(x_nhwc ? 0 : xbytes);
  P.gx = ws.add(need_data && !x_nhwc ? xbytes : 0);
  P.gt_px = ws.add(need_data ? (size_t)d.N * d.tiles_img * d.SG * d.nks * 2 * kTile : 0);
  P.wt = ws.add(need_data ? (size_t)d.SG * d.MC * d.nks * 2 * kTile : 0);
  P.gt_oc = ws.add(need_weight ? (size_t)d.N * d.stages_img * d.SG * P.k3.noct * 2 * P.k3.BN * 128 : 0);
  P.gw = ws.add(need_weight ? P.gw_bytes : 0);
  P.total = ws.total;
  P.split = precision == 1 ? 1 : 0;
  return true;
}

// ------------------------------------------------------------------------------------------------ sampling taps
// One 16-byte entry per (deformable group, kernel point, pixel): {code, lh, lw, mask} with
// code = ((pos0 + W + 1) << 4) | valid-corner bits, pos0 = floor(h)*W + floor(w) (may be "virtual": row/col -1).
// An entry of zeros means "sample outside (-1,H)x(-1,W)": contributes nothing (deform_conv_cuda_kernel.cu:273).
struct TapRaw {
  float oh, ow, m;
};

// the three global loads of a tap (issued early so that their latency overlaps other work)
__device__ __forceinline__ TapRaw tap_loads(const TC& d, const float* __restrict__ offset, const float* __restrict__ mask,
                                            int b, int dg, int kp, int p) {
  TapRaw r = {0.f, 0.f, 1.f};
  if (p < d.HoWo) {
    const size_t ob = (size_t)b * d.off_bs + ((size_t)dg * 2 * d.KK) * d.HoWo;
    r.oh = __ldg(offset + ob + (size_t)(2 * kp) * d.HoWo + p);       // deform_conv_cuda_kernel.cu:263-269
    r.ow = __ldg(offset + ob + (size_t)(2 * kp + 1) * d.HoWo + p);
    if (mask) r.m = __ldg(mask + (size_t)b * d.mask_bs + ((size_t)dg * d.KK + kp) * d.HoWo + p);
  }
  return r;
}

__device__ __forceinline__ int4 tap_finish(const TC& d, const TapRaw& r, bool has_mask, int kp, int p) {
  int4 t = make_int4(0, 0, 0, 0);
  if (p < d.HoWo) {
    const int ho = p / d.Wo, wo = p - ho * d.Wo;
    const int ki = kp / d.kw, kj = kp - ki * d.kw;
    const float hf = (float)(ho * d.sh - d.ph + ki * d.dh) + r.oh;
    const float wf = (float)(wo * d.sw - d.pw + kj * d.dw) + r.ow;
    float m = r.m;
    if (has_mask && d.mask_sigmoid) m = 1.f / (1.f + expf(-m));  // resnet.py:311 mask.sigmoid()
    if (hf > -1.f && wf > -1.f && hf < (float)d.H && wf < (float)d.W) {
      const float hfl = floorf(hf), wfl = floorf(wf);
      const int hl = (int)hfl, wl = (int)wfl;
      const bool t0 = hl >= 0, t1 = hl + 1 <= d.H - 1, l0 = wl >= 0, l1 = wl + 1 <= d.W - 1;
      const int flags = (t0 && l0 ? 1 : 0) | (t0 && l1 ? 2 : 0) | (t1 && l0 ? 4 : 0) | (t1 && l1 ? 8 : 0);
      t.x = ((hl * d.W + wl + d.W + 1) << 4) | flags;
      t.y = __float_as_int(hf - hfl);
      t.z = __float_as_int(wf - wfl);
      t.w = __float_as_int(m);
    }
  }
  return t;
}

__device__ __forceinline__ int4 make_tap(const TC& d, const float* __restrict__ offset, const float* __restrict__ mask,
                                         int b, int dg, int kp, int p) {
  return tap_finish(d, tap_loads(d, offset, mask, b, dg, kp, p), mask != nullptr, kp, p);
}

struct Taps4 {
  float4 v0, v1, v2, v3;
};

// the four corner pixels (4 channels each) of one tap entry; corners outside the image read as 0.
// `xcb` is the channel pointer biased by -(W + 1) pixels so that the tap's (pos0 + W + 1) indexes it directly; all offsets
// are 32-bit element counts (H * W * Cin < 2^30 is part of the shape gate), `rs` = W * Cin.
__device__ __forceinline__ void load_corners(const float* __restrict__ xcb, uint32_t Cin, uint32_t rs, int code, Taps4& t) {
  const float* __restrict__ p = xcb + (uint32_t)(code >> 4) * Cin;
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  t.v0 = (code & 1) ? __ldg(reinterpret_cast<const float4*>(p)) : z;
  t.v1 = (code & 2) ? __ldg(reinterpret_cast<const float4*>(p + Cin)) : z;
  t.v2 = (code & 4) ? __ldg(reinterpret_cast<const float4*>(p + rs)) : z;
  t.v3 = (code & 8) ? __ldg(reinterpret_cast<const float4*>(p + (rs + Cin))) : z;
}

__device__ __forceinline__ void interp4(const Taps4& t, float w0, float w1, float w2, float w3, float (&v)[4]) {
  const F2 z = f2_pack(0.f, 0.f), p0 = f2_pack(w0, w0), p1 = f2_pack(w1, w1), p2 = f2_pack(w2, w2), p3 = f2_pack(w3, w3);
  F2 a = f2_fma(p0, f2_pack(t.v0.x, t.v0.y), z), b = f2_fma(p0, f2_pack(t.v0.z, t.v0.w), z);
  a = f2_fma(p1, f2_pack(t.v1.x, t.v1.y), a);
  b = f2_fma(p1, f2_pack(t.v1.z, t.v1.w), b);
  a = f2_fma(p2, f2_pack(t.v2.x, t.v2.y), a);
  b = f2_fma(p2, f2_pack(t.v2.z, t.v2.w), b);
  a = f2_fma(p3, f2_pack(t.v3.x, t.v3.y), a);
  b = f2_fma(p3, f2_pack(t.v3.z, t.v3.w), b);
  f2_unpack(a, v[0], v[1]);
  f2_unpack(b, v[2], v[3]);
}

// gather 4 channels of one (pixel, unit) and store them as bf16 hi / lo into a swizzled 128-byte row
__device__ __forceinline__ void gather_store(const Taps4& t, int4 tap, uint8_t* a_hi, uint8_t* a_lo, uint32_t off,
                                             bool split) {
  const float lh = __int_as_float(tap.y), lw = __int_as_float(tap.z), m = __int_as_float(tap.w);
  const float hh = 1.f - lh, hw = 1.f - lw;
  float v[4];
  interp4(t, hh * hw * m, hh * lw * m, lh * hw * m, lh * lw * m, v);
  uint2 hi, lo;
  split4(v, hi, lo);
  *reinterpret_cast<uint2*>(a_hi + off) = hi;
  if (split) *reinterpret_cast<uint2*>(a_lo + off) = lo;
}

// ================================================================================================ wgmma helpers
// Stage of a 128-row x BN tile: warpgroup g multiplies rows [64 (g & 1), +64) of A by columns [(g >> 1) BN / 2, +BN / 2)
// of B over the stage's 64 k (four k16 steps); bf16x3 adds hi*lo and lo*hi.  A K-major: 16 k = 32 bytes along the swizzled
// row; A MN-major (kTransA): 16 k = two 8-row atoms, 2048 bytes.
template <int BN, int kTransA, int kSplit>
__device__ __forceinline__ void mma_stage_(float (&acc)[BN / 4], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo) {
  const int g = (threadIdx.x >> 7);
  const uint32_t ao = kTransA ? (uint32_t)(g & 1) * 8192u : (uint32_t)(g & 1) * 64u * 128u;
  const uint32_t bo = (uint32_t)(g >> 1) * (uint32_t)(BN / 2) * 128u;
  const uint32_t lbo = kTransA ? 8192u : 0u;
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    const uint32_t ak = ao + (kTransA ? (uint32_t)kk * 2048u : (uint32_t)kk * 32u), bk = bo + (uint32_t)kk * 32u;
    Wgmma<BN / 2, kTransA>::mma(acc, wgmma_desc(a_hi + ak, lbo, 1024), wgmma_desc(b_hi + bk, 0, 1024), 1);
    if (kSplit) {
      Wgmma<BN / 2, kTransA>::mma(acc, wgmma_desc(a_hi + ak, lbo, 1024), wgmma_desc(b_lo + bk, 0, 1024), 1);
      Wgmma<BN / 2, kTransA>::mma(acc, wgmma_desc(a_lo + ak, lbo, 1024), wgmma_desc(b_hi + bk, 0, 1024), 1);
    }
  }
  wgmma_commit();
}
// The precision is chosen outside the wgmma sequence: a branch between the MMAs of one accumulator makes ptxas insert
// warpgroup fences around each of them.
template <int BN, int kTransA>
__device__ __forceinline__ void mma_stage(float (&acc)[BN / 4], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                          int split) {
  if (split) mma_stage_<BN, kTransA, 1>(acc, a_hi, a_lo, b_hi, b_lo);
  else mma_stage_<BN, kTransA, 0>(acc, a_hi, a_lo, b_hi, b_lo);
}

// tile row / column of accumulator element i of this thread (see Wgmma in tc_common.cuh)
template <int BN>
__device__ __forceinline__ int acc_row(int i) {
  const int t = threadIdx.x & 127;
  return (threadIdx.x >> 7 & 1) * 64 + (t >> 5) * 16 + ((t & 31) >> 2) + ((i >> 1) & 1) * 8;
}
template <int BN>
__device__ __forceinline__ int acc_col(int i) {
  return (threadIdx.x >> 8) * (BN / 2) + (i >> 2) * 8 + (threadIdx.x & 3) * 2 + (i & 1);
}

// Forward epilogue of K1 and K1c: accumulator tile [128 px][BN oc] -> scale / shift / ReLU -> NCHW out.  With a k-split
// (k.red) the partial sums meet through red.add in the zero-filled output and dcn_epilogue_kernel applies scale / ReLU once
// all of them are in; the shift is added here by the first split only when nothing else is to be applied after it.
template <int BN>
__device__ __forceinline__ void fwd_epilogue(const float (&acc)[BN / 4], const Epi& ep, const TC& d, const K1P& k,
                                             float* __restrict__ out, int b, int p0, int oc0) {
  const bool add_shift = ep.shift != nullptr && blockIdx.z == 0;
#pragma unroll
  for (int i = 0; i < BN / 4; ++i) {
    const int p = p0 + acc_row<BN>(i);
    if (p >= d.HoWo) continue;
    const int oc = oc0 + acc_col<BN>(i);
    float* dst = out + ((size_t)b * d.Cout + oc) * d.HoWo + p;
    float v = acc[i];
    if (k.red) {
      red_add(dst, v + ((add_shift && !ep.scale && !ep.relu) ? __ldg(ep.shift + oc) : 0.f));
    } else {
      if (ep.scale) v *= __ldg(ep.scale + oc);
      if (ep.shift) v += __ldg(ep.shift + oc);
      if (ep.relu) v = fmaxf(v, 0.f);
      *dst = v;
    }
  }
}

// ================================================================================================ K1: forward
// grid (N * tiles_img, SG * k.goct, k splits); split z reduces over units [z * k.uper, +k.uper), which may begin and end
// inside a kernel point's channel blocks: the tap table holds the kernel points the range touches.  Warp 17 is the SAVER,
// which (when the caller keeps the sampled columns for the weight gradient) copies every finished A stage -- already bf16
// hi | lo in the tensor core's swizzled tile layout -- to global memory with one bulk store, so that the backward streams
// the tiles back instead of sampling x a second time (dcn_bwd_weight_cols_kernel).  Column tile of (image tile,
// super-group, unit): 16 KB hi [+ 16 KB lo].  The workers issue the MMAs of stage t right after gathering it and release
// stage t - 1 once its MMAs are done, so the gather of a stage overlaps the MMAs of the previous one.
template <int BN>
__global__ void __launch_bounds__(kThreads, 1) dcn_fwd_tc_kernel(const float* __restrict__ xh,
                                                                   const float* __restrict__ offset,
                                                                   const float* __restrict__ mask,
                                                                   const uint8_t* __restrict__ wt, const Epi ep, const TC d,
                                                                   const K1P k, const int split, float* __restrict__ out,
                                                                   uint8_t* __restrict__ cols) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // offset form keeps the shared address space
  int4* taps = reinterpret_cast<int4*>(smem + k.S * k.stage_bytes);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(taps) + k.tap_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + k.S;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = blockIdx.x / d.tiles_img, p0 = (blockIdx.x - b * d.tiles_img) * 128;
  const int sg = blockIdx.y / k.goct, oct = blockIdx.y - sg * k.goct;
  const int u0 = blockIdx.z * k.uper, nt = min(d.U, u0 + k.uper) - u0;
  const int kp0 = u0 / d.cbs, nkp = (u0 + nt - 1) / d.cbs - kp0 + 1;
  const int dg0 = (sg * d.cps) / d.cpdg;
  const bool saving = cols != nullptr && oct == 0;  // CTAs of the other output-channel tiles build the same columns

  if (tid == 0) {
    for (int s = 0; s < k.S; ++s) {
      mbar_init(&full_bar[s], kWorkerWarps + 1);
      mbar_init(&empty_bar[s], kWorkerWarps + (saving ? 1 : 0));  // every worker warp's MMAs [+ the saver's copy] are done
    }
    mbar_init_fence();
  }
  if (tid < kWorkers) {
    const int ndg = ((sg + 1) * d.cps - 1) / d.cpdg - dg0 + 1;
    for (int i = tid; i < ndg * nkp * 128; i += kWorkers) {
      const int row = i & 127, r = i >> 7;
      const int dgl = r / nkp, kpl = r - dgl * nkp;
      taps[i] = make_tap(d, offset, mask, b, dg0 + dgl, kp0 + kpl, p0 + row);
    }
  }
  __syncthreads();
  if (warp < kWorkerWarps) reg_alloc<kWorkerRegs>();
  else reg_dealloc<kSideRegs>();

  if (warp < kWorkerWarps) {
    // =============================================================== GATHER: A tile [128 px][64 k'] K-major, hi + lo; MMA
    const int half = lane >> 4, q = lane & 15;
    const float* __restrict__ ximg = xh + (size_t)b * d.H * d.W * d.Cin - (size_t)(d.W + 1) * d.Cin;  // biased: load_corners
    const uint32_t ucin = (uint32_t)d.Cin, urs = (uint32_t)(d.W * d.Cin);
    float acc[BN / 4];
#pragma unroll
    for (int i = 0; i < BN / 4; ++i) acc[i] = 0.f;
    int kpl = 0, cb = u0 - kp0 * d.cbs;
    // gather stage t, then issue its MMAs (one wgmma group)
    auto stage = [&](int t) {
      const int s = t % k.S;
      const uint32_t par = (uint32_t)((t / k.S) & 1);
      const int cbase = sg * d.cps + cb * 64;
      const int4* __restrict__ tp = taps + ((cbase / d.cpdg - dg0) * nkp + kpl) * 128;
      const float* __restrict__ xc = ximg + cbase + q * 4;
      uint8_t* a_hi = smem + s * k.stage_bytes;
      uint8_t* a_lo = a_hi + kTile;
      mbar_wait(&empty_bar[s], par ^ 1u);
      {  // the half-warp's pixel rows in ONE batch: all their corner loads are in flight before the first use
        int4 tap[kRowsPerHalf];
        Taps4 c[kRowsPerHalf];
#pragma unroll
        for (int j = 0; j < kRowsPerHalf; ++j) tap[j] = tp[warp * 2 * kRowsPerHalf + j * 2 + half];
#pragma unroll
        for (int j = 0; j < kRowsPerHalf; ++j) load_corners(xc, ucin, urs, tap[j].x, c[j]);
#pragma unroll
        for (int j = 0; j < kRowsPerHalf; ++j) {
          const uint32_t r = (uint32_t)(warp * 2 * kRowsPerHalf + j * 2 + half);
          gather_store(c[j], tap[j], a_hi, a_lo, swz128(r, (uint32_t)(q >> 1)) + (uint32_t)(q & 1) * 8u, split != 0);
        }
      }
      fence_proxy_async();  // generic-proxy writes -> visible to the tensor core (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(&full_bar[s]);
      mbar_wait(&full_bar[s], par);  // every warp's rows and the weight tile are in
      const uint32_t sa = smem_u32(a_hi), sb = sa + 2 * kTile;
      mma_stage<BN, 0>(acc, sa, sa + kTile, sb, sb + (uint32_t)BN * 128u, split);
      if (++cb == d.cbs) { cb = 0; ++kpl; }
    };
    // The first stage is issued before the loop so that every pass through the loop head has exactly one wgmma group in
    // flight; otherwise ptxas waits for it there and the gather of stage t no longer overlaps the MMAs of stage t - 1.
    stage(0);
    for (int t = 1; t < nt; ++t) {
      stage(t);
      wgmma_wait<1>();  // stage t - 1's MMAs are done: release it
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[(t - 1) % k.S]);
    }
    wgmma_wait<0>();
    fwd_epilogue<BN>(acc, ep, d, k, out, b, p0, sg * d.ops + oct * k.BN);
  } else if (warp == kWorkerWarps) {
    // =============================================================== TMA producer: weight tile of every chunk
    if (lane == 0) {
      const uint32_t bytes = (uint32_t)(split ? 2 : 1) * (uint32_t)k.BN * 128u;
      for (int t = 0; t < nt; ++t) {
        const int s = t % k.S;
        const uint32_t par = (uint32_t)((t / k.S) & 1);
        mbar_wait(&empty_bar[s], par ^ 1u);
        const size_t tile = ((size_t)(sg * k.noct + oct) * d.U + u0 + t);
        mbar_arrive_expect_tx(&full_bar[s], bytes);
        bulk_g2s(smem + s * k.stage_bytes + 2 * kTile, wt + tile * (size_t)(2 * k.BN * 128), bytes, &full_bar[s]);
      }
    }
  } else if (warp == kWorkerWarps + 1) {
    // =============================================================== SAVER: finished A stages -> column tiles in global memory
    if (saving && lane == 0) {
      const uint32_t tile_bytes = (uint32_t)(split ? 2 : 1) * (uint32_t)kTile;
      for (int t = 0; t < nt; ++t) {
        const int s = t % k.S;
        const uint32_t par = (uint32_t)((t / k.S) & 1);
        mbar_wait(&full_bar[s], par);  // the workers' writes are fenced to the async proxy before they arrive
        const size_t tile = ((size_t)blockIdx.x * d.SG + sg) * d.U + u0 + t;
        bulk_s2g(cols + tile * tile_bytes, smem + s * k.stage_bytes, tile_bytes);
        bulk_commit();
        bulk_wait_read0();
        mbar_arrive(&empty_bar[s]);
      }
      bulk_wait0();
    }
  }
}

// ================================================================================================ K1c: forward from saved columns
// Output-channel tiles 1..noct-1 of a forward that saves its columns: K1 gathers and saves them once (tile 0), and this kernel
// streams each stage's column tile back with one bulk copy (hi [+ lo], already in K1's swizzled A layout) next to K1's weight
// tile of its output-channel tile: a pure TMA -> wgmma pipeline like K3c, with K1's epilogue.  grid ((N * tiles_img) *
// (noct - 1), SG, k splits over units as in K1), the output-channel tile fastest: the CTAs that read one column tile run
// together and share it in L2.
template <int BN>
__global__ void __launch_bounds__(kThreads, 1) dcn_fwd_cols_kernel(const uint8_t* __restrict__ cols,
                                                                   const uint8_t* __restrict__ wt, const Epi ep, const TC d,
                                                                   const K1P k, const int split, float* __restrict__ out) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + k.S * k.stage_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + k.S;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile = blockIdx.x / k.goct, oct = 1 + (blockIdx.x - tile * k.goct);
  const int b = tile / d.tiles_img, p0 = (tile - b * d.tiles_img) * 128;
  const int sg = blockIdx.y;
  const int u0 = blockIdx.z * k.uper, nt = min(d.U, u0 + k.uper) - u0;

  if (tid == 0) {
    for (int s = 0; s < k.S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kWorkerWarps);
    }
    mbar_init_fence();
  }
  __syncthreads();
  if (warp < kWorkerWarps) reg_alloc<kWorkerRegs>();
  else reg_dealloc<kSideRegs>();

  if (warp < kWorkerWarps) {
    float acc[BN / 4];
#pragma unroll
    for (int i = 0; i < BN / 4; ++i) acc[i] = 0.f;
    auto issue = [&](int t) {
      const int s = t % k.S;
      mbar_wait(&full_bar[s], (uint32_t)((t / k.S) & 1));
      const uint32_t sa = smem_u32(smem + s * k.stage_bytes), sb = sa + 2 * kTile;
      mma_stage<BN, 0>(acc, sa, sa + kTile, sb, sb + (uint32_t)BN * 128u, split);
    };
    issue(0);  // as in K1: one wgmma group in flight at every pass through the loop head
    for (int t = 1; t < nt; ++t) {
      issue(t);
      wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[(t - 1) % k.S]);
    }
    wgmma_wait<0>();
    fwd_epilogue<BN>(acc, ep, d, k, out, b, p0, sg * d.ops + oct * k.BN);
  } else if (warp == kWorkerWarps) {
    // =============================================================== TMA producer: column tile + weight tile per stage
    if (lane == 0) {
      const uint32_t parts = split ? 2u : 1u;
      // pointers and ring position advance with the stage (this warp runs on kSideRegs registers)
      const uint32_t abytes = parts * (uint32_t)kTile;
      const uint8_t* asrc = cols + (((size_t)tile * d.SG + sg) * d.U + u0) * abytes;  // as K1's saver wrote them
      const uint8_t* bsrc = wt + ((size_t)(sg * k.noct + oct) * d.U + u0) * (size_t)(2 * BN * 128);
      int s = 0;
      uint32_t par = 1u;
      for (int t = nt; t > 0; --t, asrc += abytes, bsrc += 2 * BN * 128) {
        mbar_wait(&empty_bar[s], par);
        mbar_arrive_expect_tx(&full_bar[s], abytes / 128u * (128u + BN));
        bulk_g2s(smem + s * k.stage_bytes, asrc, abytes, &full_bar[s]);
        bulk_g2s(smem + s * k.stage_bytes + 2 * kTile, bsrc, abytes / 128u * BN, &full_bar[s]);
        if (++s == k.S) {
          s = 0;
          par ^= 1u;
        }
      }
    }
  }
}

// ================================================================================================ K2: backward data
// grid (N * tiles_img, SG, macro-chunk splits).  Per macro-chunk (2 units = 128 k'): gcol[128 px][128] = gout . W over the
// super-group's output channels (register accumulators of the four worker warpgroups, operand stages double buffered by
// TMA), drained to shared memory, then scattered:
//   grad_x   += gcol * mask * bilinear weight      (deform_conv_cuda_kernel.cu:313-362, :923-975) red.global.add.v4 (NHWC)
//   grad_off += gcol * mask * d(sample)/d(h,w)     (:390-451, :977-1064)                           red.global.add
//   grad_msk += gcol * sample                      (:1053-1064)
// The body takes its block coordinates so that the fused backward (dcn_bwd_fused_kernel) can run it too; smem is the
// 1024-byte aligned dynamic shared memory.
template <int kSide>
__device__ __forceinline__ void bwd_data_body(uint8_t* smem, int bx, int by, int bz, const float* __restrict__ xh,
                                              const float* __restrict__ offset, const float* __restrict__ mask,
                                              const uint8_t* __restrict__ gt, const uint8_t* __restrict__ wt, const TC& d,
                                              const K2P& k, const int split, float* __restrict__ gxh,
                                              float* __restrict__ goff, float* __restrict__ gmask) {
  constexpr int kStage = 4 * kTile;  // A hi | A lo | B hi | B lo
  float* gcol = reinterpret_cast<float*>(smem + 2 * kStage);
  int4* taps = reinterpret_cast<int4*>(smem + 2 * kStage + 128 * kGcolPitch * 4);
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(taps) + k.tap_bytes);
  uint64_t* full_bar = bars;         // [2]
  uint64_t* empty_bar = bars + 2;    // [2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b = bx / d.tiles_img, pt = bx - b * d.tiles_img, p0 = pt * 128;
  const int sg = by;
  const int m0 = bz * k.mper, m1 = min(d.MC, m0 + k.mper), nm = m1 - m0;
  const int u_begin = 2 * m0, u_end = min(d.U, 2 * m1);
  const int kp0 = u_begin / d.cbs, nkp = (u_end - 1) / d.cbs - kp0 + 1;
  const int dg0 = (sg * d.cps) / d.cpdg;

  if (tid == 0) {
    for (int s = 0; s < 2; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kWorkerWarps);
    }
    mbar_init_fence();
  }
  if (tid < kWorkers) {
    const int ndg = ((sg + 1) * d.cps - 1) / d.cpdg - dg0 + 1;
    for (int i = tid; i < ndg * nkp * 128; i += kWorkers) {
      const int row = i & 127, r = i >> 7;
      const int dgl = r / nkp, kpl = r - dgl * nkp;
      taps[i] = make_tap(d, offset, mask, b, dg0 + dgl, kp0 + kpl, p0 + row);
    }
  }
  __syncthreads();
  if (warp < kWorkerWarps) reg_alloc<kWorkerRegs>();
  else reg_dealloc<kSide>();

  if (warp < kWorkerWarps) {
    const int half = lane >> 4, q = lane & 15;
    // both image pointers are biased by -(W + 1) pixels (see load_corners)
    const size_t img_off = (size_t)b * d.H * d.W * d.Cin - (size_t)(d.W + 1) * d.Cin;
    const float* __restrict__ ximg = xh + img_off;
    float* __restrict__ gimg = gxh ? gxh + img_off : nullptr;
    const uint32_t ucin = (uint32_t)d.Cin, urs = (uint32_t)(d.W * d.Cin);
    constexpr int R = kRowsPerHalf;  // pixel rows of the tile owned by this half-warp (fixed for the whole kernel)
    float sh[R], sw[R], sm[R];
#pragma unroll
    for (int j = 0; j < R; ++j) sh[j] = sw[j] = sm[j] = 0.f;
    int cur_kp = -1, cur_dg = -1;

    auto flush = [&]() {
      if (cur_kp < 0) return;
      // 12 partial sums (4 rows x {d/dh, d/dw, d/dmask}) per lane, to be summed over the 16 lanes of the half-warp.
      // Recursive halving: at each step a lane keeps one half of its values and hands the other half to its partner,
      // so 6 + 3 + 2 + 1 shuffles replace 12 butterflies of 4; lane q ends up owning value (row = q >> 2, which = q & 3).
      static_assert(R == 4, "the reduction below is written for 4 rows per half-warp");
      float v12[12];
#pragma unroll
      for (int j = 0; j < R; ++j) {
        v12[3 * j] = sh[j];
        v12[3 * j + 1] = sw[j];
        v12[3 * j + 2] = sm[j];
      }
      const bool b8 = q & 8, b4 = q & 4, b2 = q & 2, b1 = q & 1;
      float v6[6], v3[3];
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        const float keep = b8 ? v12[i + 6] : v12[i], send = b8 ? v12[i] : v12[i + 6];
        v6[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
      }
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        const float keep = b4 ? v6[i + 3] : v6[i], send = b4 ? v6[i] : v6[i + 3];
        v3[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
      }
      // {v3[0], v3[1]} | {v3[2], -}
      const float k0 = b2 ? v3[2] : v3[0], s0 = b2 ? v3[0] : v3[2];
      const float k1 = b2 ? 0.f : v3[1], s1 = b2 ? v3[1] : 0.f;
      const float u0 = k0 + __shfl_xor_sync(0xffffffffu, s0, 2);
      const float u1 = k1 + __shfl_xor_sync(0xffffffffu, s1, 2);
      float v = (b1 ? u1 : u0) + __shfl_xor_sync(0xffffffffu, b1 ? u0 : u1, 1);
      {
        const int j = q >> 2, which = q & 3;
        const int row = warp * 2 * R + j * 2 + half;
        const int p = p0 + row;
        if (which < 3 && p < d.HoWo) {
          if (which < 2) {
            if (goff) red_add(goff + (size_t)b * d.off_bs + ((size_t)cur_dg * 2 * d.KK + 2 * cur_kp + which) * d.HoWo + p, v);
          } else if (gmask) {
            if (d.mask_sigmoid) {  // gradient w.r.t. the logit: m (1 - m)
              const float m = __int_as_float(taps[((cur_dg - dg0) * nkp + (cur_kp - kp0)) * 128 + row].w);
              v *= m * (1.f - m);
            }
            red_add(gmask + (size_t)b * d.mask_bs + ((size_t)cur_dg * d.KK + cur_kp) * d.HoWo + p, v);
          }
        }
      }
#pragma unroll
      for (int j = 0; j < R; ++j) sh[j] = sw[j] = sm[j] = 0.f;
    };

    for (int ml = 0; ml < nm; ++ml) {
      const int buf = ml & 1;
      const int m = m0 + ml;
      const int nu = (2 * m + 1 < d.U) ? 2 : 1;
      {  // ---- gcol tile on the tensor cores: 128 columns (the second unit's are zero when nu == 1), then drained to gcol[px][col]
        float acc[32];
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[i] = 0.f;
        for (int ks = 0; ks < d.nks; ++ks) {
          const int c = ml * d.nks + ks, s = c & 1;
          mbar_wait(&full_bar[s], (uint32_t)((c >> 1) & 1));
          const uint32_t sa = smem_u32(smem + s * kStage);
          mma_stage<128, 0>(acc, sa, sa + kTile, sa + 2 * kTile, sa + 3 * kTile, split);
          wgmma_wait<0>();
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[s]);
        }
#pragma unroll
        for (int i = 0; i < 32; i += 2)
          *reinterpret_cast<float2*>(gcol + acc_row<128>(i) * kGcolPitch + acc_col<128>(i)) = make_float2(acc[i], acc[i + 1]);
      }
      named_bar_sync(1, kWorkers);
      // ---- scatter
      for (int ul = 0; ul < nu; ++ul) {
        const int u = 2 * m + ul;
        const int kp = u / d.cbs, cb = u - kp * d.cbs;
        const int cbase = sg * d.cps + cb * 64;
        const int dg = cbase / d.cpdg;
        if (kp != cur_kp || dg != cur_dg) {
          flush();
          cur_kp = kp;
          cur_dg = dg;
        }
        const int4* __restrict__ tp = taps + ((dg - dg0) * nkp + (kp - kp0)) * 128;
        const float* __restrict__ xc = ximg + cbase + q * 4;
        float* __restrict__ gc = gimg + cbase + q * 4;
        constexpr int kB2 = 2;  // pixel rows per batch: 4 * kB2 loads in flight per lane, then up to 4 * kB2 reductions
#pragma unroll
        for (int it = 0; it < R / kB2; ++it) {
          int4 tap[kB2];
          Taps4 c[kB2];
#pragma unroll
          for (int e = 0; e < kB2; ++e) tap[e] = tp[warp * 2 * R + (it * kB2 + e) * 2 + half];
#pragma unroll
          for (int e = 0; e < kB2; ++e) load_corners(xc, ucin, urs, tap[e].x, c[e]);
#pragma unroll
          for (int e = 0; e < kB2; ++e) {
            if ((tap[e].x & 15) == 0) continue;  // sample outside the image: no gradient anywhere
            const int j = it * kB2 + e;
            const int row = warp * 2 * R + j * 2 + half;
            const float4 g4 = *reinterpret_cast<const float4*>(gcol + row * kGcolPitch + ul * 64 + q * 4);
            const float lh = __int_as_float(tap[e].y), lw = __int_as_float(tap[e].z), mk = __int_as_float(tap[e].w);
            const float hh = 1.f - lh, hw = 1.f - lw;
            const float w0 = hh * hw, w1 = hh * lw, w2 = lh * hw, w3 = lh * lw;
            const F2 LH = f2_pack(lh, lh), LW = f2_pack(lw, lw), HH = f2_pack(hh, hh), HW = f2_pack(hw, hw);
            const F2 W0 = f2_pack(w0, w0), W1 = f2_pack(w1, w1), W2 = f2_pack(w2, w2), W3 = f2_pack(w3, w3);
            const F2 MK = f2_pack(mk, mk);
            // channel pairs: pair 0 = channels 0,1; pair 1 = channels 2,3
            const F2 G[2] = {f2_pack(g4.x, g4.y), f2_pack(g4.z, g4.w)};
            const F2 A0[2] = {f2_pack(c[e].v0.x, c[e].v0.y), f2_pack(c[e].v0.z, c[e].v0.w)};
            const F2 A1[2] = {f2_pack(c[e].v1.x, c[e].v1.y), f2_pack(c[e].v1.z, c[e].v1.w)};
            const F2 A2[2] = {f2_pack(c[e].v2.x, c[e].v2.y), f2_pack(c[e].v2.z, c[e].v2.w)};
            const F2 A3[2] = {f2_pack(c[e].v3.x, c[e].v3.y), f2_pack(c[e].v3.z, c[e].v3.w)};
            F2 GM[2];
            F2 th2 = f2_pack(0.f, 0.f), tw2 = th2, tm2 = th2;
#pragma unroll
            for (int i = 0; i < 2; ++i) {
              GM[i] = f2_mul(G[i], MK);
              // d val / d h = (1-lw)(v2-v0) + lw (v3-v1);  d val / d w = (1-lh)(v1-v0) + lh (v3-v2)
              const F2 dh = f2_fma(LW, f2_sub(A3[i], A1[i]), f2_mul(HW, f2_sub(A2[i], A0[i])));
              const F2 dw = f2_fma(LH, f2_sub(A3[i], A2[i]), f2_mul(HH, f2_sub(A1[i], A0[i])));
              const F2 val = f2_fma(W3, A3[i], f2_fma(W2, A2[i], f2_fma(W1, A1[i], f2_mul(W0, A0[i]))));
              th2 = f2_fma(GM[i], dh, th2);
              tw2 = f2_fma(GM[i], dw, tw2);
              tm2 = f2_fma(G[i], val, tm2);
            }
            {
              float e0, e1;
              f2_unpack(th2, e0, e1);
              sh[j] += e0 + e1;
              f2_unpack(tw2, e0, e1);
              sw[j] += e0 + e1;
              f2_unpack(tm2, e0, e1);
              sm[j] += e0 + e1;
            }
            if (gimg) {
              float* gp = gc + (uint32_t)(tap[e].x >> 4) * ucin;
              red_add_v4_if(tap[e].x & 1, gp, f2_mul(GM[0], W0), f2_mul(GM[1], W0));
              red_add_v4_if(tap[e].x & 2, gp + ucin, f2_mul(GM[0], W1), f2_mul(GM[1], W1));
              red_add_v4_if(tap[e].x & 4, gp + urs, f2_mul(GM[0], W2), f2_mul(GM[1], W2));
              red_add_v4_if(tap[e].x & 8, gp + (urs + ucin), f2_mul(GM[0], W3), f2_mul(GM[1], W3));
            }
          }
        }
      }
      named_bar_sync(1, kWorkers);  // everyone is done reading gcol before the next drain overwrites it
    }
    flush();
  } else if (warp == kWorkerWarps) {
    // =============================================================== TMA producer: gout tile + W^T tile per K stage
    if (lane == 0) {
      const uint32_t half_bytes = (uint32_t)(split ? 2 : 1) * (uint32_t)kTile;
      int c = 0;
      for (int ml = 0; ml < nm; ++ml) {
        const int m = m0 + ml;
        for (int ks = 0; ks < d.nks; ++ks, ++c) {
          const int s = c & 1;
          const uint32_t par = (uint32_t)((c >> 1) & 1);
          mbar_wait(&empty_bar[s], par ^ 1u);
          mbar_arrive_expect_tx(&full_bar[s], 2 * half_bytes);
          const size_t atile = (((size_t)b * d.tiles_img + pt) * d.SG + sg) * d.nks + ks;
          const size_t btile = ((size_t)sg * d.MC + m) * d.nks + ks;
          bulk_g2s(smem + s * kStage, gt + atile * (size_t)(2 * kTile), half_bytes, &full_bar[s]);
          bulk_g2s(smem + s * kStage + 2 * kTile, wt + btile * (size_t)(2 * kTile), half_bytes, &full_bar[s]);
        }
      }
    }
  }
}

__device__ __forceinline__ uint8_t* aligned_smem() {
  extern __shared__ uint8_t smem_raw[];
  return smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // offset form keeps the shared address space
}

// grid (N * tiles_img, SG, macro-chunk splits)
__global__ void __launch_bounds__(kThreads, 1) dcn_bwd_data_tc_kernel(const float* __restrict__ xh,
                                                                      const float* __restrict__ offset,
                                                                      const float* __restrict__ mask,
                                                                      const uint8_t* __restrict__ gt,
                                                                      const uint8_t* __restrict__ wt, const TC d,
                                                                      const K2P k, const int split,
                                                                      float* __restrict__ gxh, float* __restrict__ goff,
                                                                      float* __restrict__ gmask) {
  bwd_data_body<kSideRegs>(aligned_smem(), blockIdx.x, blockIdx.y, blockIdx.z, xh, offset, mask, gt, wt, d, k, split, gxh,
                           goff, gmask);
}

// ================================================================================================ weight-gradient epilogue
// The accumulator tile of a K3 CTA is [128 k' rows][BN oc]; in the weight tensor [Cout][Cin/G][KK] one unit's 64 rows are
// 36 bytes apart (one kernel point of 64 channels), so writing it directly costs one 32-byte sector atomic per ELEMENT and
// per pixel split.  Instead every CTA adds its tile with 8-byte vector reductions (a thread's accumulator holds column pairs)
// into the zero-filled staging matrix `part` [SG][MC*128][ops], and a small second kernel moves it into the weight tensor's
// layout.
template <int BN>
__device__ __forceinline__ void gw_tile_store(const float (&acc)[BN / 4], float* __restrict__ tile, int pitch) {
#pragma unroll
  for (int i = 0; i < BN / 4; i += 2) red_add_v2(tile + (size_t)acc_row<BN>(i) * pitch + acc_col<BN>(i), acc[i], acc[i + 1]);
}

// one thread per (super-group, unit row, oc of the super-group); oc fastest: the reads of `part` are coalesced
__global__ void dcn_gw_reduce_kernel(const float* __restrict__ part, const TC d, float* __restrict__ gw) {
  const long long total = (long long)d.SG * d.U * 64 * d.ops;
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int ocl = (int)(idx % d.ops);
  const long long r = idx / d.ops;
  const int rowu = (int)(r % ((long long)d.U * 64)), sg = (int)(r / ((long long)d.U * 64));
  const int u = rowu >> 6, ch = rowu & 63;
  const int kp = u / d.cbs, cb = u - kp * d.cbs;
  const int ec = sg * d.cps + cb * 64 + ch, egrp = ec / d.cpg, ecin = ec - egrp * d.cpg;
  const int oc = sg * d.ops + ocl;
  if (oc / d.opg != egrp) return;  // block-diagonal padding of a packed super-group
  gw[((size_t)oc * d.cpg + ecin) * d.KK + kp] = __ldg(part + ((size_t)sg * d.MC * 128 + rowu) * d.ops + ocl);
}

// The same sum with coalesced writes for small kernels (KK <= 9): one block owns (super-group, 16 channels, 16 output
// channels), stages the KK x 16 x 16 sums in shared memory and writes, per output channel, the run of 16 * KK floats that the
// block's channels occupy in the weight tensor.
constexpr int kRedOc = 16, kRedCh = 16;
__global__ void __launch_bounds__(256) dcn_gw_reduce_tile_kernel(const float* __restrict__ part, const TC d,
                                                                  float* __restrict__ gw) {
  __shared__ float tile[9 * kRedCh][kRedOc + 1];
  const int per_sg = d.cps / kRedCh;
  const int sg = blockIdx.x / per_sg, c0 = (blockIdx.x - sg * per_sg) * kRedCh;  // first channel inside the super-group
  const int cb = c0 >> 6, ch0 = c0 & 63;
  const int ocl0 = blockIdx.y * kRedOc;
  const int tid = threadIdx.x;
  {
    const int j = tid & (kRedOc - 1), r0 = tid / kRedOc;  // 16 rows per pass
    for (int row = r0; row < d.KK * kRedCh; row += 256 / kRedOc) {
      const int kp = row / kRedCh, ch = row - kp * kRedCh;
      tile[row][j] = __ldg(part + ((size_t)sg * d.MC * 128 + (size_t)(kp * d.cbs + cb) * 64 + ch0 + ch) * d.ops + ocl0 + j);
    }
  }
  __syncthreads();
  const int ec0 = sg * d.cps + c0;
  for (int i = tid; i < kRedOc * kRedCh * d.KK; i += 256) {
    const int j = i / (kRedCh * d.KK), e = i - j * (kRedCh * d.KK);
    const int ch = e / d.KK, kp = e - ch * d.KK;
    const int oc = sg * d.ops + ocl0 + j, grp = oc / d.opg;
    const int ec = ec0 + ch;
    if (ec / d.cpg == grp) gw[((size_t)oc * d.cpg + (ec - grp * d.cpg)) * d.KK + kp] = tile[kp * kRedCh + ch][j];
  }
}

// ================================================================================================ K3: backward weight
// grid (SG * oc tiles, M blocks = pairs of units, pixel splits).  D[128 k'][BN oc] += col^T[128 k'][64 px] . gout[64 px][BN oc]
// per 64-pixel stage; the gathered tile is written [unit half][pixel][64 ch] = MN-major for the tensor core.  As in K1 the
// workers issue the MMAs of a stage after gathering it and release the previous stage once its MMAs are done.
template <int BN>
__global__ void __launch_bounds__(kThreads, 1) dcn_bwd_weight_tc_kernel(const float* __restrict__ xh,
                                                                        const float* __restrict__ offset,
                                                                        const float* __restrict__ mask,
                                                                        const uint8_t* __restrict__ gt, const TC d,
                                                                        const K3P k, const int split,
                                                                        float* __restrict__ gw) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);  // offset form keeps the shared address space
  int4* tap_s = reinterpret_cast<int4*>(smem + k.S * k.stage_bytes);  // [16 warps][8]
  uint64_t* bars = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(tap_s) + 4096);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + k.S;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mb = blockIdx.y;
  const int sg = blockIdx.x / k.noct, oct = blockIdx.x - sg * k.noct;
  const int total = d.N * d.stages_img;
  const int gs0 = blockIdx.z * k.sper, gs1 = min(total, gs0 + k.sper), ns = gs1 - gs0;

  if (tid == 0) {
    for (int s = 0; s < k.S; ++s) {
      mbar_init(&full_bar[s], kWorkerWarps + 1);
      mbar_init(&empty_bar[s], kWorkerWarps);
    }
    mbar_init_fence();
  }
  __syncthreads();
  if (warp < kWorkerWarps) reg_alloc<kWorkerRegs>();
  else reg_dealloc<kSideRegs>();

  if (warp < kWorkerWarps) {
    // =============================================================== GATHER: A tile [2 units][64 px][64 ch], hi + lo
    const int half = lane >> 4, q = lane & 15;
    const int u = 2 * mb + half;             // this half-warp's unit
    const bool u_ok = u < d.U;
    const int kp = u_ok ? u / d.cbs : 0, cb = u_ok ? u - kp * d.cbs : 0;
    const int cbase = sg * d.cps + cb * 64;
    const int dg = cbase / d.cpdg;
    // lanes 0..15 build the taps of this warp's 8 pixels x 2 units; the loads of the NEXT stage's offsets / mask are issued
    // before this stage's gather and consumed after it, so that their latency is hidden behind the gather
    constexpr int PX = 64 / kWorkerWarps;  // pixels of a stage per warp: 8
    const int tl_half = (lane / PX) & 1, tl_j = lane % PX;
    const int tl_u = 2 * mb + tl_half;
    const bool tl_ok = lane < 2 * PX && tl_u < d.U;
    const int tl_kp = tl_ok ? tl_u / d.cbs : 0;
    const int tl_dg = tl_ok ? (sg * d.cps + (tl_u - tl_kp * d.cbs) * 64) / d.cpdg : 0;
    int4* my_taps = tap_s + warp * 2 * (2 * PX);  // [2 buffers][2 units][PX]
    auto stage_of = [&](int i, int& b, int& pbase) {
      const int gs = gs0 + i;
      b = gs / d.stages_img;
      pbase = (gs - b * d.stages_img) * 64;
    };
    if (ns > 0) {
      int b0, pb0;
      stage_of(0, b0, pb0);
      if (lane < 2 * PX) my_taps[lane] = tl_ok ? make_tap(d, offset, mask, b0, tl_dg, tl_kp, pb0 + warp * PX + tl_j) : make_int4(0, 0, 0, 0);
    }
    __syncwarp();
    float acc[BN / 4];
#pragma unroll
    for (int i = 0; i < BN / 4; ++i) acc[i] = 0.f;
    auto stage = [&](int i) {  // gather stage i, then issue its MMAs
      const int s = i % k.S;
      const uint32_t par = (uint32_t)((i / k.S) & 1);
      int b, pbase, bn = 0, pbn = 0;
      stage_of(i, b, pbase);
      const bool have_next = i + 1 < ns;
      TapRaw raw = {0.f, 0.f, 1.f};
      if (have_next) {
        stage_of(i + 1, bn, pbn);
        if (tl_ok) raw = tap_loads(d, offset, mask, bn, tl_dg, tl_kp, pbn + warp * PX + tl_j);
      }
      const float* __restrict__ xc = xh + ((size_t)b * d.H * d.W - (size_t)(d.W + 1)) * d.Cin + cbase + q * 4;  // biased
      const uint32_t ucin = (uint32_t)d.Cin, urs = (uint32_t)(d.W * d.Cin);
      uint8_t* a_hi = smem + s * k.stage_bytes + half * 8192;
      uint8_t* a_lo = a_hi + kTile;
      const int4* cur = my_taps + (i & 1) * (2 * PX) + half * PX;
      mbar_wait(&empty_bar[s], par ^ 1u);
      {
        int4 tap[PX];
        Taps4 c[PX];
#pragma unroll
        for (int j = 0; j < PX; ++j) tap[j] = cur[j];
#pragma unroll
        for (int j = 0; j < PX; ++j) load_corners(xc, ucin, urs, tap[j].x, c[j]);
#pragma unroll
        for (int j = 0; j < PX; ++j) {
          const uint32_t r = (uint32_t)(warp * PX + j);
          gather_store(c[j], tap[j], a_hi, a_lo, swz128(r, (uint32_t)(q >> 1)) + (uint32_t)(q & 1) * 8u, split != 0);
        }
      }
      if (have_next && lane < 2 * PX)
        my_taps[((i + 1) & 1) * (2 * PX) + lane] =
            tl_ok ? tap_finish(d, raw, mask != nullptr, tl_kp, pbn + warp * PX + tl_j) : make_int4(0, 0, 0, 0);
      fence_proxy_async();
      __syncwarp();
      if (lane == 0) mbar_arrive(&full_bar[s]);
      mbar_wait(&full_bar[s], par);
      const uint32_t sa = smem_u32(smem + s * k.stage_bytes), sb = sa + 2 * kTile;
      mma_stage<BN, 1>(acc, sa, sa + kTile, sb, sb + (uint32_t)BN * 128u, split);
    };
    stage(0);  // as in K1: one wgmma group in flight at every pass through the loop head (ns >= 1 by construction)
    for (int i = 1; i < ns; ++i) {
      stage(i);
      wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % k.S]);
    }
    wgmma_wait<0>();
    // =============================================================== EPILOGUE: registers [k' row][oc col] -> this split's partial tile
    gw_tile_store<BN>(acc, gw + ((size_t)sg * d.MC * 128 + (size_t)mb * 128) * d.ops + (size_t)oct * k.BN, d.ops);
  } else if (warp == kWorkerWarps) {
    if (lane == 0) {
      const uint32_t bytes = (uint32_t)(split ? 2 : 1) * (uint32_t)k.BN * 128u;
      for (int i = 0; i < ns; ++i) {
        const int s = i % k.S;
        const uint32_t par = (uint32_t)((i / k.S) & 1);
        mbar_wait(&empty_bar[s], par ^ 1u);
        mbar_arrive_expect_tx(&full_bar[s], bytes);
        const size_t tile = ((size_t)(gs0 + i) * d.SG + sg) * k.noct + oct;
        bulk_g2s(smem + s * k.stage_bytes + 2 * kTile, gt + tile * (size_t)(2 * k.BN * 128), bytes, &full_bar[s]);
      }
    }
  }
}

// ================================================================================================ K3c: backward weight from saved columns
// Same grid, tiles and epilogue as K3, but the A operand is streamed back from the column tiles the forward saved
// (dcn_fwd_tc_kernel's saver warp) instead of being sampled from x again: a pure TMA -> wgmma pipeline.  A 64-pixel stage of
// a unit is one contiguous 8 KB half of its [128 px][64 ch] tile (the 128-byte swizzle repeats every 8 rows).
template <int BN, int kSide>
__device__ __forceinline__ void bwd_weight_cols_body(uint8_t* smem, int bx, int by, int bz, const uint8_t* __restrict__ cols,
                                                     const uint8_t* __restrict__ gt, const TC& d, const K3P& k, const int S,
                                                     const int split, float* __restrict__ gw) {
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + S * k.stage_bytes);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + S;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int mb = by;
  const int sg = bx / k.noct, oct = bx - sg * k.noct;
  const int total = d.N * d.stages_img;
  const int gs0 = bz * k.sper, gs1 = min(total, gs0 + k.sper), ns = gs1 - gs0;
  const int nu = (2 * mb + 1 < d.U) ? 2 : 1;

  if (tid == 0) {
    for (int s = 0; s < S; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kWorkerWarps);
    }
    mbar_init_fence();
  }
  if (nu == 1 && tid < kWorkers) {  // odd unit count: the second 64 rows of A are never loaded; keep them finite
    for (int s = 0; s < S; ++s)
      for (int i = tid; i < 2 * 512; i += kWorkers) {
        const int part = i >> 9, w = i & 511;
        reinterpret_cast<uint4*>(smem + s * k.stage_bytes + part * kTile + 8192)[w] = make_uint4(0, 0, 0, 0);
      }
    fence_proxy_async();
  }
  __syncthreads();
  if (warp < kWorkerWarps) reg_alloc<kWorkerRegs>();
  else reg_dealloc<kSide>();

  if (warp < kWorkerWarps) {
    // =============================================================== MMA (as K3), then registers -> this split's partial tile
    float acc[BN / 4];
#pragma unroll
    for (int i = 0; i < BN / 4; ++i) acc[i] = 0.f;
    auto issue = [&](int i) {
      const int s = i % S;
      mbar_wait(&full_bar[s], (uint32_t)((i / S) & 1));
      const uint32_t sa = smem_u32(smem + s * k.stage_bytes), sb = sa + 2 * kTile;
      mma_stage<BN, 1>(acc, sa, sa + kTile, sb, sb + (uint32_t)BN * 128u, split);
    };
    issue(0);  // as in K1: one wgmma group in flight at every pass through the loop head
    for (int i = 1; i < ns; ++i) {
      issue(i);
      wgmma_wait<1>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[(i - 1) % S]);
    }
    wgmma_wait<0>();
    gw_tile_store<BN>(acc, gw + ((size_t)sg * d.MC * 128 + (size_t)mb * 128) * d.ops + (size_t)oct * k.BN, d.ops);
  } else if (warp == kWorkerWarps) {
    // =============================================================== TMA producer: column halves + grad_out tile per stage
    if (lane == 0) {
      const uint32_t parts = split ? 2u : 1u;
      const uint32_t tile_bytes = parts * (uint32_t)kTile;
      const uint32_t gbytes = parts * (uint32_t)k.BN * 128u;
      for (int i = 0; i < ns; ++i) {
        const int s = i % S;
        const uint32_t par = (uint32_t)((i / S) & 1);
        const int gs = gs0 + i;
        const int b = gs / d.stages_img, st = gs - b * d.stages_img;
        mbar_wait(&empty_bar[s], par ^ 1u);
        mbar_arrive_expect_tx(&full_bar[s], (uint32_t)nu * parts * 8192u + gbytes);
        uint8_t* stage = smem + s * k.stage_bytes;
        const uint8_t* src =
            cols + ((((size_t)b * d.tiles_img + (st >> 1)) * d.SG + sg) * d.U + 2 * mb) * tile_bytes + (size_t)(st & 1) * 8192;
        for (int ul = 0; ul < nu; ++ul)
          for (uint32_t part = 0; part < parts; ++part)
            bulk_g2s(stage + part * kTile + ul * 8192, src + (size_t)ul * tile_bytes + (size_t)part * kTile, 8192u, &full_bar[s]);
        const size_t tile = ((size_t)gs * d.SG + sg) * k.noct + oct;
        bulk_g2s(stage + 2 * kTile, gt + tile * (size_t)(2 * k.BN * 128), gbytes, &full_bar[s]);
      }
    }
  }
}

// grid (SG * noct, unit pairs, pixel splits)
template <int BN>
__global__ void __launch_bounds__(kThreads, 1) dcn_bwd_weight_cols_kernel(const uint8_t* __restrict__ cols,
                                                                          const uint8_t* __restrict__ gt, const TC d,
                                                                          const K3P k, const int S, const int split,
                                                                          float* __restrict__ gw) {
  bwd_weight_cols_body<BN, kSideRegs>(aligned_smem(), blockIdx.x, blockIdx.y, blockIdx.z, cols, gt, d, k, S, split, gw);
}

// ================================================================================================ fused backward: K2 + K3c
// One launch for a backward that wants both gradients from saved columns: the first N * tiles_img * SG * msplit CTAs of the
// 1-D grid run K2's body, the rest K3c's.  The two read only what the pre-passes wrote and write disjoint outputs, so the
// K3c CTAs fill the SMs that K2's grid leaves idle and its last wave runs beside K2's CTAs instead of after them.  K2's CTAs
// come first: they are the long ones.  Dynamic shared memory is the larger of the two bodies' needs.
template <int BN>
__global__ void __launch_bounds__(kThreads, 1) dcn_bwd_fused_kernel(const float* __restrict__ xh,
                                                                    const float* __restrict__ offset,
                                                                    const float* __restrict__ mask,
                                                                    const uint8_t* __restrict__ gt_px,
                                                                    const uint8_t* __restrict__ wt, const K2P k2,
                                                                    float* __restrict__ gxh, float* __restrict__ goff,
                                                                    float* __restrict__ gmask,
                                                                    const uint8_t* __restrict__ cols,
                                                                    const uint8_t* __restrict__ gt_oc, const K3P k3,
                                                                    const int S3, float* __restrict__ gw, const TC d,
                                                                    const int split) {
  const int nx2 = d.N * d.tiles_img, n2 = nx2 * d.SG * k2.msplit;
  int id = blockIdx.x;
  if (id < n2) {
    const int bx = id % nx2, r = id / nx2;
    bwd_data_body<kSideRegsMax>(aligned_smem(), bx, r % d.SG, r / d.SG, xh, offset, mask, gt_px, wt, d, k2, split, gxh, goff,
                                gmask);
  } else {
    id -= n2;
    const int nx3 = d.SG * k3.noct, r = id / nx3;
    bwd_weight_cols_body<BN, kSideRegsMax>(aligned_smem(), id % nx3, r % d.MC, r / d.MC, cols, gt_oc, d, k3, S3, split,
                                           gw);
  }
}

// ================================================================================================ operand pre-tiling
__device__ __forceinline__ void split8(const float (&v)[8], uint4& hi, uint4& lo) {
  split2(v[0], v[1], hi.x, lo.x);
  split2(v[2], v[3], hi.y, lo.y);
  split2(v[4], v[5], hi.z, lo.z);
  split2(v[6], v[7], hi.w, lo.w);
}

// weight element of (global output channel, global input channel, kernel point); 0 across original groups
__device__ __forceinline__ float w_elem(const float* __restrict__ w, const TC& d, int oc, int c, int kp) {
  const int g = c / d.cpg;
  if (oc / d.opg != g) return 0.f;
  return __ldg(w + ((size_t)oc * d.cpg + (c - g * d.cpg)) * d.KK + kp);
}

// K1 B tiles: [sg][oc tile][unit] -> [BN rows = oc][64 k' = channels of the unit], K-major swizzled, hi then lo
__global__ void dcn_wtile_fwd_kernel(const float* __restrict__ w, const TC d, int BN, int noct, uint8_t* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)d.SG * noct * d.U * BN * 8;
  if (idx >= total) return;
  const int c16 = (int)(idx & 7);
  const int r = (int)((idx >> 3) % BN);
  const long long tile = idx / (8LL * BN);
  const int u = (int)(tile % d.U);
  const int oct = (int)((tile / d.U) % noct);
  const int sg = (int)(tile / ((long long)d.U * noct));
  const int kp = u / d.cbs, cb = u - kp * d.cbs;
  const int oc = sg * d.ops + oct * BN + r;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = w_elem(w, d, oc, sg * d.cps + cb * 64 + c16 * 8 + e, kp);
  uint4 hi, lo;
  split8(v, hi, lo);
  uint8_t* base = dst + tile * (size_t)(2 * BN * 128);
  *reinterpret_cast<uint4*>(base + swz128((uint32_t)r, (uint32_t)c16)) = hi;
  *reinterpret_cast<uint4*>(base + BN * 128 + swz128((uint32_t)r, (uint32_t)c16)) = lo;
}

// K2 B tiles: [sg][macro-chunk][K stage] -> [128 rows = k' of the 2 units][64 oc of the stage], hi then lo
__global__ void dcn_wtile_bwd_kernel(const float* __restrict__ w, const TC d, uint8_t* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)d.SG * d.MC * d.nks * 128 * 8;
  if (idx >= total) return;
  const int c16 = (int)(idx & 7);
  const int r = (int)((idx >> 3) & 127);
  const long long tile = idx >> 10;
  const int ks = (int)(tile % d.nks);
  const int m = (int)((tile / d.nks) % d.MC);
  const int sg = (int)(tile / ((long long)d.nks * d.MC));
  const int u = 2 * m + (r >> 6);
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) v[e] = 0.f;
  if (u < d.U) {
    const int kp = u / d.cbs, cb = u - kp * d.cbs;
    const int c = sg * d.cps + cb * 64 + (r & 63);
#pragma unroll
    for (int e = 0; e < 8; ++e) v[e] = w_elem(w, d, sg * d.ops + ks * 64 + c16 * 8 + e, c, kp);
  }
  uint4 hi, lo;
  split8(v, hi, lo);
  uint8_t* base = dst + tile * (size_t)(2 * kTile);
  *reinterpret_cast<uint4*>(base + swz128((uint32_t)r, (uint32_t)c16)) = hi;
  *reinterpret_cast<uint4*>(base + kTile + swz128((uint32_t)r, (uint32_t)c16)) = lo;
}

// K2 A tiles: gout [N,Cout,HoWo] -> [b][pixel tile][sg][K stage] -> [128 rows = px][64 oc], hi then lo.  One CTA per tile.
// grad w.r.t. the convolution result when the forward ended in y = relu(acc * scale + shift)
__device__ __forceinline__ float gout_elem(const float* __restrict__ gout, const float* __restrict__ ysaved, const Epi& ep,
                                           size_t idx, int oc) {
  float g = __ldg(gout + idx);
  if (ep.relu && !(__ldg(ysaved + idx) > 0.f)) g = 0.f;
  if (ep.scale) g *= __ldg(ep.scale + oc);
  return g;
}

// Also writes the K3 B tiles (oc-row layout, see dcn_gout_oc_tiles_kernel) of the same elements when dst_oc != nullptr, so
// that a backward that needs both gradients reads grad_out once.
__global__ void __launch_bounds__(256) dcn_gout_px_tiles_kernel(const float* __restrict__ gout,
                                                                const float* __restrict__ ysaved, const Epi ep, const TC d,
                                                                uint8_t* __restrict__ dst, uint8_t* __restrict__ dst_oc,
                                                                int BN, int noct) {
  // grid (tiles, 4): a CTA converts 32 of the tile's 128 pixel rows -- 4x the CTAs of a tile-per-CTA layout, which matters for
  // the small maps (res5: 144 tiles on an H100 SXM's 132 SMs)
  __shared__ float t[64][33];
  const long long tile = blockIdx.x;
  const int ks = (int)(tile % d.nks);
  const int sg = (int)((tile / d.nks) % d.SG);
  const int pt = (int)((tile / ((long long)d.nks * d.SG)) % d.tiles_img);
  const int b = (int)(tile / ((long long)d.nks * d.SG * d.tiles_img));
  const int r0 = blockIdx.y * 32;
  const int p0 = pt * 128 + r0, oc0 = sg * d.ops + ks * 64;
  const int tid = threadIdx.x;
#pragma unroll
  for (int i = 0; i < 8; ++i) {  // 8 independent loads per thread: 32 pixels (one 128-byte run) of 64 channels
    const int e = tid + i * 256;
    const int o = e >> 5, pp = e & 31;
    const int p = p0 + pp;
    t[o][pp] = p < d.HoWo ? gout_elem(gout, ysaved, ep, ((size_t)b * d.Cout + oc0 + o) * d.HoWo + p, oc0 + o) : 0.f;
  }
  __syncthreads();
  uint8_t* base = dst + tile * (size_t)(2 * kTile);
  {
    const int r = tid >> 3, c16 = tid & 7;  // 32 rows x 8 chunks = 256 threads
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = t[c16 * 8 + i][r];
    uint4 hi, lo;
    split8(v, hi, lo);
    *reinterpret_cast<uint4*>(base + swz128((uint32_t)(r0 + r), (uint32_t)c16)) = hi;
    *reinterpret_cast<uint4*>(base + kTile + swz128((uint32_t)(r0 + r), (uint32_t)c16)) = lo;
  }
  if (dst_oc) {  // rows = output channels, 64-pixel stages: this CTA's 32 pixels are chunks [c0, c0 + 4) of one stage
    const int o = tid >> 2, ch = tid & 3;  // 64 channel rows x 4 chunks of 8 pixels
    const int ocs = ks * 64 + o;           // channel inside the super-group
    const int oct = ocs / BN, row = ocs - oct * BN;
    const int pglob = pt * 128 + r0;       // first pixel of this CTA inside the image
    const int ps = pglob >> 6, c16 = ((pglob & 63) >> 3) + ch;
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = t[o][ch * 8 + i];
    uint4 hi, lo;
    split8(v, hi, lo);
    if (ps < d.stages_img) {
      const size_t tile_oc = (((size_t)b * d.stages_img + ps) * d.SG + sg) * noct + oct;
      uint8_t* bo = dst_oc + tile_oc * (size_t)(2 * BN * 128);
      *reinterpret_cast<uint4*>(bo + swz128((uint32_t)row, (uint32_t)c16)) = hi;
      *reinterpret_cast<uint4*>(bo + BN * 128 + swz128((uint32_t)row, (uint32_t)c16)) = lo;
    }
  }
}

// K3 B tiles: gout -> [b][64-pixel stage][sg][oc tile] -> [BN rows = oc][64 px], K-major swizzled, hi then lo
__global__ void dcn_gout_oc_tiles_kernel(const float* __restrict__ gout, const float* __restrict__ ysaved, const Epi ep,
                                         const TC d, int BN, int noct, uint8_t* __restrict__ dst) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)d.N * d.stages_img * d.SG * noct * BN * 8;
  if (idx >= total) return;
  const int c16 = (int)(idx & 7);
  const int r = (int)((idx >> 3) % BN);
  const long long tile = idx / (8LL * BN);
  const int oct = (int)(tile % noct);
  const int sg = (int)((tile / noct) % d.SG);
  const int ps = (int)((tile / ((long long)noct * d.SG)) % d.stages_img);
  const int b = (int)(tile / ((long long)noct * d.SG * d.stages_img));
  const int oc = sg * d.ops + oct * BN + r;
  const size_t src = ((size_t)b * d.Cout + oc) * d.HoWo;
  float v[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int p = ps * 64 + c16 * 8 + e;
    v[e] = p < d.HoWo ? gout_elem(gout, ysaved, ep, src + p, oc) : 0.f;
  }
  uint4 hi, lo;
  split8(v, hi, lo);
  uint8_t* base = dst + tile * (size_t)(2 * BN * 128);
  *reinterpret_cast<uint4*>(base + swz128((uint32_t)r, (uint32_t)c16)) = hi;
  *reinterpret_cast<uint4*>(base + BN * 128 + swz128((uint32_t)r, (uint32_t)c16)) = lo;
}

// y = relu(y * scale + shift) in place: the forward's epilogue when the reduction was split over kernel points
__global__ void dcn_epilogue_kernel(float* __restrict__ y, long long total, int Cout, int HoWo, const Epi ep) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int oc = (int)((i / HoWo) % Cout);
  float v = y[i];
  if (ep.scale) v *= __ldg(ep.scale + oc);
  if (ep.shift) v += __ldg(ep.shift + oc);
  if (ep.relu) v = fmaxf(v, 0.f);
  y[i] = v;
}

// x and grad_x change layout through the library's pyramid layout change (roi_align.cu), as a one-level pyramid
int change_layout(const float* src, const TC& d, float* dst, bool to_nhwc, cudaStream_t stream) {
  d2b_pyramid P = {};
  P.num_levels = 1;
  P.feat[0] = src;
  P.H[0] = d.H;
  P.W[0] = d.W;
  P.scale[0] = 1.f;
  float* dsts[1] = {dst};
  return to_nhwc ? d2b_pyramid_nchw_to_nhwc(&P, d.N, d.Cin, dsts, D2B_F32, (void*)stream)
                 : d2b_pyramid_nhwc_to_nchw(&P, d.N, d.Cin, reinterpret_cast<void* const*>(dsts), D2B_F32, (void*)stream);
}

// Launches one of the warp-specialised kernels, which need more than 48 KB of dynamic shared memory.  Every kernel is its
// own instantiation, so each keeps its own opt-in record.
template <auto kernel, class... Args>
int launch_big_smem(dim3 grid, int smem_bytes, cudaStream_t stream, Args... args) {
  D2B_ALLOW_BIG_SMEM(kernel);
  kernel<<<grid, kThreads, smem_bytes, stream>>>(args...);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}

// The GEMM kernels are instantiated per output-channel tile width: calls launch(std::integral_constant<int, W>()) for the
// plan's width BN, W one of the widths the kernel is instantiated for (the last when BN is none of the others).
template <int W, int... More, class Launch>
int with_tile_width(int BN, Launch launch) {
  if constexpr (sizeof...(More) > 0)
    if (BN != W) return with_tile_width<More...>(BN, launch);
  return launch(std::integral_constant<int, W>());
}

}  // namespace

// ------------------------------------------------------------------------------------------------ host entry points
// 1 when the plan of the direction builds: the tensor-core kernels take the shape
D2B_API int d2b_deform_conv_tc_shape_supported(const d2b_dcn_params* p, int backward) {
  FwdPlan f;
  BwdPlan b;
  return backward ? plan_bwd(p, 1, 1, 1, 1, b) : plan_fwd(p, 1, 1, false, f);
}

// (library-internal, declared in deform_conv_tc.cuh for deform_conv.cu)
size_t d2b_deform_conv_tc_fwd_workspace(const d2b_dcn_params* p, int precision, int x_nhwc) {
  FwdPlan P;
  return plan_fwd(p, precision, x_nhwc, false, P) ? P.total : 0;
}

size_t d2b_deform_conv_tc_bwd_workspace(const d2b_dcn_params* p, int precision, int x_nhwc, int need_data, int need_weight) {
  BwdPlan P;
  return plan_bwd(p, precision, x_nhwc, need_data, need_weight, P) ? P.total : 0;
}

// the forward writes the columns and the backward reads them: 0 unless both plans build
size_t d2b_deform_conv_tc_cols_bytes(const d2b_dcn_params* p, int precision) {
  FwdPlan f;
  BwdPlan b;
  return plan_fwd(p, precision, 1, false, f) && plan_bwd(p, precision, 1, 0, 0, b) ? f.cols_bytes : 0;
}

// tcflags: bit 0 = x is NHWC, bit 1 = `offset` is the fused [N, 3*DG*KK, Ho, Wo] offset + mask-logit tensor (mask must be null)
// cols: optional, d2b_deform_conv_tc_cols_bytes() bytes, 16-byte aligned: receives the sampled columns (see the saver warp)
int d2b_deform_conv_forward_tc(const float* x, const float* offset, const float* mask, const float* weight,
                               const float* scale, const float* shift, int relu, const d2b_dcn_params* p, int precision,
                               int tcflags, float* out, void* cols, void* workspace, size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int x_nhwc = tcflags & 1;
  FwdPlan P;  // argument validity was checked by the caller
  if (!plan_fwd(p, precision, x_nhwc, cols != nullptr, P)) return D2B_EUNSUPPORTED;
  TC& d = P.d;
  const K1P& k = P.k1;
  if (d.N == 0) return D2B_OK;
  if (tcflags & 2) {
    if (mask) return D2B_EINVAL;
    mask = use_fused_offset_mask(d, offset);
  }
  if (!workspace || workspace_bytes < P.total) return D2B_EWORKSPACE;
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) || (x_nhwc && (reinterpret_cast<uintptr_t>(x) & 15)) ||
      (reinterpret_cast<uintptr_t>(cols) & 15))
    return D2B_EINVAL;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  uint8_t* wt = ws + P.wt;
  const float* xh = x;
  if (!x_nhwc) {
    float* xn = reinterpret_cast<float*>(ws + P.x);
    if (int rc = change_layout(x, d, xn, true, stream)) return rc;
    xh = xn;
  }
  {
    const long long total = (long long)d.SG * k.noct * d.U * k.BN * 8;
    dcn_wtile_fwd_kernel<<<d2b_cdiv(total, 256), 256, 0, stream>>>(weight, d, k.BN, k.noct, wt);
    D2B_CHECK_LAUNCH();
  }
  if (k.red) D2B_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)d.N * d.Cout * d.HoWo, stream));
  const Epi ep = {scale, shift, relu};
  const dim3 grid(d.N * d.tiles_img, d.SG * k.goct, k.ksplit);
  const int smem_bytes = k.S * k.stage_bytes + k.tap_bytes + 1024 + 128;
  int rc = with_tile_width<16, 32, 64, 128>(k.BN, [&](auto bn) {
    return launch_big_smem<dcn_fwd_tc_kernel<decltype(bn)::value>>(grid, smem_bytes, stream, xh, offset, mask, wt, ep, d, k,
                                                                    P.split, out, reinterpret_cast<uint8_t*>(cols));
  });
  if (rc) return rc;
  if (P.colfed) {
    const K1P& kc = P.kc;
    const dim3 grid_c(d.N * d.tiles_img * kc.goct, d.SG, kc.ksplit);
    const int smem_c = kc.S * kc.stage_bytes + 1024 + 128;
    const uint8_t* cl = reinterpret_cast<const uint8_t*>(cols);
    rc = with_tile_width<16, 32, 64, 128>(kc.BN, [&](auto bn) {
      return launch_big_smem<dcn_fwd_cols_kernel<decltype(bn)::value>>(grid_c, smem_c, stream, cl, wt, ep, d, kc, P.split,
                                                                        out);
    });
    if (rc) return rc;
  }
  if (k.red && (scale || relu)) {
    const long long total = (long long)d.N * d.Cout * d.HoWo;
    dcn_epilogue_kernel<<<d2b_cdiv(total, 256), 256, 0, stream>>>(out, total, d.Cout, d.HoWo, ep);
    D2B_CHECK_LAUNCH();
  }
  return D2B_OK;
}

// grad_x: NCHW (or NHWC when x_nhwc) fully written; grad_offset / grad_mask / grad_weight fully written.
// With the fused offset + mask-logit tensor (tcflags bit 1) grad_offset is its [N, 3*DG*KK, Ho, Wo] gradient (mask part through
// the sigmoid) and grad_mask must be null.  scale / y_saved / relu: transpose of the forward's epilogue.
int d2b_deform_conv_backward_tc(const float* x, const float* offset, const float* mask, const float* weight,
                                const float* grad_out, const float* scale, const float* y_saved, int relu,
                                const d2b_dcn_params* p, int precision, int tcflags, const void* cols, float* grad_x,
                                float* grad_offset, float* grad_mask, float* grad_weight, void* workspace,
                                size_t workspace_bytes, void* stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  const int x_nhwc = tcflags & 1;
  const int need_data = (grad_x || grad_offset || grad_mask) ? 1 : 0, need_weight = grad_weight ? 1 : 0;
  BwdPlan P;
  if (!plan_bwd(p, precision, x_nhwc, need_data, need_weight, P)) return D2B_EUNSUPPORTED;
  TC& d = P.d;
  const K2P& k2 = P.k2;
  const K3P& k3 = P.k3;
  const bool fused_om = (tcflags & 2) != 0;
  if (fused_om && (mask || grad_mask)) return D2B_EINVAL;
  if (relu && !y_saved) return D2B_EINVAL;
  const size_t nx = (size_t)d.N * d.H * d.W * d.Cin, noff = (size_t)d.N * d.DG * (fused_om ? 3 : 2) * d.KK * d.HoWo;
  const size_t nm = (size_t)d.N * d.DG * d.KK * d.HoWo, nw = (size_t)d.Cout * d.cpg * d.KK;
  if (fused_om) {
    mask = use_fused_offset_mask(d, offset);
    if (grad_offset) grad_mask = grad_offset + (size_t)d.DG * 2 * d.KK * d.HoWo;
  }
  const Epi ep = {scale, nullptr, relu};
  if (d.N == 0 || (!need_data && !need_weight)) {
    void* zp[3] = {grad_offset, fused_om ? nullptr : grad_mask, grad_weight};
    size_t zb[3] = {noff * 4, nm * 4, nw * 4};
    return d2b_zero_buffers(zp, zb, 3, stream);
  }
  if (!workspace || workspace_bytes < P.total) return D2B_EWORKSPACE;
  if ((reinterpret_cast<uintptr_t>(workspace) & 255) || (x_nhwc && (reinterpret_cast<uintptr_t>(x) & 15)) ||
      (x_nhwc && grad_x && (reinterpret_cast<uintptr_t>(grad_x) & 15)) || (reinterpret_cast<uintptr_t>(cols) & 15))
    return D2B_EINVAL;
  uint8_t* ws = reinterpret_cast<uint8_t*>(workspace);
  const float* xh = x;
  if (!x_nhwc) {
    float* xn = reinterpret_cast<float*>(ws + P.x);
    if (int rc = change_layout(x, d, xn, true, stream)) return rc;
    xh = xn;
  }
  float* gxh = grad_x ? (x_nhwc ? grad_x : reinterpret_cast<float*>(ws + P.gx)) : nullptr;
  uint8_t* gt_oc = need_weight ? ws + P.gt_oc : nullptr;
  float* gw_part = need_weight ? reinterpret_cast<float*>(ws + P.gw) : nullptr;
  {  // every accumulated output of the call zero-filled by one launch (grad_mask of the fused layout lives inside grad_offset;
    // grad_weight is accumulated in the staging matrix and then written element by element)
    void* zp[4] = {grad_offset, fused_om ? nullptr : grad_mask, gxh, gw_part};
    size_t zb[4] = {noff * 4, nm * 4, nx * 4, P.gw_bytes};
    int rc = d2b_zero_buffers(zp, zb, 4, stream);
    if (rc) return rc;
  }
  // With saved columns and both gradients wanted, K2 and K3c run as one launch (dcn_bwd_fused_kernel) on a 1-D grid.
  const long long fused_ctas = (long long)d.N * d.tiles_img * d.SG * k2.msplit + (long long)d.SG * k3.noct * d.MC * k3.nsplit;
  const bool fused = need_data && need_weight && cols && fused_ctas <= 0x7fffffffLL;
  const uint8_t* cl = reinterpret_cast<const uint8_t*>(cols);
  const int S3 = std::min(6, (kMaxSmem - 2048) / k3.stage_bytes);  // K3c's operand ring
  const int smem3 = S3 * k3.stage_bytes + 1024 + 128;
  if (need_data) {
    uint8_t* gt_px = ws + P.gt_px;
    uint8_t* wt = ws + P.wt;
    // grad_out is read once: pixel-row tiles for K2 and (when the weight gradient is wanted too) channel-row tiles for K3
    dcn_gout_px_tiles_kernel<<<dim3((unsigned)((size_t)d.N * d.tiles_img * d.SG * d.nks), 4), 256, 0, stream>>>(
        grad_out, y_saved, ep, d, gt_px, gt_oc, k3.BN, k3.noct);
    D2B_CHECK_LAUNCH();
    {
      const long long total = (long long)d.SG * d.MC * d.nks * 128 * 8;
      dcn_wtile_bwd_kernel<<<d2b_cdiv(total, 256), 256, 0, stream>>>(weight, d, wt);
      D2B_CHECK_LAUNCH();
    }
    const int smem2 = 2 * 4 * kTile + 128 * kGcolPitch * 4 + k2.tap_bytes + 1024 + 128;
    float* gm = mask ? grad_mask : nullptr;
    int rc;
    if (fused) {
      rc = with_tile_width<64, 128>(k3.BN, [&](auto bn) {
        return launch_big_smem<dcn_bwd_fused_kernel<decltype(bn)::value>>(
            dim3((unsigned)fused_ctas), std::max(smem2, smem3), stream, xh, offset, mask, gt_px, wt, k2, gxh, grad_offset, gm,
            cl, gt_oc, k3, S3, gw_part, d, P.split);
      });
    } else {
      rc = launch_big_smem<dcn_bwd_data_tc_kernel>(dim3(d.N * d.tiles_img, d.SG, k2.msplit), smem2, stream, xh, offset, mask,
                                                   gt_px, wt, d, k2, P.split, gxh, grad_offset, gm);
    }
    if (rc) return rc;
    if (grad_x && !x_nhwc) {
      if (int rc = change_layout(gxh, d, grad_x, false, stream)) return rc;
    }
  }
  if (need_weight) {
    if (!need_data) {
      const long long total = (long long)d.N * d.stages_img * d.SG * k3.noct * k3.BN * 8;
      dcn_gout_oc_tiles_kernel<<<d2b_cdiv(total, 256), 256, 0, stream>>>(grad_out, y_saved, ep, d, k3.BN, k3.noct, gt_oc);
      D2B_CHECK_LAUNCH();
    }
    if (!fused) {  // (the fused launch ran the weight gradient's CTAs already)
      // output-channel tile fastest, then the unit pair: the CTAs that read one column (or gathered) tile and those that read
      // one grad_out tile run in the same wave and share them in L2
      const dim3 grid(d.SG * k3.noct, d.MC, k3.nsplit);
      int rc;
      if (cols) {  // the forward kept its sampled columns: stream them back (no second pass over x)
        rc = with_tile_width<64, 128>(k3.BN, [&](auto bn) {
          return launch_big_smem<dcn_bwd_weight_cols_kernel<decltype(bn)::value>>(grid, smem3, stream, cl, gt_oc, d, k3, S3,
                                                                                   P.split, gw_part);
        });
      } else {
        const int smem_bytes = k3.S * k3.stage_bytes + 4096 + 1024 + 128;
        rc = with_tile_width<64, 128>(k3.BN, [&](auto bn) {
          return launch_big_smem<dcn_bwd_weight_tc_kernel<decltype(bn)::value>>(grid, smem_bytes, stream, xh, offset, mask,
                                                                                 gt_oc, d, k3, P.split, gw_part);
        });
      }
      if (rc) return rc;
    }
    if (d.KK <= 9) {  // d.ops is a multiple of 16 (shape gate)
      dcn_gw_reduce_tile_kernel<<<dim3(d.SG * (d.cps / kRedCh), d.ops / kRedOc), 256, 0, stream>>>(gw_part, d, grad_weight);
    } else {
      const long long total = (long long)d.SG * d.U * 64 * d.ops;
      dcn_gw_reduce_kernel<<<d2b_cdiv(total, 256), 256, 0, stream>>>(gw_part, d, grad_weight);
    }
    D2B_CHECK_LAUNCH();
  }
  return D2B_OK;
}

