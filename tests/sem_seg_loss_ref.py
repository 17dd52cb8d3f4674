"""Float64 reference of the semantic segmentation loss (detectron2_b200/csrc/sem_seg_loss.cu), its error bounds and its path
model.

Reference.  F.interpolate(logits.float(), scale_factor=stride, mode="bilinear", align_corners=False) followed by the
per-pixel cross-entropy, in torch float64 on the CPU or on CUDA.  The taps are part of the operation: PyTorch's CUDA source
index with the fp32 scale (float)(1.0 / stride), r = fp32(scale * (d + 0.5) - 0.5) clamped at 0, i0 = (int)r, i1 = i0 + 1
clamped at in - 1, l1 = r - i0 (exact), l0 = fp32(1 - l1).  In float64 the product of two fp32 numbers and the subtraction
are exact at these sizes, so one rounding to fp32 reproduces the fused multiply-add.  At odd strides this matters: at
stride 3 and d = 1 the fp32 index is 1.49e-8, not 0, so row 1 gets a weight that exact arithmetic gives it none.  The
upsampled value is l0y (l0x a + l1x b) + l1y (l0x d + l1x e), gathered (not a dense matrix product), so that a zero weight
times a non-finite logit is NaN where PyTorch's and the kernel's are.  Everything after the taps is float64: logsumexp as
log_softmax writes it (max, then log of the sum of exp(v - max): NaN when a channel is +inf), ignore / bad-label skipping,
weights, the mean, top-k 1.0 and the top-k sum over a given selection.  Gradients are autograd of that forward.

Error bounds.  The tracker `T` and `sum_bound` come from tests/box_loss_ref.py: u = 2^-24 per fp32 rounding,
TINY per rounding for underflow, SELF for float64's own rounding.  sem_seg_loss.cu is compiled with -fmad=false and uses
two fast intrinsics, whose maximum errors the CUDA C++ Programming Guide tabulates ("Intrinsic Functions"):
    __expf(x)   "The maximum ulp error is 2 + floor(abs(1.173 * x))"
    __logf(x)   "For x in [0.5, 2], the maximum absolute error is 2^-21.41, otherwise, the maximum ulp error is 3."
__expf flushes results below 2^-126 to 0, which adds 2^-126 absolute.
  * Upsampled value: four fp32 roundings (two products, two FMAs) on the worst path of a tap, each within u of a partial
    sum bounded by M = sum of |tap weight * logit|: e_v = 4 u (1 + 8 u) M.  Stride 1 is a copy: exact.
  * lse: the online logsumexp is compared with the exact logsumexp of the kernel's own values v~ (1-Lipschitz: within
    max_c e_v of the reference's).  Its sum s carries, relative: per rescale of the running max 2 ulp + 1 rounding of the
    product, plus (1.173 ulp + u) |gap| summed over the gaps (at most the range R of the pixel's values); the term's own
    __expf (2 + 1.173 R) ulp + u R; the C additions C u.  A rescale is counted for every channel that may raise the running
    max.  Then log(1 + theta), the __logf bound, and the final rounding.
  * loss = lse - v_t, x = loss * w: one rounding each.
  * Sums: fp32 per thread over kPixPerThread = 4 pixels, 5 butterfly levels and 8 warps in order, double over the CTA
    partials in the 1024-thread tree, one fp32 rounding: sum_bound(terms, errs, 4, nb).  Top-k adds (k - #{x > t}) * t in
    double, which is the sum of the tied selected values.
  * Backward: p = __expf(v - lse), D = g (p - [t = c]) with g = fp32(grad_sum * w), then per logit an FMA chain over the
    columns of each row (weight sums wx rounded) and one over the rows (wy rounded): gamma_n (|D| + e_D) with n = rows +
    columns + 2 of the logit, carried back through the transposed taps.
Top-k selection is decided for a pixel when its value is provably among (or outside) the k largest: lo(p) = x - e above
the (k+1)-th largest hi = x + e, or hi(p) below the k-th largest lo.  NaN ranks above +inf, as torch.topk orders it.

Path model.  `fwd_paths` restates the forward's launch arithmetic (kChunk = 1024 pixels per CTA, nb CTAs, the finish and
tie-prefix loops over 1024 partials per pass, 4 radix levels); `bwd_plan` restates the backward's tiling (tile side T,
region bounds RBY / RBX, channels per CTA CC, channel chunks, shared memory).  `shape_labels` turns a call's shapes into
the paths it reaches; the GPU test adds the labels its values reach.
"""
import math

import torch

from box_loss_ref import SELF, TINY, U, ULP, T, f32, sum_bound

F64 = torch.float64
K_CHUNK = 1024
K_FINISH = 1024
K_LEVELS = 4
SMEM_TARGET = 100 * 1024
SMEM_OPTIN = 227 * 1024
SMEM_TWO_PER_SM = 114 * 1024
MAX_STRIDE = 32
FTZ = 2.0 ** -126
LOGF_ABS = 2.0 ** -21.41
STATUS_BAD_LABEL = 1


# ---- taps and the upsampling ----------------------------------------------------------------------------------------
def taps(stride, out_size, in_size, device="cpu"):
    """(i0, i1, l0, l1) of output rows 0 .. out_size - 1: long indices, float64 weights that are fp32 numbers."""
    d = torch.arange(out_size, dtype=F64, device=device)
    if stride == 1:
        i = d.long()
        return i, i, torch.ones_like(d), torch.zeros_like(d)
    scale = f32(1.0 / stride)
    r = (scale * (d + 0.5) - 0.5).to(torch.float32).to(F64).clamp_min(0.0)
    i0 = r.floor().long()
    i1 = i0 + (i0 < in_size - 1).long()
    l1 = r - i0
    l0 = (1.0 - l1).to(torch.float32).to(F64)
    return i0, i1, l0, l1


def upsample(x, stride):
    """x [N, C, Hp, Wp] float64 -> [N, C, Hp * stride, Wp * stride]: the gathered bilinear taps (autograd flows)."""
    if stride == 1:
        return x
    hp, wp = x.shape[-2:]
    y0, y1, a0, a1 = taps(stride, hp * stride, hp, x.device)
    x0, x1, b0, b1 = taps(stride, wp * stride, wp, x.device)
    r0, r1 = x[:, :, y0], x[:, :, y1]
    top = r0[..., x0] * b0 + r0[..., x1] * b1
    bot = r1[..., x0] * b0 + r1[..., x1] * b1
    return top * a0[:, None] + bot * a1[:, None]


def upsample_adjoint(e, stride, hp, wp):
    """The transpose of `upsample` applied to e [N, C, H, W] >= 0: per logit, the tap-weighted sum over its output pixels."""
    if stride == 1:
        return e
    with torch.enable_grad():
        x = torch.zeros(e.shape[:2] + (hp, wp), dtype=F64, device=e.device, requires_grad=True)
        (g,) = torch.autograd.grad(upsample(x, stride), x, grad_outputs=e)
    return g


def taps_per_logit(stride, in_size):
    """The most output rows whose taps reach one low-res row (zero weights included): the FMA chain length per axis."""
    i0, i1, _, _ = taps(stride, in_size * stride, in_size)
    hit = torch.zeros(in_size, dtype=torch.long)
    hit.index_add_(0, i0, torch.ones_like(i0))
    hit.index_add_(0, i1, (i1 != i0).long())
    return int(hit.max())


# ---- the float64 reference and its bounds ---------------------------------------------------------------------------
def _lse(v):
    """log_softmax's logsumexp over dim 1: NaN when a channel is NaN or +inf."""
    m = v.detach().amax(1, keepdim=True)
    return (m + torch.log(torch.exp(v - m).sum(1, keepdim=True)))[:, 0]


def fast_exp(t):
    """__expf of a tracked argument (v may be -inf with e = 0: exactly 0)."""
    v = torch.exp(t.v)
    hi, lo = torch.exp(t.v + t.e), torch.exp(t.v - t.e)
    ulps = 2.0 + torch.floor(1.173 * (t.v.abs() + t.e))
    e = torch.maximum(hi - v, v - lo) + ulps * ULP * hi + FTZ + TINY
    return T(v, torch.where(t.v == -math.inf, 0.0, e))


class Ref:
    """The float64 reference of one call, its bounds, and the path labels its values reach.

    logits [N, C, Hp, Wp] (any float dtype: converted to fp32 first), targets [N, H, W] int64, weights [N, H, W] fp32 or
    None, top_k None (mean) / 1.0 / a fraction.  `grad(selected, grad_sum)` gives the reference gradient of
    grad_sum * loss_sum over the given selection (None: every valid pixel) and its per-element bound."""

    def __init__(self, logits, targets, stride, ignore, top_k=None, weights=None):
        self.stride, self.ignore, self.top_k = stride, ignore, top_k
        self.dev = logits.device
        x32 = logits.float()
        self.x = x32.to(F64)
        self.N, self.C, self.Hp, self.Wp = x32.shape
        P = targets.numel()
        self.P = P
        self.mode = "mean" if top_k is None else "all" if top_k == 1.0 else "select"
        self.k = 0 if top_k is None else P if top_k == 1.0 else int(top_k * P)
        t = targets.to(self.dev, torch.int64)
        self.t = t
        in_range = (t >= 0) & (t < self.C)
        self.valid = (t != ignore) & in_range
        self.status = STATUS_BAD_LABEL if bool(((t != ignore) & ~in_range).any()) else 0
        self.count = int(self.valid.sum())
        self.w = None if weights is None else weights.to(self.dev, torch.float32).to(F64)
        self.tc = torch.where(self.valid, t, 0)
        with torch.no_grad():
            v = upsample(self.x, stride)
            ev = torch.zeros_like(v) if stride == 1 else 4 * U * (1 + 8 * U) * upsample(self.x.abs(), stride)
            ev = torch.where(torch.isfinite(v), ev, 0.0)
            self.v, self.ev = v, ev
            self._forward_bounds()

    def _forward_bounds(self):
        v, ev, C = self.v, self.ev, self.C
        fin = torch.isfinite(v)
        vm = torch.where(fin, v, -math.inf)
        m = vm.amax(1)
        vmin = torch.where(fin, v, math.inf).amin(1)
        evm = ev.amax(1)
        R = torch.where(m > -math.inf, m - vmin, 0.0) + 2 * evm
        prev = torch.cat([torch.full_like(vm[:, :1], -math.inf), vm.cummax(1).values[:, :-1]], 1)
        resc = ((vm + 2 * evm[:, None] >= prev) & fin & (prev > -math.inf)).sum(1).to(F64)
        rho = resc * (2 * ULP + 2 * U) + (1.173 * ULP + U) * R + (2 + 1.173 * R) * ULP + U * R + C * U + C * FTZ
        theta = torch.expm1(rho)
        lse = _lse(v)
        s_hi = torch.exp(lse - m + 2 * evm) * (1 + theta)
        e_log = -torch.log1p(-theta) + torch.clamp_min(3 * ULP * torch.log(s_hi).abs(), LOGF_ABS)
        e_lse = evm + e_log
        e_lse = e_lse + U * (lse.abs() + e_lse) + TINY
        okl = torch.isfinite(lse) & self.valid
        self.lse = torch.where(self.valid, lse, 0.0)
        self.e_lse = torch.where(okl, e_lse, 0.0) * SELF
        vt = v.gather(1, self.tc[:, None])[:, 0]
        evt = ev.gather(1, self.tc[:, None])[:, 0]
        loss = torch.where(self.valid, lse - vt, 0.0)
        e_loss = self.e_lse + evt
        e_loss = e_loss + U * (loss.abs() + e_loss) + TINY
        self.loss = loss
        self.e_loss = torch.where(torch.isfinite(loss) & self.valid, e_loss, 0.0) * SELF
        if self.w is None:
            self.xv, self.ex = loss, self.e_loss
        else:
            xv = loss * self.w
            self.xv = xv
            self.ex = torch.where(torch.isfinite(xv),
                                  self.w.abs() * self.e_loss + U * (xv.abs() + self.w.abs() * self.e_loss) + TINY, 0.0)

    # -- sums and the selection --
    def nb(self):
        return -(-self.P // K_CHUNK)

    def loss_sum(self, selected=None):
        """(float64 sum, bound) of what the kernel adds: every valid loss (mean), every x (top-k 1.0), or the x of the
        selected pixels."""
        if self.mode == "mean":
            keep = self.valid
            terms, errs = self.loss[keep], self.e_loss[keep]
        elif self.mode == "all":
            terms, errs = self.xv.reshape(-1), self.ex.reshape(-1)
        else:
            keep = selected.reshape(-1).bool()
            terms, errs = self.xv.reshape(-1)[keep], self.ex.reshape(-1)[keep]
        if terms.numel() == 0:
            return 0.0, 0.0
        return float(terms.sum()), sum_bound(terms, errs, 4, self.nb())

    def decided(self):
        """(above, below): pixels that must be / must not be among the k largest of the kernel's values."""
        x = self.xv.reshape(-1)
        e = self.ex.reshape(-1)
        big = 1e300
        key = torch.where(torch.isnan(x), math.inf, torch.where(torch.isinf(x), x.sign() * big, x))
        lo, hi = key - e, key + e
        k, P = self.k, self.P
        hs = torch.sort(hi, descending=True).values
        ls = torch.sort(lo, descending=True).values
        h_k1 = hs[k] if k < P else torch.tensor(-math.inf, dtype=F64, device=x.device)
        l_k = ls[k - 1] if k > 0 else torch.tensor(math.inf, dtype=F64, device=x.device)
        return lo > h_k1, hi < l_k

    # -- the gradient --
    def use(self, selected=None):
        u = self.valid
        if selected is not None and selected.numel():
            u = u & selected.to(self.dev).bool()
        return u

    def grad(self, selected=None, grad_sum=1.0):
        """(reference gradient [N, C, Hp, Wp] float64, bound, reached): grad_sum * d loss_sum / d logits over the pixels
        in `use(selected)`; `reached` marks the logits a used pixel's taps reach."""
        gs = f32(grad_sum)
        use = self.use(selected)
        x = self.x.clone().requires_grad_(True)
        v = upsample(x, self.stride)
        v = torch.where(use[:, None], v, 0.0)
        lse = _lse(v)
        loss = lse - v.gather(1, self.tc[:, None])[:, 0]
        if self.w is not None:
            loss = loss * self.w
        total = torch.where(use, loss, 0.0).sum() * gs
        (g,) = torch.autograd.grad(total, x)
        with torch.no_grad():
            ok = use & torch.isfinite(self.lse)
            arg = self.v - self.lse[:, None]
            e_arg = self.ev + self.e_lse[:, None]
            e_arg = torch.where(torch.isfinite(arg), e_arg + U * (arg.abs() + e_arg), 0.0)
            p = fast_exp(T(torch.where(ok[:, None], arg, -math.inf), torch.where(ok[:, None], e_arg, 0.0)))
            onehot = torch.arange(self.C, device=self.dev)[None, :, None, None] == self.tc[:, None]
            q_v = p.v - onehot.to(F64)
            e_q = p.e + torch.where(onehot, U * (q_v.abs() + p.e), 0.0)
            if self.w is None:
                gv, e_g = torch.full_like(self.lse, gs), torch.zeros_like(self.lse)
            else:
                gv = gs * self.w
                e_g = U * gv.abs() + TINY
            gv, e_g = torch.where(ok, gv, 0.0)[:, None], torch.where(ok, e_g, 0.0)[:, None]
            d_v = gv * q_v
            e_d = gv.abs() * e_q + q_v.abs() * e_g + e_g * e_q
            e_d = torch.where(ok[:, None], e_d + U * (d_v.abs() + e_d) + TINY, 0.0)
            d_v = torch.where(ok[:, None], d_v, 0.0)
            e_d = torch.where(torch.isfinite(e_d), e_d, 0.0)
            d_v = torch.where(torch.isfinite(d_v), d_v, 0.0)
            n = taps_per_logit(self.stride, self.Hp) + taps_per_logit(self.stride, self.Wp) + 2
            gam = n * U / (1 - n * U)
            e_grid = e_d * (1 + gam) + gam * d_v.abs() + n * TINY * ok[:, None]
            bound = upsample_adjoint(e_grid, self.stride, self.Hp, self.Wp) * SELF
            reach = upsample_adjoint(ok[:, None].expand(-1, self.C, -1, -1).to(F64), self.stride, self.Hp, self.Wp) > 0
        return g, bound, reach


# ---- the kernel's exact per-pixel values and its selection rule -----------------------------------------------------
def order_keys(x32):
    """order_key() of sem_seg_loss.cu as int64: every NaN above +inf, -0.0 and +0.0 one key."""
    x = torch.where(x32 == 0, torch.zeros_like(x32), x32)
    u = x.view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    k = torch.where(u >= 2 ** 31, (~u) & 0xFFFFFFFF, u | 2 ** 31)
    return torch.where(torch.isnan(x32), 0xFFFFFFFF, k)


def select_top_k(x32, k):
    """The documented selection of the k largest fp32 values: ties taken in ascending flat index."""
    keys = order_keys(x32.reshape(-1))
    sel = torch.zeros(keys.numel(), dtype=torch.uint8, device=keys.device)
    if k:
        sel[torch.sort(keys, descending=True, stable=True).indices[:k]] = 1
    return sel.view(x32.shape)


# ---- the path model -------------------------------------------------------------------------------------------------
def bwd_smem(T_, rby, rbx, cc):
    rbq = rby * rbx
    return cc * rbq * 4 + rbq * 12 + (rby + rbx) * 16 + T_ * 16


def bwd_plan(C, Hp, Wp, stride):
    """bwd_plan() of sem_seg_loss.cu: dict(T, RBY, RBX, CC, nchunks, smem, rb) (rb: the unclamped region bound)."""
    T_ = max(2, 32 // stride)
    rb = (T_ + 1) * stride + 2
    rby, rbx = min(rb, Hp * stride), min(rb, Wp * stride)
    fixed, per = bwd_smem(T_, rby, rbx, 0), rby * rbx * 4
    cc = (SMEM_TARGET - fixed) // per if SMEM_TARGET > fixed + per else 1
    cc = max(1, min(cc, C))
    return dict(T=T_, RBY=rby, RBX=rbx, CC=cc, nchunks=-(-C // cc), smem=bwd_smem(T_, rby, rbx, cc), rb=rb)


def fwd_paths(N, Hp, Wp, stride):
    P = N * Hp * stride * Wp * stride
    nb = -(-P // K_CHUNK)
    return dict(P=P, nb=nb, passes=-(-nb // K_FINISH))


def region_spare(stride, size):
    """Least spare rows (rb - true region) over the tiles of one axis of `size` low-res rows."""
    i0, i1, _, _ = taps(stride, size * stride, size)
    T_ = max(2, 32 // stride)
    rb = (T_ + 1) * stride + 2
    spare = rb
    for y0 in range(0, size, T_):
        y1 = min(y0 + T_, size)
        lo = int(torch.searchsorted(i1, torch.tensor(y0)))
        hi = int(torch.searchsorted(i0, torch.tensor(y1)))
        spare = min(spare, rb - (hi - lo))
    return spare


def shape_labels(N, C, Hp, Wp, stride, dtype, top_k):
    """The kernel paths a call's shapes reach."""
    out = set()
    f = fwd_paths(N, Hp, Wp, stride)
    b = bwd_plan(C, Hp, Wp, stride)
    if stride == 1:
        out.add("stride1_copy")
    elif f32(1.0 / stride) != 1.0 / stride:
        out.add("odd_stride_fp32_taps")
    if stride > 1:
        out.add("last_logit_both_taps")
    if b["T"] == 2 and b["CC"] == 1:
        out.add("T2_cc1")
    if b["smem"] > SMEM_TWO_PER_SM:
        out.add("smem_one_cta_per_sm")
    if Hp % b["T"] or Wp % b["T"]:
        out.add("ragged_tile")
    if Hp < b["T"] or Wp < b["T"]:
        out.add("map_smaller_than_tile")
    if b["RBY"] < b["rb"] or b["RBX"] < b["rb"]:
        out.add("region_clamped_to_map")
    if stride > 1 and min(region_spare(stride, Hp), region_spare(stride, Wp)) <= 1:
        out.add("region_spare_1")
    out.add("single_chunk" if b["nchunks"] == 1 else "multi_chunk")
    if C % b["CC"] and b["nchunks"] > 1:
        out.add("ragged_channel_chunk")
    if f["P"] % K_CHUNK:
        out.add("tail_cta")
    if N > 1 and (f["P"] // N) % K_CHUNK:
        out.add("image_boundary_in_cta")
    if f["passes"] > 1:
        out.add("finish_multi_pass")
        if top_k is not None and top_k != 1.0 and int(top_k * f["P"]) > 0:
            out.add("tie_prefix_multi_pass")
    if top_k is None:
        out.add("mean")
    elif top_k == 1.0:
        out.add("top_k_all")
    else:
        k = int(top_k * f["P"])
        out.add("select_k0" if k == 0 else "select_k1" if k == 1 else "select")
    if dtype == torch.float16:
        out.add("f16")
    if dtype == torch.bfloat16:
        out.add("bf16")
    return out


SHAPE_LABELS = {"stride1_copy", "odd_stride_fp32_taps", "last_logit_both_taps", "T2_cc1", "smem_one_cta_per_sm",
                "ragged_tile", "map_smaller_than_tile", "region_clamped_to_map", "region_spare_1", "single_chunk",
                "multi_chunk", "ragged_channel_chunk", "tail_cta", "image_boundary_in_cta", "finish_multi_pass",
                "tie_prefix_multi_pass", "mean", "top_k_all", "select", "select_k0", "select_k1", "f16", "bf16"}
# reached by the values of a call: asserted by the GPU test, which sees the kernel's own per-pixel values
VALUE_LABELS = {"threshold_zero_with_ignored_ties", "threshold_nan", "radix_level_3_decides", "ties_split_at_threshold",
                "ignore_in_class_range", "bad_label", "all_ignored", "weights_zero_or_negative", "pos_inf_logit",
                "neg_inf_logit", "nan_logit", "exp_underflow"}
