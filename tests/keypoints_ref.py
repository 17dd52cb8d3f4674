"""Float64 reference of the keypoint head kernels (detectron2_b200/csrc/keypoints.cu), their error bounds and path model.

Decoding.  Per output column (and row) d of a ceil(w) x ceil(h) resize of an S x S map, the taps restate the kernel's fp32
arithmetic, which is PyTorch's upsample_bicubic2d (align_corners=False): scale = fp32(S / out), real = fma(scale, d + 0.5,
-0.5), in = floor(real), t = fp32(real - in), source indices in - 1 .. in + 2 clamped to [0, S - 1].  Python has no fma:
scale * (d + 0.5) is exact in float64 (two fp32 numbers), the float64 addition of -0.5 is checked to be exact (TwoSum), so
one rounding to fp32 is the fused operation.  The A = -0.75 cubic coefficients are evaluated in float64 from the fp32 t.
The reference value of a pixel is the float64 gathered separable sum over those 4 x 4 taps (gathered, so that a zero tap
weight times a non-finite value is NaN as in PyTorch and the kernel); a same-size resize is PyTorch's copy.

Bound.  `T` and the form of `sum_bound` come from tests/box_loss_ref.py (u = 2^-24 per fp32 rounding, TINY for underflow, SELF for
float64's own rounding); `fma` adds a fused multiply-add with one rounding.  The tracker carries the kernel's sequence:
conv1(x) = fma(fma(1.25, x, -2.25) * x, x, 1), conv2(x) = fma(fma(fma(-0.75, x, 3.75), x, -6), x, 3), c0 = conv2(t + 1),
c1 = conv1(t), c2 = conv1(1 - t), c3 = conv2((1 - t) + 1) (the coefficients' errors are measured against the exact
polynomials of the fp32 t), and the four-tap sums fma(x3, c3, fma(x2, c2, fma(x0, c0, x1 * c1))), first along each of the
S source rows, then down the columns.  The result is a bound per output pixel.

Score.  1 / sum_i exp(m_i - L) over the S x S map, L the kernel's reported logit (the map value at its pixel).  Each term
is one fp32 subtraction and expf (2 ulp); one lane adds ceil(S^2 / 32) terms in order, then 5 butterfly levels; the
division rounds once.  A sum past FLT_MAX is inf in fp32 and the score 0: an absolute 2^-126 covers it and subnormal
scores.  Position: (ox + 0.5) * cw + x1 in fp32 from the pixel, bit for bit.

Loss.  The per-row loss is float64 logsumexp(x) - x_t of the fp32 up-cast logits, with log_softmax's NaN rule (NaN when a
logit is NaN or +inf); the gradient is autograd of that forward times grad_scale.  The kernel's sequence: m = max (exact),
expf(x - m) per term, ceil(S^2 / 256) terms per thread then 5 shuffle levels and 8 warps in order (sum_bound's + 13,
here per row), logf (1 ulp), x_t - m and the final subtraction one rounding each; the gradient ((p / sum) - onehot) * grad_scale rounds
the division, the subtraction and the product once each.

Targets.  The exact cell floor((c - x1) S / (x2 - x1)) as a Fraction of the fp32 inputs.  The kernel's (and PyTorch's)
sequence rcp(x2 - x1) * S, (c - x1) * that, four roundings, is within 4u (1 + 4u) relative of it when every step is a
normal finite number; a cell is *decided* when that interval holds no integer other than at an exact 0.

Path model.  `decode_paths` restates the decode's launch arithmetic (kTile = 4096 pixels, tiles per ROI, the copy flag,
shared memory S^2 * 4 against 48 KB and the 227 KB opt-in, the prep chunk ceil(R / 1024), the persistent grid of 4 CTAs
per SM); `decode_shape_labels` / `loss_shape_labels` turn a call's shapes into the paths it reaches; the GPU test adds the
labels its values reach.
"""
import math
from fractions import Fraction

import torch

from box_loss_ref import SELF, TINY, U, T

F64 = torch.float64
F32 = torch.float32
A = -0.75
K_TILE = 4096
K_THREADS = 256
K_BLOCKS_PER_SM = 4
K_PREP = 1024
MAX_S = 241
SMEM_DEFAULT = 48 * 1024
SMEM_OPTIN = 227 * 1024
MAX_PIXELS = 2 ** 32
H100_SMS = 132
SCORE_ABS = 2.0 ** -126


def fma(a, b, c):
    """fp32 fma(a, b, c) of tracked quantities: the exact a * b + c, rounded once."""
    v = a.v * b.v + c.v
    e = a.v.abs() * b.e + b.v.abs() * a.e + a.e * b.e + c.e
    return T._round(v, e, (e == 0) & (v.to(F32).to(F64) == v))


def _const(c, like):
    return T(torch.full_like(like, c))


def two_sum_exact(a, b):
    """True where the float64 a + b is exact (Knuth's TwoSum error term is 0)."""
    s = a + b
    bb = s - a
    return ((a - (s - bb)) + (b - bb)) == 0


# ---- the bicubic taps -----------------------------------------------------------------------------------------------
def axis_taps(S, out, device="cpu"):
    """Taps of output rows 0 .. out - 1 of a resize from S: (index [out, 4] long, t [out] float64 holding the fp32 t).
    Asserts that the emulated fma was exact in float64."""
    scale = float(torch.tensor(float(S), dtype=F32) / torch.tensor(float(out), dtype=F32))
    d = torch.arange(out, dtype=F64, device=device) + 0.5  # exact in fp32 for out < 2^23
    prod = scale * d  # two fp32 numbers: exact in float64
    assert bool(two_sum_exact(prod, torch.full_like(prod, -0.5)).all()), (S, out)
    real = (prod - 0.5).to(F32).to(F64)
    base = real.floor()
    t = (real - base).to(F32).to(F64)
    idx = (base.long()[:, None] + torch.arange(-1, 3, device=device)[None]).clamp(0, S - 1)
    return idx, t


def coeffs_exact(t):
    """[out, 4] float64 A = -0.75 cubic convolution coefficients of t."""
    def c1(x):
        return ((A + 2) * x - (A + 3)) * x * x + 1

    def c2(x):
        return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A

    return torch.stack([c2(t + 1), c1(t), c1(1 - t), c2(2 - t)], dim=1)


def coeffs_tracked(t, fused=True):
    """The kernel's fp32 coefficients as tracked quantities: a list of 4 T of shape [out] (value exact, see module doc).
    fused False: every product and sum rounded on its own."""
    tt = T(t)
    f = fma if fused else (lambda a, b, c: a * b + c)  # noqa: E731

    def conv1(x):
        return f(f(_const(1.25, t), x, _const(-2.25, t)) * x, x, _const(1.0, t))

    def conv2(x):
        return f(f(f(_const(-0.75, t), x, _const(3.75, t)), x, _const(-6.0, t)), x, _const(3.0, t))

    t2 = 1 - tt
    got = [conv2(tt + 1), conv1(tt), conv1(t2), conv2(t2 + 1)]
    exact = coeffs_exact(t)
    # the tracker's values are the polynomials of the rounded arguments; measure against the exact ones of t
    return [T(exact[:, k], g.e + (g.v - exact[:, k]).abs()) for k, g in enumerate(got)]


def interp_t(c, x):
    """fma(x3, c3, fma(x2, c2, fma(x0, c0, x1 * c1))) of tracked coefficients c and values x (lists of 4 T)."""
    return fma(x[3], c[3], fma(x[2], c[2], fma(x[0], c[0], x[1] * c[1])))


def interp_unfused_t(c, x):
    """((x0 * c0 + x1 * c1) + x2 * c2) + x3 * c3 with every product and sum rounded."""
    return ((x[0] * c[0] + x[1] * c[1]) + x[2] * c[2]) + x[3] * c[3]


def _rounded(t):
    """t with one rounding charged even where the tracker found the magnitude's result exact (the signed one may not be)."""
    return T(t.v, t.e + U * t.v.abs() + TINY)


def interp_mag_t(c, x):
    """interp_t on magnitudes, every operation charged a rounding."""
    return _rounded(fma(x[3], c[3], _rounded(fma(x[2], c[2], _rounded(fma(x[0], c[0], _rounded(x[1] * c[1])))))))


def interp_unfused_mag_t(c, x):
    """interp_unfused_t on magnitudes, every operation charged a rounding."""
    r = _rounded
    return r(r(r(r(x[0] * c[0]) + r(x[1] * c[1])) + r(x[2] * c[2])) + r(x[3] * c[3]))


def bicubic(maps, out_h, out_w, any_order=False):
    """(value, bound) [..., out_h, out_w] float64 of the kernel's resize of maps [..., S, S] (fp32 values in any dtype).
    any_order: bound any evaluation of the same taps that rounds every product and sum (PyTorch's CPU kernel), either
    axis first, instead of the kernel's fused sequence."""
    m = maps.to(F64)
    S = m.shape[-1]
    if out_h == S and out_w == S:
        return m.clone(), torch.zeros_like(m)
    ix, tx = axis_taps(S, out_w, m.device)
    iy, ty = axis_taps(S, out_h, m.device)
    cx, cy = coeffs_tracked(tx), coeffs_tracked(ty)

    def resize(x, interp, cx, cy, ix, iy):
        xs = [T(x[..., ix[:, k]]) for k in range(4)]  # along the columns, for every source row: [..., S, out_w]
        rows = interp(cx, xs)
        ys = [T(rows.v[..., iy[:, k], :], rows.e[..., iy[:, k], :]) for k in range(4)]  # down the rows
        return interp([T(c.v[:, None], c.e[:, None]) for c in cy], ys)

    v = resize(m, interp_t, cx, cy, ix, iy).v
    # the bound runs the same sequence on the magnitudes: every partial sum is then at its largest, so the bound does
    # not depend on cancellation within a sum
    if any_order:
        cx, cy = coeffs_tracked(tx, False), coeffs_tracked(ty, False)
    mag = [T(c.v.abs(), c.e) for c in cx], [T(c.v.abs(), c.e) for c in cy]
    if any_order:
        e = resize(m.abs(), interp_unfused_mag_t, *mag, ix, iy).e
        e_t = resize(m.abs().transpose(-1, -2), interp_unfused_mag_t, mag[1], mag[0], iy, ix).e
        e = torch.maximum(e, e_t.transpose(-1, -2))
    else:
        e = resize(m.abs(), interp_mag_t, *mag, ix, iy).e
    e = torch.where(torch.isfinite(v), e, 0.0) * SELF
    return v, torch.where(torch.isnan(e), math.inf, e)


# ---- decode ---------------------------------------------------------------------------------------------------------
def roi_geometry(roi):
    """The kernel's fp32 ROI geometry: dict(x1, y1, cw, ch, wo, ho, ok) with Python floats / ints."""
    r = torch.as_tensor(roi, dtype=F32).cpu()
    w = (r[2] - r[0]).clamp(min=1)
    h = (r[3] - r[1]).clamp(min=1)
    wc, hc = w.ceil(), h.ceil()
    ok = bool(torch.isfinite(wc) & torch.isfinite(hc)) and float(wc) * float(hc) <= MAX_PIXELS
    return dict(x1=r[0], y1=r[1], cw=w / wc, ch=h / hc, wo=int(wc) if ok else 0, ho=int(hc) if ok else 0, ok=ok)


def positions(g):
    """fp32 (x [wo], y [ho]) of every output column / row: (o + 0.5) * cw + x1, as the kernel rounds it."""
    ox = torch.arange(g["wo"], dtype=F32) + 0.5
    oy = torch.arange(g["ho"], dtype=F32) + 0.5
    return ox * g["cw"] + g["x1"], oy * g["ch"] + g["y1"]


def score(maps, logit):
    """(score, bound) [K] float64 of 1 / sum exp(m - L) over each S x S map [K, S, S] for the kernel's logits L [K]."""
    m = maps.to(F64).reshape(maps.shape[0], -1)
    L = logit.to(F64)[:, None]
    n = m.shape[1]
    with torch.no_grad():
        d = T(m) - T(L.expand_as(m))
        fin = torch.isfinite(d.v)
        d = T(torch.where(fin, d.v, torch.where(torch.isnan(d.v), d.v, d.v)), torch.where(fin, d.e, 0.0))
        ex = d.exp()
        terms = ex.v
        errs = torch.where(torch.isfinite(ex.e), ex.e, 0.0)
        total = terms.sum(1)
        absum = terms.abs().sum(1)
        k = -(-n // 32) + 5
        gam = k * U / (1 - k * U)
        e_sum = errs.sum(1) + gam * (absum + errs.sum(1))
        s = 1.0 / total
        lo = (total - e_sum).clamp_min(1e-300)
        e = (1.0 / lo - s) + U * s + SCORE_ABS
        e = torch.where(torch.isfinite(total), e, SCORE_ABS)  # an infinite sum: the score is 0 in both
        return s, torch.where(torch.isfinite(s), e * SELF, 0.0)


# ---- the loss -------------------------------------------------------------------------------------------------------
def _lse(x):
    """log_softmax's logsumexp over the last dim: NaN when a value is NaN or +inf."""
    m = x.detach().amax(-1, keepdim=True)
    return (m + torch.log(torch.exp(x - m).sum(-1, keepdim=True)))[..., 0]


class LossRef:
    """Float64 reference of one keypoint loss call on logits [N, K, S, S] (any float dtype, read as fp32) with the
    kernel's targets / valid: per-row loss and bound, and `grad(grad_scale)` (gradient and per-element bound)."""

    def __init__(self, logits, target, valid):
        x = logits.float().to(F64)
        self.N, self.K, self.S = x.shape[0], x.shape[1], x.shape[2]
        self.x = x.reshape(self.N * self.K, -1)
        self.t = target.reshape(-1).long()
        self.valid = valid.reshape(-1).bool()
        n = self.x.shape[1]
        self.items = -(-n // K_THREADS)
        with torch.no_grad():
            x, t = self.x, self.t
            m = x.amax(1, keepdim=True)
            nan_row = torch.isnan(x).any(1, keepdim=True)
            m = torch.where(nan_row, math.nan, m)
            self.m = m
            d = x - m
            ninf = x == -math.inf
            e_d = torch.where(ninf | ~torch.isfinite(d), 0.0, U * d.abs())
            ex = T(torch.where(ninf, -math.inf, d), e_d).exp()
            self.p_num = ex
            terms = ex.v
            errs = torch.where(torch.isfinite(ex.e), ex.e, 0.0)
            s = terms.sum(1)
            a = terms.abs().sum(1)
            k = self.items + 13
            gam = k * U / (1 - k * U)
            es = errs.sum(1)
            e_s = es + gam * (a + es) + (len(terms[0]) + 8) * 2.0 ** -53 * a
            self.sum = T(s, e_s)
            lg = self.sum.log()
            xt = x.gather(1, t.clamp(0, n - 1)[:, None])[:, 0]
            dt = T(xt) - T(m[:, 0])
            dt = T(dt.v, torch.where(torch.isfinite(dt.v), dt.e, 0.0))
            loss_t = lg - dt
            loss = _lse(x) - xt
            self.loss = torch.where(self.valid, loss, 0.0)
            eb = torch.where(torch.isfinite(loss), loss_t.e, 0.0) * SELF
            self.e_loss = torch.where(self.valid, eb, 0.0)

    def grad(self, grad_scale):
        """(gradient [rows, S*S] float64, bound) of sum_rows grad_scale[row] * loss[row] over the valid rows."""
        gs = grad_scale.reshape(-1).float().to(F64)
        x = self.x.clone().requires_grad_(True)
        loss = _lse(x) - x.gather(1, self.t.clamp(0, x.shape[1] - 1)[:, None])[:, 0]
        loss = torch.where(self.valid, loss, 0.0)
        (g,) = torch.autograd.grad((loss * torch.where(self.valid, gs, 0.0)).sum(), x)
        with torch.no_grad():
            p = self.p_num / T(self.sum.v[:, None].expand_as(self.x), self.sum.e[:, None].expand_as(self.x))
            onehot = (torch.arange(self.x.shape[1], device=self.x.device)[None] == self.t[:, None]).to(F64)
            q = p - T(onehot)
            gq = q * T(gs[:, None].expand_as(self.x))
            e = torch.where(self.valid[:, None] & torch.isfinite(g), gq.e, 0.0) * SELF
            g = torch.where(self.valid[:, None], g, 0.0)
        return g, e


def total_bound(terms, errs):
    """Bound of torch's fp32 sum of `terms` in any order (each carrying errs): gamma_n (sum |t| + sum e) + sum e."""
    n = max(terms.numel(), 1)
    gam = n * U / (1 - n * U)
    e = float(errs.sum())
    return e + gam * (float(terms.abs().sum()) + e)


# ---- targets --------------------------------------------------------------------------------------------------------
def exact_cells(c, lo, hi, S):
    """(cell [..] long, decided [..] bool) of floor((c - lo) S / (hi - lo)) for fp32 inputs (any shape, broadcast).
    c == hi gives S - 1 (decided); a cell is decided when every fp32 step is a finite normal number and the 4-rounding
    interval around the exact value holds no integer boundary (an exact 0 stays 0).  The exact value is taken in float64
    (4 roundings of 2^-53) and, where that leaves the decision open, as a Fraction."""
    c, lo, hi = torch.broadcast_tensors(c.float().cpu(), lo.float().cpu(), hi.float().cpu())
    width = hi - lo
    scale = width.reciprocal() * S
    num = c - lo
    f = num * scale
    normal = lambda z: torch.isfinite(z) & ((z == 0) | (z.abs() >= 2.0 ** -126))  # noqa: E731
    ok = normal(width) & (width != 0) & normal(scale) & normal(num) & normal(f) & torch.isfinite(c)
    delta = 4 * U * (1 + 4 * U)
    ex = (c.double() - lo.double()) * S / (hi.double() - lo.double())
    ex = torch.where(ok, ex, 0.0)
    b = ex.abs() * (delta + 8 * 2.0 ** -53)
    cell = ex.floor()
    dec = ok & ((ex == 0) | ((ex - b).floor() == cell) & ((ex + b).floor() == cell) & (ex != cell))
    cell = cell.long()
    open_ = ok & ~dec & (ex != 0)
    dexact = Fraction(4) * Fraction(2) ** -24 * (1 + Fraction(4) * Fraction(2) ** -24)
    for i in torch.nonzero(open_.reshape(-1))[:, 0].tolist():
        e = (Fraction(float(c.reshape(-1)[i])) - Fraction(float(lo.reshape(-1)[i]))) * S / (
            Fraction(float(hi.reshape(-1)[i])) - Fraction(float(lo.reshape(-1)[i])))
        fl = math.floor(e)
        bb = abs(e) * dexact
        cell.view(-1)[i] = fl
        dec.view(-1)[i] = e != fl and math.floor(e - bb) == fl and math.floor(e + bb) == fl
    on_hi = c == hi
    return torch.where(on_hi, S - 1, cell), dec | on_hi


# ---- the path model -------------------------------------------------------------------------------------------------
def smem_bytes(S):
    return S * S * 4


def needs_optin(S):
    return smem_bytes(S) > SMEM_DEFAULT


def tiles(npix):
    return -(-npix // K_TILE)


def decode_paths(rois, S, K, sms=H100_SMS):
    """dict of the decode's launch arithmetic for rois [R, 4] (fp32 values)."""
    geo = [roi_geometry(r) for r in rois.float().cpu()]
    t = [tiles(g["wo"] * g["ho"]) for g in geo]
    items = sum(t) * K
    grid = sms * K_BLOCKS_PER_SM
    R = len(geo)
    return dict(geo=geo, tiles=t, items=items, grid=grid, per_cta=-(-items // grid), chunk=-(-R // K_PREP) if R else 0,
                smem=smem_bytes(S))


def decode_shape_labels(rois, S, K, dtype=F32, sms=H100_SMS):
    """The decode paths a call's shapes reach."""
    p = decode_paths(rois, S, K, sms)
    out = set()
    for g, nt in zip(p["geo"], p["tiles"]):
        if not g["ok"]:
            finite = all(math.isfinite(float(g[k])) for k in ("x1", "y1", "cw", "ch"))
            out.add("nan_row_pixels" if finite else "nan_row_box")
            continue
        wo, ho, npix = g["wo"], g["ho"], g["wo"] * g["ho"]
        if wo == S and ho == S:
            out.add("copy")
        elif wo == S or ho == S:
            out.add("one_axis_equals_S")
        for n, ax in ((wo, "x"), (ho, "y")):
            if n > S:
                out.add("upsample_" + ax)
            elif n < S:
                out.add("downsample_" + ax)
        if npix == 1:
            out.add("one_pixel")
        if npix % K_TILE == K_TILE - 1:
            out.add("tile_minus_1")
        if npix % K_TILE == 0:
            out.add("tile_exact")
        if npix % K_TILE == 1 and npix > 1:
            out.add("tile_plus_1")
        if nt > 1:
            out.add("multi_tile")
    if p["per_cta"] > 1:
        out.add("items_exceed_grid")
    if p["chunk"] > 1:
        out.add("prep_chunk_%d" % min(p["chunk"], 3))
    if needs_optin(S):
        out.add("smem_optin")
    if S == MAX_S:
        out.add("smem_max")
    if S * S < 32:
        out.add("finish_idle_lanes")
    if dtype == torch.float16:
        out.add("f16_maps")
    return out


def roi_labels(rois):
    """Labels of the boxes themselves (fp32): sub-pixel and reversed boxes, far coordinates."""
    out = set()
    r = rois.float().cpu()
    fin = torch.isfinite(r).all(1)
    r = r[fin]
    w, h = r[:, 2] - r[:, 0], r[:, 3] - r[:, 1]
    if bool(((w < 1) & (w >= 0) & (h >= 1)).any()):
        out.add("w_below_1")
    if bool(((h < 1) & (h >= 0) & (w >= 1)).any()):
        out.add("h_below_1")
    if bool(((w < 1) & (h < 1)).any()):
        out.add("w_h_below_1")
    if bool((w < 0).any()):
        out.add("x2_below_x1")
    if bool((r.abs() > 5e3).any()):
        out.add("far_coordinates")
    return out


def loss_shape_labels(N, K, S, dtype):
    out = set()
    n = S * S
    out.add("row_lt_cta" if n < K_THREADS else "row_eq_cta" if n == K_THREADS else "row_gt_cta")
    if n > 32 * K_THREADS:
        out.add("row_many_per_thread")
    if dtype == torch.float16:
        out.add("f16_logits")
    if dtype == torch.bfloat16:
        out.add("bf16_logits")
    if N * K > 4096:
        out.add("many_rows")
    return out


DECODE_SHAPE_LABELS = {"copy", "one_axis_equals_S", "upsample_x", "upsample_y", "downsample_x", "downsample_y",
                       "one_pixel", "tile_minus_1", "tile_exact", "tile_plus_1", "multi_tile", "items_exceed_grid",
                       "prep_chunk_2", "prep_chunk_3", "smem_optin", "smem_max", "finish_idle_lanes", "f16_maps",
                       "nan_row_box", "nan_row_pixels", "w_below_1", "h_below_1", "w_h_below_1", "x2_below_x1",
                       "far_coordinates"}
DECODE_VALUE_LABELS = {"ties_first_pixel", "signed_zero_max", "nan_copy", "nan_arith", "pos_inf_cell", "all_neg_inf",
                       "one_ulp_maxima", "score_underflow"}
LOSS_SHAPE_LABELS = {"row_lt_cta", "row_eq_cta", "row_gt_cta", "row_many_per_thread", "f16_logits", "bf16_logits",
                     "many_rows"}
LOSS_VALUE_LABELS = {"kp_on_x2", "kp_outside", "v0", "zero_width", "nan_cell", "nan_logit", "pos_inf_logit",
                     "neg_inf_logit", "nan_invalid_row", "big_logits", "uniform_row", "grad_scale_edge", "no_valid",
                     "undecided_cell"}
