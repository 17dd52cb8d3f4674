"""Float64 reference of the box-branch losses (detectron2_b200/csrc/losses.cu), its error bounds and its path model.

Reference.  The per-row terms are written from the reference functions, in torch float64, so that they run on the CPU and
on CUDA: fvcore sigmoid_focal_loss (binary_cross_entropy_with_logits itself for gamma = 0), smooth_l1_loss (beta < 1e-5 is
L1), giou_loss (eps 1e-7) of Box2BoxTransform.apply_deltas with clamp(max=scale_clamp), Box2BoxTransform[Rotated].get_deltas
with the (da + 180) % 360 - 180 wrap, FCOS's Box2BoxTransformLinear decode + GIoU and compute_ctrness_targets + BCE, and the
Fast R-CNN cross_entropy, _log_classification_stats and the delta gather.  Gradients are autograd of that float64 forward,
so they do not depend on the kernel's hand-derived backward.  Parameters (alpha, gamma, beta, scale_clamp, the weights) are
taken at the fp32 values the kernel receives; formula constants (eps, pi / 180) are exact.  Where pow's backward meets
0 * inf at q = 1 - p_t = 0 (gamma < 1, |x| > 37 in float64) the gradient is its limit 0.

Error bounds.  losses.cu is compiled with -fmad=false and without fast math, so every fp32 +, -, *, / and sqrtf rounds once,
to within u = 2^-24 relative.  CUDA documents these maximum errors, in ulp (an ulp is at most 2^-23 relative): expf 2,
logf 1, log1pf 1, powf 4; expf(0) = 1 and logf(1) = 0 are exact.  The bound of a value is a forward error analysis of the
kernel's own sequence of operations, carried out by `T` below: each quantity holds its float64 value v and a bound e on
|fp32 result - v|.
  * a +- b:  e = ea + eb + u |v|;   a * b:  |a| eb + |b| ea + ea eb + u |v|;   a / b:  (ea + |v| eb) / (|b| - eb) + u |v|.
    The rounding term is dropped where the result is exact: exact operands whose float64 result is an fp32 number, an
    exact 0 added, an exact power of two (or 0) multiplied.
  * f = expf / logf / log1pf / powf / sqrtf:  e = max |f(v +- ea) - f(v)| + k ulp, monotone f, so the extremes are at
    the ends of the interval.
  * A compare a < b is *decided* when |a - b| > ea + eb or when both sides are exact; otherwise the element is undecided.
    Values are continuous across every compare here (sign, n < beta, clamp, relu, inter, min / max, argmax of equal
    values), so the loss bound holds either way; undecided gradient elements are left out of the gradient check.
Float64 itself rounds at 2^-53: the same analysis with u = 2^-53 bounds the reference's own error by e 2^-29, so each
bound is e (1 + 2^-28).  Underflow adds at most 2^-149 per operation; TINY = 2^-140 per rounding covers it.

Focal loss.  fvcore's q = 1 - p_t cancels in fp32 by design and the reference does the same in float64.  p = 1 / (1 +
expf(-x)) is within 4.5 u relative; the product with a binary t is exact, 1 - p and 1 - (...) each round once, so q is
off by at most (4.5 p + 2) u <= 6.5 u: an absolute bound, in 2^-24 units, not a relative one.  ce = (1 - t) x -
(min(x, 0) - log1pf(expf(-|x|))) is off by at most about 3 u (|x| + ce).  The loss ce q^gamma then carries
ce d(q^gamma) + q^gamma 3 u (|x| + ce): for |x| <= 100 that is at most 6.5 u (gamma + 1) |x| + 300 u <= 2e-5 absolute,
and it goes to 0 with the loss where q -> 0 (ce ~ q there).  For gamma < 1 the tracker takes (q + 6.5 u)^gamma - q^gamma,
which stays finite at q = 0.

Sums.  Each classification thread adds at most kItems * V::N = 16 (fp32) or 32 (fp16 / bf16) terms in order; a
regression thread adds D smooth-L1 terms, one GIoU term or one centerness term; a Fast R-CNN lane adds one.  Then come 5
butterfly levels and the 8 warps in order, so a CTA's partial has error at most gamma_n sum |t_i| with n = items + 13 and
gamma_n = n u / (1 - n u).  The CTA partials are added in double (at most ceil(P / 256) + 8 adds each, 2^-53 relative) and
the total is rounded to fp32 once (u |S|).  With E_i the per-term bounds:
    |S_kernel - S_ref| <= sum E_i + gamma_n (sum |t_i| + sum E_i) + (ceil(P / 256) + 8 + len) 2^-53 sum |t_i| + u |S|.

Path model.  `dense_shape_labels` / `frcnn_shape_labels` turn a call's shapes into the kernel paths it reaches;
`Result.labels` adds the paths the values reach (decided edges, status bits).  `dense_ctas` / `frcnn_ctas` restate the
launch arithmetic (kThreads = 256, kItems = 4, V::N = 16 / sizeof(T)); `dense_refuses` the argument rules.
"""
import math
from collections import namedtuple

import torch
import torch.nn.functional as F

F64 = torch.float64
U = 2.0 ** -24
ULP = 2.0 ** -23
TINY = 2.0 ** -140
SELF = 1.0 + 2.0 ** -28  # the reference's own float64 rounding, see above
K_THREADS, K_ITEMS, K_WARPS = 256, 4, 8
STATUS_WIDTH, STATUS_CLASS, STATUS_ORDER = 1, 2, 4
SL1, GIOU, LIN = 0, 1, 2


def f32(x):
    """The fp32 value of a Python float, as a Python float."""
    return float(torch.tensor(x, dtype=torch.float32))


# ---- the error tracker ----------------------------------------------------------------------------------------------
def _ok32(v):
    return v.to(torch.float32).to(F64) == v


def _pow2_or_zero(t):
    m, _ = torch.frexp(t.v)
    return (t.e == 0) & ((t.v == 0) | (m.abs() == 0.5))


class T:
    """A quantity of the kernel: v its float64 value, e a bound on |fp32 result - v| (see the module docstring)."""
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v = v
        self.e = torch.zeros_like(v) if e is None else e

    @staticmethod
    def const(c, like):
        """A constant the kernel holds in fp32: exact if c is an fp32 number, else off by |fp32(c) - c|."""
        v = torch.full_like(like, c, dtype=F64)
        return T(v, torch.full_like(v, abs(f32(c) - c)))

    def _lift(self, o):
        return o if isinstance(o, T) else T.const(float(o), self.v)

    @staticmethod
    def _round(v, e, exact):
        return T(v, e + torch.where(exact, 0.0, U * v.abs() + TINY))

    def __add__(self, o):
        o = self._lift(o)
        v = self.v + o.v
        e = self.e + o.e
        z = lambda t: (t.e == 0) & (t.v == 0)  # noqa: E731
        return T._round(v, e, z(self) | z(o) | ((e == 0) & _ok32(v)))

    __radd__ = __add__

    def __neg__(self):
        return T(-self.v, self.e)

    def __sub__(self, o):
        return self + (-self._lift(o))

    def __rsub__(self, o):
        return self._lift(o) + (-self)

    def __mul__(self, o):
        o = self._lift(o)
        v = self.v * o.v
        e = self.v.abs() * o.e + o.v.abs() * self.e + self.e * o.e
        return T._round(v, e, _pow2_or_zero(self) | _pow2_or_zero(o) | ((e == 0) & _ok32(v)))

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = self._lift(o)
        v = self.v / o.v
        den = o.v.abs() - o.e
        e = torch.where(den > 0, (self.e + v.abs() * o.e) / den.clamp_min(1e-300), math.inf)
        e = torch.where((self.e == 0) & (o.e == 0), 0.0, e)
        return T._round(v, e, (e == 0) & _ok32(v) & (v * o.v == self.v))

    def __rtruediv__(self, o):
        return self._lift(o) / self

    def abs(self):
        return T(self.v.abs(), self.e)

    def _mono(self, f, ulps, exact_at=None, lo=-math.inf):
        v = f(self.v)
        hi = f(self.v + self.e)
        low = f((self.v - self.e).clamp_min(lo))
        e = torch.maximum((hi - v).abs(), (v - low).abs())
        e = e + ulps * ULP * torch.maximum(hi.abs(), low.abs()) + TINY
        e = torch.where(torch.isnan(e), math.inf, e)
        if exact_at is not None:
            e = torch.where((self.e == 0) & (self.v == exact_at), 0.0, e)
        return T(v, e)

    def exp(self):
        return self._mono(torch.exp, 2, 0.0)

    def log(self):
        return self._mono(torch.log, 1, 1.0, lo=0.0)

    def log1p(self):
        return self._mono(torch.log1p, 1, 0.0, lo=-1.0)

    def sqrt(self):
        t = self._mono(torch.sqrt, 1, None, lo=0.0)  # correctly rounded: 0.5 ulp
        ex = (self.e == 0) & _ok32(t.v) & (t.v * t.v == self.v)
        return T(t.v, torch.where(ex, 0.0, t.e))

    def pow(self, g):
        return self._mono(lambda x: x.clamp_min(0) ** g, 4, None, lo=0.0)


def tmax(a, b):
    return T(torch.maximum(a.v, b.v), torch.maximum(a.e, b.e))


def tmin(a, b):
    return T(torch.minimum(a.v, b.v), torch.maximum(a.e, b.e))


def where(c, a, b):
    return T(torch.where(c, a.v, b.v), torch.where(c, a.e, b.e))


def undecided(a, b):
    """a < b (or a > b, a == b) cannot be told from the bounds."""
    m = a.e + b.e
    return ((a.v - b.v).abs() <= m) & (m > 0)


def share(a, b, larger):
    """share_max (larger=True) / share_min: 1, 0.5 at a tie, 0 -- autograd's split of torch.maximum / minimum."""
    w = a.v > b.v if larger else a.v < b.v
    return torch.where(w, 1.0, torch.where(a.v == b.v, 0.5, 0.0)).to(F64), undecided(a, b)


def sum_bound(terms, errs, items, parts):
    """Bound of the kernel's fixed-order sum of `terms` (float64, the reference) whose elements carry `errs`."""
    a = float(terms.abs().sum())
    e = float(errs.sum())
    s = float(terms.sum())
    n = items + 13
    gam = n * U / (1 - n * U)
    return e + gam * (a + e) + (math.ceil(parts / 256) + 8 + terms.numel()) * 2.0 ** -53 * a + U * abs(s)


# ---- the kernel's operation sequences under the tracker -------------------------------------------------------------
def focal_t(x, t, gamma, alpha):
    """losses.cu focal(): (loss, d loss / d x) of the fp32 logit x (T, exact) and the target t (T)."""
    ce = (1 - t) * x - (T(torch.minimum(x.v, torch.zeros_like(x.v)), x.e) - (-x.abs()).exp().log1p())
    p = 1 / (1 + (-x).exp())
    if gamma == 0:
        loss, g = ce, p - t
    else:
        q = 1 - (p * t + (1 - p) * (1 - t))
        m = q * q if gamma == 2 else q.pow(gamma)
        loss = ce * m
        d = m * (q + gamma * (1 - q) * ce)
        g = where(t.v > 0.5, -d, d)
    if alpha >= 0:
        at = alpha * t + (1 - alpha) * (1 - t)
        loss, g = at * loss, at * g
    return loss, g


def smooth_l1_t(diff, beta):
    """smooth_l1(): (loss, gradient, undecided) of the difference diff (T)."""
    n = diff.abs()
    sgn = torch.sign(diff.v)
    und = undecided(diff, T(torch.zeros_like(diff.v)))
    if beta < f32(1e-5):
        return n, T(sgn), und
    bt = T.const(beta, diff.v)
    quad = n.v < beta
    und = und | undecided(n, bt)
    lq, gq = 0.5 * (n * n) / bt, n / bt * T(sgn)
    ll = n - 0.5 * bt
    loss = where(quad, lq, ll)
    loss = T(loss.v, torch.where(und, torch.maximum(lq.e, ll.e), loss.e))
    return loss, where(quad, gq, T(sgn)), und


def get_deltas_t(s, t, w):
    """Box2BoxTransform[Rotated].get_deltas in the kernel's order (boxes.cuh); s, t: lists of T, w: fp32 weights."""
    if len(s) == 5:
        d = [w[0] * (t[0] - s[0]) / s[2], w[1] * (t[1] - s[1]) / s[3], w[2] * (t[2] / s[2]).log(),
             w[3] * (t[3] / s[3]).log()]
        a = t[4] - s[4]
        r = a + 180.0
        m = T(torch.remainder(r.v, 360.0), r.e)  # fmodf is exact; the + 360 of a negative remainder rounds
        m = T(m.v, m.e + torch.where(torch.fmod(r.v, 360.0) < 0, U * m.v.abs(), 0.0))
        und = ((m.v <= m.e) | (360.0 - m.v <= m.e)) & (m.e > 0)
        wa = T.const(w[4] * math.pi / 180.0, a.v)
        return d + [(m - 180.0) * wa], und
    sw, sh = s[2] - s[0], s[3] - s[1]
    scx, scy = s[0] + 0.5 * sw, s[1] + 0.5 * sh
    tw, th = t[2] - t[0], t[3] - t[1]
    tcx, tcy = t[0] + 0.5 * tw, t[1] + 0.5 * th
    d = [w[0] * (tcx - scx) / sw, w[1] * (tcy - scy) / sh, w[2] * (tw / sw).log(), w[3] * (th / sh).log()]
    return d, torch.zeros_like(sw.v, dtype=torch.bool)


def giou_t(p, q):
    """giou_loss() of losses.cu: (loss, d loss / d p [4], undecided, flags) for boxes p, q (lists of T)."""
    eps = T.const(1e-7, p[0].v)
    xk1, yk1, xk2, yk2 = tmax(p[0], q[0]), tmax(p[1], q[1]), tmin(p[2], q[2]), tmin(p[3], q[3])
    und = undecided(yk2, yk1) | undecided(xk2, xk1)
    inter = (yk2.v > yk1.v) & (xk2.v > xk1.v)
    iw, ih = xk2 - xk1, yk2 - yk1
    zero = T(torch.zeros_like(iw.v))
    I = where(inter, iw * ih, zero)
    pw, ph = p[2] - p[0], p[3] - p[1]
    Un = pw * ph + (q[2] - q[0]) * (q[3] - q[1]) - I
    iou = I / (Un + eps)
    xc1, yc1, xc2, yc2 = tmin(p[0], q[0]), tmin(p[1], q[1]), tmax(p[2], q[2]), tmax(p[3], q[3])
    cw, ch = xc2 - xc1, yc2 - yc1
    Cc = cw * ch
    loss = 1 - (iou - (Cc - Un) / (Cc + eps))
    dU = I / ((Un + eps) * (Un + eps)) - 1 / (Cc + eps)
    dI = -1 / (Un + eps) - dU
    dC = (Un + eps) / ((Cc + eps) * (Cc + eps))
    g = [-dU * ph, -dU * pw, dU * ph, dU * pw]
    ties = torch.zeros_like(inter)
    for i, (a, b, big, s, m) in enumerate(((p[0], q[0], True, -1, ih), (p[1], q[1], True, -1, iw),
                                           (p[2], q[2], False, 1, ih), (p[3], q[3], False, 1, iw))):
        sh, u = share(a, b, big)
        und = und | (u & inter)
        ties = ties | ((sh == 0.5) & inter)
        g[i] = where(inter, g[i] + s * dI * m * T(sh), g[i])
    for i, (a, b, big, s, m) in enumerate(((p[0], q[0], False, -1, ch), (p[1], q[1], False, -1, cw),
                                           (p[2], q[2], True, 1, ch), (p[3], q[3], True, 1, cw))):
        sh, u = share(a, b, big)
        und = und | u
        ties = ties | (sh == 0.5)
        g[i] = g[i] + s * dC * m * T(sh)
    exact = lambda a, b: (a.e == 0) & (b.e == 0) & (a.v == b.v)  # noqa: E731
    flags = dict(inter=inter & ~und, disjoint=((xk2.v < xk1.v) | (yk2.v < yk1.v)) & ~und,
                 touching=exact(xk2, xk1) | exact(yk2, yk1), tie=ties & ~und)
    return loss, g, und, flags


def decode_t(an, d, w, clamp):
    """apply_deltas() of boxes.cuh and the chain of giou_row(): (p, dp/dd factors, undecided, flags)."""
    widths, heights = an[2] - an[0], an[3] - an[1]
    ctr_x, ctr_y = an[0] + 0.5 * widths, an[1] + 0.5 * heights
    dx, dy, dw, dh = d[0] / w[0], d[1] / w[1], d[2] / w[2], d[3] / w[3]
    c = T(torch.full_like(dw.v, clamp))
    und = undecided(dw, c) | undecided(dh, c)
    pass_w, pass_h = ~(dw.v > clamp), ~(dh.v > clamp)
    flags = dict(clamp_equal=((dw.v == clamp) & (dw.e == 0)) | ((dh.v == clamp) & (dh.e == 0)),
                 clamp_above=(~pass_w | ~pass_h) & ~und)
    dw, dh = where(pass_w, dw, c), where(pass_h, dh, c)
    pcx, pcy = dx * widths + ctr_x, dy * heights + ctr_y
    ew, eh = dw.exp(), dh.exp()
    pw, ph = ew * widths, eh * heights
    p = [pcx - 0.5 * pw, pcy - 0.5 * ph, pcx + 0.5 * pw, pcy + 0.5 * ph]
    return p, (widths, heights, ew, eh, pass_w, pass_h), und, flags


def giou_row_t(an, d, gt, w, clamp):
    p, (widths, heights, ew, eh, pass_w, pass_h), und, flags = decode_t(an, d, w, clamp)
    loss, gp, u2, f2 = giou_t(p, gt)
    gcx, gcy = gp[0] + gp[2], gp[1] + gp[3]
    gpw, gph = 0.5 * gp[2] - 0.5 * gp[0], 0.5 * gp[3] - 0.5 * gp[1]
    zero = T(torch.zeros_like(gcx.v))
    g = [gcx * widths / w[0], gcy * heights / w[1], where(pass_w, gpw * widths * ew / w[2], zero),
         where(pass_h, gph * heights * eh / w[3], zero)]
    flags.update(f2)
    ordered = (p[2].v >= p[0].v) & (p[3].v >= p[1].v) & (gt[2].v >= gt[0].v) & (gt[3].v >= gt[1].v)
    return loss, g, und | u2, flags, ordered


def giou_row_linear_t(an, d, gt):
    ctr_x, ctr_y = 0.5 * (an[0] + an[2]), 0.5 * (an[1] + an[3])
    sw, sh = an[2] - an[0], an[3] - an[1]
    r = [T(torch.clamp_min(x.v, 0.0)) for x in d]
    p = [ctr_x - r[0] * sw, ctr_y - r[1] * sh, ctr_x + r[2] * sw, ctr_y + r[3] * sh]
    loss, gp, und, flags = giou_t(p, gt)
    zero = T(torch.zeros_like(sw.v))
    g = [where(d[0].v <= 0, zero, -gp[0] * sw), where(d[1].v <= 0, zero, -gp[1] * sh),
         where(d[2].v <= 0, zero, gp[2] * sw), where(d[3].v <= 0, zero, gp[3] * sh)]
    ordered = (p[2].v >= p[0].v) & (p[3].v >= p[1].v) & (gt[2].v >= gt[0].v) & (gt[3].v >= gt[1].v)
    return loss, g, und, flags, ordered


def ctrness_t(an, gt):
    cx, cy = 0.5 * (an[0] + an[2]), 0.5 * (an[1] + an[3])
    sw, sh = an[2] - an[0], an[3] - an[1]
    l, t, r, b = (cx - gt[0]) / sw, (cy - gt[1]) / sh, (gt[2] - cx) / sw, (gt[3] - cy) / sh
    c = ((tmin(l, r) / tmax(l, r)) * (tmin(t, b) / tmax(t, b))).sqrt()
    tie = ((l.v == r.v) & (l.e == 0) & (r.e == 0)) | ((t.v == b.v) & (t.e == 0) & (b.e == 0)) | \
          (((l.v == 0) | (r.v == 0) | (t.v == 0) | (b.v == 0)) & (c.e == 0))
    return c, tie


# ---- the float64 reference (autograd) -------------------------------------------------------------------------------
def focal_ref(x, t, gamma, alpha):
    """fvcore sigmoid_focal_loss per element (binary_cross_entropy_with_logits for gamma = 0)."""
    ce = F.binary_cross_entropy_with_logits(x, t, reduction="none")
    if gamma == 0:
        loss = ce
    else:
        p = torch.sigmoid(x)
        p_t = p * t + (1 - p) * (1 - t)
        loss = ce * ((1 - p_t) ** gamma)
    if alpha >= 0:
        loss = (alpha * t + (1 - alpha) * (1 - t)) * loss
    return loss


def get_deltas_ref(src, tgt, w):
    if src.shape[-1] == 5:
        sx, sy, sw, sh, sa = src.unbind(-1)
        tx, ty, tw, th, ta = tgt.unbind(-1)
        da = (ta - sa + 180.0) % 360.0 - 180.0
        return torch.stack([w[0] * (tx - sx) / sw, w[1] * (ty - sy) / sh, w[2] * torch.log(tw / sw),
                            w[3] * torch.log(th / sh), da * (w[4] * math.pi / 180.0)], -1)
    sw, sh = src[..., 2] - src[..., 0], src[..., 3] - src[..., 1]
    sx, sy = src[..., 0] + 0.5 * sw, src[..., 1] + 0.5 * sh
    tw, th = tgt[..., 2] - tgt[..., 0], tgt[..., 3] - tgt[..., 1]
    tx, ty = tgt[..., 0] + 0.5 * tw, tgt[..., 1] + 0.5 * th
    return torch.stack([w[0] * (tx - sx) / sw, w[1] * (ty - sy) / sh, w[2] * torch.log(tw / sw),
                        w[3] * torch.log(th / sh)], -1)


def smooth_l1_ref(x, t, beta):
    if beta < f32(1e-5):
        return torch.abs(x - t)
    n = torch.abs(x - t)
    return torch.where(n < beta, 0.5 * n ** 2 / beta, n - 0.5 * beta)


def giou_ref(b1, b2, eps=1e-7):
    x1, y1, x2, y2 = b1.unbind(-1)
    x1g, y1g, x2g, y2g = b2.unbind(-1)
    xk1, yk1 = torch.max(x1, x1g), torch.max(y1, y1g)
    xk2, yk2 = torch.min(x2, x2g), torch.min(y2, y2g)
    inter = torch.zeros_like(x1)
    mask = (yk2 > yk1) & (xk2 > xk1)
    inter[mask] = (xk2[mask] - xk1[mask]) * (yk2[mask] - yk1[mask])
    union = (x2 - x1) * (y2 - y1) + (x2g - x1g) * (y2g - y1g) - inter
    iou = inter / (union + eps)
    xc1, yc1 = torch.min(x1, x1g), torch.min(y1, y1g)
    xc2, yc2 = torch.max(x2, x2g), torch.max(y2, y2g)
    area_c = (xc2 - xc1) * (yc2 - yc1)
    return 1 - (iou - (area_c - union) / (area_c + eps))


def apply_deltas_ref(d, an, w, clamp):
    widths, heights = an[:, 2] - an[:, 0], an[:, 3] - an[:, 1]
    ctr_x, ctr_y = an[:, 0] + 0.5 * widths, an[:, 1] + 0.5 * heights
    dx, dy = d[:, 0] / w[0], d[:, 1] / w[1]
    dw, dh = torch.clamp(d[:, 2] / w[2], max=clamp), torch.clamp(d[:, 3] / w[3], max=clamp)
    pcx, pcy = dx * widths + ctr_x, dy * heights + ctr_y
    pw, ph = torch.exp(dw) * widths, torch.exp(dh) * heights
    return torch.stack([pcx - 0.5 * pw, pcy - 0.5 * ph, pcx + 0.5 * pw, pcy + 0.5 * ph], -1)


def apply_deltas_linear_ref(d, an):
    d = F.relu(d)
    ctr_x, ctr_y = 0.5 * (an[:, 0] + an[:, 2]), 0.5 * (an[:, 1] + an[:, 3])
    sw, sh = an[:, 2] - an[:, 0], an[:, 3] - an[:, 1]
    d = d * torch.stack([sw, sh, sw, sh], -1)
    return torch.stack([ctr_x - d[:, 0], ctr_y - d[:, 1], ctr_x + d[:, 2], ctr_y + d[:, 3]], -1)


def ctrness_ref(an, gt):
    cx, cy = 0.5 * (an[:, 0] + an[:, 2]), 0.5 * (an[:, 1] + an[:, 3])
    sw, sh = an[:, 2] - an[:, 0], an[:, 3] - an[:, 1]
    reg = torch.stack([cx - gt[:, 0], cy - gt[:, 1], gt[:, 2] - cx, gt[:, 3] - cy], -1) / torch.stack([sw, sh, sw, sh], -1)
    lr, tb = reg[:, [0, 2]], reg[:, [1, 3]]
    return torch.sqrt((lr.min(dim=-1).values / lr.max(dim=-1).values) * (tb.min(dim=-1).values / tb.max(dim=-1).values))


# ---- results --------------------------------------------------------------------------------------------------------
Result = namedtuple("Result", "sums sum_bounds counts status grads bounds und labels n_und n_dec")


def _rows(t, i):
    return [T(t[:, q]) for q in range(t.shape[1])] if i is None else [T(t[i, q]) for q in range(t.shape[1])]


def dense(logits, deltas, ctr, anchors, gt_boxes, labels, K, rpn, gamma, alpha, beta, loss_type, scale_clamp, weights,
          grad_sums, pin=None):
    """d2b_dense_loss_forward + _backward in float64.  logits[l] [N, R_l, K], deltas[l] [N, R_l, D], ctr[l] [N, R_l]
    (LIN only), anchors [R, D], gt_boxes [N, R, D], labels [N, R], grad_sums: the three fp32 values.  pin: bool [N, R, D]
    marking deltas known to equal the kernel's own fp32 target (the difference is exactly 0 there).
    Gradients are those of sums . grad_sums: every level's logits, then deltas, then centerness."""
    dev = anchors.device
    gamma, alpha, beta, clamp = f32(gamma), f32(alpha), f32(beta), f32(scale_clamp)
    w = None if weights is None else [f32(x) for x in weights]
    gs = [float(torch.tensor(grad_sums, dtype=torch.float32)[i]) for i in range(3)]
    N, D = gt_boxes.shape[0], anchors.shape[-1]
    Rl = [int(x.shape[1]) for x in logits]
    R = sum(Rl)
    lab = labels.to(dev).long()
    an = anchors.to(dev, F64)
    gt = gt_boxes.to(dev, F64)
    labels_out, status = set(), 0
    vec = 4 if logits[0].dtype == torch.float32 else 8
    nparts = dense_ctas(N, K, Rl, vec)
    # classification
    x = torch.cat([t.to(dev, F64).reshape(N, r, K) for t, r in zip(logits, Rl)], 1).requires_grad_(True)
    valid = lab >= 0
    tgt = (lab == 1).to(F64)[..., None] if rpn else (lab[..., None] == torch.arange(K, device=dev)).to(F64)
    xv = torch.where(valid[..., None], x, torch.zeros_like(x))
    lc = focal_ref(xv, tgt, gamma, alpha) * valid[..., None]
    if bool(torch.isnan(x.detach()[~valid]).any()):
        labels_out.add("ignored_nan")
    gx, = torch.autograd.grad(lc.sum() * gs[0], x) if R * N else (torch.zeros_like(x),)
    gx = torch.where(torch.isnan(gx) & torch.isfinite(x.detach()), 0.0, gx)
    xd = x.detach()
    vm = valid[..., None].expand_as(xd)
    loss_t, g_t = focal_t(T(xd[vm]), T(tgt.expand_as(xd)[vm]), gamma, alpha)
    gb = torch.zeros_like(xd)
    gb[vm] = ((g_t * gs[0]).e * SELF)
    s_cls = sum_bound(lc.detach()[vm], loss_t.e * SELF, K_ITEMS * vec, nparts)
    sums = [float(lc.detach().sum()), 0.0, 0.0]
    bnds = [s_cls, 0.0, 0.0]
    # regression
    in_range = (lab >= -1) & (lab <= (1 if rpn else K))
    if not bool(in_range.all()):
        status |= STATUS_CLASS
    pos = (lab == 1) if rpn else ((lab >= 0) & (lab < K))
    counts = [int(pos.sum()), int((lab == 0).sum() if rpn else (lab == K).sum())]
    giou = loss_type in (GIOU, LIN)
    w32 = (anchors[:, 2] - anchors[:, 0]) if D == 4 else anchors[:, 2]  # get_deltas' assertion, in fp32, every anchor
    if not giou and N > 0 and not bool((w32 > 0).all()):
        status |= STATUS_WIDTH
    dl = torch.cat([t.to(dev, F64).reshape(N, r, D) for t, r in zip(deltas, Rl)], 1).requires_grad_(True)
    n_i, a_i = torch.nonzero(pos, as_tuple=True)
    dp = dl[n_i, a_i]
    anp, gtp = an[a_i], gt[n_i, a_i]
    gd_b = torch.zeros_like(dl.detach())
    und_d = torch.zeros_like(dl.detach(), dtype=torch.bool)
    ctr_x = [t.to(dev, F64).reshape(N, r).requires_grad_(True) for t, r in zip(ctr, Rl)]
    if loss_type == SL1:
        tg = get_deltas_ref(anp, gtp, w)
        d_t, wrap_und = get_deltas_t(_rows(anp, None), _rows(gtp, None), w)
        tg_t = [T(tg[:, q].clone(), d_t[q].e) for q in range(D)]
        if pin is not None:
            pp = pin.to(dev)[n_i, a_i]
            tg = torch.where(pp, dp.detach(), tg)
            tg_t = [where(pp[:, q], T(dp.detach()[:, q]), tg_t[q]) for q in range(D)]
        lr = smooth_l1_ref(dp, tg, beta)
        terms_e, und_rows = [], []
        for q in range(D):
            lq, gq, uq = smooth_l1_t(T(dp.detach()[:, q]) - tg_t[q], beta)
            uq = uq | wrap_und
            terms_e.append(lq.e)
            gd_b[n_i, a_i, q] = (gq * gs[1]).e * SELF
            und_d[n_i, a_i, q] = uq
            diff = T(dp.detach()[:, q]) - tg_t[q]
            if bool(((diff.v == 0) & (diff.e == 0)).any()):
                labels_out.add("diff_zero")
            if beta >= f32(1e-5):
                n = diff.v.abs()
                if bool(((n < beta) & ~uq).any()):
                    labels_out.add("sl1_quadratic")
                if bool(((n >= beta) & ~uq).any()):
                    labels_out.add("sl1_linear")
        if beta < f32(1e-5) and len(n_i):
            labels_out.add("sl1_l1")
        if D == 5 and bool((((gtp[:, 4] - anp[:, 4]) >= 180) | ((gtp[:, 4] - anp[:, 4]) < -180)).any()):
            labels_out.add("angle_wrap")
        terms = lr.detach().reshape(-1)
        e_terms = torch.stack(terms_e, 1).reshape(-1) * SELF
        sums[1] = float(terms.sum())
        bnds[1] = sum_bound(terms, e_terms, D, nparts)
        loss_reg = lr.sum()
        loss_ctr = None
    else:
        a_rows, g_rows, d_rows = _rows(anp, None), _rows(gtp, None), [T(dp.detach()[:, q]) for q in range(4)]
        if loss_type == GIOU:
            lr = giou_ref(apply_deltas_ref(dp, anp, w, clamp), gtp)
            lt, gt_t, und, flags, ordered = giou_row_t(a_rows, d_rows, g_rows, w, clamp)
        else:
            lr = giou_ref(apply_deltas_linear_ref(dp, anp), gtp)
            lt, gt_t, und, flags, ordered = giou_row_linear_t(a_rows, d_rows, g_rows)
            if bool((dp.detach() <= 0).any()):
                labels_out.add("fcos_relu_zero")
        if not bool(ordered.all()):
            status |= STATUS_ORDER
        for name in ("inter", "disjoint", "touching", "tie", "clamp_equal", "clamp_above"):
            if name in flags and bool(flags[name].any()):
                labels_out.add("giou_" + name if name in ("inter", "disjoint", "touching", "tie") else name)
        for q in range(4):
            gd_b[n_i, a_i, q] = (gt_t[q] * gs[1]).e * SELF
            und_d[n_i, a_i, q] = und
        sums[1] = float(lr.detach().sum())
        bnds[1] = sum_bound(lr.detach(), lt.e * SELF, 1, nparts)
        loss_reg = lr.sum()
        loss_ctr = None
        if loss_type == LIN:
            xc = torch.cat(ctr_x, 1)[n_i, a_i]
            ct = ctrness_ref(anp, gtp)
            lcr = F.binary_cross_entropy_with_logits(xc, ct, reduction="none")
            ct_t, tie = ctrness_t(a_rows, g_rows)
            if bool(tie.any()):
                labels_out.add("fcos_ctr_tie")
            lct, gct = focal_t(T(xc.detach()), ct_t, 0.0, -1.0)
            sums[2] = float(lcr.detach().sum())
            bnds[2] = sum_bound(lcr.detach(), lct.e * SELF, 1, nparts)
            loss_ctr = lcr.sum()
            gc_b = torch.zeros((N, R), dtype=F64, device=dev)
            gc_b[n_i, a_i] = (gct * gs[2]).e * SELF
    total = loss_reg * gs[1] + (loss_ctr * gs[2] if loss_ctr is not None else 0.0)
    leaves = [dl] + ctr_x
    grads = torch.autograd.grad(total, leaves, allow_unused=True) if total.requires_grad else [None] * len(leaves)
    gdl = grads[0] if grads[0] is not None else torch.zeros_like(dl)
    out_g = [t for t in gx.split(Rl, 1)] + [t for t in gdl.split(Rl, 1)]
    out_b = [t for t in gb.split(Rl, 1)] + [t for t in gd_b.split(Rl, 1)]
    out_u = [torch.zeros_like(t, dtype=torch.bool) for t in gx.split(Rl, 1)] + [t for t in und_d.split(Rl, 1)]
    if loss_type == LIN:
        for l, g in enumerate(grads[1:]):
            out_g.append(g if g is not None else torch.zeros_like(ctr_x[l]))
        out_b += list(gc_b.split(Rl, 1))
        out_u += [torch.zeros_like(t, dtype=torch.bool) for t in gc_b.split(Rl, 1)]
    if status & STATUS_WIDTH:
        labels_out.add("status_width")
    if status & STATUS_CLASS:
        labels_out.add("status_class")
    if status & STATUS_ORDER:
        labels_out.add("status_order")
    n_und = int(und_d.sum())
    return Result(sums, bnds, counts, status, out_g, out_b, out_u, labels_out, n_und, int(pos.sum()) * D - n_und)


def frcnn(scores, deltas, proposals, gt_boxes, gt_classes, beta, loss_type, scale_clamp, weights, grad_sums, pin=None):
    """d2b_frcnn_loss_forward + _backward in float64: scores [R, K+1], deltas [R, kreg * D], proposals / gt_boxes [R, D],
    gt_classes [R].  Returns the two sums, the four counts of _log_classification_stats and the status, and the
    gradients of sums . grad_sums."""
    dev = proposals.device
    beta, clamp = f32(beta), f32(scale_clamp)
    w = [f32(x) for x in weights]
    gs = [float(torch.tensor(grad_sums, dtype=torch.float32)[i]) for i in range(2)]
    R, K1 = scores.shape
    K, D = K1 - 1, proposals.shape[-1]
    kreg = deltas.shape[1] // D
    sc = scores.to(dev, F64).requires_grad_(True)
    dl = deltas.to(dev, F64).requires_grad_(True)
    cls = gt_classes.to(dev).long()
    labels_out, status = set(), 0
    ok = (cls >= 0) & (cls <= K)
    if not bool(ok.all()):
        status |= STATUS_CLASS
    fg = (cls >= 0) & (cls < K)
    if bool((cls == K).any()):
        labels_out.add("background_row")
    s = sc.detach()
    pred = s.argmax(dim=1) if R else cls
    counts = [int(fg.sum()), int((pred == cls).sum()), int((fg & (pred == cls)).sum()), int((fg & (pred == K)).sum())]
    mx = s.max(dim=1, keepdim=True).values if R else s[:, :1]
    at_max = (s == mx).nonzero()
    if len(at_max):
        lanes = torch.zeros((R, 32), dtype=torch.bool, device=dev)
        lanes[at_max[:, 0], at_max[:, 1] % 32] = True
        if bool((lanes.sum(1) >= 2).any()):
            labels_out.add("argmax_tie_across_lanes")
    ci = torch.where(ok, cls, 0)
    ce = F.cross_entropy(sc, ci, reduction="none") * ok
    # the kernel's log-sum-exp under the tracker: lane sums of ceil(K1 / 32) terms, 5 butterfly levels
    t = (T(s) - T(mx)).exp()
    nl = math.ceil(K1 / 32) + 5
    se_v = t.v.sum(1)
    se = T(se_v, t.e.sum(1) + (nl * U / (1 - nl * U)) * (t.v.abs().sum(1) + t.e.sum(1)))
    lse = se.log()
    xc = T(s.gather(1, ci[:, None])[:, 0]) - T(mx[:, 0])
    lce = lse - xc
    p = (T(s) - T(mx) - T(lse.v[:, None], lse.e[:, None])).exp()
    onehot = (torch.arange(K1, device=dev)[None] == cls[:, None]).to(F64)
    gsc_b = torch.where(ok[:, None], ((p - T(onehot)) * gs[0]).e * SELF, 0.0)
    sums = [float(ce.detach().sum()), 0.0]
    parts = frcnn_ctas(R)
    bnds = [sum_bound(ce.detach(), torch.where(ok, lce.e, 0.0) * SELF, 1, parts), 0.0]
    gd_b = torch.zeros_like(dl.detach())
    und_d = torch.zeros_like(dl.detach(), dtype=torch.bool)
    rows = torch.nonzero(fg)[:, 0]
    cols = (torch.zeros_like(rows) if kreg == 1 else cls[rows] * D)[:, None] + torch.arange(D, device=dev)[None]
    dp = dl[rows[:, None], cols]
    pr, gt = proposals.to(dev, F64)[rows], gt_boxes.to(dev, F64)[rows]
    if loss_type == SL1:
        w32 = (proposals[:, 2] - proposals[:, 0]) if D == 4 else proposals[:, 2]
        if bool((~(w32.to(dev)[rows] > 0)).any()):
            status |= STATUS_WIDTH
        tg = get_deltas_ref(pr, gt, w)
        d_t, wrap_und = get_deltas_t(_rows(pr, None), _rows(gt, None), w)
        tg_t = [T(tg[:, q].clone(), d_t[q].e) for q in range(D)]
        if pin is not None:
            pp = pin.to(dev)[rows]
            tg = torch.where(pp, dp.detach(), tg)
            tg_t = [where(pp[:, q], T(dp.detach()[:, q]), tg_t[q]) for q in range(D)]
        lr = smooth_l1_ref(dp, tg, beta)
        e_terms = []
        for q in range(D):
            lq, gq, uq = smooth_l1_t(T(dp.detach()[:, q]) - tg_t[q], beta)
            e_terms.append(lq.e)
            gd_b[rows, cols[:, q]] = (gq * gs[1]).e * SELF
            und_d[rows, cols[:, q]] = uq | wrap_und
        sums[1] = float(lr.detach().sum())
        bnds[1] = sum_bound(lr.detach().reshape(-1), torch.stack(e_terms, 1).reshape(-1) * SELF, 1, parts)
    else:
        lr = giou_ref(apply_deltas_ref(dp, pr, w, clamp), gt)
        lt, g_t, und, _, ordered = giou_row_t(_rows(pr, None), [T(dp.detach()[:, q]) for q in range(4)], _rows(gt, None),
                                              w, clamp)
        if not bool(ordered.all()):
            status |= STATUS_ORDER
        for q in range(4):
            gd_b[rows, cols[:, q]] = (g_t[q] * gs[1]).e * SELF
            und_d[rows, cols[:, q]] = und
        sums[1] = float(lr.detach().sum())
        bnds[1] = sum_bound(lr.detach(), lt.e * SELF, 1, parts)
    total = ce.sum() * gs[0] + lr.sum() * gs[1]
    if total.requires_grad:
        gsc, gdl = torch.autograd.grad(total, [sc, dl], allow_unused=True)
    else:
        gsc, gdl = None, None
    gsc = torch.zeros_like(s) if gsc is None else gsc
    gdl = torch.zeros_like(dl.detach()) if gdl is None else gdl
    if status & STATUS_CLASS:
        labels_out.add("status_class")
    n_und = int(und_d.sum())
    return Result(sums, bnds, counts, status, [gsc, gdl], [gsc_b, gd_b],
                  [torch.zeros_like(s, dtype=torch.bool), und_d], labels_out, n_und, len(rows) * D - n_und)


# ---- the path model ---------------------------------------------------------------------------------------------------
def vec_elems(dtype):
    return 4 if dtype == torch.float32 else 8


def dense_ctas(N, K, R_levels, vec):
    """Classification CTAs (kThreads * kItems * V::N elements each, per level) plus regression CTAs (kThreads rows)."""
    chunk = K_THREADS * K_ITEMS * vec
    return sum(-(-(N * r * K) // chunk) for r in R_levels) + -(-(N * sum(R_levels)) // K_THREADS)


def frcnn_ctas(R):
    return -(-R // K_WARPS) if R > 0 else 0


def dense_refuses(K, box_dim, label_kind_i8, loss_type, aligned=True):
    """The argument rules of dense_setup that the cases here touch: True where the library returns EINVAL."""
    if label_kind_i8 and K != 1:
        return True
    if loss_type == GIOU and box_dim != 4:
        return True
    if loss_type == LIN and (box_dim != 4 or label_kind_i8):
        return True
    return not aligned


def dense_shape_labels(N, K, R_levels, dtype, rpn, gamma, alpha, loss_type=SL1):
    v = vec_elems(dtype)
    chunk = K_THREADS * K_ITEMS * v
    out = {"vec4" if v == 4 else "vec8", "labels_i8" if rpn else "labels_i64"}
    for r in R_levels:
        el = N * r * K
        if el == 0:
            out.add("empty_level")
            continue
        if el % v:
            out.add("tail_partial")
        if K % v:
            out.add("row_ends_in_vector")
        if K < v:
            out.add("rows_per_vector_gt1")
        if N > 1 and (r * K) % v:
            out.add("image_boundary_in_vector")
        if (-el) % chunk >= v:  # the last CTA has whole vectors past the end: their threads leave the loop
            out.add("cta_early_break")
    g = f32(gamma)
    out.add("gamma0_alpha" if g == 0 and alpha >= 0 else "gamma0" if g == 0 else "gamma2" if g == 2 else "gamma_pow")
    rows = N * sum(R_levels)
    if rows % K_THREADS:
        out.add("reg_tail_cta")
    out.add("finish_multi_pass" if dense_ctas(N, K, R_levels, v) > K_THREADS else "finish_single_pass")
    return out


def frcnn_shape_labels(R, K, kreg, D, dtype, loss_type):
    k1 = K + 1
    out = set()
    if k1 < 32:
        out.add("k1_lt_32")
    elif k1 == 32:
        out.add("k1_eq_32")
    elif k1 == 33:
        out.add("k1_33")
    if k1 > 64:
        out.add("k1_many_passes")
    if R % K_WARPS:
        out.add("rows_ragged_cta")
    out.add("agnostic" if kreg == 1 and K > 1 else "class_specific")
    if D == 5:
        out.add("rot5")
    if loss_type == GIOU:
        out.add("giou")
    if dtype == torch.float16:
        out.add("f16")
    if dtype == torch.bfloat16:
        out.add("bf16")
    return out
