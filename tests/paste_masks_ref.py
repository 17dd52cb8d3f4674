"""Float64 reference, error bound and path model of the paste kernels (detectron2_b200/csrc/paste_masks.cu).

Reference: the GPU branch of detectron2's _do_paste_mask (mask_ops.py:17-69, skip_empty=False: every pixel of the image),
i.e. grid_sample with bilinear sampling, zero padding and align_corners=False, computed in float64 from the fp32 box and mask
values.  Pixel p of an axis with box edges b0, b1 samples the mask at

    q = (p + 0.5 - b0) / (b1 - b0),   i = ((2 q - 1 + 1) M - 1) / 2 = q M - 1/2,

and the bilinear weight of mask column j is max(0, 1 - |i - j|) -- zero padding makes the four taps of a sample outside
(-1, M) zero.  The map is separable: v = Ay @ mask @ Ax.T with Ax[p, j] the weight of mask column j at image column p.  A
sample coordinate that is not finite (a zero or negative extent where a pixel centre meets b0, a NaN or infinite corner)
gives v = 0: that is the kernel's contract (paste_value, :33-34).  The one exception is left as it is: at threshold exactly 0 a
NaN coordinate gives 0 >= 0, a pixel set, where grid_sample's NaN would compare False.

Bound.  paste_masks.cu is compiled with -fmad=false, so sample_coord (:24-27) rounds each step once.  With eps = 2^-24 and
p + 0.5 exact (p < 2^23): p + 0.5 - b0 and b1 - b0 are single roundings of exact differences, the quotient a third, so q is
within 3 eps |q|; 2q is exact; 2q - 1 and + 1 round within eps (|2q| + 1) in total, which M / 2 scales; * M and - 1 round
within eps |2 q M| + eps (|2 q M| + 1), which / 2 (exact) halves.  To first order

    |ix - i| <= eps (3 M |q| + M |q| + M / 2 + 2 M |q| + 1 / 2) <= eps (7 M |q| + M / 2 + 1 / 2),

and the bound used, delta = eps (7 M |q| + M + 1), keeps M / 2 + 1 / 2 for the second-order terms.  The error grows with
M |p + 0.5 - b0| / |b1 - b0|, so sub-pixel boxes get a large delta far from the box (where v is 0 anyway).
v is piecewise bilinear in (ix, iy) and continuous, zero padding included, so a coordinate error moves it by at most
L (delta_x + delta_y), L = the largest step between neighbouring values of the zero-padded mask.  paste_value (:30-45) then
forms each of the four terms m * (wx * wy) with four roundings (wx0 = xe - ix, wy0, the product, the scaling by m; wx1 =
ix - fx is exact) and adds them with three more: within 7 eps sum |terms| <= 7 eps A, A = the reference on |mask|.  So

    |v32 - v64| <= b = 8 eps A + L (delta_x + delta_y),

and b = 0 where a coordinate lies more than its delta beyond the support (i + delta <= -1 or i - delta >= M) or is not
finite: there v32 = v64 = 0 exactly.

A boolean pixel (threshold t >= 0, compared in fp32) is decidable when v64 - b >= t (set) or v64 + b < t (clear).  A uint8
pixel (t < 0: (uint8) fl(255 v)) is decidable when floor(255 (v64 -+ b) -+ 255 eps |v64|) agree; an undecidable one may
take either of the two values.

Path model: the launch decisions of d2b_paste_masks / d2b_paste_masks_packed (:319-368) for a given SM count, paste_rect
(:59-71), the CTAs paste_assign (:77-128) gives each mask, each mask's head, its ragged tail, the chunks of phase 1 that
wrap a row (:177-183) and the row spills of phase 2a (:194-235), restated in numpy float32 and Python integers.
"""
import numpy as np

from roi_align_ref import EPS32, cdiv

K_THREADS = 256      # kThreads
K_PIX = 16           # kPix: output bytes per phase-1 chunk
K_MAX_M = 64         # kMaxM
K_MAX_GRID_Y = 65535  # kMaxGridY: masks per launch of a (CTAs per mask, N) grid
TAB_MAX_BYTES = 30 * 1024
C_VAL = 8


# =========================================================================================== reference
def axis(n, b0, b1, m):
    """Sample coordinates of pixels 0..n-1 of one axis: (i, delta, weights [n, m], zero) -- zero marks the pixels whose
    coordinate lies beyond the support by more than delta, or is not finite, where v is exactly 0."""
    assert n <= 1 << 23
    b0, b1 = float(np.float32(b0)), float(np.float32(b1))
    p = np.arange(n, dtype=np.float64)
    with np.errstate(all="ignore"):
        q = (p + 0.5 - b0) / (b1 - b0)
        i = q * m - 0.5
    fin = np.isfinite(i)
    d = np.where(fin, EPS32 * (7.0 * m * np.abs(np.where(fin, q, 0.0)) + m + 1.0), 0.0)
    zero = ~fin | (i + d <= -1.0) | (i - d >= m)
    ic = np.where(fin, i, -2.0)
    w = np.maximum(0.0, 1.0 - np.abs(ic[:, None] - np.arange(m)[None, :]))
    return ic, d, w, zero


def max_step(mask):
    """L: the largest difference between neighbouring values of the zero-padded mask."""
    p = np.pad(np.asarray(mask, dtype=np.float64), 1)
    return float(max(np.abs(np.diff(p, axis=0)).max(), np.abs(np.diff(p, axis=1)).max()))


class Paste:
    """One mask pasted into an H x W image: the window [r0, r1) x [c0, c1) outside which v = b = 0 exactly, and v64, the
    bound b and A inside it."""

    def __init__(self, mask, box, h, w):
        mask = np.asarray(mask, dtype=np.float32).astype(np.float64)
        m = mask.shape[-1]
        ix, dx, ax, zx = axis(w, box[0], box[2], m)
        iy, dy, ay, zy = axis(h, box[1], box[3], m)
        cols, rows = np.nonzero(~zx)[0], np.nonzero(~zy)[0]
        if len(cols) and len(rows):
            self.c0, self.c1, self.r0, self.r1 = int(cols[0]), int(cols[-1]) + 1, int(rows[0]), int(rows[-1]) + 1
            assert len(cols) == self.c1 - self.c0 and len(rows) == self.r1 - self.r0  # i is monotonic in p
        else:
            self.c0 = self.c1 = self.r0 = self.r1 = 0
        ays, axs = ay[self.r0:self.r1], ax[self.c0:self.c1]
        self.v = ays @ mask @ axs.T
        self.a = ays @ np.abs(mask) @ axs.T
        self.b = C_VAL * EPS32 * self.a + max_step(mask) * (dy[self.r0:self.r1, None] + dx[None, self.c0:self.c1])
        self.h, self.w = h, w

    def full(self, what="v"):
        out = np.zeros((self.h, self.w))
        out[self.r0:self.r1, self.c0:self.c1] = getattr(self, what)
        return out


def soft(masks, boxes, h, w):
    """v64 and b of every mask: two [N, H, W] float64 arrays (small images only)."""
    ps = [Paste(mk, bx, h, w) for mk, bx in zip(np.asarray(masks), np.asarray(boxes, dtype=np.float32))]
    return np.stack([p.full("v") for p in ps]), np.stack([p.full("b") for p in ps])


def decide(v, b, threshold):
    """(expected byte, decidable, lowest, highest allowed byte) of pixels with reference value v and bound b."""
    t = float(np.float32(threshold))
    if t >= 0:
        hi, lo = v - b >= t, v + b < t
        want = hi.astype(np.int64)
        return want, hi | lo, want * (hi | lo), np.where(hi | lo, want, 1)
    lo = np.floor(255.0 * (v - b) - 255.0 * EPS32 * np.abs(v)).astype(np.int64)
    hi = np.floor(255.0 * (v + b) + 255.0 * EPS32 * np.abs(v)).astype(np.int64)
    return lo, lo == hi, lo, hi


def outside_byte(threshold):
    """The value of a pixel that cannot see its mask (v = 0): zbyte / zbit (:154, :296)."""
    t = float(np.float32(threshold))
    return (1 if 0.0 >= t else 0) if t >= 0 else 0


# =========================================================================================== path model
def status(n, m, h, w, threshold=0.5, packed=False):
    """The refusals of both entry points (:321-326, :339-343) on valid pointers: 'ok', 'einval' or 'unsupported'."""
    if n == 0 or h == 0 or w == 0:
        return "ok"
    if n < 0 or m <= 0 or h < 0 or w < 0 or (packed and not threshold >= 0):
        return "einval"
    if m > K_MAX_M or h * w >= 1 << 30:
        return "unsupported"
    return "ok"


def paste_rect(box, m, h, w):
    """paste_rect (:59-71) in float32: ((cx0, cx1, ry0, ry1), kind), kind = narrowed, clipped (narrowed, then cut by an
    image border), full_narrow (W < 32), full_nonfinite, full_degenerate (extent <= 0) or full_huge (extent or |x0|, |y0|
    >= 1e8)."""
    f = np.float32
    x0, y0, x1, y1 = (f(v) for v in box)
    with np.errstate(all="ignore"):
        bw, bh = f(x1 - x0), f(y1 - y0)
        big = f(1e8)
        if w >= 2 * K_PIX and bw > 0 and bh > 0 and bw < big and bh < big and abs(x0) < big and abs(y0) < big:
            fm = f(m)
            fx0, fx1 = f(np.floor(f(x0 - f(bw / fm)))) - f(2), f(np.ceil(f(x1 + f(bw / fm)))) + f(2)
            fy0, fy1 = f(np.floor(f(y0 - f(bh / fm)))) - f(2), f(np.ceil(f(y1 + f(bh / fm)))) + f(2)
            r = (int(max(fx0, f(0))), int(min(fx1, f(w - 1))), int(max(fy0, f(0))), int(min(fy1, f(h - 1))))
            cut = fx0 < 0 or fy0 < 0 or fx1 > w - 1 or fy1 > h - 1
            return r, "clipped" if cut and not rect_empty(r) else "narrowed"
    full = (0, w - 1, 0, h - 1)
    if w < 2 * K_PIX:
        return full, "full_narrow"
    if not all(np.isfinite(v) for v in (x0, y0, x1, y1)):
        return full, "full_nonfinite"
    if not (bw > 0 and bh > 0):
        return full, "full_degenerate"
    return full, "full_huge"


def rect_empty(r):
    return r[1] < r[0] or r[3] < r[2]


def rect_pixels(r):
    return 0 if rect_empty(r) else (r[1] - r[0] + 1) * (r[3] - r[2] + 1)


def cta_counts(rects, h, w, sms):
    """paste_assign (:77-128): the CTAs of a balanced launch each mask gets -- one plus a share of the spare CTAs in
    proportion to its cost (zero fill of the plane + exact evaluation of its rectangle), in integer arithmetic."""
    total = 8 * sms
    fill = (h * w // K_PIX) * 24
    cost = [((fill + (0 if rect_empty(r) else (r[3] - r[2] + 1) * (r[1] - r[0] + 32) * 44)) >> 8) + 1 for r in rects]
    tot, spare, prefix, out = sum(cost), total - len(rects), 0, []
    for k, c in enumerate(cost):
        b0 = k + spare * prefix // tot
        b1 = k + 1 + spare * (prefix + c) // tot
        out.append(b1 - b0)
        prefix += c
    assert sum(out) == total
    return out


def launch(n, m, h, w, sms):
    """d2b_paste_masks (:344-368): dict(balanced, tab, gx (CTAs per mask of a uniform launch), capped, launches)."""
    plane = h * w
    chunks = cdiv(plane, K_PIX)
    tab = w >= 2 * K_PIX and 4 * (w + h + 2) <= TAB_MAX_BYTES
    total = 8 * sms
    if 2 * n <= total:
        return dict(balanced=True, tab=tab, gx=None, capped=False, launches=1)
    gx = cdiv(chunks + 1, K_THREADS)
    want = cdiv(8 * sms, n)
    capped = gx > want
    if capped:
        gx = max(want, 1)
    return dict(balanced=False, tab=tab, gx=gx, capped=capped, launches=cdiv(n, K_MAX_GRID_Y))


def launch_packed(n, h, w, sms):
    """d2b_paste_masks_packed (:327-335): dict(gx, capped, launches)."""
    words = h * cdiv(w, 32)
    want = max(1, cdiv(16 * sms, n))
    gx = min(cdiv(words, K_THREADS), want)
    return dict(gx=gx, capped=gx < cdiv(words, K_THREADS), launches=cdiv(n, K_MAX_GRID_Y))


def head_of(k, plane):
    """Bytes before the first 16-byte boundary of plane k (:159), the output itself 16-byte aligned."""
    return (16 - (k * plane) % 16) % 16


def mask_geometry_labels(k, rect, h, w, tab):
    """Head, tail, phase-1 row wraps and phase-2a row spills of mask k with rectangle `rect`."""
    out = set()
    plane = h * w
    head = head_of(k, plane)
    if head and plane > 0:
        out.add("head_unaligned")
    if plane > head and (plane - head) % K_PIX:
        out.add("ragged_tail")
    if rect_empty(rect):
        return out
    cx0, cx1, ry0, ry1 = rect
    # phase 1: chunks active only through the row they wrap into (:181-182)
    s = head + K_PIX * np.arange((plane - head) // K_PIX, dtype=np.int64)
    py, px = s // w, s % w
    pxe = px + K_PIX - 1
    wrap = pxe >= w
    same = (py >= ry0) & (py <= ry1) & (px <= cx1)
    nxt = (py + 1 >= ry0) & (py + 1 <= ry1) & (pxe - w >= cx0)
    if (wrap & ~same & nxt).any():
        out.add("chunk_wrap_active")
    if (wrap & ~same & nxt & (pxe - w == cx0)).any():
        out.add("chunk_wrap_at_cx0")
    if tab:  # phase 2a: a widened row reaching columns the rectangle's own table range [c_lo, c_hi] does not hold
        r = np.arange(ry0, ry1 + 1, dtype=np.int64)
        lo, hi = r * w + cx0, r * w + cx1
        a = np.where(lo < head, head, ((lo - head) & ~(K_PIX - 1)) + head)
        b = np.where(hi < head, head, (((hi - head) >> 4) + 1) * K_PIX + head)
        b = np.minimum(b, head + (plane - head) // K_PIX * K_PIX)
        c_lo, c_hi = max(cx0 - (K_PIX - 1), 0), min(cx1 + (K_PIX - 1), w - 1)
        if ((a < r * w) & (a < b)).any() and c_hi < w - 1:
            out.add("spill_prev_row")
        if ((b > (r + 1) * w) & (a < b)).any() and c_lo > 0:
            out.add("spill_next_row")
    return out


def packed_labels(rects, h, w):
    out = {"packed"}
    if w % 32:
        out.add("packed_partial_word")
    for cx0, cx1, ry0, ry1 in rects:
        if cx1 >= cx0 and ry1 >= ry0 and cx1 % 32 == 0:
            out.add("packed_word_at_cx1")  # a word starting on the rectangle's last column (:305)
    return out


def path_labels(masks_m, boxes, h, w, threshold, sms, packed=True):
    """Every path label one call reaches on a device with `sms` SMs."""
    n = len(boxes)
    out = set()
    L = launch(n, masks_m, h, w, sms)
    out.add("byte_balanced" if L["balanced"] else "byte_uniform")
    out.add("tab" if L["tab"] else "notab_narrow" if w < 2 * K_PIX else "notab_large")
    if L["capped"]:
        out.add("uniform_gx_capped")
    if n > K_MAX_GRID_Y:
        out.add("n_over_65535")
    rects, kinds = zip(*(paste_rect(b, masks_m, h, w) for b in boxes))
    counts = cta_counts(rects, h, w, sms) if L["balanced"] else [L["gx"]] * n
    if max(counts) >= 2:
        out.add("mask_multi_cta")
    for r, kind in zip(rects, kinds):
        out.add("rect_empty" if kind == "narrowed" and rect_empty(r) else "rect_" + kind)
    # masks with the same head see the same geometry: one of each head is enough
    seen = set()
    for k, r in enumerate(rects):
        key = (head_of(k, h * w), r)
        if key in seen:
            continue
        seen.add(key)
        out |= mask_geometry_labels(k, r, h, w, L["tab"])
    t = float(np.float32(threshold))
    if t == 0.0:
        out.add("thr_zero")
    if t < 0:
        out.add("u8")
    if masks_m == 1:
        out.add("M1")
    if masks_m == K_MAX_M:
        out.add("M64")
    if packed and t >= 0:
        out |= packed_labels(rects, h, w)
        if launch_packed(n, h, w, sms)["capped"]:
            out.add("packed_gx_capped")
    return out


def known_constant(c, box, m, h, w):
    """Closed form for a constant mask c: v = c tri(ix) tri(iy), tri(i) = clip(min(i + 1, m - i), 0, 1) -- the weights of
    the columns that exist sum to 1 inside [0, m - 1] and fall linearly to 0 at -1 and m."""
    def tri(n, b0, b1):
        i = (np.arange(n) + 0.5 - float(np.float32(b0))) / (float(np.float32(b1)) - float(np.float32(b0))) * m - 0.5
        return np.clip(np.minimum(i + 1.0, m - i), 0.0, 1.0)

    return c * np.outer(tri(h, box[1], box[3]), tri(w, box[0], box[2]))
