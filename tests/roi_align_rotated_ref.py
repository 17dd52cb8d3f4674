"""Float64 reference and path model of the rotated RoIAlign kernels (detectron2_b200/csrc/roi_align.cu).

Reference: forward and backward of ROIAlignRotated, one RoI at a time.  The geometry is restated in fp32 in load_geom<true>'s
expression order (:86-121): centre = roi * scale - 0.5, sides = roi * scale, theta = (float)((double)angle * pi / 180),
bin = side / P, grid = sr or ceil(side / P) clamped at 0, count = max(gh * gw, 1), a dead RoI (NaN level) has an empty grid.
The sampling grid and the level come out bit-identical to the kernels'.  Every sample position is then computed in float64
from those fp32 values and from cos / sin of the fp32 theta (rot_xy, :179-184), and make_tap2 (:160-177) is applied in
float64: a sample outside [-1, H] x [-1, W] contributes nothing, coordinates are clamped at 0, lo >= size - 1 collapses to the
last row / column.  The weights of one RoI form a sparse [bins, H * W] matrix W (duplicate taps summed, divided by the count);
the forward is W x and the backward is W^T g, so the two cannot drift apart.

Besides the value, every output element carries A = the same operator applied to |x| (forward) or |grad_out| (backward),
m = the number of fp32 terms the kernel sums into it, and P, a position-error term:

    |got - ref| <= (m + 5) 2^-24 A + P        (+ half an ulp of fp16 / bf16 outputs)

The first term is the rounding of the fp32 sums and of the weights (as for the axis-aligned kernels, tests/roi_align_ref.py).
The second exists because rotated sample positions are not exact in fp32: the kernels rotate with sincosf (at most 2 ulp of
error, CUDA C Programming Guide, "Mathematical Functions": sinf / cosf / sincosf) and roi_align.cu is compiled with FMA
contraction.  Per sample, with eps = 2^-24, Y = |start_h| + |ph bin_h| + |(iy + .5) bin_h / gh| (the terms of yy), X the same
for xx, and ctr = max(|ctr_h|, |ctr_w|), the kernel's fp32 y differs from the float64 one by at most
    yy:      5 roundings (ph*bin, +start, (iy+.5)*bin, /g, +), each <= eps times a quantity <= Y, times |cos| <= 1   5 eps Y
    cos:     2 ulp <= 4 eps |cos|, times |yy| <= Y                                                                    4 eps Y
    xx, sin: the same for the second term                                                                         9 eps X
    centre:  roi * scale - 0.5 rounded once (contracted) or twice (the reference): <= eps |roi s| + 2 eps |ctr|    3 eps (ctr + 1/2)
    y:       two products and two sums, each <= eps (Y + X + ctr)                                                4 eps (Y + X + ctr)
that is eps (13 (Y + X) + 7 ctr + 3/2), and the same for x.  Second-order terms are below eps^2 * 200 (Y + X + ctr); the bound
    delta_s = C_POS 2^-24 (Y + X + ctr + 1),  C_POS = 14
covers both with the one unit of slack.  A bilinear patch has slope at most L_s = max(|v3 - v1|, |v4 - v2|) + max(|v2 - v1|,
|v4 - v3|) over its four taps, and clamping to the map keeps it continuous except at y = -1, y = H, x = -1, x = W, so the
forward's P = (1 / count) sum_s delta_s L_s, L_s taken over every cell the delta_s-box around the sample touches.  A bilinear
weight moves by at most delta in y plus delta in x, so the backward's P at a pixel is sum_s |g| 2 delta_s / count over the
samples whose delta_s-box reaches the pixel.  At angle 0 (sincosf(0) is exact) with every fp32 intermediate exact (dyadic
geometry), delta_s = 0 and the bound reduces to the axis-aligned one.

A sample within delta_s of one of the four discontinuities is ambiguous: the kernel and the reference may legitimately take
different branches there.  Roi.ambiguous counts them.

Path model: the per-RoI and per-launch decisions of the rotated kernels and their launchers, restated with line references:
  roi_align_rot_fwd_kernel<1024>   NCHW forward     table / on the fly (:204), channel slabs of pick_c_per_cta (:730, :1702)
  roi_align_rot_bwd_kernel         NCHW backward    early return on an empty grid (:256), the same slabs (:1729)
  roi_align_rot_nhwc_kernel        channels-last    table / on the fly (:1424), 128-channel slabs and lane_live (:1411-1423)
  nhwc_supported                   D2B_ROI_ROTATED  [128][bins | 1] fp32 tile <= 150 KB (:1511-1513)
  ops._pick_layout                 layout of a call
"""
import math
from collections import namedtuple

import numpy as np
import scipy.sparse as sp

from roi_align_ref import EPS32, cdiv, half_ulp

K_ROT_MAXTAP = 1024  # kRotMaxTap (:1399) and roi_align_rot_fwd_kernel<1024> (:1704)
K_NHWC_CH = 128      # kNhwcCh (:742)
C_POS = 14           # position-error constant, derived in the module docstring

Geom = namedtuple("Geom", "b ctr_h ctr_w rh rw theta start_h start_w bin_h bin_w gh gw count")


def geom(roi, scale, ph, pw, sr, dead=False):
    """load_geom<true> (:86-121) in fp32.  roi = (b, cx, cy, w, h, angle) in image coordinates."""
    f = np.float32
    s = f(scale)
    ctr_w, ctr_h = f(f(roi[1]) * s) - f(0.5), f(f(roi[2]) * s) - f(0.5)
    rw, rh = f(f(roi[3]) * s), f(f(roi[4]) * s)
    theta = f(float(f(roi[5])) * math.pi / 180.0)
    bin_h, bin_w = f(rh / f(ph)), f(rw / f(pw))
    gh = sr if sr > 0 else max(int(math.ceil(bin_h)), 0)
    gw = sr if sr > 0 else max(int(math.ceil(bin_w)), 0)
    if dead:
        gh = gw = 0
    return Geom(int(roi[0]), float(ctr_h), float(ctr_w), float(rh), float(rw), float(theta), float(-rh / f(2)),
                float(-rw / f(2)), float(bin_h), float(bin_w), gh, gw, max(gh * gw, 1))


def _exact32(*vals):
    return all(np.all(np.float32(v) == v) for v in vals)


def _terms(start, bin_, p, i, g):
    """The three terms of rot_xy's yy (or xx) in float64, and whether each fp32 step of the kernel is exact."""
    a = p * bin_
    q = (i + 0.5) * bin_
    d = q / g
    exact = _exact32(a, start + a, q, d, start + a + d) and np.all(d * g == q)
    return start + a + d, np.abs(start) + np.abs(a) + np.abs(d), exact


def _tap1(v, size):
    """make_tap1 (:130-152) after the range test, in float64: (lo, hi, weight of hi)."""
    v = np.maximum(v, 0.0)
    lo = np.floor(v).astype(np.int64)
    last = lo >= size - 1
    lo = np.where(last, size - 1, lo)
    hi = np.where(last, size - 1, lo + 1)
    return lo, hi, np.where(last, 0.0, v - lo)


class Roi:
    """One rotated RoI on one level: every sample's float64 position, its taps and delta_s, the sparse weight matrices."""

    def __init__(self, roi, scale, ph, pw, sr, h, w, dead=False):
        self.g = g = geom(roi, scale, ph, pw, sr, dead)
        self.ph, self.pw, self.h, self.w = ph, pw, h, w
        bins = ph * pw
        P, Q, I, J = np.meshgrid(np.arange(ph), np.arange(pw), np.arange(g.gh), np.arange(g.gw), indexing="ij")
        P, Q, I, J = (a.ravel().astype(np.float64) for a in (P, Q, I, J))
        self.bin = (P * pw + Q).astype(np.int64)
        yy, ty, ey = _terms(g.start_h, g.bin_h, P, I, g.gh if g.gh else 1)
        xx, tx, ex = _terms(g.start_w, g.bin_w, Q, J, g.gw if g.gw else 1)
        th = np.float64(g.theta)
        c, s = math.cos(th), math.sin(th)
        self.y = yy * c - xx * s + g.ctr_h
        self.x = yy * s + xx * c + g.ctr_w
        exact = (g.theta == 0.0 and ey and ex and _exact32(self.y, self.x)
                 and _exact32(float(np.float32(roi[1])) * scale, float(np.float32(roi[2])) * scale))
        ctr = max(abs(g.ctr_h), abs(g.ctr_w))
        self.delta = np.zeros_like(self.y) if exact else C_POS * EPS32 * (ty + tx + ctr + 1.0)
        self.inside = (self.y >= -1) & (self.y <= h) & (self.x >= -1) & (self.x <= w)
        d = self.delta
        self.ambiguous = int(sum(((np.abs(v - e) <= d).sum() for v, e in
                                  ((self.y, -1.0), (self.y, float(h)), (self.x, -1.0), (self.x, float(w))))))
        # the four taps of every in-map sample: weights / count in a sparse [bins, H * W] matrix
        yl, yh, ly = _tap1(self.y, h)
        xl, xh, lx = _tap1(self.x, w)
        cols = np.stack([yl * w + xl, yl * w + xh, yh * w + xl, yh * w + xh])
        wts = np.stack([(1 - ly) * (1 - lx), (1 - ly) * lx, ly * (1 - lx), ly * lx]) / g.count
        keep = np.broadcast_to(self.inside, cols.shape)
        rows = np.broadcast_to(self.bin, cols.shape)
        shape = (bins, h * w)
        self.W = sp.csr_matrix((wts[keep], (rows[keep], cols[keep])), shape=shape)
        self.absW = abs(self.W)
        self.M = sp.csr_matrix((np.ones(keep.sum()), (rows[keep], cols[keep])), shape=shape)  # terms per (bin, pixel)
        # the delta-box of every in-map sample: its corners' taps, and the block of pixels it reaches
        box = []
        for dy in (-1, 1):
            for dx in (-1, 1):
                cy, cx = np.clip(self.y + dy * d, -1, h), np.clip(self.x + dx * d, -1, w)
                a, b, _ = _tap1(cy, h)
                e, f, _ = _tap1(cx, w)
                box.append((a, b, e, f))
        self.corners = box
        r0, r1 = np.minimum(box[0][0], box[1][0]), np.maximum(box[2][1], box[3][1])
        c0, c1 = np.minimum(box[0][2], box[2][2]), np.maximum(box[1][3], box[3][3])
        blk_r, blk_c, blk_v = [], [], []
        for i in range(3):
            for j in range(3):
                live = self.inside & (r0 + i <= r1) & (c0 + j <= c1)
                blk_r.append(self.bin[live])
                blk_c.append(((r0 + i) * w + c0 + j)[live])
                blk_v.append(2 * d[live] / g.count)
        self.Pb = sp.csr_matrix((np.concatenate(blk_v), (np.concatenate(blk_r), np.concatenate(blk_c))), shape=shape)
        self.Pf = sp.csr_matrix((d[self.inside] / g.count, (self.bin[self.inside], np.nonzero(self.inside)[0])),
                                shape=(bins, len(self.y)))

    @property
    def samples(self):
        return self.g.gh * self.g.gw

    def forward(self, img):
        """img: [C, H, W] -> (out, A, m, P), each [C, PH, PW] float64."""
        x = _np(img).reshape(img.shape[0], -1)
        out = (self.W @ x.T).T
        a = (self.absW @ np.abs(x).T).T
        m = np.full_like(out, 4.0 * self.samples)
        p = np.zeros_like(out)
        if self.inside.any():
            slope = np.zeros((x.shape[0], len(self.y)))
            for a0, a1, b0, b1 in self.corners:
                v1, v2, v3, v4 = x[:, a0 * self.w + b0], x[:, a0 * self.w + b1], x[:, a1 * self.w + b0], x[:, a1 * self.w + b1]
                slope = np.maximum(slope, np.maximum(np.abs(v3 - v1), np.abs(v4 - v2)) + np.maximum(np.abs(v2 - v1), np.abs(v4 - v3)))
            p = (self.Pf @ slope.T).T
        shp = (x.shape[0], self.ph, self.pw)
        return out.reshape(shp), a.reshape(shp), m.reshape(shp), p.reshape(shp)

    def backward(self, go):
        """go: [C, PH, PW] -> (grad, A, m, P), each [C, H, W] float64."""
        g = _np(go).reshape(go.shape[0], -1)
        shp = (g.shape[0], self.h, self.w)
        res = ((self.W.T @ g.T).T, (self.absW.T @ np.abs(g).T).T,
               np.broadcast_to(np.asarray(self.M.sum(0)), (g.shape[0], self.h * self.w)), (self.Pb.T @ np.abs(g).T).T)
        return tuple(np.asarray(r).reshape(shp) for r in res)


def _np(t):
    return t.detach().double().cpu().numpy() if hasattr(t, "detach") else np.asarray(t, dtype=np.float64)


def forward(feats, rois, scales, lv, ph, pw, sr):
    """The pooled output of every RoI: feats = the levels [N, C, H, W], lv[k] = level of RoI k (-1: none, zero output)."""
    k, c = len(rois), feats[0].shape[1]
    out = [np.zeros((k, c, ph, pw)) for _ in range(4)]
    for i, r in enumerate(np.asarray(rois, dtype=np.float32)):
        l = max(lv[i], 0)  # the kernels sample a RoI without a level on level 0, with an empty grid
        f = feats[l]
        R = Roi(r, scales[l], ph, pw, sr, f.shape[2], f.shape[3], dead=lv[i] < 0)
        for o, v in zip(out, R.forward(f[R.g.b])):
            o[i] = v
    return tuple(out)


def backward(go, shapes, rois, scales, lv, ph, pw, sr):
    """Gradients of every level (shapes: [N, C, H, W] each) for grad_out `go` [K, C, PH, PW]: (grad, A, m, P) per level."""
    go = _np(go)
    res = [tuple(np.zeros(s) for _ in range(4)) for s in shapes]
    for i, r in enumerate(np.asarray(rois, dtype=np.float32)):
        l = max(lv[i], 0)
        s = shapes[l]
        R = Roi(r, scales[l], ph, pw, sr, s[2], s[3], dead=lv[i] < 0)
        for arr, v in zip(res[l], R.backward(go[i])):
            arr[R.g.b] += v
    return res


def tolerance(ref, a, m, p, dtype=None):
    tol = (np.asarray(m) + 5) * EPS32 * a + p
    if dtype is not None:
        tol = tol + half_ulp(np.abs(ref) + tol, dtype)
    return tol


def check(got, ref, a, m, p, dtype=None, what=""):
    got = _np(got)
    tol = tolerance(ref, a, m, p, dtype)
    err = np.abs(got - ref)
    bad = err > tol
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), 0)), err.shape)
        raise AssertionError("%s: %d of %d elements outside (m + 5) 2^-24 A + P%s; worst at %s: got %r ref %r tol %r"
                             % (what, bad.sum(), bad.size, " + half ulp" if dtype else "", i, got[i], ref[i], tol[i]))


# =========================================================================================== path model
def pick_c_per_cta(k, c, sms):
    """pick_c_per_cta (:730-734): channels per CTA of both NCHW rotated kernels."""
    cpc = c
    while cpc > 16 and k * cdiv(c, cpc) < 4 * sms:
        cpc = (cpc + 1) // 2
    return cpc


def nhwc_supported(c, hw, ph, pw):
    """nhwc_supported (:1506-1513) for D2B_ROI_ROTATED, forward and backward alike."""
    if c % 4:
        return False
    if any(h * w * (c // 4) >= 1 << 28 for h, w in hw):
        return False
    return 4 * K_NHWC_CH * ((ph * pw) | 1) <= 150 * 1024


def pick_layout(setting, c, hw, ph, pw, channels_last):
    """ops._pick_layout for a rotated call with POOLER_LAYOUT = "nchw" or "nhwc"."""
    if setting == "nchw" or not nhwc_supported(c, hw, ph, pw):
        return "nchw"
    return "cl" if channels_last else "xpose"


def slabs(c):
    """Channel slabs of roi_align_rot_nhwc_kernel (grid.y): (first channel, channels); lanes with lane * 4 >= channels are
    not lane_live (:1422-1423)."""
    return [(c0, min(K_NHWC_CH, c - c0)) for c0 in range(0, c, K_NHWC_CH)]


def roi_labels(R, nhwc):
    """Paths of the rotated kernels for one RoI: table or taps on the fly, the same test in both kernels (:204, :1424)."""
    taps = R.ph * R.pw * R.samples
    if taps == 0:
        return {"empty_grid"}  # no taps; roi_align_rot_bwd_kernel returns early (:256)
    kinds = {"table_1024" if taps == K_ROT_MAXTAP else "table" if taps < K_ROT_MAXTAP else "onfly"}
    out = {"nchw_" + t for t in kinds}
    if nhwc:
        out |= {"nhwc_" + t for t in kinds}
    return out


def launch_labels(k, c, ph, pw, hw, sms):
    out = set()
    cpc = pick_c_per_cta(k, c, sms)
    out.add("cpc_whole" if cpc == c else ("cpc_ragged" if c % cpc else "cpc_split"))
    if c % 4:
        out.add("c_not_4")
    elif not nhwc_supported(c, hw, ph, pw):
        out.add("nhwc_refused")
    else:
        sl = slabs(c)
        out.add("slab_full" if c == K_NHWC_CH else "slab_partial" if c < K_NHWC_CH
                else "slab_ragged" if sl[-1][1] < K_NHWC_CH else "slab_multi")
        if ph * pw == 299:
            out.add("nhwc_largest_pooled")
    if ph != pw:
        out.add("non_square")
    return out


ANGLES = {0.0: "angle0", 90.0: "angle90", -90.0: "angle-90", 180.0: "angle180", -180.0: "angle-180", 45.0: "angle45"}


def boundary_labels(R, roi, sr):
    """Sampling-ratio, angle, position and box-shape labels of one RoI."""
    g = R.g
    out = {"sr%d" % sr, ANGLES.get(float(roi[5]), "angle_other")}
    if g.b == 1:
        out.add("batch1")
    if R.samples:
        n_in = int(R.inside.sum())
        out.add("outside_whole" if n_in == 0 else "outside_partial" if n_in < len(R.y) else "inside")
    if sr > 0 and (g.rh < 0 or g.rw < 0):
        out.add("mirrored")
    if 0 < g.rh < 1 and 0 < g.rw < 1:
        out.add("sub_pixel")
    if R.samples and not R.delta.any():
        for name, v in (("-1", lambda n: -1.0), ("0", lambda n: 0.0), ("H-1", lambda n: n - 1.0), ("H", lambda n: float(n))):
            if (R.y == v(R.h)).any() and (R.x == v(R.w)).any():
                out.add("pos_" + name)
    return out
