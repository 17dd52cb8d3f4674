"""Float64 reference and path model of the axis-aligned RoIAlign kernels (detectron2_b200/csrc/roi_align.cu).

Reference: forward and backward of roi_align(aligned=True/False), one RoI at a time from its footprint crop.  Sample positions
are computed in fp32 in the kernels' expression order (load_geom, make_tap1 callers); weights, products and sums in float64;
the backward is the exact transpose.  Besides the values it returns, per output element, A = the same operator applied to
|input| and m = the number of terms the kernel's fp32 sum is made of, for the bound |got - ref| <= (m + 5) 2^-24 A.

Path model: the per-RoI and per-launch decisions of the three kernels and their launchers, restated with line references:
  roi_align_nhwc_kernel      channels-last forward      nhwc_fwd_labels, launch_fwd_nhwc
  roi_align_bwd_nhwc_kernel  channels-last backward     nhwc_bwd_labels, launch_bwd_nhwc
  roi_align_v3_kernel        NCHW forward and backward  v3_labels, launch_fwd
"""
import math
from collections import namedtuple

import numpy as np

from test_roi_align_column_walk import sample_pos, tap_list

# roi_align.cu constants
K_MAXE, K_MAXP, K_CAPPX, K_ROWOFF = 32, 16, 448, 1536  # :295-301
K_COLCAP = 192                                          # :814
K_NHWC_CH, K_NHWC_CHUNK = 128, 64                       # :742-743
K_BWD_BAND, K_BWD_MAXFW, K_BWD_WARPS = 64, 96, 8        # :1123-1125
EPS32 = 2.0 ** -24

Geom = namedtuple("Geom", "b start_h start_w bin_h bin_w gh gw count raw_h raw_w")


def geom(roi, scale, ph, pw, sr, aligned):
    """load_geom<false> (:80-122) in fp32.  raw_h / raw_w: the box sides before the aligned=False clamp to one pixel."""
    f = np.float32
    s, off = f(scale), f(0.5 if aligned else 0.0)
    sw, sh = f(f(roi[1]) * s) - off, f(f(roi[2]) * s) - off
    ew, eh = f(f(roi[3]) * s) - off, f(f(roi[4]) * s) - off
    raw_w, raw_h = f(ew - sw), f(eh - sh)
    rw, rh = (raw_w, raw_h) if aligned else (max(raw_w, f(1)), max(raw_h, f(1)))
    bin_h, bin_w = f(rh / f(ph)), f(rw / f(pw))
    gh = sr if sr > 0 else max(int(math.ceil(bin_h)), 0)
    gw = sr if sr > 0 else max(int(math.ceil(bin_w)), 0)
    return Geom(int(roi[0]), float(sh), float(sw), float(bin_h), float(bin_w), gh, gw, gh * gw, float(raw_h), float(raw_w))


def lists(g, ph, pw, h, w):
    """The per-bin-row and per-bin-column tap lists (add_tap, :308-322) without the kMaxE cap: [(index, weight)] each."""
    ys = [tap_list(g.start_h, g.bin_h, g.gh, p, h, fp32=True) for p in range(ph)]
    xs = [tap_list(g.start_w, g.bin_w, g.gw, p, w, fp32=True) for p in range(pw)]
    return ys, xs


def positions(g, ph, pw):
    """Every fp32 sample row and column of the RoI."""
    ys = {sample_pos(g.start_h, g.bin_h, g.gh, p, i, True) for p in range(ph) for i in range(g.gh)}
    xs = {sample_pos(g.start_w, g.bin_w, g.gw, p, i, True) for p in range(pw) for i in range(g.gw)}
    return ys, xs


def _dense(lsts):
    idx = [i for l in lsts for i, _ in l]
    if not idx:
        return None, 0
    lo = min(idx)
    m = np.zeros((len(lsts), max(idx) - lo + 1))
    for p, l in enumerate(lsts):
        for i, wt in l:
            m[p, i - lo] += wt
    return m, lo


def _np(t):
    return t.detach().double().cpu().numpy() if hasattr(t, "detach") else np.asarray(t, dtype=np.float64)


class Roi:
    """One RoI on one level: geometry, tap lists, dense weights over the footprint."""

    def __init__(self, roi, scale, ph, pw, sr, aligned, h, w):
        self.g = geom(roi, scale, ph, pw, sr, aligned)
        self.ph, self.pw, self.h, self.w = ph, pw, h, w
        self.ylists, self.xlists = lists(self.g, ph, pw, h, w)
        self.wy, self.y0 = _dense(self.ylists)
        self.wx, self.x0 = _dense(self.xlists)
        self.empty = self.wy is None or self.wx is None
        # taps on the fly in both layouts (pooled size > 16 or a list longer than kMaxE), or the channels-last backward's
        # per-sample scatter (footprint wider than kBwdMaxFw): every sample is its own fp32 term
        self.onfly = (ph > K_MAXP or pw > K_MAXP or any(len(l) > K_MAXE for l in self.ylists + self.xlists)
                      or (not self.empty and self.wx.shape[1] > K_BWD_MAXFW))
        self.inv = 1.0 / max(self.g.count, 1)

    def rows(self):
        return slice(self.y0, self.y0 + self.wy.shape[1]), slice(self.x0, self.x0 + self.wx.shape[1])

    def forward(self, img):
        """img: [C, H, W] (numpy or torch, any device) -> (out, A, m), each [C, PH, PW] float64."""
        c = img.shape[0]
        if self.empty:
            z = np.zeros((c, self.ph, self.pw))
            return z, z, z
        ys, xs = self.rows()
        crop = _np(img[:, ys, xs])
        out = np.einsum("py,cyx,qx->cpq", self.wy, crop, self.wx, optimize=True) * self.inv
        a = np.einsum("py,cyx,qx->cpq", np.abs(self.wy), np.abs(crop), np.abs(self.wx), optimize=True) * self.inv
        ny, nx = (self.wy != 0).sum(1), (self.wx != 0).sum(1)
        m = np.maximum(ny[:, None] * nx[None, :], ny[:, None] + nx[None, :]).astype(np.float64)
        if self.onfly:
            m[:] = 4 * self.g.count
        return out, a, np.broadcast_to(m, out.shape)

    def backward(self, go):
        """go: [C, PH, PW] -> (footprint slices, grad, A, m) of the footprint crop."""
        go = _np(go)
        if self.empty:
            return None
        gx = np.einsum("py,cpq,qx->cyx", self.wy, go, self.wx, optimize=True) * self.inv
        a = np.einsum("py,cpq,qx->cyx", np.abs(self.wy), np.abs(go), np.abs(self.wx), optimize=True) * self.inv
        m = ((self.wy != 0).astype(np.float64).T @ np.ones((self.ph, self.pw)) @ (self.wx != 0).astype(np.float64))
        if self.onfly:
            m = m * self.g.count
        return self.rows(), gx, a, np.broadcast_to(m, gx.shape)


def forward(feats, rois, scales, lv, ph, pw, sr, aligned):
    """The pooled output of every RoI: feats = the levels [N, C, H, W], lv[k] = level of RoI k (-1: none, zero output)."""
    k, c = len(rois), feats[0].shape[1]
    out, a, m = (np.zeros((k, c, ph, pw)) for _ in range(3))
    for i, r in enumerate(np.asarray(rois, dtype=np.float32)):
        if lv[i] < 0:
            continue
        f = feats[lv[i]]
        R = Roi(r, scales[lv[i]], ph, pw, sr, aligned, f.shape[2], f.shape[3])
        out[i], a[i], m[i] = R.forward(f[R.g.b])
    return out, a, m


def backward(go, shapes, rois, scales, lv, ph, pw, sr, aligned):
    """Gradients of every level (shapes: [N, C, H, W] each) for grad_out `go` [K, C, PH, PW]: (grad, A, m) per level."""
    go = _np(go)
    res = [tuple(np.zeros(s) for _ in range(3)) for s in shapes]
    for i, r in enumerate(np.asarray(rois, dtype=np.float32)):
        if lv[i] < 0:
            continue
        s = shapes[lv[i]]
        R = Roi(r, scales[lv[i]], ph, pw, sr, aligned, s[2], s[3])
        t = R.backward(go[i])
        if t is None:
            continue
        (ys, xs), gx, a, m = t
        yi, xi = np.arange(ys.start, ys.stop)[:, None], np.arange(xs.start, xs.stop)[None, :]
        for arr, v in zip(res[lv[i]], (gx, a, m)):
            np.add.at(arr[R.g.b], (slice(None), yi, xi), v)
    return res


def half_ulp(x, dtype):
    """Half a unit in the last place of `dtype` ('float16' / 'bfloat16') at |x| (normal and subnormal range)."""
    mant, emin = {"float16": (10, -14), "bfloat16": (7, -126)}[dtype]
    e = np.floor(np.log2(np.maximum(np.abs(x), 2.0 ** emin)))
    return 0.5 * 2.0 ** (e - mant)


def tolerance(ref, a, m, dtype=None):
    tol = (np.asarray(m) + 5) * EPS32 * a
    if dtype is not None:
        tol = tol + half_ulp(np.abs(ref) + tol, dtype)
    return tol


def check(got, ref, a, m, dtype=None, what=""):
    got = _np(got)
    tol = tolerance(ref, a, m, dtype)
    err = np.abs(got - ref)
    bad = err > tol
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), 0)), err.shape)
        raise AssertionError("%s: %d of %d elements outside (m + 5) 2^-24 A%s; worst at %s: got %r ref %r tol %r"
                             % (what, bad.sum(), bad.size, " + half ulp" if dtype else "", i, got[i], ref[i], tol[i]))


# =========================================================================================== path model
def cdiv(a, b):
    return -(-a // b)


def launch_fwd_nhwc(k, c, ph, pw, sms):
    """launch_fwd_nhwc (:1101-1105): (nchunks, chunk) of the channels-last forward's grid.z."""
    bins, slabs = ph * pw, cdiv(c, K_NHWC_CH)
    want = cdiv(8 * sms, k * slabs)
    nchunks = max(cdiv(bins, K_NHWC_CHUNK), min(want, cdiv(bins, 8)))
    chunk = cdiv(bins, nchunks)
    if nchunks > 1:
        chunk = min(K_NHWC_CHUNK - 1, cdiv(chunk, 7) * 7)
    return cdiv(bins, chunk), chunk


def bwd_nhwc_smem(rows, pw):  # :1369-1371
    return 4 * K_NHWC_CH * (rows * pw + K_BWD_WARPS * pw)


def launch_bwd_nhwc(k, c, ph, pw, sms):
    """launch_bwd_nhwc (:1378-1382): bin rows per CTA of the channels-last backward."""
    slabs, rows = cdiv(c, K_NHWC_CH), ph
    while (rows > 4 and (bwd_nhwc_smem(rows, pw) > 100 * 1024 or k * slabs * cdiv(ph, rows) < 4 * sms)
           and bwd_nhwc_smem(rows, pw) > 56 * 1024):
        rows = (rows + 1) // 2
    return rows


def nhwc_bwd_supported(ph, pw):
    """nhwc_supported's backward branch (:1514-1519): the tile at the deepest split launch_bwd_nhwc may take fits 180 KB."""
    rows = ph
    while rows > 4 and bwd_nhwc_smem(rows, pw) > 100 * 1024:
        rows = (rows + 1) // 2
    return bwd_nhwc_smem(rows, pw) <= 180 * 1024


def launch_fwd(k, c, sms):
    """launch_fwd (:718-721): channel groups of 4 per CTA of the NCHW kernel."""
    ngroup = cdiv(c, 4)
    gpc = ngroup
    while gpc > 8 and k * cdiv(ngroup, gpc) < 24 * sms:
        gpc = (gpc + 1) // 2
    return gpc


def slabs(c):
    """Channel slabs of the channels-last kernels (grid.y): (first channel, channels)."""
    return [(c0, min(K_NHWC_CH, c - c0)) for c0 in range(0, c, K_NHWC_CH)]


def _padded_x(n):  # :982 (table) and :1011 (per-bin loop): lists padded to 4, or to a multiple of 8 when longer
    return 0 if n == 0 else (4 if n <= 4 else (n + 7) & ~7)


def walk_refusals(R, chunk):
    """Why roi_align_nhwc_kernel does not take the column walk for this RoI (:970-986, :1023): a subset of
    {three_bins, colcap, profit, nymax, pw7}; empty = the walk runs."""
    xl, pw = R.xlists, R.pw
    why = set()
    total = padded = 0
    for b in range(pw):
        own = 0
        for c, _ in xl[b]:
            in1 = b >= 1 and any(q[0] == c for q in xl[b - 1])
            in2 = b >= 2 and any(q[0] == c for q in xl[b - 2])
            if in1 and in2:
                why.add("three_bins")
            own += not in1
        total += max(own, 1)
        padded += _padded_x(len(xl[b]))
    if total + 4 > K_COLCAP:
        why.add("colcap")
    if total * 5 > padded * 4:
        why.add("profit")
    if max(len(l) for l in R.ylists) > 6:
        why.add("nymax")
    if pw % 7 or chunk % 7:
        why.add("pw7")
    return why


def nhwc_fwd_labels(R, chunk, nchunks):
    """Paths of roi_align_nhwc_kernel for one RoI (:1017-1082)."""
    bins = R.ph * R.pw
    if R.ph > K_MAXP or R.pw > K_MAXP:
        return {"fwd_onfly_pooled"}
    if any(len(l) > K_MAXE for l in R.ylists + R.xlists):
        return {"fwd_onfly_overflow"}
    why = walk_refusals(R, chunk)
    out = set()
    if not why:
        for z in range(nchunks):
            b0 = z * chunk
            for u in range(0, min(chunk, bins - b0), 7):
                fb = b0 + u
                ph, pw0 = fb // R.pw, fb % R.pw
                ny = len(R.ylists[ph])
                if ny == 0:
                    out.add("walk_empty_row")
                    continue
                out.add("walk_ry%d" % ny)  # ny <= 6: one chunk of ny tap rows (:1038)
                if pw0 > 0:
                    out.add("walk_carry_in")
        return out
    if len(why) == 1:
        out.add("refuse_" + next(iter(why)))
    for ph in range(R.ph):
        ny = len(R.ylists[ph])
        if ny == 0:
            out.add("bin_empty_row")
            continue
        for pw in range(R.pw):
            nx = len(R.xlists[pw])
            if nx == 0:
                continue
            form = "bin42" if _padded_x(nx) <= 4 else "bin81"
            out.add(form)
            if ny % 2 and nx % (4 if form == "bin42" else 8):  # padding taps on both axes (:934, :1011)
                out.add(form + "_padded")
    return out


def nhwc_bwd_labels(R, rows):
    """Paths of roi_align_bwd_nhwc_kernel for one RoI, over its grid.z CTAs of `rows` bin rows (:1181-1365)."""
    if R.ph > K_MAXP or R.pw > K_MAXP:
        return {"bwd_per_sample_pooled"}
    out = set()
    xcols = [i for l in R.xlists for i, _ in l]
    for ph0 in range(0, R.ph, rows):
        yl = R.ylists[ph0:ph0 + rows]
        yrows = [i for l in yl for i, _ in l]
        if not xcols or not yrows:
            out.add("bwd_empty")  # :1228
            continue
        fw = max(xcols) - min(xcols) + 1
        if fw > K_BWD_MAXFW:
            out.add("bwd_per_sample_wide")  # :1229
            continue
        ymin, ymax = min(yrows), max(yrows)
        nb = cdiv(ymax - ymin + 1, K_BWD_BAND)
        out.add("bwd_bands%d" % min(nb, 3))
        for b in range(1, nb):  # a band edge inside the footprint rows of one bin row
            edge = ymin + b * K_BWD_BAND
            if any(min(i for i, _ in l) < edge <= max(i for i, _ in l) for l in yl if l):
                out.add("bwd_band_edge_in_bin_row")
        colcnt = max(sum(any(i == x for i, _ in l) for l in R.xlists) for x in set(xcols))
        rowcnt = max(sum(any(i == y for i, _ in l) for l in yl) for y in set(yrows))
        out.add("bwd_general" if max(colcnt, rowcnt) > 2 else "bwd_separable")  # s_wide (:1266, :1299)
    return out


def v3_labels(R):
    """Mode of roi_align_v3_kernel for one RoI (:353-464): the same in the forward and the backward."""
    if R.ph > K_MAXP or R.pw > K_MAXP or any(len(l) > K_MAXE for l in R.ylists + R.xlists):
        return {"v3_onfly"}
    xs = [i for l in R.xlists for i, _ in l]
    ys = [i for l in R.ylists for i, _ in l]
    if not xs or not ys:
        return {"v3_empty"}
    xmin, fw = min(xs), max(xs) - min(xs) + 1
    ymin, ymax = min(ys), max(ys)
    if (ymax - ymin + 1) * fw > K_ROWOFF:
        return {"v3_direct_rowoff"}
    nb, ph0 = 0, 0
    while ph0 < R.ph:  # greedy bands of bin rows (:411-433)
        yb, ye, ph1 = 1 << 30, -1, ph0
        while ph1 < R.ph:
            l = R.ylists[ph1]
            nyb, nye = (min(yb, min(i for i, _ in l)), max(ye, max(i for i, _ in l))) if l else (yb, ye)
            if nye >= nyb and (nye - nyb + 1) * fw > K_CAPPX:
                if ph1 == ph0:
                    return {"v3_direct_row"}
                break
            yb, ye, ph1 = nyb, nye, ph1 + 1
        nb, ph0 = nb + 1, ph1
    sy, sx = sum(len(l) for l in R.ylists), sum(len(l) for l in R.xlists)
    if 2 * sy * sx < (ymax - ymin + 1) * fw:
        return {"v3_direct_sparse"}
    return {"v3_staged_1band" if nb == 1 else "v3_staged_bands"}


def launch_labels(k, c, ph, pw, sms, nhwc=True):
    out = set()
    gpc = launch_fwd(k, c, sms)
    out.add("v3_groups_split" if gpc < cdiv(c, 4) else "v3_groups_whole")
    if c % 4:
        out.add("v3_ragged_group")
    if not nhwc:
        return out
    nchunks, chunk = launch_fwd_nhwc(k, c, ph, pw, sms)
    out.add("fwd_nchunks1" if nchunks == 1 else ("fwd_nchunks_ragged" if (ph * pw) % chunk else "fwd_nchunks_even"))
    sl = slabs(c)
    out.add("slab_full" if c == K_NHWC_CH else ("slab_partial" if c < K_NHWC_CH else "slab_ragged" if sl[-1][1] < K_NHWC_CH
                                                 else "slab_multi"))
    if len(sl) > 2:
        out.add("slab_many")
    if nhwc_bwd_supported(ph, pw):
        rows = launch_bwd_nhwc(k, c, ph, pw, sms)
        if rows < ph:
            out.add("bwd_rows_split_ragged" if ph % rows else "bwd_rows_split")
    return out


def boundary_labels(R, sr, aligned):
    out = {"sr%d" % sr}
    if not aligned and (R.g.raw_h < 1 or R.g.raw_w < 1):
        out.add("unaligned_clamp")
    ys, xs = positions(R.g, R.ph, R.pw)
    for name, v in (("-1", lambda n: -1.0), ("0", lambda n: 0.0), ("H-1", lambda n: n - 1.0), ("H", lambda n: float(n))):
        if v(R.h) in ys and v(R.w) in xs:
            out.add("pos_" + name)
    return out
