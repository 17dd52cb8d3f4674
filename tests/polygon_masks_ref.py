"""Reference of the polygon mask rasterizer (detectron2_b200/csrc/polygon_raster.cuh): a literal restatement of pycocotools'
rleFrPoly + merge + decode, and of detectron2's rasterize_polygons_within_box (structures/masks.py:39-85).

pycocotools is not needed: the restatement below walks every lattice point of every edge, like the C code, and is pinned
by checks that do not come from itself (tests/test_polygon_masks_host.py): the reference's own known answers, an
independent even-odd test at pixel centres, and the even toggle count of every column.

Rasterizing one polygon on an h x w grid (C double / int semantics, no fused multiply-add):
  1. X = (int)(5 x + 0.5), truncation toward zero (Python int() / numpy astype), then the ring is closed;
  2. each edge is walked by the DDA: dx = |Xe - Xs|, dy = |Ye - Ys|, flip = (dx >= dy and Xs > Xe) or (dx < dy and
     Ys > Ye) swaps the ends; x-major edges emit (t + Xs, (int)(Ys + s t + 0.5)) with s = (Ye - Ys) / dx, y-major edges
     ((int)(Xs + s t + 0.5), t + Ys) with s = (Xe - Xs) / dy, for t = flip ? D - d : d, d = 0..D, into one list;
  3. each consecutive pair with u[j] != u[j-1] and xd = ((u[j] < u[j-1] ? u[j] : u[j] - 1) + 0.5) / 5 - 0.5 an integer in
     [0, w - 1] toggles index xd h + ceil(clamp((min v + 0.5) / 5 - 0.5, 0, h));
  4. pixel (r, c) is the parity of the toggles at indices <= c h + r.
An instance is the union of its polygons.  Contracts of the library where the reference is undefined: a polygon with a
non-finite vertex or a lattice value 5 x + 0.5 outside (-2^30, 2^30) adds nothing, and so does a non-finite box.

numpy evaluates `ys + s * t + .5` elementwise in IEEE double, each operation rounded once, exactly like the C expression;
astype(np.int64) truncates toward zero, like the C cast.
"""
import math

import numpy as np

LATTICE_LIMIT = 2.0 ** 30


def snap(xy):
    """Lattice coordinates (int array of 2k) of the flat float64 polygon, or None when the library skips it."""
    v = 5.0 * np.asarray(xy, dtype=np.float64) + 0.5
    if not (np.abs(v) < LATTICE_LIMIT).all():
        return None
    return v.astype(np.int64)


def _edge_points(xs, ys, xe, ye):
    """The DDA's points of one edge, in emission order (vectorised: the same double expressions per point)."""
    dx, dy = abs(xe - xs), abs(ys - ye)
    flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
    if flip:
        xs, xe, ys, ye = xe, xs, ye, ys
    if dx >= dy:
        d = np.arange(dx + 1, dtype=np.int64)
        t = dx - d if flip else d
        if dx == 0:  # one point; C evaluates the 0/0 slope here, but the point forms no kept pair
            return t + xs, np.array([ys], np.int64)
        s = float(ye - ys) / dx
        return t + xs, (ys + s * t.astype(np.float64) + 0.5).astype(np.int64)
    d = np.arange(dy + 1, dtype=np.int64)
    t = dy - d if flip else d
    s = float(xe - xs) / dy
    return (xs + s * t.astype(np.float64) + 0.5).astype(np.int64), t + ys


def walk(X, Y):
    """u, v of the whole ring (steps 1-2), X / Y the k lattice vertices."""
    k = len(X)
    us, vs = [], []
    for j in range(k):
        u, v = _edge_points(int(X[j]), int(Y[j]), int(X[(j + 1) % k]), int(Y[(j + 1) % k]))
        us.append(u)
        vs.append(v)
    return np.concatenate(us), np.concatenate(vs)


def toggles(u, v, h, w):
    """Step 3: (column, row) of every kept pair, in list order."""
    j = np.nonzero(u[1:] != u[:-1])[0] + 1
    xd = np.where(u[j] < u[j - 1], u[j], u[j] - 1).astype(np.float64)
    xd = (xd + 0.5) / 5.0 - 0.5
    keep = (np.floor(xd) == xd) & (xd >= 0) & (xd <= w - 1)
    j, xd = j[keep], xd[keep]
    yd = np.minimum(v[j], v[j - 1]).astype(np.float64)
    yd = (yd + 0.5) / 5.0 - 0.5
    yd = np.ceil(np.clip(yd, 0, h))
    return xd.astype(np.int64), yd.astype(np.int64)


def decode(cols, rows, h, w):
    """Step 4: parity of the toggles at column-major indices <= c h + r."""
    tog = np.zeros(h * w + 1, np.int64)
    np.add.at(tog, cols * h + rows, 1)
    return (np.cumsum(tog[:h * w]) & 1).astype(bool).reshape(w, h).T


def fr_poly(xy, h, w):
    """One polygon (flat float64 x0, y0, x1, ...) on an h x w grid -> bool [h, w]."""
    L = snap(xy)
    if L is None:
        return np.zeros((h, w), bool)
    c, r = toggles(*walk(L[0::2], L[1::2]), h, w)
    return decode(c, r, h, w)


def fr_poly_literal(xy, h, w):
    """fr_poly one point at a time with Python ints and floats: the C loops line by line (slow; small polygons)."""
    k = len(xy) // 2
    x = [int(5.0 * float(xy[2 * j]) + .5) for j in range(k)] + [0]
    y = [int(5.0 * float(xy[2 * j + 1]) + .5) for j in range(k)] + [0]
    x[k], y[k] = x[0], y[0]
    u, v = [], []
    for j in range(k):
        xs, xe, ys, ye = x[j], x[j + 1], y[j], y[j + 1]
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe, ys, ye = xe, xs, ye, ys
        if dx >= dy:
            s = (ye - ys) / dx if dx else 0.0
            for d in range(dx + 1):
                t = dx - d if flip else d
                u.append(t + xs)
                v.append(int(ys + s * t + .5))
        else:
            s = (xe - xs) / dy
            for d in range(dy + 1):
                t = dy - d if flip else d
                v.append(t + ys)
                u.append(int(xs + s * t + .5))
    tog = [0] * (h * w + 1)
    for j in range(1, len(u)):
        if u[j] != u[j - 1]:
            xd = (float(u[j] if u[j] < u[j - 1] else u[j] - 1) + .5) / 5.0 - .5
            if math.floor(xd) != xd or xd < 0 or xd > w - 1:
                continue
            yd = (float(v[j] if v[j] < v[j - 1] else v[j - 1]) + .5) / 5.0 - .5
            yd = math.ceil(0.0 if yd < 0 else (float(h) if yd > h else yd))
            tog[int(xd) * h + int(yd)] ^= 1
    m = np.zeros(h * w, bool)
    acc = 0
    for i in range(h * w):
        acc ^= tog[i]
        m[i] = acc
    return m.reshape(w, h).T


def to_bitmask(polygons, h, w):
    """polygons_to_bitmask: the union of the instance's polygons; no polygon -> all zeros."""
    out = np.zeros((h, w), bool)
    for p in polygons:
        out |= fr_poly(np.asarray(p, np.float64), h, w)
    return out


def transform(polygons, box, s):
    """rasterize_polygons_within_box's steps 1-2 with numpy's dtypes: box float32, w / h float32, ratio = s / max(w, 0.1)
    (float32 division, or the Python float s / 0.1), polygons float64.  Returns the transformed polygons."""
    box = np.asarray(box, dtype=np.float32)
    w, h = box[2] - box[0], box[3] - box[1]
    out = []
    for p in polygons:
        p = np.array(p, dtype=np.float64)
        p[0::2] = p[0::2] - box[0]
        p[1::2] = p[1::2] - box[1]
        out.append(p)
    with np.errstate(all="ignore"):
        ratio_h = s / max(h, 0.1)
        ratio_w = s / max(w, 0.1)
        for p in out:
            p[0::2] *= ratio_w
            p[1::2] *= ratio_h
    return out


def crop_and_resize(instances, boxes, s, mask_index=None):
    """PolygonMasks.crop_and_resize: instances = list of polygon lists; boxes [K, 4]; mask_index [K] (None: k <-> k; outside
    [0, G): all zeros).  Returns bool [K, s, s]."""
    boxes = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    out = np.zeros((len(boxes), s, s), bool)
    for k, box in enumerate(boxes):
        g = k if mask_index is None else int(mask_index[k])
        if not 0 <= g < len(instances) or not np.isfinite(box).all():
            continue
        with np.errstate(all="ignore"):
            out[k] = to_bitmask(transform(instances[g], box, s), s, s)
    return out


# ------------------------------------------------------------------------------------------- the kernel's closed form
def _floor5(a):
    return a // 5  # Python floor division


def closed_form_edge(xs, ys, xe, ye, c_lo, c_hi):
    """polygon_raster.cuh poly_edge_toggles in Python: {column: lower v of the kept pair} for columns in [c_lo, c_hi]."""
    out = {}
    dx, dy = abs(xe - xs), abs(ys - ye)
    flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
    if flip:
        xs, xe, ys, ye = xe, xs, ye, ys
    if dx >= dy:
        if dx == 0:
            return out
        s = float(ye - ys) / dx
        for c in range(max(c_lo, -_floor5(-xs + 2)), min(c_hi, _floor5(xe - 3)) + 1):
            t = 5 * c + 2 - xs
            out[c] = min(int(ys + s * t + .5), int(ys + s * (t + 1) + .5))
        return out
    s = float(xe - xs) / dy

    def u(t):
        return int(xs + s * t + .5)

    ua, ub = u(0), u(dy)
    up = ub > ua
    lo, hi = min(ua, ub), max(ua, ub)
    for c in range(max(c_lo, -_floor5(-lo + 2)), min(c_hi, _floor5(hi - 3)) + 1):
        m = 5 * c + (3 if up else 2)

        def past(t):
            return u(t) >= m if up else u(t) <= m

        est = math.ceil((m - (0.5 if up else -0.5) - xs) / s)
        t = int(min(max(est, 1), dy))
        while t > 1 and past(t - 1):
            t -= 1
        while t < dy and not past(t):
            t += 1
        if min(u(t - 1), u(t)) == 5 * c + 2:
            out[c] = ys + t - 1
    return out


def walk_edge_toggles(xs, ys, xe, ye, w):
    """The literal walk's kept pairs inside one edge: {column: lower v}, and how many pairs each column got."""
    u, v = _edge_points(xs, ys, xe, ye)
    out, count = {}, {}
    for j in range(1, len(u)):
        if u[j] != u[j - 1]:
            m = int(u[j] if u[j] < u[j - 1] else u[j] - 1)
            if m % 5 == 2 and 0 <= (m - 2) // 5 <= w - 1:
                c = (m - 2) // 5
                out[c] = int(min(v[j], v[j - 1]))
                count[c] = count.get(c, 0) + 1
    return out, count
