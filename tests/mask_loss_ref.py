"""Float64 reference of the Mask R-CNN mask loss (detectron2_b200/csrc/postproc.cu: mask_loss_fwd_kernel, mask_loss_bwd_kernel).

Targets: BitMasks.crop_and_resize -- RoIAlign(S x S, spatial_scale 1, sampling_ratio 0, aligned=True) of the proposal's
ground-truth mask read as `mask != 0`, thresholded at `>= 0.5`.  The geometry and the tap weights are tests/roi_align_ref.py's
(`Roi`: sample positions in fp32 in the kernels' expression order, weights in float64).  The threshold is decided on the
un-normalised sum, `sum >= count / 2`, so it is exact in float64.  A mask index outside [0, G) gives an all-zero target.
Loss: per proposal, the sum over its S*S bins of softplus(x) - t x (np.logaddexp(0, x) - t x, stable at any |x|) on its
class channel; 0 for a class outside [0, C).  Gradient: (sigmoid(x) - t) * scale on the class channel, exactly 0 elsewhere.

Error bounds, from the kernels' fp32 arithmetic (postproc.cu is compiled with -fmad=false and without fast math):
  * Targets.  With dyadic geometry (box corners on multiples of 1/8 pixel, each bin a dyadic multiple of its sampling grid)
    every sample position, bilinear weight, weight product and partial sum is exact in fp32: the sum is a multiple of at
    least 2^-8 and below 2^12.  `v / count >= 0.5` then rounds the right way, since 0.5 is representable and a sum one
    step below count / 2 is at least 2^-8 / count below it.  So the targets equal the reference bit for bit.
    Elsewhere the kernel's v is a sum of 4 count non-negative terms, each a product of two rounded weights, then divided
    by count: |v - v_ref| <= (4 count + 8) 2^-24 for v <= 1.  Only a bin that close to 0.5 may take the other target.
  * Per-proposal loss.  Every term is non-negative.  Each is exact to a few ulps relative, plus an absolute error of about
    2^-24 from rounding 1 + exp(-|x|) before logf.  The kernel adds the terms in n = ceil(S^2 / 256) + 5 + 8 steps:
    its thread's share of the bins, 5 warp shuffles, then the 8 warp partials.  So
        |got - ref| <= (n + 8) 2^-24 (ref_k + S^2).
  * Gradient.  sigmoid(x) = 1 / (1 + expf(-x)): expf is within 2 ulp, the add and the division are rounded once.  That
    gives an absolute error of at most 2.25 2^-24 in sigmoid.  Add the subtraction of t (exact for t = 0, and at most
    2^-25 for t = 1) and the product with scale.  The total is below 4 2^-24 scale per element.  This is an absolute
    bound, because sigmoid(x) - 1 cancels for large x.  `scale` is the fp32 value the kernel is given.
"""
import math
from collections import namedtuple

import numpy as np

import roi_align_ref as ra

EPS32 = 2.0 ** -24

Targets = namedtuple("Targets", "t v near rois")


def roi(box, s, h, w):
    """roi_align_ref.Roi of a proposal box (x1, y1, x2, y2) on an h x w mask: scale 1, S x S, sampling_ratio 0, aligned."""
    return ra.Roi(np.array([0.0] + [float(c) for c in box], dtype=np.float32), 1.0, s, s, 0, True, h, w)


def pooled_sum(R, mask):
    """The un-normalised RoIAlign sum [S, S] of `mask != 0` (numpy [H, W], any dtype) and the kernel's divisor count."""
    count = max(R.g.count, 1)
    if R.empty:
        return np.zeros((R.ph, R.pw)), count
    ys, xs = R.rows()
    crop = (np.asarray(mask)[ys, xs] != 0).astype(np.float64)
    return R.wy @ crop @ R.wx.T, count


def targets(gt, boxes, mask_index, s):
    """gt: numpy [G, H, W] masks of one image; boxes [K, 4]; mask_index [K] or None (proposal k <-> mask k).
    Returns Targets: t [K, S, S] bool, v [K, S, S] float64 pooled values, near [K, S, S] bool (|v - 0.5| within the
    non-dyadic bound above), rois [K] (the Roi of each proposal)."""
    gt = np.asarray(gt)
    k = len(boxes)
    t, v, near = np.zeros((k, s, s), bool), np.zeros((k, s, s)), np.zeros((k, s, s), bool)
    rois = []
    for i, box in enumerate(np.asarray(boxes, dtype=np.float32)):
        R = roi(box, s, gt.shape[1], gt.shape[2])
        rois.append(R)
        mi = i if mask_index is None else int(mask_index[i])
        if not 0 <= mi < gt.shape[0]:
            continue
        sm, count = pooled_sum(R, gt[mi])
        t[i] = sm >= 0.5 * count
        v[i] = sm / count
        near[i] = np.abs(v[i] - 0.5) <= (4 * count + 8) * EPS32
    return Targets(t, v, near, rois)


def class_ok(classes, k, c):
    cl = np.zeros(k, np.int64) if classes is None else np.asarray(classes, np.int64)
    return cl, (cl >= 0) & (cl < c)


def class_channel(logits, classes):
    """logits [K, C, S, S] -> the proposal's class channel [K, S, S] float64 (zeros for a class outside [0, C))."""
    x = np.asarray(logits, dtype=np.float64)
    cl, ok = class_ok(classes, x.shape[0], x.shape[1])
    return np.where(ok[:, None, None], x[np.arange(len(x)), np.where(ok, cl, 0)], 0.0), ok


def loss_per_roi(logits, t, classes):
    """(loss sum per proposal [K], its bound [K]) of the fp32 logits [K, C, S, S] against the targets t [K, S, S]."""
    x, ok = class_channel(logits, classes)
    s2 = x.shape[1] * x.shape[2]
    ref = np.where(ok, (np.logaddexp(0.0, x) - t * x).sum(axis=(1, 2)), 0.0)
    n = math.ceil(s2 / 256) + 5 + 8
    return ref, np.where(ok, (n + 8) * EPS32 * (ref + s2), 0.0)


def grad(logits, t, classes, scale):
    """d loss / d logits [K, C, S, S] for d loss / d loss_per_roi[k] = scale[k] (the fp32 values), and the bound per element."""
    lg = np.asarray(logits, dtype=np.float64)
    x, ok = class_channel(lg, classes)
    scale = np.broadcast_to(np.asarray(scale, np.float64), (len(lg),))
    g = np.zeros_like(lg)
    cl, _ = class_ok(classes, lg.shape[0], lg.shape[1])
    sig = np.exp(-np.logaddexp(0.0, -x))
    rows = np.nonzero(ok)[0]
    g[rows, cl[rows]] = ((sig - t) * scale[:, None, None])[rows]
    return g, 4 * EPS32 * scale


def check(got, ref, tol, what):
    got = np.asarray(got, dtype=np.float64)
    err = np.abs(got - ref)
    bad = ~(err <= tol)
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), 0)), err.shape)
        raise AssertionError("%s: %d of %d outside the bound; worst at %s: got %r ref %r tol %r"
                             % (what, bad.sum(), bad.size, i, got[i], ref[i], np.broadcast_to(tol, err.shape)[i]))
