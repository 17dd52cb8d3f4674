"""Rotated RoIAlign (roi_align.cu) path by path against the float64 reference of tests/roi_align_rotated_ref.py.

Every case runs forward and backward through layers.ROIAlignRotated (ROIPooler(..., "ROIAlignRotated") for the pyramid
cases) three ways: NCHW input with ops.POOLER_LAYOUT = "nchw" (roi_align_rot_fwd_kernel / roi_align_rot_bwd_kernel), NCHW
input with "nhwc" (layout change + roi_align_rot_nhwc_kernel) and channels_last input in place (the same channels-last
kernel).  C % 4 != 0 and pooled sizes above the channels-last kernel's tile run the NCHW kernels in every setting.  The
bound is elementwise |got - ref| <= (m + 5) 2^-24 A + P (plus half an ulp of fp16 / bf16 outputs): A = the reference on |x|
(forward) or |grad_out| (backward), m = the fp32 terms summed, P = the derived position-error term (the reference module's
docstring).  No element is exempt.  tests/test_roi_align_rotated_paths_host.py checks on the CPU that each case reaches the
paths listed here, at 132 and at 114 SMs, and that no sample of a case lies within its position error of the map edge,
except in the angle-0 lattice case, whose positions are exact.

case             reaches
lattice_a0       angle 0 on a dyadic lattice: samples exactly on -1, 0, H-1 and H; tap table in both kernels
angles_7x7       angles 90, -90, 180, -180, 45 and arbitrary; boxes partly and wholly outside the map; image 1 of 2;
                 C = 128 (one full slab), channel slabs of 16 in the NCHW kernels
nonsquare_7x5    7 x 5 bins, sampling_ratio 2
nonsquare_5x9    5 x 9 bins, sampling_ratio 3
pooled_13x23     299 bins, the largest pooled area the channels-last kernel takes; table and taps on the fly
pooled_20x15     300 bins: refused by the channels-last kernel, NCHW in every setting
taps_1024        8 x 8 bins with a 4 x 4 grid (exactly 1 024 taps: table) and a 4 x 5 grid (1 280: on the fly)
empty_sr0        zero width, zero height and negative sides at sampling_ratio 0: an empty grid, zero output, no gradient
mirrored_sr2     the same boxes at sampling_ratio 2: the grid is mirrored and still sampled
sub_pixel        RoIs smaller than one level pixel (no clamp of the sides to 1)
c6_nchw          C = 6: NCHW kernels only
c132             C = 132: a ragged second channels-last slab (4 channels), ragged NCHW channel slabs
c200_k4          C = 200 at K = 4: NCHW slabs of 13 channels, the last one of 5
c256_k4          C = 256: two full channels-last slabs
box_head_k600    600 RoIs: one NCHW channel slab per RoI
f16_layer        fp16 features through the layer: up-cast to fp32, as in the reference
bf16_layer       bf16 features: bf16 outputs of the channels-last kernel, bf16 grad_out read in place
pyramid          four FPN levels through ROIPooler: RoIs on every level, the exact level boundaries sqrt(wh) = 112 / 224 /
                 448, a negative-area RoI (no level: zero output, no gradient), a large RoI on the coarsest level (on the fly)
pyramid_f16      the same in fp16: fp16 outputs and fp16 grad_out in the channels-last kernel

Properties: P1 the forward of a RoI is bitwise the same pooled alone and among 4 000 others, in every layout (the NCHW channel
slabs change with K); P2 the "nhwc" and channels_last forwards are bitwise equal (every case); P3 adjointness sum(y g) =
sum(x dx) in float64, within the summed tolerances (every case and layout).
"""
import functools
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

import roi_align_rotated_ref as rr

pytestmark = pytest.mark.gpu
DEV = "cuda"

# rois: (image, ctr_x, ctr_y, w, h, angle) in level pixels -- ctr = the kernel's centre, roi * scale - 0.5 -- or, for the
# pyramid cases (img=True), the image-coordinate boxes themselves
Case = namedtuple("Case", "name c n levels ph pw sr rois k dtype img labels")
S4 = 0.25
PYR = [(64, 96, 1 / 4), (32, 48, 1 / 8), (16, 24, 1 / 16), (8, 12, 1 / 32)]


def _c(name, c, hw, ph, pw, rois, sr=0, n=1, k=None, dtype=torch.float32, labels=(), scale=S4, levels=None):
    lv = levels or [(hw[0], hw[1], scale)]
    return Case(name, c, n, lv, ph, pw, sr, [(0,) * (6 - len(r)) + tuple(r) for r in rois], k, dtype, levels is not None,
                frozenset(labels))


# zero width, zero height, negative width, negative height, both negative, and an ordinary box
_EDGE = [(8.3, 9.1, 0, 6.2, 25), (10.7, 7.9, 7.4, 0, -40), (20.2, 12.6, -5.3, 6.1, 70), (9.6, 20.4, 6.6, -4.2, 0),
         (15.1, 15.3, -3.1, -2.7, -135), (22.35, 19.65, 5.9, 7.7, 10)]
_PYR_ROIS = [(0, 40.3, 37.7, 112, 112, 31.0), (0, 160.6, 100.2, 224, 224, -47.0), (0, 190.1, 130.3, 448, 448, 12.5),
             (0, 250.7, 80.9, 56, 224, 97.0), (0, 60.9, 200.3, 40.4, 30.2, -160.0), (1, 300.2, 150.6, 1400.3, 1200.7, 21.0),
             (1, 120.4, 90.2, -30.0, 40.0, 15.0), (1, 330.8, 44.6, 150.3, 80.7, 63.0), (1, 20.2, 30.6, 300.9, 200.5, -35.0)]

CASES = [
    _c("lattice_a0", 8, (12, 12), 7, 7, [(2, 2, 7, 7, 0), (9, 9, 7, 7, 0), (9, 2, 7, 7, 0), (2.5, 9.25, 3.5, 1.75, 0),
                                         (5, 5, 14, 14, 0)], sr=1, scale=0.5,
       labels={"angle0", "pos_-1", "pos_0", "pos_H-1", "pos_H", "sr1", "nchw_table", "nhwc_table", "cpc_whole",
               "slab_partial", "inside"}),
    _c("angles_7x7", 128, (40, 48), 7, 7,
       [(0, 20.37, 15.29, 14.6, 9.3, 90), (1, 3.41, 37.13, 18.2, 12.7, -90), (0, 44.71, 2.33, 20.1, 11.4, 180),
        (1, 24.19, 20.57, 10.9, 16.3, -180), (0, 1.83, 1.61, 22.3, 14.9, 45), (1, 30.77, 25.43, 12.6, 7.9, 33.7),
        (0, -30.3, 60.7, 10.2, 8.6, -123.4), (1, 70.1, -20.9, 6.3, 4.1, 45)], n=2,
       labels={"angle90", "angle-90", "angle180", "angle-180", "angle45", "angle_other", "outside_partial", "outside_whole",
               "batch1", "sr0", "cpc_split", "slab_full"}),
    _c("nonsquare_7x5", 32, (40, 40), 7, 5, [(20.3, 18.7, 17.1, 12.2, 30), (9.6, 30.2, 9.9, 21.3, -60),
                                             (31.4, 6.8, 14.3, 8.6, 150.3)], sr=2, labels={"non_square", "sr2"}),
    _c("nonsquare_5x9", 12, (40, 40), 5, 9, [(20.3, 18.7, 17.1, 12.2, 120), (33.6, 35.2, 19.9, 11.3, -15.5)], sr=3,
       labels={"non_square", "sr3"}),
    _c("pooled_13x23", 16, (48, 56), 13, 23, [(28.3, 24.6, 18.4, 16.9, 22), (26.1, 23.7, 40.3, 30.2, -8.5)],
       labels={"nhwc_largest_pooled", "nchw_table", "nchw_onfly", "nhwc_table", "nhwc_onfly"}),
    _c("pooled_20x15", 16, (48, 56), 20, 15, [(28.3, 24.6, 18.4, 16.9, 22), (26.1, 23.7, 31.3, 45.2, -118.5)],
       labels={"nhwc_refused"}),
    _c("taps_1024", 32, (64, 64), 8, 8, [(30.3, 29.6, 30.1, 28.3, 17), (33.9, 31.2, 35.2, 27.7, -71)],
       labels={"nchw_table_1024", "nhwc_table_1024", "nchw_onfly", "nhwc_onfly"}),
    _c("empty_sr0", 8, (32, 32), 7, 7, _EDGE, labels={"empty_grid"}),
    _c("mirrored_sr2", 8, (32, 32), 7, 7, _EDGE, sr=2, labels={"mirrored"}),
    _c("sub_pixel", 8, (32, 32), 7, 7, [(10.3, 12.6, 0.5, 0.75, 30), (20.8, 6.1, 0.3, 0.9, -100.2)], labels={"sub_pixel"}),
    _c("c6_nchw", 6, (32, 40), 7, 7, [(15.3, 14.6, 12.2, 9.1, 40), (30.1, 20.4, 33.7, 20.2, -12)], labels={"c_not_4"}),
    _c("c132", 132, (32, 40), 7, 7, [(15.3, 14.6, 12.2, 9.1, 40), (30.1, 20.4, 33.7, 20.2, -12)],
       labels={"slab_ragged", "cpc_ragged"}),
    _c("c200_k4", 200, (32, 40), 7, 7, [(15.3, 14.6, 12.2, 9.1, 40), (30.1, 20.4, 33.7, 20.2, -12)], k=4,
       labels={"slab_ragged", "cpc_ragged"}),
    _c("c256_k4", 256, (24, 32), 7, 7, [(15.3, 14.6, 12.2, 9.1, 40), (20.1, 10.4, 23.7, 10.2, -12)], k=4,
       labels={"slab_multi"}),
    _c("box_head_k600", 32, (24, 32), 7, 7, [(15.3, 14.6, 12.2, 9.1, 40), (20.1, 10.4, 23.7, 10.2, -12), (9.2, 8.8, 6.1, 4.3, 5)],
       k=600, labels={"cpc_whole"}),
    _c("f16_layer", 64, (32, 40), 7, 7, [(15.3, 14.6, 12.2, 9.1, 40), (30.1, 20.4, 33.7, 20.2, -12)], dtype=torch.float16,
       labels={"f16_layer_upcast"}),
    _c("bf16_layer", 64, (32, 40), 14, 14, [(15.3, 14.6, 12.2, 9.1, 40), (30.1, 20.4, 33.7, 20.2, -12)],
       dtype=torch.bfloat16, labels={"out_bf16", "go_bf16"}),
    _c("pyramid", 8, None, 7, 7, _PYR_ROIS, n=2, levels=PYR, labels={"pyramid", "dead_level", "level_boundary", "nchw_onfly"}),
    _c("pyramid_f16", 16, None, 7, 7, _PYR_ROIS, n=2, levels=PYR, dtype=torch.float16, labels={"out_f16", "go_f16"}),
]
BY_NAME = {c.name: c for c in CASES}
ids = [c.name for c in CASES]


def image_rois(case):
    """The case's RoIs as a [K, 6] fp32 array of image-coordinate rotated boxes, tiled to K with integer level-pixel shifts."""
    base, k = case.rois, case.k or len(case.rois)
    s = case.levels[0][2]
    out = []
    for j in range(k):
        b, cx, cy, w, h, a = base[j % len(base)]
        cx, cy = cx + (j // len(base)) % 3, cy + (j // len(base)) % 2
        out.append([b, cx, cy, w, h, a] if case.img else [b, (cx + 0.5) / s, (cy + 0.5) / s, w / s, h / s, a])
    return np.array(out, dtype=np.float32)


def levels_of(case, rois):
    """assign_boxes_to_levels (detectron2 poolers.py) with RotatedBoxes.area = w * h, in fp32; -1 = no level (NaN)."""
    if len(case.levels) == 1:
        return np.zeros(len(rois), dtype=np.int64)
    r = torch.from_numpy(rois)
    lv = torch.floor(4 + torch.log2(torch.sqrt(r[:, 3] * r[:, 4]) / 224 + 1e-8)).clamp(2, 5) - 2
    return torch.where(torch.isnan(lv), -1, lv).long().numpy()


def roi_objects(case):
    """(roi, level, Roi) for every distinct RoI of the case; a RoI without a level has the empty grid of level 0."""
    rois = image_rois(case)
    out, seen = [], set()
    for r, l in zip(rois, levels_of(case, rois)):
        key = tuple(r.tolist())
        if key in seen:
            continue
        seen.add(key)
        h, w, s = case.levels[max(l, 0)]
        out.append((r, int(l), rr.Roi(r, s, case.ph, case.pw, case.sr, h, w, dead=l < 0)))
    return out


def path_labels(case, sms):
    """Every path label the case reaches on a device with `sms` SMs (tests/roi_align_rotated_ref.py's model)."""
    rois = image_rois(case)
    hw = [(h, w) for h, w, _ in case.levels]
    nhwc = rr.nhwc_supported(case.c, hw, case.ph, case.pw)
    out = rr.launch_labels(len(rois), case.c, case.ph, case.pw, hw, sms)
    lv = levels_of(case, rois)
    for r, l, R in roi_objects(case):
        out |= rr.roi_labels(R, nhwc) | rr.boundary_labels(R, r, case.sr)
        if l < 0:
            out.add("dead_level")
        if case.img and l >= 0 and float(np.sqrt(np.float32(r[3]) * np.float32(r[4]))) in (112.0, 224.0, 448.0):
            out.add("level_boundary")
    if case.dtype == torch.float16 and not case.img:
        out.add("f16_layer_upcast")  # layers/roi_align_rotated.py: the kernel sees fp32
    elif case.dtype != torch.float32 and nhwc:
        t = {torch.float16: "f16", torch.bfloat16: "bf16"}[case.dtype]
        out |= {"out_" + t, "go_" + t}
    if len(case.levels) > 1 and set(lv.tolist()) >= set(range(len(case.levels))):
        out.add("pyramid")
    return out


@functools.lru_cache(maxsize=None)
def _inputs(name):
    """Features, grad_out (CPU, in the case's dtype), RoIs, levels, and the float64 reference forward / backward."""
    case = BY_NAME[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    feats = [torch.randn(case.n, case.c, h, w, generator=g).to(case.dtype) for h, w, _ in case.levels]
    rois = image_rois(case)
    lv = levels_of(case, rois)
    go = torch.randn(len(rois), case.c, case.ph, case.pw, generator=g).to(case.dtype)
    scales = [s for _, _, s in case.levels]
    fwd = rr.forward(feats, rois, scales, lv, case.ph, case.pw, case.sr)
    bwd = rr.backward(go, [tuple(f.shape) for f in feats], rois, scales, lv, case.ph, case.pw, case.sr)
    return feats, go, rois, lv, fwd, bwd


def _half_name(dt):
    return {torch.float16: "float16", torch.bfloat16: "bfloat16"}.get(dt)


def _run(case, xs, rois):
    import detectron2_b200.layers as L
    from detectron2_b200.poolers import ROIPooler

    if len(case.levels) == 1:
        return L.ROIAlignRotated((case.ph, case.pw), case.levels[0][2], case.sr)(xs[0], torch.from_numpy(rois).to(DEV))
    assert (np.diff(rois[:, 0]) >= 0).all()  # ROIPooler orders its output by image
    boxes = [torch.from_numpy(rois[rois[:, 0] == b, 1:]).to(DEV) for b in range(case.n)]
    return ROIPooler((case.ph, case.pw), [s for _, _, s in case.levels], case.sr, "ROIAlignRotated")(xs, boxes)


@pytest.mark.parametrize("name", ids)
def test_roi_align_rotated_path_case(name, monkeypatch):
    from detectron2_b200 import ops
    from detectron2_b200.poolers import assign_boxes_to_levels

    case = BY_NAME[name]
    feats, go, rois, lv, (yref, ya, ym, yp), bwd = _inputs(name)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert case.labels <= path_labels(case, sms)
    if case.img:
        got = assign_boxes_to_levels([torch.from_numpy(rois[rois[:, 0] == b, 1:]).to(DEV) for b in range(case.n)], 2, 5, 224, 4)
        live = lv >= 0
        assert (got.cpu().numpy()[live] == lv[live]).all()
    hd = _half_name(case.dtype)
    hw = [(h, w) for h, w, _ in case.levels]
    outs = {}
    for layout in ("nchw", "nhwc", "cl") if case.c % 4 == 0 else ("nchw",):
        monkeypatch.setattr(ops, "POOLER_LAYOUT", "nchw" if layout == "nchw" else "nhwc")
        xs = [f.to(DEV) for f in feats]
        if layout == "cl":
            xs = [x.contiguous(memory_format=torch.channels_last) for x in xs]
        want = rr.pick_layout(ops.POOLER_LAYOUT, case.c, hw, case.ph, case.pw, layout == "cl")
        assert ops._pick_layout(xs, 1, (case.ph, case.pw), rotated=True) == want
        assert ops._pick_layout(xs, 1, (case.ph, case.pw), rotated=True, backward=True, channels_last=layout == "cl") == want
        xs = [x.requires_grad_(True) for x in xs]
        y = _run(case, xs, rois)
        assert y.dtype == case.dtype
        rr.check(y, yref, ya, ym, yp, hd, "%s %s forward" % (name, layout))
        y.backward(go.to(DEV))
        adj_lhs = (y.detach().double().cpu() * go.double()).sum().item()
        adj_rhs, adj_tol = 0.0, float((rr.tolerance(yref, ya, ym, yp, hd) * np.abs(go.double().numpy())).sum())
        for l, (x, (gref, ga, gm, gp)) in enumerate(zip(xs, bwd)):
            rr.check(x.grad, gref, ga, gm, gp, hd, "%s %s backward level %d" % (name, layout, l))
            adj_rhs += (x.detach().double().cpu() * x.grad.double().cpu()).sum().item()
            adj_tol += float((rr.tolerance(gref, ga, gm, gp, hd) * np.abs(feats[l].double().numpy())).sum())
        # P3: sum(y g) = sum(x dx) -- the GPU forward and backward of one call sample the same points
        assert abs(adj_lhs - adj_rhs) <= adj_tol, (layout, adj_lhs, adj_rhs, adj_tol)
        outs[layout] = y.detach()
    if "cl" in outs:  # P2: both channels-last routes run the same kernel on the same NHWC values
        assert torch.equal(outs["nhwc"], outs["cl"])


def _realistic_rotated(g, k, h, w, scale):
    s = torch.exp(torch.rand(k, generator=g) * (math.log(400) - math.log(8)) + math.log(8))
    ar = torch.exp((torch.rand(k, generator=g) - 0.5) * 1.4)
    ctr = torch.rand(k, 2, generator=g) * torch.tensor([w / scale, h / scale])
    ang = 180.0 - torch.rand(k, generator=g) * 360.0
    return torch.cat([torch.zeros(k, 1), ctr, (s * ar.sqrt())[:, None], (s / ar.sqrt())[:, None], ang[:, None]], 1)


@pytest.mark.parametrize("ph", [7, 14])
def test_rotated_forward_of_a_roi_is_bitwise_independent_of_k(ph, monkeypatch):
    """P1: no atomics in the forward; the NCHW kernel's channel slabs (pick_c_per_cta) change with K and the channels-last
    kernel's do not, so 64 RoIs pooled one at a time and among 4 000 others give the same bits, in every layout."""
    from detectron2_b200 import layers as L, ops

    g = torch.Generator().manual_seed(100 + ph)
    x = torch.randn(1, 256, 100, 152, generator=g).to(DEV)
    probe = _realistic_rotated(g, 64, 100, 152, S4)
    others = _realistic_rotated(g, 4000, 100, 152, S4)
    pos = torch.randperm(4064, generator=g)[:64]
    keep = torch.ones(4064, dtype=torch.bool)
    keep[pos] = False
    big = torch.empty(4064, 6)
    big[pos], big[keep] = probe, others
    op = L.ROIAlignRotated((ph, ph), S4, 0)
    for layout in ("nchw", "nhwc", "cl"):
        monkeypatch.setattr(ops, "POOLER_LAYOUT", "nchw" if layout == "nchw" else "nhwc")
        xi = x.contiguous(memory_format=torch.channels_last) if layout == "cl" else x
        yb = op(xi, big.to(DEV))[pos.to(DEV)]
        for i in range(64):
            y1 = op(xi, probe[i:i + 1].to(DEV))
            assert torch.equal(y1[0], yb[i]), (layout, i)
