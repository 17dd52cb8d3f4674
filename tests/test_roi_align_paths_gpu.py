"""Axis-aligned RoIAlign (roi_align.cu) path by path against the float64 reference of tests/roi_align_ref.py.

Every case runs forward and backward through layers.ROIAlign (ROIPooler for the pyramid case) three ways: NCHW input with
ops.POOLER_LAYOUT = "nchw" (roi_align_v3_kernel), NCHW input with "nhwc" (layout change + roi_align_nhwc_kernel /
roi_align_bwd_nhwc_kernel) and channels_last input in place (the same channels-last kernels); C % 4 != 0 runs the NCHW
kernel only.  The geometry is dyadic (power-of-two scales, box corners on multiples of 1/8 level pixels, bins a dyadic
multiple of their sampling grid), so every sample position is exact in fp32 and the only error left is the rounding of the
fp32 sums: |got - ref| <= (m + 5) 2^-24 A elementwise, A = the reference on |x| (forward) or |grad_out| (backward), m = the
terms summed (plus half an ulp of fp16 / bf16 outputs).  tests/test_roi_align_paths_host.py checks on the CPU that each case
reaches the paths listed here, at 132 and at 114 SMs.

case              reaches
walk_ry_7x7       column walk with 1..6 tap rows, a bin row outside the map; 7 chunks of 7 bins; C = 128 (one full slab);
                  v3 staged in one and in several bands, channel groups split; backward separable, one band
walk_14x14_k100   walk at PW = 14 with the carry-in unit; 10 output chunks, 9 of 21 bins and a last one of 7
walk_14x14_c132   walk at PW = 14; ragged last chunk; C = 132 (ragged second slab); backward 4 rows per CTA, last CTA 2
refusals_7x7      walk refused for three bins on one column, s_nymax > 6, the profitability test; per-bin <4,2> with padding
                  taps on both axes; backward general form (bins narrower than a pixel); C = 4
per_bin_8x8       walk refused for PW % 7; per-bin <4,2> and <8,1> with odd ny and nx not a multiple of 4 / 8; backward
                  4 rows per CTA; v3 channel groups whole
colcap_14x14      walk refused for kColCap alone (17 owned columns per bin); per-bin <8,1>; backward per sample
                  (footprint wider than kBwdMaxFw); v3 mode 1 (footprint above kRowoffCap)
overflow_7x7      taps on the fly after a 33-entry column list; backward per sample (wide); v3 mode 2
pooled_17x5       taps on the fly for a pooled size above 16, forward and backward (per sample); v3 mode 2
bands_7x7         backward in 1, 2 and 3 bands of 64 rows, band edges inside a bin row; v3 mode 1 (footprint)
sparse_sr1        v3 mode 1 through sparse sampling (sampling_ratio 1); a RoI outside the map: v3 without a valid
                  sample, the channels-last backward's early return, an all-empty per-bin RoI
c6_nchw           C = 6: a ragged channel group of the NCHW kernel (only layout that takes it)
c388_7x7          C = 388: four slabs, the last one of 4 channels; channel groups split
c256_k24          C = 256 at small K: channel groups split, two full slabs
box_head_k1100    1 100 RoIs at 7x7: one output chunk per RoI
rows_10x10_k20    10x10 at K = 20: 3 bin rows per backward CTA, the last CTA 1
f16_7x7           fp16 features: fp16 outputs of the channels-last forward and fp16 grad_out in its backward
bf16_14x14        the same in bf16, at 14x14
unaligned_8x8     aligned=False, boxes below one pixel (the max(rw, 1) clamp)
lattice_7x7       sample rows and columns exactly on -1, 0, H-1 and H
sr2, sr3, sr4     sampling_ratio 2, 3 and 4
pyramid_7x7       four FPN levels through ROIPooler, RoIs on every level

Properties: P1 the forward of a RoI is bitwise the same pooled alone and among 4 000 others, in every layout; P2 the "nhwc"
and channels_last forwards are bitwise equal (every case); P3 the backward matches the reference at K on both sides of the
channels-last backward's rows-per-CTA thresholds (8x8, 10x10); P4 adjointness sum(y g) = sum(x dx) in float64 (every case);
P5 a 2.2 GB-per-image channels-last map, RoIs on image 1's bottom rows (byte offsets above 2^31), forward and backward.
"""
import functools
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

import roi_align_ref as ra

pytestmark = pytest.mark.gpu
DEV = "cuda"

# rois: (level, image, start_w, start_h, bin_w, bin_h) in level pixels -- start = the kernel's start_w / start_h after the
# aligned offset; the box side is the bin times the pooled size
Case = namedtuple("Case", "name c n levels ph pw sr aligned rois k dtype labels")
S4 = 0.25


def _c(name, c, hw, ph, pw, rois, sr=0, aligned=True, n=1, k=None, dtype=torch.float32, labels=(), scale=S4, levels=None):
    lv = levels or [(hw[0], hw[1], scale)]
    return Case(name, c, n, lv, ph, pw, sr, aligned, [(0,) * (6 - len(r)) + tuple(r) for r in rois], k, dtype,
                frozenset(labels))


CASES = [
    _c("walk_ry_7x7", 128, (64, 48), 7, 7, [(0, 2, 1.5, 2, 1), (1, 3, 2, 2, 1), (0, 4, 3, 2, 2), (1, 2, 1, 2, 3),
                                            (0, 5, 2, 2, 4), (1, 2, 3, 2, 5), (0, 3, -9, 2, 2)], n=2,
       labels={"walk_ry1", "walk_ry2", "walk_ry3", "walk_ry4", "walk_ry5", "walk_ry6", "walk_empty_row",
               "fwd_nchunks_even", "slab_full", "v3_staged_1band", "v3_staged_bands", "v3_groups_split", "bwd_separable",
               "bwd_bands1", "sr0"}),
    _c("walk_14x14_k100", 64, (48, 48), 14, 14, [(0, 1, 2, 2, 1), (0, 3, 1, 2, 2)], k=100,
       labels={"walk_ry2", "walk_ry3", "walk_carry_in", "fwd_nchunks_ragged", "slab_partial", "bwd_rows_split_ragged"}),
    _c("walk_14x14_c132", 132, (48, 48), 14, 14, [(0, 1, 2, 2, 1), (1, 3, 1, 2, 2)], n=2, k=100,
       labels={"walk_ry2", "walk_carry_in", "fwd_nchunks_ragged", "slab_ragged", "bwd_rows_split_ragged"}),
    _c("refusals_7x7", 4, (40, 40), 7, 7, [(2, 1.5, 0.5, 1), (2, 1, 2, 6), (1.5, 1.5, 4, 1), (2, 2, 2, 1)],
       labels={"refuse_three_bins", "refuse_nymax", "refuse_profit", "bin42", "bin42_padded", "bwd_general"}),
    _c("per_bin_8x8", 12, (40, 40), 8, 8, [(2, 3, 2, 2), (2, 3, 4, 2)],
       labels={"refuse_pw7", "bin42_padded", "bin81", "bin81_padded", "bwd_rows_split", "v3_groups_whole"}),
    _c("colcap_14x14", 8, (24, 272), 14, 14, [(7.5, 1.5, 17, 1), (2, 2, 2, 1)],
       labels={"refuse_colcap", "bin81_padded", "bwd_per_sample_wide", "v3_direct_rowoff"}),
    _c("overflow_7x7", 8, (24, 272), 7, 7, [(4, 2, 32, 1), (2, 2, 2, 2)],
       labels={"fwd_onfly_overflow", "bwd_per_sample_wide", "v3_onfly"}),
    _c("pooled_17x5", 8, (48, 40), 17, 5, [(2, 2, 2, 1), (1.5, 3, 4, 2)],
       labels={"fwd_onfly_pooled", "bwd_per_sample_pooled", "v3_onfly"}),
    _c("bands_7x7", 4, (200, 40), 7, 7, [(2, 3, 2, 18), (3, 2, 2, 27), (2, 2, 2, 2)],
       labels={"bwd_bands1", "bwd_bands2", "bwd_bands3", "bwd_band_edge_in_bin_row", "v3_direct_rowoff"}),
    _c("sparse_sr1", 8, (48, 48), 7, 7, [(2, 2, 5, 5), (2, 2, 1, 1), (-30, -30, 2, 2)], sr=1,
       labels={"v3_direct_sparse", "v3_staged_1band", "v3_empty", "bwd_empty", "bin_empty_row", "sr1"}),
    _c("c6_nchw", 6, (48, 48), 7, 7, [(2, 2, 5, 5), (2, 2, 2, 2), (4, 2, 32, 1)], labels={"v3_ragged_group"}),
    _c("c388_7x7", 388, (32, 40), 7, 7, [(2, 2, 2, 2), (3, 1.5, 3, 1)], labels={"slab_ragged", "slab_many"}),
    _c("c256_k24", 256, (32, 40), 7, 7, [(2, 2, 2, 2), (3, 1.5, 3, 1), (1, 2, 1, 3)], k=24,
       labels={"slab_multi", "v3_groups_split"}),
    _c("box_head_k1100", 4, (48, 64), 7, 7, [(2, 2, 2, 2), (3, 1.5, 1, 1), (5, 3, 3, 2)], n=2, k=1100,
       labels={"fwd_nchunks1"}),
    _c("rows_10x10_k20", 8, (48, 48), 10, 10, [(2, 2, 2, 2), (3, 1.5, 1, 3)], k=20, labels={"bwd_rows_split_ragged"}),
    _c("f16_7x7", 128, (40, 48), 7, 7, [(1.5, 2, 2, 2), (3, 1.5, 1, 3), (4, 4, 4, 1)], dtype=torch.float16,
       labels={"fwd_out_f16", "bwd_go_f16"}),
    _c("bf16_14x14", 64, (40, 40), 14, 14, [(1.5, 1.5, 1, 2), (3, 2, 2, 1)], dtype=torch.bfloat16,
       labels={"fwd_out_bf16", "bwd_go_bf16", "walk_carry_in"}),
    _c("unaligned_8x8", 8, (32, 32), 8, 8, [(2, 3, 1 / 16, 1 / 16), (2.5, 3, 1 / 16, 2), (2, 2, 2, 2)], aligned=False,
       labels={"unaligned_clamp", "bwd_general"}),
    _c("lattice_7x7", 8, (12, 12), 7, 7, [(-1.5, -1.5, 1, 1), (5.5, 5.5, 1, 1), (-1.5, 5.5, 1, 1), (-2, -2, 2, 2)],
       scale=0.5, labels={"pos_-1", "pos_0", "pos_H-1", "pos_H"}),
    _c("sr2", 8, (48, 48), 7, 7, [(2, 2, 8, 1), (2, 2, 2, 2)], sr=2, labels={"sr2"}),
    _c("sr3", 8, (48, 48), 7, 7, [(2, 2, 3, 3), (1.5, 1.5, 3, 6)], sr=3, labels={"sr3"}),
    _c("sr4", 8, (48, 48), 7, 7, [(2, 2, 2, 2), (1.5, 1.5, 4, 1)], sr=4, labels={"sr4"}),
    _c("pyramid_7x7", 8, None, 7, 7, [(l, b, 2 + b, 3, 2, 4) for b in range(2) for l in range(4)], n=2,
       levels=[(64, 96, 1 / 4), (32, 48, 1 / 8), (16, 24, 1 / 16), (8, 12, 1 / 32)], labels={"pyramid"}),
]
BY_NAME = {c.name: c for c in CASES}
ids = [c.name for c in CASES]


def image_rois(case):
    """The case's RoIs as a [K, 5] fp32 array of image-coordinate boxes, tiled to K with integer level-pixel shifts."""
    off = 0.5 if case.aligned else 0.0
    base = case.rois
    k = case.k or len(base)
    out = []
    for j in range(k):
        lvl, b, sx, sy, bw, bh = base[j % len(base)]
        sx, sy = sx + (j // len(base)) % 3, sy + (j // len(base)) % 2
        s = case.levels[lvl][2]
        out.append([b, (sx + off) / s, (sy + off) / s, (sx + bw * case.pw + off) / s, (sy + bh * case.ph + off) / s])
    out = np.array(out, dtype=np.float64)
    assert (out.astype(np.float32) == out).all()
    return out.astype(np.float32)


def levels_of(case, rois):
    """assign_boxes_to_levels (detectron2 poolers.py) in fp32; a single-level case has every RoI on level 0."""
    if len(case.levels) == 1:
        return np.zeros(len(rois), dtype=np.int64)
    r = torch.from_numpy(rois)
    size = torch.sqrt((r[:, 3] - r[:, 1]) * (r[:, 4] - r[:, 2]))
    return (torch.floor(4 + torch.log2(size / 224 + 1e-8)).clamp(2, 5) - 2).long().numpy()


def path_labels(case, sms):
    """Every path label the case reaches on a device with `sms` SMs (tests/roi_align_ref.py's model)."""
    rois = image_rois(case)
    lv = levels_of(case, rois)
    k, nhwc = len(rois), case.c % 4 == 0
    nchunks, chunk = ra.launch_fwd_nhwc(k, case.c, case.ph, case.pw, sms)
    rows = ra.launch_bwd_nhwc(k, case.c, case.ph, case.pw, sms)
    out = ra.launch_labels(k, case.c, case.ph, case.pw, sms, nhwc)
    seen = set()
    for r, l in zip(rois, lv):
        key = (tuple(r[1:]), int(l))
        if key in seen:
            continue
        seen.add(key)
        h, w, s = case.levels[l]
        R = ra.Roi(r, s, case.ph, case.pw, case.sr, case.aligned, h, w)
        out |= ra.v3_labels(R) | ra.boundary_labels(R, case.sr, case.aligned)
        if nhwc:
            out |= ra.nhwc_fwd_labels(R, chunk, nchunks) | ra.nhwc_bwd_labels(R, rows)
    if case.dtype != torch.float32 and nhwc:
        t = {torch.float16: "f16", torch.bfloat16: "bf16"}[case.dtype]
        out |= {"fwd_out_" + t, "bwd_go_" + t}
    if len(case.levels) > 1 and len(set(lv.tolist())) == len(case.levels):
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
    fwd = ra.forward(feats, rois, scales, lv, case.ph, case.pw, case.sr, case.aligned)
    bwd = ra.backward(go, [tuple(f.shape) for f in feats], rois, scales, lv, case.ph, case.pw, case.sr, case.aligned)
    return feats, go, rois, lv, fwd, bwd


def _half_name(dt):
    return {torch.float16: "float16", torch.bfloat16: "bfloat16"}.get(dt)


def _run(case, xs, rois):
    import detectron2_b200.layers as L
    from detectron2_b200.poolers import ROIPooler

    if len(case.levels) == 1:
        return L.ROIAlign((case.ph, case.pw), case.levels[0][2], case.sr, case.aligned)(xs[0], torch.from_numpy(rois).to(DEV))
    boxes = [torch.from_numpy(rois[rois[:, 0] == b, 1:]).to(DEV) for b in range(case.n)]
    assert (np.diff(rois[:, 0]) >= 0).all()  # ROIPooler orders its output by image
    pooler = ROIPooler((case.ph, case.pw), [s for _, _, s in case.levels], case.sr, "ROIAlignV2" if case.aligned else "ROIAlign")
    return pooler(xs, boxes)


@pytest.mark.parametrize("name", ids)
def test_roi_align_path_case(name, monkeypatch):
    from detectron2_b200 import ops

    case = BY_NAME[name]
    feats, go, rois, lv, (yref, ya, ym), bwd = _inputs(name)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert case.labels <= path_labels(case, sms)
    r32 = torch.from_numpy(rois)
    assert torch.equal(r32.to(case.dtype).float(), r32)  # ROIAlign samples with the boxes in the feature dtype
    hd = _half_name(case.dtype)
    outs = {}
    for layout in ("nchw", "nhwc", "cl") if case.c % 4 == 0 else ("nchw",):
        monkeypatch.setattr(ops, "POOLER_LAYOUT", "nchw" if layout == "nchw" else "nhwc")
        xs = [f.to(DEV) for f in feats]
        if layout == "cl":
            xs = [x.contiguous(memory_format=torch.channels_last) for x in xs]
        assert ops._pick_layout(xs, 1, (case.ph, case.pw)) == {"nchw": "nchw", "nhwc": "xpose", "cl": "cl"}[layout]
        xs = [x.requires_grad_(True) for x in xs]
        y = _run(case, xs, rois)
        assert y.dtype == case.dtype
        ra.check(y, yref, ya, ym, hd, "%s %s forward" % (name, layout))
        y.backward(go.to(DEV))
        adj_lhs = (y.detach().double().cpu() * go.double()).sum().item()
        adj_rhs, adj_tol = 0.0, float((ra.tolerance(yref, ya, ym, hd) * np.abs(go.double().numpy())).sum())
        for l, (x, (gref, ga, gm)) in enumerate(zip(xs, bwd)):
            ra.check(x.grad, gref, ga, gm, hd, "%s %s backward level %d" % (name, layout, l))
            adj_rhs += (x.detach().double().cpu() * x.grad.double().cpu()).sum().item()
            adj_tol += float((ra.tolerance(gref, ga, gm, hd) * np.abs(feats[l].double().numpy())).sum())
        # P4: sum(y g) = sum(x dx) -- the GPU forward and backward of one call are each other's transpose
        assert abs(adj_lhs - adj_rhs) <= adj_tol, (layout, adj_lhs, adj_rhs, adj_tol)
        outs[layout] = y.detach()
    if "cl" in outs:  # P2: both channels-last routes run the same kernel on the same NHWC bytes
        assert torch.equal(outs["nhwc"], outs["cl"])


def _realistic_rois(g, k, h, w, scale):
    s = torch.exp(torch.rand(k, generator=g) * (math.log(400) - math.log(8)) + math.log(8))
    ar = torch.exp((torch.rand(k, generator=g) - 0.5) * 1.4)
    ctr = torch.rand(k, 2, generator=g) * torch.tensor([w / scale, h / scale])
    wh = torch.stack([s * ar.sqrt(), s / ar.sqrt()], 1)
    return torch.cat([torch.zeros(k, 1), ctr - wh / 2, ctr + wh / 2], 1)


@pytest.mark.parametrize("ph", [7, 14])
def test_forward_of_a_roi_is_bitwise_independent_of_k(ph, monkeypatch):
    """P1: no atomics in the forward; output chunks (grid.z), channel slabs and channel-group splits only move work between
    CTAs, so 64 RoIs pooled one at a time and among 4 000 others give the same bits, in every layout."""
    from detectron2_b200 import layers as L, ops

    g = torch.Generator().manual_seed(ph)
    x = torch.randn(1, 256, 100, 152, generator=g).to(DEV)
    probe = _realistic_rois(g, 64, 100, 152, S4)
    others = _realistic_rois(g, 4000, 100, 152, S4)
    pos = torch.randperm(4064, generator=g)[:64]
    keep = torch.ones(4064, dtype=torch.bool)
    keep[pos] = False
    big = torch.empty(4064, 5)
    big[pos], big[keep] = probe, others
    op = L.ROIAlign((ph, ph), S4, 0, True)
    for layout in ("nchw", "nhwc", "cl"):
        monkeypatch.setattr(ops, "POOLER_LAYOUT", "nchw" if layout == "nchw" else "nhwc")
        xi = x.contiguous(memory_format=torch.channels_last) if layout == "cl" else x
        yb = op(xi, big.to(DEV))[pos.to(DEV)]
        for i in range(64):
            y1 = op(xi, probe[i:i + 1].to(DEV))
            assert torch.equal(y1[0], yb[i]), (layout, i)


@pytest.mark.parametrize("p", [8, 10])
def test_backward_is_independent_of_k_across_rows_per_cta(p, monkeypatch):
    """P3: the channels-last backward's bin rows per CTA change with K (launch_bwd_nhwc); the gradient of a fixed set of RoIs,
    padded with RoIs whose grad_out is zero, matches the reference at K on both sides of every threshold."""
    from detectron2_b200 import layers as L, ops

    sms = torch.cuda.get_device_properties(0).multi_processor_count
    ks = sorted({kk for kk in range(8, 1200) if ra.launch_bwd_nhwc(kk, 8, p, p, sms) != ra.launch_bwd_nhwc(kk - 1, 8, p, p, sms)})
    assert ks  # 8x8: K = 4 * sms; 10x10: 2 * sms and 4 * sms
    ks = sorted({8} | {kk + d for kk in ks for d in (-1, 0)})
    assert len({ra.launch_bwd_nhwc(kk, 8, p, p, sms) for kk in ks}) >= 2
    g = torch.Generator().manual_seed(p)
    x = torch.randn(1, 8, 48, 48, generator=g)
    base = np.array([[0, (sx + 0.5) / S4, (sy + 0.5) / S4, (sx + bw * p + 0.5) / S4, (sy + bh * p + 0.5) / S4]
                     for sx, sy, bw, bh in [(2, 2, 2, 2), (1.5, 3, 1, 3), (3, 1.5, 4, 1), (2, 2, 0.5, 1)]], dtype=np.float32)
    go = torch.randn(4, 8, p, p, generator=g)
    (gref, ga, gm), = ra.backward(go, [(1, 8, 48, 48)], base, [S4], [0] * 4, p, p, 0, True)
    pad = _realistic_rois(g, max(ks), 48, 48, S4)
    monkeypatch.setattr(ops, "POOLER_LAYOUT", "nhwc")
    for kk in ks:
        rois = torch.cat([torch.from_numpy(base), pad[:kk - 4]])
        gfull = torch.cat([go, torch.zeros(kk - 4, 8, p, p)])
        xg = x.to(DEV).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        y = L.ROIAlign((p, p), S4, 0, True)(xg, rois.to(DEV))
        y.backward(gfull.to(DEV))
        ra.check(xg.grad, gref, ga, gm, None, "K=%d rows=%d" % (kk, ra.launch_bwd_nhwc(kk, 8, p, p, sms)))


def test_offsets_past_2_31_bytes():
    """P5: one channels-last N = 2 map of 2.2 GB per image (C = 256, 1536 x 1400; H*W*C/4 < 2^28 is the channels-last
    kernels' limit).  RoIs on image 1's bottom rows, whose byte offsets exceed 2^31, through the column walk, the per-bin
    loop and taps on the fly, forward and backward, compared with the reference on the footprint crops."""
    if torch.cuda.mem_get_info()[0] < 12 * 2 ** 30:
        pytest.skip("needs 12 GB of free device memory")
    from detectron2_b200 import layers as L

    n, c, h, w = 2, 256, 1536, 1400
    assert h * w * c // 4 < 2 ** 28 and h * w * c * 4 > 2 ** 31
    g = torch.Generator(device=DEV).manual_seed(5)
    x = torch.empty(n, h, w, c, device=DEV).normal_(generator=g).permute(0, 3, 1, 2)  # channels_last storage
    x.requires_grad_(True)
    # (pooled, start_w, start_h, bin_w, bin_h) in level pixels (scale 1/4), disjoint footprints on the last rows
    specs = [(7, 8, h - 16, 2, 2), (8, 40, h - 18, 2, 2), (7, 80, h - 8, 33, 1), (17, 400, h - 20, 1, 1)]
    for ph, sx, sy, bw, bh in specs:
        r = np.array([[1, (sx + 0.5) / S4, (sy + 0.5) / S4, (sx + bw * ph + 0.5) / S4, (sy + bh * ph + 0.5) / S4]],
                     dtype=np.float32)
        R = ra.Roi(r[0], S4, ph, ph, 0, True, h, w)
        x.grad = None
        y = L.ROIAlign((ph, ph), S4, 0, True)(x, torch.from_numpy(r).to(DEV))
        ref, a, m = R.forward(x.detach()[1])
        ra.check(y[0], ref, a, m, None, "P5 forward pooled %d" % ph)
        go = torch.randn(1, c, ph, ph, device=DEV, generator=g)
        y.backward(go)
        (ys, xs), gref, ga, gm = R.backward(go[0])
        grow = slice(ys.start - 1, min(ys.stop + 1, h)), slice(xs.start - 1, min(xs.stop + 1, w))  # one pixel of zeros around
        pad = lambda t: np.pad(t, ((0, 0), (1, grow[0].stop - ys.stop), (1, grow[1].stop - xs.stop)))  # noqa: E731
        ra.check(x.grad[1][:, grow[0], grow[1]], pad(gref), pad(ga), pad(gm), None, "P5 backward pooled %d" % ph)
        assert x.grad[0].abs().sum().item() == 0
    del x
    torch.cuda.empty_cache()
