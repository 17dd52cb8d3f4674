"""Keypoint head kernels (keypoints.cu) path by path against the float64 reference of tests/keypoints_ref.py.

Decoding: each case runs d2b_keypoints_from_heatmaps through keypoints_from_heatmaps_op and asserts, per ROI:
  1. F.interpolate(maps, bicubic) on CUDA lies within the reference's bound at every pixel (pins the tap model to PyTorch);
  2. the kernel's pixel is the first argmax, NaN first, of that CUDA fp32 map: no tolerance (the bit-exactness claim);
  3. against float64 alone: no pixel is decidedly above the kernel's pixel, no earlier pixel decidedly equal or above it;
     with a NaN in the float64 map, the first NaN;
  4. the logit is bitwise the CUDA map at the pixel, the position bit-exact, the score within its bound, NaN exactly where
     the reference has it; non-finite and over-2^32-pixel boxes give NaN rows and leave the other rows as they are;
  5. fp16 maps give the outputs of their fp32 up-cast;
  6. the declared labels are reached.
The loss: keypoint_loss_op / keypoint_loss_backward_op with a per-row grad_scale; targets, valid and num_valid exactly (the
fp32 restatement on CUDA, and the exact cell wherever it is decided); each row's loss within its bound and 0 on invalid
rows; every gradient element within its own bound, 0 on invalid rows, NaN exactly where the reference has it; fp16 / bf16
equal to the fp32 run of the same values with the gradient rounded once.

decode case     reaches
coco            1 x 100 detections, K 17, S 56, one full-image box: 261 tiles in one ROI, more items than CTAs
r1025 .. r2049  small boxes: prep chunks of 2 and 3 ROIs per thread; S 5 leaves finish lanes idle
tile_edges      ceil(h) ceil(w) = 1, 4095, 4096, 4097, 8192
copy_axes       56 x 56 (copy), 56 x 57 and 57 x 56 (one axis = S), w < 1, h < 1, both, x2 < x1
far             coordinates near 1e4, fractional offsets, up and down sampling on each axis
s1, s2, s17, s112, s241   the map sizes: S 112 needs the shared-memory opt-in, S 241 232 324 of its 232 448 bytes
const, signed_zero, nan_copy, nan_arith, inf_cells, corner_block, one_ulp, spread, f16, nan_rows: the value edges

loss case       reaches
train_*         16 x 128 proposals, K 17, S 56 in fp32, bf16, fp16
s1 .. s241      S^2 below, at and above the 256-thread CTA; S 241 takes 227 logits per thread
edges           keypoints on x2 / y2, outside, v 0 / 1 / 2, a zero-width box, a subnormal-width box (0 * inf: invalid),
                a NaN coordinate, and undecided cells
nonfinite       NaN, +inf, -inf logits in valid rows and NaN in invalid ones
big, uniform, gs_edges: +-1e4 logits, a constant row (loss log S^2), grad_scale 0, negative and subnormal
"""
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

import keypoints_ref as R
from detectron2_b200 import keypoint_head as kh

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16
NAN, INF = math.nan, math.inf

Dec = namedtuple("Dec", "name S K dtype labels")
DECODE = [
    Dec("coco", 56, 17, F32, {"multi_tile", "items_exceed_grid", "upsample_x", "upsample_y", "downsample_x",
                              "downsample_y"}),
    Dec("r1025", 17, 1, F32, {"prep_chunk_2", "upsample_x", "downsample_y"}),
    Dec("r1600", 17, 3, F32, {"prep_chunk_2"}),
    Dec("r2049", 5, 1, F32, {"prep_chunk_3", "finish_idle_lanes"}),
    Dec("tile_edges", 56, 3, F32, {"one_pixel", "tile_minus_1", "tile_exact", "tile_plus_1", "multi_tile"}),
    Dec("copy_axes", 56, 17, F32, {"copy", "one_axis_equals_S", "w_below_1", "h_below_1", "w_h_below_1",
                                   "x2_below_x1"}),
    Dec("far", 56, 3, F32, {"far_coordinates", "upsample_x", "downsample_y", "downsample_x", "upsample_y"}),
    Dec("s1", 1, 3, F32, {"finish_idle_lanes", "copy", "upsample_x"}),
    Dec("s2", 2, 17, F32, {"finish_idle_lanes", "copy", "one_pixel"}),
    Dec("s17", 17, 17, F32, {"copy", "upsample_x"}),
    Dec("s112", 112, 3, F32, {"smem_optin", "copy", "multi_tile"}),
    Dec("s241", 241, 1, F32, {"smem_optin", "smem_max", "copy", "multi_tile"}),
    Dec("const", 56, 3, F32, {"ties_first_pixel"}),
    Dec("signed_zero", 56, 2, F32, {"signed_zero_max", "copy"}),
    Dec("nan_copy", 56, 3, F32, {"nan_copy"}),
    Dec("nan_arith", 56, 3, F32, {"nan_arith"}),
    Dec("inf_cells", 17, 3, F32, {"pos_inf_cell", "all_neg_inf"}),
    Dec("corner_block", 17, 2, F32, {"upsample_x", "upsample_y"}),
    Dec("one_ulp", 56, 2, F32, {"one_ulp_maxima", "copy"}),
    Dec("spread", 56, 3, F32, {"score_underflow", "downsample_x"}),
    Dec("f16", 56, 17, F16, {"f16_maps"}),
    Dec("nan_rows", 20, 3, F32, {"nan_row_box", "nan_row_pixels"}),
]


def _boxes_from_sizes(sizes, g, origin=(0.0, 0.0), jitter=True):
    """[R, 4] boxes of the given (w, h) at random (fractional) positions."""
    wh = torch.tensor(sizes, dtype=torch.float64)
    xy = torch.rand(len(sizes), 2, generator=g, dtype=torch.float64) * 500 + torch.tensor(origin, dtype=torch.float64)
    if not jitter:
        xy = xy.floor()
    return torch.cat([xy, xy + wh], 1).float()


def decode_inputs(c):
    """(maps [R, K, S, S] on the GPU in the case dtype, rois [R, 4] fp32 on the GPU)."""
    g = torch.Generator().manual_seed(DECODE.index(c) + 11)
    S, K = c.S, c.K

    def sides(n, lo, hi):
        return torch.randint(lo, hi, (n, 2), generator=g).double() - torch.rand(n, 2, generator=g, dtype=torch.float64)

    if c.name == "coco":
        side = torch.exp(torch.empty(100, 2, dtype=torch.float64).uniform_(math.log(16.0), math.log(600.0), generator=g))
        ctr = torch.rand(100, 2, generator=g, dtype=torch.float64) * torch.tensor([1333.0, 800.0], dtype=torch.float64)
        rois = torch.cat([ctr - side / 2, ctr + side / 2], 1).float()
        rois[0] = torch.tensor([0.0, 0.0, 1333.0, 800.0])
    elif c.name in ("r1025", "r1600", "r2049"):
        n = int(c.name[1:])
        rois = _boxes_from_sizes(sides(n, 2, 7).tolist(), g)  # few distinct output sizes: the checks run per size
        rois[:8, 2] = rois[:8, 0] + 40.5                      # and a few wider than the map
    elif c.name == "tile_edges":
        rois = _boxes_from_sizes([(1, 1), (63, 65), (64, 64), (17, 241), (128, 64), (0.5, 0.25)], g, jitter=False)
    elif c.name == "copy_axes":
        rois = torch.tensor([[3.25, 4.5, 59.25, 60.5], [10.0, 10.0, 66.0, 66.0], [0.5, 7.0, 56.5, 63.5],
                             [0.0, 0.0, 56.75, 55.5], [7.0, 3.0, 7.5, 40.0], [7.0, 3.0, 90.0, 3.25],
                             [5.2, 5.1, 5.4, 5.9], [30.0, 40.0, 20.0, 35.0], [100.0, 50.0, 100.0, 50.0]])
    elif c.name == "far":
        rois = torch.tensor([[9999.3, 9998.6, 10030.1, 10100.9], [-10020.7, 9900.25, -9900.5, 9930.125],
                             [12345.6, -7777.7, 12399.9, -7700.1], [9990.0, 9990.0, 10000.5, 10000.5]])
    elif c.name in ("s1", "s2", "s17", "s112", "s241"):
        big = {1: 40, 2: 9, 17: 60, 112: 150, 241: 300}[S]
        sizes = [(S, S), (1, 1), (big, max(S // 2, 1)), (big, big // 2 + 1), (max(S // 3, 1), big)]
        rois = _boxes_from_sizes(sizes, g)
        rois[0] = torch.tensor([2.0, 3.0, 2.0 + S, 3.0 + S])
    elif c.name in ("const", "corner_block", "inf_cells"):
        rois = torch.tensor([[0.0, 0.0, 4.0 * S, 4.0 * S], [1.5, 2.5, 40.0, 20.5], [0.0, 0.0, 2.0 * S, 2.0 * S]])
    elif c.name in ("signed_zero", "one_ulp"):
        rois = torch.tensor([[2.0, 3.0, 2.0 + S, 3.0 + S], [0.25, 0.5, 90.75, 71.0]])
    elif c.name in ("nan_copy", "nan_arith", "spread"):
        rois = torch.tensor([[2.0, 3.0, 2.0 + S, 3.0 + S], [10.3, 20.7, 55.9, 99.2],
                             [4.0, 4.0, 8.0, 8.0] if c.name == "spread" else [4.0, 4.0, 24.0, 24.0]])
    elif c.name == "f16":
        rois = _boxes_from_sizes(sides(20, 2, 200).tolist(), g)
    elif c.name == "nan_rows":
        rois = torch.tensor([[0.0, 0.0, 30.0, 20.0], [NAN, 0.0, 5.0, 5.0], [0.0, 0.0, INF, 9.0],
                             [0.0, 0.0, 70000.0, 70000.0], [1.0, 2.0, 9.0, 40.0], [0.0, -INF, 3.0, 3.0]])
    R_ = rois.shape[0]
    maps = torch.randn((R_, K, S, S), generator=g) * 3
    if c.name == "const":
        maps[:] = 0.375
    elif c.name == "signed_zero":
        maps[0, 1] = -maps[0, 1].abs() - 1.0
        maps[0, 1, 0, 1] = -0.0
        maps[0, 1, 0, 3] = 0.0
    elif c.name == "nan_copy":
        maps[0, 1, 7, 9] = NAN
        maps[0, 2, 30, 40] = NAN
        maps[0, 2, 31, 2] = NAN
    elif c.name == "nan_arith":
        maps[1, 0, 30, 17] = NAN
        maps[2, 2, 10, 10] = NAN
        maps[2, 2, 40, 1] = NAN
    elif c.name == "inf_cells":
        maps[0, 0, 0, 5] = INF   # on the border: the clamped taps add inf * c0 + inf * c1 of opposite signs
        maps[1, 1, 8, 8] = INF   # inside: +-inf pixels, a NaN where a zero weight meets it
        maps[2, 2] = -INF
    elif c.name == "corner_block":
        maps = -maps.abs() - 1.0
        maps[:, :, :4, :4] = 2.5  # a block in the corner: the clamped border taps and the ringing next to the block
    elif c.name == "one_ulp":
        for r in range(R_):
            for k in range(K):
                maps[r, k] = -maps[r, k].abs()
                maps[r, k, 20, 30] = 1.0
                maps[r, k, 40, 5] = float(torch.nextafter(torch.tensor(1.0), torch.tensor(2.0)))
    elif c.name == "spread":
        maps = torch.where(torch.rand(maps.shape, generator=g) < 0.5, -1e4, 1e4) + torch.randn(maps.shape, generator=g)
        maps[2] = -1e4 + torch.randn(maps[2].shape, generator=g)
        maps[2, :, 0, 0] = 1e4  # the 4 x 4 resize never reads cell (0, 0): exp(2e4) overflows, the score is 0
    return maps.to(DEV, c.dtype), rois.to(DEV)


def same(a, b):
    """Bitwise-equal values, NaN equal to NaN."""
    return a.shape == b.shape and a.dtype == b.dtype and bool(((a == b) | (torch.isnan(a) & torch.isnan(b))).all())


def within(got, want, bound, what):
    """Finite reference: |got - want| <= bound; non-finite: the same value (NaN for NaN)."""
    got = got.to(torch.float64)
    nan_w, nan_g = torch.isnan(want), torch.isnan(got)
    assert torch.equal(nan_w, nan_g), "%s: NaN at %d elements, the reference at %d" % (what, int(nan_g.sum()),
                                                                                       int(nan_w.sum()))
    inf = torch.isinf(want)
    assert torch.equal(got[inf], want[inf]), "%s: infinite values differ" % what
    bad = torch.isfinite(want) & ~((got - want).abs() <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError("%s: %d elements outside their bound; first at %s: got %r, want %r, bound %.3g"
                             % (what, int(bad.sum()), tuple(torch.unravel_index(torch.tensor(i), want.shape)),
                                float(got.reshape(-1)[i]), float(want.reshape(-1)[i]), float(bound.reshape(-1)[i])))


def first_argmax(flat):
    """[n, P] -> [n]: torch's CUDA argmax rule: any NaN wins (the first), else the first of the largest (-0 == +0)."""
    nan = torch.isnan(flat)
    fl = torch.where(nan, -INF, flat)
    top = fl.amax(1, keepdim=True)
    first_max = (fl == top).to(torch.uint8).argmax(1)
    return torch.where(nan.any(1), nan.to(torch.uint8).argmax(1), first_max)


def check_group(maps32, rois, out, idx, ho, wo, copy, labels, what):
    """Assertions 1-4 for the ROIs `idx` (all of output size ho x wo); adds the value labels they reach."""
    m = maps32[idx]                                           # [n, K, S, S]
    n, K, S = m.shape[0], m.shape[1], m.shape[2]
    o = out[idx]                                              # [n, K, 4]
    cu = F.interpolate(m, size=(ho, wo), mode="bicubic", align_corners=False)  # PyTorch's CUDA op
    v, e = R.bicubic(m, ho, wo)
    within(cu, v, e, what + " F.interpolate")                                  # 1
    flat = cu.reshape(n * K, -1)
    want = first_argmax(flat)
    rb = rois[idx].float()
    w = (rb[:, 2] - rb[:, 0]).clamp(min=1)
    h = (rb[:, 3] - rb[:, 1]).clamp(min=1)
    cw, ch = w / w.ceil(), h / h.ceil()
    px = (torch.arange(wo, device=DEV, dtype=F32)[None] + 0.5) * cw[:, None] + rb[:, 0:1]  # [n, wo]
    py = (torch.arange(ho, device=DEV, dtype=F32)[None] + 0.5) * ch[:, None] + rb[:, 1:2]
    x, y = o[..., 0].reshape(-1), o[..., 1].reshape(-1)
    pxk, pyk = px.repeat_interleave(K, 0), py.repeat_interleave(K, 0)
    wx, wy = want % wo, want // wo
    ok = (x == pxk.gather(1, wx[:, None])[:, 0]) & (y == pyk.gather(1, wy[:, None])[:, 0])
    if not bool(ok.all()):                                                     # 2
        j = int(torch.nonzero(~ok)[0])
        kx = int((pxk[j] == x[j]).to(torch.uint8).argmax())
        ky = int((pyk[j] == y[j]).to(torch.uint8).argmax())
        raise AssertionError("%s: map %d: kernel pixel (%d, %d) value %r, CUDA argmax (%d, %d) value %r"
                             % (what, j, ky, kx, float(cu.reshape(n * K, ho, wo)[j, ky, kx]), int(wy[j]), int(wx[j]),
                                float(flat[j, want[j]])))
    # 3: the kernel's pixel recovered from its position alone, against float64
    mx, my = pxk == x[:, None], pyk == y[:, None]
    assert bool((mx.sum(1) == 1).all() and (my.sum(1) == 1).all()), what + ": position not on the pixel grid"
    p = my.to(torch.uint8).argmax(1) * wo + mx.to(torch.uint8).argmax(1)
    vf, ef = v.reshape(n * K, -1), e.reshape(n * K, -1)
    nan64 = torch.isnan(vf)
    has_nan = nan64.any(1)
    assert torch.equal(p[has_nan], nan64.to(torch.uint8).argmax(1)[has_nan]), what + ": not the first float64 NaN"
    lo = torch.where(nan64, -INF, vf - ef)
    hi_p = (vf + ef).gather(1, p[:, None])
    earlier = torch.arange(vf.shape[1], device=DEV)[None] < p[:, None]
    bad = ((lo > hi_p) | (earlier & (lo >= hi_p))) & ~has_nan[:, None]
    assert not bool(bad.any()), "%s: %d pixels decidedly above (or earlier and not below) the kernel's" % (
        what, int(bad.sum()))
    # 4: the logit, the score
    assert same(o[..., 2].reshape(-1), flat.gather(1, p[:, None])[:, 0]), what + ": logit"
    s_ref, s_e = R.score(m.reshape(n * K, S, S), o[..., 2].reshape(-1))
    within(o[..., 3].reshape(-1), s_ref, s_e, what + " score")
    # value labels
    fl = torch.where(torch.isnan(flat), -INF, flat)
    top = fl.amax(1, keepdim=True)
    ties = (fl == top).sum(1)
    src = m.reshape(n * K, -1)
    if bool(((ties > 1) & ~has_nan).any()):
        labels.add("ties_first_pixel")
    if bool(((top[:, 0] == 0) & ((fl == top) & (torch.signbit(fl))).any(1) & ((fl == top) & ~torch.signbit(fl)).any(1)).any()):
        labels.add("signed_zero_max")
    if bool(has_nan.any()):
        labels.add("nan_copy" if copy else "nan_arith")
    if bool((src == INF).any()):
        labels.add("pos_inf_cell")
    if bool((src == -INF).all(1).any()):
        labels.add("all_neg_inf")
    second = torch.where(fl == top, -INF, fl).amax(1)
    if bool((torch.isfinite(top[:, 0]) & (torch.nextafter(second, top[:, 0]) == top[:, 0])).any()):
        labels.add("one_ulp_maxima")
    if bool((o[..., 3] == 0).any()):
        labels.add("score_underflow")


def check_decode(c, maps, rois):
    out = kh.keypoints_from_heatmaps_op(maps, rois)
    if c.dtype != F32:
        assert same(out, kh.keypoints_from_heatmaps_op(maps.float(), rois)), c.name + ": fp16 != its fp32 up-cast"  # 5
    labels = set()
    maps32 = maps.float()
    groups = {}
    rc = rois.cpu()
    bad_rows = []
    for i in range(rois.shape[0]):
        g = R.roi_geometry(rc[i])
        if not g["ok"]:
            bad_rows.append(i)
            continue
        groups.setdefault((g["ho"], g["wo"]), []).append(i)
    for i in bad_rows:
        assert bool(torch.isnan(out[i]).all()), (c.name, i)
    if bad_rows:
        good = [i for i in range(rois.shape[0]) if i not in bad_rows]
        assert same(out[good], kh.keypoints_from_heatmaps_op(maps[good], rois[good])), c.name + ": NaN rows leak"
    for (ho, wo), idx in groups.items():
        idx_t = torch.tensor(idx, device=DEV)
        check_group(maps32, rois, out, idx_t, ho, wo, ho == c.S and wo == c.S, labels,
                    "%s [%d x %d, ROI %d]" % (c.name, ho, wo, idx[0]))
    return labels


@pytest.mark.parametrize("c", DECODE, ids=lambda c: c.name)
def test_decode_case(c):
    maps, rois = decode_inputs(c)
    got = check_decode(c, maps, rois)
    got |= R.decode_shape_labels(rois, c.S, c.K, c.dtype, torch.cuda.get_device_properties(0).multi_processor_count)
    got |= R.roi_labels(rois)
    assert c.labels <= got, (c.name, sorted(c.labels - got))


# ---- loss -------------------------------------------------------------------------------------------------------------
Loss = namedtuple("Loss", "name N K S dtype labels")
LOSS = [
    Loss("train_f32", 2048, 17, 56, F32, {"row_gt_cta", "many_rows", "kp_on_x2", "kp_outside", "v0"}),
    Loss("train_bf16", 2048, 17, 56, BF16, {"bf16_logits", "many_rows"}),
    Loss("train_f16", 2048, 17, 56, F16, {"f16_logits", "many_rows"}),
    Loss("s1", 6, 3, 1, F32, {"row_lt_cta"}),
    Loss("s5", 6, 17, 5, F32, {"row_lt_cta"}),
    Loss("s16", 6, 17, 16, BF16, {"row_eq_cta", "bf16_logits"}),
    Loss("s17", 6, 17, 17, F16, {"row_gt_cta", "f16_logits"}),
    Loss("s241", 3, 2, 241, F32, {"row_gt_cta", "row_many_per_thread"}),
    Loss("edges", 8, 17, 56, F32, {"kp_on_x2", "kp_outside", "v0", "zero_width", "nan_cell", "undecided_cell"}),
    Loss("nonfinite", 4, 17, 56, F32, {"nan_logit", "pos_inf_logit", "neg_inf_logit", "nan_invalid_row"}),
    Loss("nonfinite_bf16", 4, 17, 16, BF16, {"nan_logit", "pos_inf_logit", "neg_inf_logit", "nan_invalid_row"}),
    Loss("big", 4, 17, 56, F32, {"big_logits"}),
    Loss("uniform", 4, 17, 56, F32, {"uniform_row"}),
    Loss("gs_edges", 4, 17, 56, F32, {"grad_scale_edge"}),
    Loss("no_valid", 3, 17, 56, F32, {"no_valid"}),
]


def loss_inputs(c):
    """(logits [N, K, S, S] in the case dtype, keypoints [N, K, 3], boxes [N, 4], grad_scale [N, K]) on the GPU."""
    g = torch.Generator().manual_seed(LOSS.index(c) + 101)
    N, K, S = c.N, c.K, c.S
    side = 4 + torch.rand(N, 2, generator=g) * 200
    x1y1 = torch.rand(N, 2, generator=g) * 600
    b = torch.cat([x1y1, x1y1 + side], 1)
    b[0] = b[0].round()
    kp = torch.empty(N, K, 3)
    kp[..., :2] = b[:, None, :2] + (torch.rand(N, K, 2, generator=g) * 1.3 - 0.15) * side[:, None]
    kp[..., 2] = torch.randint(0, 3, (N, K), generator=g).float()
    kp[:, 0, 0], kp[:, min(1, K - 1), 1] = b[:, 2], b[:, 3]
    kp[:, :2, 2] = 2.0
    logits = torch.randn((N, K, S, S), generator=g) * 2
    gs = 0.25 + torch.rand(N, K, generator=g)
    if c.name == "edges":
        b[1, 2] = b[1, 0]                                   # zero width
        kp[1, 3, 0] = b[1, 0] + 1.0
        b[2] = torch.tensor([0.0, 5.0, 1e-40, 60.0])        # subnormal width
        kp[2, :, 0] = 0.0                                   # at x1: (0 - 0) * inf = NaN: not valid
        kp[2, :, 1] = 20.0
        kp[2, :, 2] = 1.0
        kp[3, 4, 0] = NAN                                   # a NaN coordinate
        kp[3, 4, 2] = 2.0
        b[4] = torch.tensor([0.0, 0.0, 3.0, 7.0])           # 56 / 3 is not exact: cells near the integer boundaries
        kp[4, :, 0] = torch.arange(K).float() * 3.0 / 56.0 * 3.0
        kp[4, :, 1] = 1.5
        kp[4, :, 2] = 2.0
        b[5] = torch.tensor([10.0, 20.0, 30.0, 40.0])
        kp[5, :, 0] = 10.0 + torch.arange(K).float() * 20.0 / 17.0 + 0.01
        kp[5, :, 1] = 50.0                                  # below the box: invalid
    elif c.name.startswith("nonfinite"):
        kp[:, :, 2] = 2.0
        kp[:, 5:, 2] = 0.0                                  # rows 5.. invalid
        kp[:, :5, :2] = b[:, None, :2] + 0.3 * side[:, None]
        logits[0, 1, 3, 3] = NAN
        logits[1, 2, 4, 4] = INF
        logits[1, 3, 4, 4] = -INF
        logits[2, 0] = -INF
        logits[2, 0, 1, 1] = 0.5                            # all but one -inf
        logits[3, 4, 0, 0] = -INF
        logits[3, 6, 2, 2] = NAN                            # invalid rows: no effect
        logits[3, 7, 3, 3] = INF
    elif c.name == "big":
        logits = torch.where(torch.rand(logits.shape, generator=g) < 0.5, -1e4, 1e4) + logits
    elif c.name == "uniform":
        logits[:] = 0.625
    elif c.name == "gs_edges":
        gs = torch.where(torch.rand(N, K, generator=g) < 0.3, 0.0, gs)
        gs[:, 1::3] *= -1.0
        gs[:, 2::5] = 1e-40
    elif c.name == "no_valid":
        kp[..., 2] = 0.0
    return logits.to(DEV, c.dtype), kp.to(DEV), b.to(DEV), gs.to(DEV)


def run_loss(logits, kp, boxes, gs):
    loss, target, valid, nv = kh.keypoint_loss_op(logits, kp, boxes)
    grad = kh.keypoint_loss_backward_op(logits, target, valid, gs)
    return loss, target, valid, nv, grad


def check_targets(kp, boxes, S, target, valid, nv, labels):
    t_host, v_host = kh._keypoints_to_heatmap_host(kp, boxes, S)  # the fp32 restatement on CUDA
    assert torch.equal(target, t_host) and torch.equal(valid.long(), v_host), "targets differ from the CUDA restatement"
    assert int(nv) == int(v_host.sum())
    cx, dx = R.exact_cells(kp[..., 0], boxes[:, None, 0], boxes[:, None, 2], S)
    cy, dy = R.exact_cells(kp[..., 1], boxes[:, None, 1], boxes[:, None, 3], S)
    vis = kp[..., 2].cpu() > 0
    inside = (cx >= 0) & (cx < S) & (cy >= 0) & (cy < S)
    dec = (dx & dy) | ~vis
    want_v = inside & vis
    assert torch.equal(valid.cpu().bool()[dec], want_v[dec]), "valid differs from the exact cell"
    want_t = torch.where(want_v, cy * S + cx, 0)
    assert torch.equal(target.cpu()[dec], want_t[dec]), "target differs from the exact cell"
    if bool((~dec).any()):
        labels.add("undecided_cell")
    b = boxes.cpu()
    kc = kp.cpu()
    if bool((kc[..., 0] == b[:, None, 2]).any()) or bool((kc[..., 1] == b[:, None, 3]).any()):
        labels.add("kp_on_x2")
    if bool((vis & ~inside & dx & dy).any()):
        labels.add("kp_outside")
    if bool((kc[..., 2] == 0).any()):
        labels.add("v0")
    w = b[:, 2] - b[:, 0]
    if bool((w == 0).any()):
        labels.add("zero_width")
    nan_cell = torch.isnan(kc[..., 0]) | ((kc[..., 0] == b[:, None, 0]) & (w[:, None] != 0) & (w[:, None].abs() < 2.0 ** -126))
    if bool((nan_cell & vis).any()):
        assert not bool(valid.cpu().bool()[nan_cell].any()), "a NaN cell is valid"
        labels.add("nan_cell")
    if int(nv) == 0:
        labels.add("no_valid")


def check_loss(c, logits, kp, boxes, gs):
    labels = set()
    loss, target, valid, nv, grad = run_loss(logits, kp, boxes, gs)
    if c.dtype != F32:
        out32 = run_loss(logits.float(), kp, boxes, gs)
        for a, b in zip((loss, target, valid, nv), out32[:4]):
            assert same(a, b), c.name
        assert grad.dtype == c.dtype and same(grad, out32[4].to(c.dtype)), c.name + ": gradient not the fp32 one rounded"
        grad = out32[4]
    check_targets(kp, boxes, c.S, target, valid, nv, labels)
    ref = R.LossRef(logits, target, valid)
    within(loss.reshape(-1), ref.loss, ref.e_loss, c.name + " loss")
    assert bool((loss.reshape(-1)[~ref.valid] == 0).all()), c.name + ": loss of an invalid row"
    g_ref, g_e = ref.grad(gs)
    within(grad.reshape(g_ref.shape), g_ref, g_e, c.name + " grad")
    assert bool((grad.reshape(g_ref.shape)[~ref.valid] == 0).all()), c.name + ": gradient of an invalid row"
    lf = logits.float().reshape(ref.x.shape)
    vr = ref.valid[:, None]
    for name, hit in (("nan_logit", torch.isnan(lf) & vr), ("pos_inf_logit", (lf == INF) & vr),
                      ("neg_inf_logit", (lf == -INF) & vr), ("nan_invalid_row", torch.isnan(lf) & ~vr)):
        if bool(hit.any()):
            labels.add(name)
    if bool((lf.abs() >= 1e4).any()):
        labels.add("big_logits")
    if bool(((lf == lf[:, :1]).all(1) & ref.valid).any()):
        labels.add("uniform_row")
        S2 = c.S * c.S
        u = (lf == lf[:, :1]).all(1) & ref.valid
        assert bool((loss.reshape(-1)[u].double() - math.log(S2)).abs().le(ref.e_loss[u] + 1e-12).all())
    gv = gs.reshape(-1)[ref.valid]
    if bool((gv == 0).any()) and bool((gv < 0).any()) and bool(((gv != 0) & (gv.abs() < 2.0 ** -126)).any()):
        labels.add("grad_scale_edge")
    return labels


@pytest.mark.parametrize("c", LOSS, ids=lambda c: c.name)
def test_loss_case(c):
    logits, kp, boxes, gs = loss_inputs(c)
    got = check_loss(c, logits, kp, boxes, gs)
    got |= R.loss_shape_labels(c.N, c.K, c.S, c.dtype)
    assert c.labels <= got, (c.name, sorted(c.labels - got))


@pytest.mark.parametrize("normalizer", [None, 7.5])
def test_loss_wrapper_total_and_gradient(normalizer):
    """keypoint_rcnn_loss_fixed: the total within its bound, the gradient with grad_scale fp32(1 / normalizer)."""
    c = LOSS[[x.name for x in LOSS].index("edges")]
    logits, kp, boxes, _ = loss_inputs(c)
    lg = logits.clone().requires_grad_(True)
    split = [3, 0, c.N - 3]
    loss, nv = kh.keypoint_rcnn_loss_fixed(lg, list(kp.split(split)), list(boxes.split(split)), normalizer)
    loss.backward()
    _, target, valid, _ = kh.keypoint_loss_op(logits, kp, boxes)
    ref = R.LossRef(logits, target, valid)
    div = float(int(nv)) if normalizer is None else normalizer
    assert int(nv) == int(valid.sum()) > 0
    terms, errs = ref.loss[ref.valid], ref.e_loss[ref.valid]
    want = float(terms.sum()) / div
    bound = R.total_bound(terms, errs) / div * (1 + 2 * R.U) + R.U * abs(want)
    assert abs(float(loss.detach()) - want) <= bound, (float(loss), want, bound)
    gs = (torch.ones(()) / torch.tensor(div, dtype=F32)).to(DEV)
    g_ref, g_e = ref.grad(gs.expand(c.N, c.K))
    within(lg.grad.reshape(g_ref.shape), g_ref, g_e, "wrapper grad")


def test_no_valid_keypoint_with_nonfinite_logits_is_zero():
    """Without a valid keypoint the loss and gradient are 0 even with NaN / inf logits (the reference's pred.sum() * 0 is
    NaN there; the sync-free loss keeps 0 rather than reduce every logit to carry it)."""
    c = LOSS[[x.name for x in LOSS].index("no_valid")]
    logits, kp, boxes, _ = loss_inputs(c)
    logits[0, 0, 0, 0], logits[1, 2, 3, 4], logits[2, 5, 6, 7] = NAN, INF, -INF
    lg = logits.clone().requires_grad_(True)
    for normalizer in (None, 7.5):
        loss, nv = kh.keypoint_rcnn_loss_fixed(lg, [kp], [boxes], normalizer)
        assert int(nv) == 0 and float(loss.detach()) == 0.0
        loss.backward()
        assert not bool(lg.grad.any()) and not bool(torch.isnan(lg.grad).any())
        lg.grad = None


def test_nan_cell_follows_the_cuda_reference():
    """The reference's floor().long() turns a NaN cell into INT64_MIN on CUDA: the keypoint is not valid."""
    kp = torch.tensor([[[NAN, 20.0, 2.0], [0.0, 20.0, 1.0], [5.0, 20.0, 2.0]]], device=DEV)
    for boxes in (torch.tensor([[0.0, 5.0, 40.0, 60.0]], device=DEV), torch.tensor([[0.0, 5.0, 1e-40, 60.0]], device=DEV)):
        t_ref, v_ref = kh._keypoints_to_heatmap_host(kp, boxes, 56)
        t, v = kh.keypoints_to_heatmap(kp, boxes, 56)
        assert torch.equal(t, t_ref) and torch.equal(v, v_ref)
        assert int(v[0, 0]) == 0 and int(t[0, 0]) == 0
        nan = torch.tensor([math.nan], device=DEV)
        assert int(nan.floor().long()) == -2 ** 63
