"""Semantic segmentation loss kernels (sem_seg_loss.cu) path by path against the float64 reference of
tests/sem_seg_loss_ref.py.

Each case runs d2b_sem_seg_loss_forward / _backward through sem_seg_loss_op / sem_seg_loss_backward_op (the raw sum, with a
grad_sum other than 1) and asserts:
  * status and count exactly; lse within its bound on every valid pixel and exactly 0 on skipped ones, NaN / inf where the
    reference's is;
  * the upsampled map of F.interpolate(logits.float()) on CUDA within the reference's interpolation bound of the gathered
    fp32 taps (this pins the tap model to PyTorch);
  * the selection: exactly k pixels, equal to the documented rule (the k largest, ties in ascending flat index, NaN first)
    applied to the kernel's own fp32 per-pixel values (lse - v_target) * w, every pixel decided above the float64 k-th
    value selected and every pixel decided below it not; undecided pixels at most the case's stated share;
  * loss_sum within its bound of the float64 sum (mean: the valid pixels; top-k: the kernel's selected set);
  * every gradient element within its own bound (no normalisation by the largest one), exactly 0 on the logits no used
    pixel reaches, and NaN exactly where the reference's is;
  * fp16 / bf16 logits: every output equal to the fp32 run of the same values, the gradient rounded once;
  * the path labels the case declares (tests/test_sem_seg_loss_paths_host.py checks the shape labels on the CPU).

case               reaches
fpn_full_*         Panoptic FPN 2 x 54 x 200 x 336 at stride 4, mean, fp32 and bf16: three finish passes
cityscapes_*       Panoptic-DeepLab 4 x 19 x 256 x 512 at stride 4, top-k 0.2 with weights over 8 192 CTAs; with 85 % of
                   the pixels ignored the threshold is 0 among the ignored ties
coco_topk          2 x 133 x 160 x 160: 10 channel chunks, the last of 7 channels
deeplab_os8_f16    DeepLab output stride 8, fp16
s16_*              stride 16, mean and top-k
s1 .. s32          the stride sweep: ragged tiles and channel chunks (C = CC + 1), maps of 1 and 2 rows, one channel per
                   CTA, one CTA per SM, and the tightest region (stride 31, Hp = 9: one spare row), whose last row alone
                   feeds a logit in the second image
nonfinite_*        NaN in channel 1, NaN in channel 0, NaN after a -inf channel, +inf and -inf logits (fp32, fp16)
c1, c2, bad_label, all_ignored, k0, k1, radix3, big_logits, weights_edge, const_ties: the other edges
"""
import math
from collections import namedtuple

import pytest
import torch
import torch.nn.functional as F

import sem_seg_loss_ref as R
from detectron2_b200 import semantic_seg as S

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
F32, F16, BF16 = torch.float32, torch.float16, torch.bfloat16

Case = namedtuple("Case", "name N C Hp Wp stride dtype top_k weights ignore gs und labels")


def _c(name, N, C, Hp, Wp, stride, dtype=F32, top_k=None, weights=False, ignore=255, gs=0.37, und=0.01, labels=()):
    return Case(name, N, C, Hp, Wp, stride, dtype, top_k, weights, ignore, gs, und, frozenset(labels))


CASES = [
    _c("fpn_full_f32", 2, 54, 200, 336, 4, labels={"mean", "finish_multi_pass", "ragged_channel_chunk"}),
    _c("fpn_full_bf16", 2, 54, 200, 336, 4, dtype=BF16, labels={"bf16", "finish_multi_pass"}),
    _c("cityscapes_topk", 4, 19, 256, 512, 4, top_k=0.2, weights=True,
       labels={"select", "tie_prefix_multi_pass", "ragged_channel_chunk"}),
    _c("cityscapes_mostly_ignored", 4, 19, 256, 512, 4, top_k=0.2, weights=True, und=0.9,
       labels={"threshold_zero_with_ignored_ties", "tie_prefix_multi_pass", "ties_split_at_threshold"}),
    _c("coco_topk", 2, 133, 160, 160, 4, top_k=0.2, weights=True, labels={"ragged_channel_chunk", "multi_chunk"}),
    _c("deeplab_os8_f16", 2, 21, 100, 100, 8, dtype=F16, top_k=0.2, labels={"f16", "ragged_channel_chunk"}),
    _c("s16_mean", 2, 19, 64, 128, 16, labels={"mean", "ragged_channel_chunk", "finish_multi_pass"}),
    _c("s16_topk", 2, 19, 64, 128, 16, top_k=0.2, gs=2.5, labels={"select", "tie_prefix_multi_pass"}),
    _c("s1", 2, 18, 36, 37, 1, labels={"stride1_copy", "ragged_tile", "ragged_channel_chunk", "tail_cta",
                                        "image_boundary_in_cta"}),
    _c("s2", 2, 16, 17, 1, 2, top_k=0.3, weights=True,
       labels={"single_chunk", "map_smaller_than_tile", "region_clamped_to_map", "last_logit_both_taps"}),
    _c("s3", 1, 18, 21, 12, 3, top_k=0.5, weights=True,
       labels={"odd_stride_fp32_taps", "ragged_channel_chunk", "ragged_tile", "tail_cta"}),
    _c("s5", 2, 7, 2, 13, 5, labels={"odd_stride_fp32_taps", "map_smaller_than_tile", "region_clamped_to_map"}),
    _c("s7", 1, 9, 9, 6, 7, ignore=0, labels={"odd_stride_fp32_taps", "ignore_in_class_range", "ragged_tile"}),
    _c("s8", 2, 12, 6, 7, 8, top_k=0.25, labels={"ragged_channel_chunk", "ragged_tile", "image_boundary_in_cta"}),
    _c("s13", 1, 5, 7, 1, 13, labels={"odd_stride_fp32_taps", "ragged_tile", "map_smaller_than_tile"}),
    _c("s20", 1, 4, 4, 5, 20, top_k=0.2, weights=True, labels={"ragged_channel_chunk", "ragged_tile"}),
    _c("s24", 1, 3, 5, 4, 24, top_k=0.1, labels={"T2_cc1", "odd_stride_fp32_taps", "multi_chunk"}),
    _c("s31", 2, 2, 9, 10, 31, labels={"T2_cc1", "smem_one_cta_per_sm", "region_spare_1", "ragged_tile"}),
    _c("s32", 2, 3, 4, 5, 32, top_k=1.0, weights=True, labels={"top_k_all", "smem_one_cta_per_sm", "ragged_tile"}),
    _c("c1", 2, 1, 6, 7, 4, top_k=0.3, ignore=-1, und=1.0,
       labels={"threshold_zero_with_ignored_ties", "ties_split_at_threshold"}),
    _c("c2", 2, 2, 8, 9, 4, ignore=2 ** 40, labels={"mean"}),
    _c("bad_label", 2, 5, 6, 7, 4, weights=True, top_k=0.5, labels={"bad_label"}),
    _c("all_ignored", 1, 5, 4, 5, 4, labels={"all_ignored", "mean"}),
    _c("k0", 1, 5, 4, 5, 4, top_k=1e-4, labels={"select_k0"}),
    _c("k1", 1, 5, 4, 5, 4, top_k=1.5 / 320, labels={"select_k1"}),
    _c("radix3", 1, 2, 40, 40, 1, top_k=0.5, weights=True, und=1.0, labels={"radix_level_3_decides"}),
    _c("big_logits", 2, 6, 8, 9, 4, top_k=0.3, weights=True, labels={"exp_underflow"}),
    _c("nonfinite_f32", 1, 4, 10, 12, 4, labels={"nan_logit", "pos_inf_logit", "neg_inf_logit"}),
    _c("nonfinite_f16", 1, 4, 10, 12, 4, dtype=F16, top_k=0.02, und=0.25,
       labels={"nan_logit", "pos_inf_logit", "neg_inf_logit", "threshold_nan", "f16"}),
    _c("weights_edge", 2, 5, 8, 10, 4, top_k=0.6, weights=True, und=0.5,
       labels={"weights_zero_or_negative", "threshold_zero_with_ignored_ties", "ties_split_at_threshold"}),
    _c("const_ties", 2, 8, 50, 60, 4, top_k=0.2, und=1.0, labels={"ties_split_at_threshold"}),
]
BY_NAME = {c.name: c for c in CASES}


def build(c, seed=0):
    """(logits, targets, weights) of a case on the GPU."""
    g = torch.Generator(device=DEV).manual_seed(seed + 1000 * CASES.index(c))
    N, C, hp, wp, s = c.N, c.C, c.Hp, c.Wp, c.stride
    h, w = hp * s, wp * s
    logits = torch.randn((N, C, hp, wp), generator=g, device=DEV) * 3.0
    targets = torch.randint(0, C, (N, h, w), generator=g, device=DEV)
    u = torch.rand((N, h, w), generator=g, device=DEV)
    targets[u < (0.85 if c.name == "cityscapes_mostly_ignored" else 0.1)] = c.ignore
    targets[:, : h // 5, : w // 4] = c.ignore
    weights = 0.5 + 2.5 * torch.rand((N, h, w), generator=g, device=DEV) if c.weights else None
    if c.name == "bad_label":
        targets[0, 3, 5], targets[1, h - 1, w - 1], targets[1, 0, w - 1] = C, -3, C + 7
    elif c.name == "all_ignored":
        targets.fill_(c.ignore)
    elif c.name == "s31":
        # image 1: only the last output row of the tightest region (the tile at low-res rows 6, 7 spans 94 rows of the
        # 95 its bound allows) is valid; that row reaches row 7 with weight 4.8e-7 and nothing else reaches row 7
        i0, _, _, _ = R.taps(s, h, hp)
        last = int(torch.searchsorted(i0, torch.tensor(8))) - 1
        targets[1] = c.ignore
        targets[1, last] = torch.randint(0, C, (w,), generator=g, device=DEV)
    elif c.name == "radix3":
        # C = 2, zero logits, stride 1: every valid loss is the same fp32 log 2, and weights 1 + j 2^-23 spread the values
        # over about 300 ulps, so that many agree with the k-th largest in their top 24 key bits
        logits.zero_()
        j = torch.randint(0, 200, (N, h, w), generator=g, device=DEV)
        weights = 1.0 + j.float() * 2.0 ** -23
    elif c.name == "big_logits":
        logits = torch.where(torch.rand(logits.shape, generator=g, device=DEV) < 0.5, -1e4, 1e4)
        logits[:, 1] = logits[:, 0] - 100.0                       # a gap beyond 88: __expf underflows to 0
        logits[:, 2] += torch.randn((N, hp, wp), generator=g, device=DEV) * 40
    elif c.name.startswith("nonfinite"):
        logits[0, 1, 3, 3] = math.nan
        logits[0, 2, 6, 8] = -math.inf
        logits[0, 0, 8, 2] = math.inf
        logits[0, 0, 1, 9] = math.nan                              # NaN in the first channel: before any finite max
        logits[0, 0, 5, 2], logits[0, 1, 5, 2] = -math.inf, math.nan  # NaN after nothing but -inf
        targets[0, 26:30, 30:36] = 2                               # targets on the -inf channel: an infinite loss
    elif c.name == "weights_edge":
        kind = torch.randint(0, 10, (N, h, w), generator=g, device=DEV)
        weights = torch.where(kind < 3, -weights, weights)         # negative: an ignored pixel's 0 * w is -0.0
        weights = torch.where(kind == 3, 0.0, weights)
        weights = torch.where(kind == 4, 1e-40, weights)           # subnormal
    elif c.name == "const_ties":
        logits.fill_(0.375)
    return logits.to(c.dtype), targets, weights


def run(c, logits, targets, weights, gs):
    loss_sum, count, status, lse, sel = S.sem_seg_loss_op(logits, targets, c.stride, c.ignore, c.top_k, weights)
    grad = S.sem_seg_loss_backward_op(logits, targets, c.stride, c.ignore, weights, sel, lse,
                                      torch.tensor(gs, dtype=torch.float32, device=DEV))
    return loss_sum, count, status, lse, sel, grad


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
    fin = torch.isfinite(want)
    err = (got - want).abs()
    bad = fin & ~(err <= bound)
    if bool(bad.any()):
        i = int(torch.nonzero(bad.reshape(-1))[0])
        raise AssertionError("%s: %d elements outside their bound; first at %s: got %r, want %r, bound %.3g"
                             % (what, int(bad.sum()), tuple(torch.unravel_index(torch.tensor(i), want.shape)),
                                float(got.reshape(-1)[i]), float(want.reshape(-1)[i]), float(bound.reshape(-1)[i])))


def upsampled32(logits, stride):
    x = logits.float()
    return x if stride == 1 else F.interpolate(x, scale_factor=stride, mode="bilinear", align_corners=False)


def kernel_values(ref, up, lse, weights):
    """The kernel's per-pixel fp32 values x = (lse - v_target) * w, 0 on skipped pixels, from its own lse."""
    vt = up.gather(1, ref.tc[:, None])[:, 0]
    x = torch.where(ref.valid, lse - vt, torch.zeros_like(lse))
    return x if weights is None else x * weights


def check(c, logits, targets, weights, gs=None):
    """Run a case and assert everything the module docstring lists; returns the labels its values reach."""
    gs = c.gs if gs is None else gs
    loss_sum, count, status, lse, sel, grad = run(c, logits, targets, weights, gs)
    if c.dtype != F32:
        out32 = run(c, logits.float(), targets, weights, gs)
        for a, b in zip((loss_sum, count, status, lse, sel), out32[:5]):
            assert same(a, b), c.name
        assert grad.dtype == c.dtype and same(grad, out32[5].to(c.dtype)), c.name
        grad = out32[5]
    ref = R.Ref(logits, targets, c.stride, c.ignore, c.top_k, weights)
    labels = set()
    assert int(status) == ref.status and int(count) == ref.count, (c.name, int(status), int(count))
    up = upsampled32(logits, c.stride)
    within(up, ref.v, ref.ev, c.name + " F.interpolate")
    within(lse, ref.lse, ref.e_lse, c.name + " lse")
    assert bool((lse[~ref.valid] == 0).all()), c.name + ": lse of a skipped pixel is not 0"
    x32 = kernel_values(ref, up, lse, weights)
    n_und = 0
    if ref.mode == "select":
        assert int(sel.sum()) == ref.k, (c.name, int(sel.sum()), ref.k)
        assert torch.equal(sel, R.select_top_k(x32, ref.k)), c.name + ": selection differs from the documented rule"
        above, below = ref.decided()
        flat = sel.reshape(-1).bool()
        assert bool(flat[above].all()) and not bool(flat[below].any()), c.name + ": a decided pixel is misselected"
        n_und = int((~(above | below)).sum())
        if ref.k:
            keys = R.order_keys(x32.reshape(-1))
            t = int(torch.sort(keys, descending=True).values[ref.k - 1])
            tied = keys == t
            if int(tied.sum()) > int((tied & flat).sum()) > 0:
                labels.add("ties_split_at_threshold")
            if t == int(R.order_keys(torch.zeros(1, device=DEV))[0]) and bool((~ref.valid).any()):
                labels.add("threshold_zero_with_ignored_ties")
            if t == 0xFFFFFFFF:
                labels.add("threshold_nan")
            if bool(((keys >> 8) == (t >> 8)).logical_and(keys != t).any()):
                labels.add("radix_level_3_decides")
    assert n_und <= c.und * ref.P, (c.name, n_und, ref.P)
    want, bound = ref.loss_sum(sel if ref.mode == "select" else None)
    got = float(loss_sum)
    if math.isfinite(want):
        assert abs(got - want) <= bound, (c.name, got, want, bound)
    else:
        assert got == want or (math.isnan(got) and math.isnan(want)), (c.name, got, want)
    g_ref, g_bound, reach = ref.grad(sel if ref.mode == "select" else None, gs)
    within(grad, g_ref, g_bound, c.name + " grad")
    assert bool((grad[~reach & ~torch.isnan(g_ref)] == 0).all()), c.name + ": a gradient no used pixel reaches is not 0"
    # the labels the values reach
    if 0 <= c.ignore < c.C:
        labels.add("ignore_in_class_range")
    if ref.status:
        labels.add("bad_label")
    if ref.count == 0:
        labels.add("all_ignored")
    if weights is not None and bool((weights <= 0).any()):
        labels.add("weights_zero_or_negative")
    lf = logits.float()
    for name, hit in (("nan_logit", torch.isnan(lf)), ("pos_inf_logit", lf == math.inf), ("neg_inf_logit", lf == -math.inf)):
        if bool(hit.any()):
            labels.add(name)
    gap = (ref.lse[:, None] - ref.v)[ref.valid[:, None].expand_as(ref.v) & torch.isfinite(ref.v)]
    if gap.numel() and bool((gap > 88).any()):
        labels.add("exp_underflow")
    return labels


@pytest.mark.parametrize("c", CASES, ids=lambda c: c.name)
def test_case(c):
    logits, targets, weights = build(c)
    got = check(c, logits, targets, weights)
    got |= R.shape_labels(c.N, c.C, c.Hp, c.Wp, c.stride, c.dtype, c.top_k)
    assert c.labels <= got, (c.name, sorted(c.labels - got))


def test_loss_weight_through_the_public_wrappers():
    """loss_weight 0.37: grad_sum = 0.37 / count (mean) or 0.37 / k (top-k) reaches the backward."""
    for c, wrap in ((BY_NAME["s3"], "fpn"), (BY_NAME["s8"], "deeplab")):
        logits, targets, weights = build(c, seed=5)
        if wrap == "fpn":
            c = c._replace(top_k=None, weights=False)
            weights = None
        ref = R.Ref(logits, targets, c.stride, c.ignore, c.top_k, weights)
        lg = logits.clone().requires_grad_(True)
        if wrap == "fpn":
            loss = S.sem_seg_fpn_losses(lg, targets, c.stride, c.ignore, 0.37)["loss_sem_seg"]
            sel, div = None, ref.count
        else:
            loss = S.deeplab_losses(lg, targets, c.stride, c.ignore, 0.37, "hard_pixel_mining", c.top_k, weights)
            loss = loss["loss_sem_seg"]
            sel, div = S.sem_seg_loss_op(logits, targets, c.stride, c.ignore, c.top_k, weights)[4], ref.k
        loss.backward()
        want, bound = ref.loss_sum(sel)
        want_loss = want / div * 0.37
        assert abs(float(loss.detach()) - want_loss) <= (bound / div * 0.37) * (1 + 4 * R.U) + 4 * R.U * abs(want_loss), wrap
        gs = float(torch.tensor(0.37, dtype=torch.float32) / torch.tensor(float(div), dtype=torch.float32))
        g_ref, g_bound, _ = ref.grad(sel, gs)
        within(lg.grad, g_ref, g_bound + 2 * R.U * g_ref.abs(), wrap + " grad")
