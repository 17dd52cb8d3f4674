"""paste_masks_in_image (paste_masks.cu) path by path against the float64 reference of tests/paste_masks_ref.py.

For every case: the byte output equals the fp32 oracle (orc.paste_masks, the kernel's expression order) bit for bit; every
pixel the float64 reference decides -- its value farther than the derived bound from the threshold, or from a uint8 step --
equals that decision, and an undecided uint8 pixel is one of the two values the bound allows; undecided pixels are a small
share of the pixels inside the masks' rectangles, so the check is not vacuous; with a threshold >= 0 the bit-packed output
unpacks to the byte output.  tests/test_paste_masks_paths_host.py checks on the CPU that each case reaches the paths listed
here, at 132 and at 114 SMs.

case                  reaches
balanced_borders      9 masks on 61 x 83 (every head after mask 0 unaligned, ragged tails): boxes inside, straddling each
                      border and wholly off each side (empty rectangle); coordinate tables, rows spilling into both
                      neighbours, phase-1 chunks active through the row they wrap into; many CTAs per mask
balanced_degenerate   zero and negative width, a 0.3 px box, |x| >= 1e8, extent >= 1e8, NaN, +inf and -inf corners
thr_zero              the borders at threshold 0: every pixel that cannot see its mask is 1
u8_borders            the borders as uint8 (threshold < 0)
thr_above_one         threshold 1.5: nothing is set
narrow_w*             W = 1, 15, 16, 17, 31: no tables, the whole image evaluated
large_3x7700          W + H > 7678: no tables on a wide image
large_2000x6000       no tables, 12 M pixels per plane
uniform_*             600 masks: the (CTAs per mask, N) launch with tables (40 x 72), without (9 x 31 and 2 x 7700), and
                      with the CTAs per mask capped (100 x 100)
m1, m7, m64           mask sides 1, 7 and 64 (the largest the kernel takes); thresholds 0.5, 0.999 and uint8
packed_last_word      W = 97: a row's last packed word holds one pixel, on the rectangle's last column
bench                 100 masks on 800 x 1333, every mask against the oracle and the reference
n65600                65 600 masks on 5 x 7: two launches of the uniform grid, byte and packed

Across launches (test_plane_is_independent_of_the_launch) a mask's plane is byte-identical pasted alone, at index 0 and 1 of a
balanced batch, and inside a batch of 600.
"""
import functools
from collections import namedtuple

import numpy as np
import pytest
import torch

import paste_masks_ref as pr
from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda"
NAN, INF = float("nan"), float("inf")

Case = namedtuple("Case", "name n m h w thr boxes masks labels")

# 61 x 83: inside, straddling left / top / right / bottom, wholly off left / top / right / bottom
BORDERS = [(20.3, 15.7, 60.2, 45.1), (-10.4, 20.2, 25.6, 50.3), (30.1, -12.6, 70.7, 18.4), (55.3, 10.1, 95.8, 40.9),
           (5.2, 40.3, 45.9, 75.6), (-60.2, 10.3, -20.7, 50.1), (10.4, -70.2, 60.3, -25.8), (110.3, 5.2, 150.6, 40.4),
           (20.1, 90.3, 60.7, 130.2)]
DEGENERATE = [(10.2, 8.7, 50.4, 40.3), (30.0, 10.0, 30.0, 40.0), (40.0, 10.0, 20.0, 40.0), (40.3, 30.35, 40.6, 30.65),
              (-1e8, 5.0, 1e8, 50.0), (5.5, 3.5, 2e8, 50.5), (NAN, 5.0, 30.0, 40.0), (10.3, 10.7, INF, 40.2),
              (-INF, -INF, 40.5, 50.5)]


def random_boxes(n, h, w, seed, lo=1.0):
    """Centres anywhere in the image (and a little beyond), sides from `lo` px to the image's."""
    g = np.random.default_rng(seed)
    ctr = g.random((n, 2)) * [w * 1.2, h * 1.2] - [w * 0.1, h * 0.1]
    wh = lo + g.random((n, 2)) * [w, h]
    return np.concatenate([ctr - wh / 2, ctr + wh / 2], 1)


def bench_boxes(n, h, w, seed):
    g = torch.Generator().manual_seed(seed)
    torch.rand(n, 28, 28, generator=g)
    ctr = torch.rand(n, 2, generator=g) * torch.tensor([float(w), float(h)])
    wh = 20 + torch.rand(n, 2, generator=g) * 500
    return torch.cat([ctr - wh / 2, ctr + wh / 2], 1).numpy()


def _c(name, n, m, h, w, thr, boxes, labels, masks="rand"):
    return Case(name, n, m, h, w, thr, boxes, masks, frozenset(labels))


_EDGE_R = [(60.3, 5.2, 110.7, 30.4), (80.1, 12.6, 99.2, 35.3), (70.6, 20.3, 130.2, 39.8), (90.2, 1.3, 103.5, 25.1),
           (40.3, 3.1, 98.6, 36.9)]
CASES = [
    _c("balanced_borders", 9, 28, 61, 83, 0.5, BORDERS,
       {"byte_balanced", "tab", "mask_multi_cta", "rect_narrowed", "rect_clipped", "rect_empty", "head_unaligned",
        "ragged_tail", "spill_prev_row", "spill_next_row", "chunk_wrap_active", "packed", "packed_partial_word"}),
    _c("balanced_degenerate", 9, 28, 61, 83, 0.5, DEGENERATE,
       {"rect_full_degenerate", "rect_full_nonfinite", "rect_full_huge", "rect_narrowed"}),
    _c("thr_zero", 9, 28, 61, 83, 0.0, BORDERS, {"thr_zero", "packed"}),
    _c("u8_borders", 9, 28, 61, 83, -1.0, BORDERS, {"u8"}),
    _c("thr_above_one", 9, 28, 61, 83, 1.5, BORDERS, {"packed"}),
] + [
    _c("narrow_w%d" % w, 5, 28, 23, w, 0.5, ("random", 10 + w), {"notab_narrow", "rect_full_narrow", "byte_balanced"})
    for w in (1, 15, 16, 17, 31)
] + [
    _c("large_3x7700", 3, 28, 3, 7700, 0.5, [(100.3, -1.2, 900.6, 2.7), (5000.2, 0.3, 7800.1, 3.9), (-200.4, -5.1, 300.3, 10.2)],
       {"notab_large", "rect_clipped"}),
    _c("large_2000x6000", 3, 28, 2000, 6000, 0.5,
       [(100.3, 200.7, 900.6, 1500.2), (4500.2, 1200.3, 6100.1, 2100.9), (-300.5, -100.2, 700.3, 400.8)],
       {"notab_large", "mask_multi_cta"}),
    _c("uniform_tab_40x72", 600, 28, 40, 72, 0.5, ("random", 1), {"byte_uniform", "tab"}),
    _c("uniform_notab_9x31", 600, 28, 9, 31, 0.5, ("random", 2), {"byte_uniform", "notab_narrow"}),
    _c("uniform_notab_2x7700", 600, 28, 2, 7700, 0.5, ("random", 3), {"byte_uniform", "notab_large"}),
    _c("uniform_capped_100x100", 600, 28, 100, 100, 0.5, ("random", 4), {"byte_uniform", "uniform_gx_capped", "mask_multi_cta"}),
    _c("m1", 6, 1, 37, 129, 0.5, ("random", 5), {"M1"}, masks="high"),
    _c("m7", 9, 7, 40, 72, 0.999, ("random", 6), {"packed"}, masks="high"),
    _c("m64", 5, 64, 50, 90, -1.0, ("random", 7), {"M64", "u8"}),
    _c("packed_last_word", 5, 28, 40, 97, 0.5, _EDGE_R, {"packed_partial_word", "packed_word_at_cx1"}, masks="high"),
    _c("bench", 100, 28, 800, 1333, 0.5, ("bench", 42), {"packed_gx_capped", "mask_multi_cta", "tab"}),
    _c("n65600", 65600, 4, 5, 7, 0.5, ("random", 8), {"n_over_65535", "byte_uniform", "packed"}),
]
BY_NAME = {c.name: c for c in CASES}
ids = [c.name for c in CASES]


def case_boxes(case):
    """[N, 4] fp32 boxes; the random recipes tile at most 1 000 distinct boxes."""
    if isinstance(case.boxes, tuple):
        kind, seed = case.boxes
        if kind == "bench":
            return bench_boxes(case.n, case.h, case.w, seed).astype(np.float32)
        base = random_boxes(min(case.n, 1000), case.h, case.w, seed)
        return np.resize(base, (case.n, 4)).astype(np.float32)
    return np.resize(np.array(case.boxes, dtype=np.float64), (case.n, 4)).astype(np.float32)


def case_masks(case):
    """[N, M, M] fp32 masks in [0, 1) ("high": [0.5, 1)); at most 1 000 distinct ones, tiled with the boxes' period."""
    g = torch.Generator().manual_seed(sum(map(ord, case.name)))
    k = min(case.n, 1000)
    if case.boxes == ("bench", 42):
        g = torch.Generator().manual_seed(42)  # the masks of tests/test_gpu_parity.py's full-size case
    m = torch.rand(k, case.m, case.m, generator=g)
    if case.masks == "high":
        m = 0.5 + 0.5 * m
    return m.repeat((case.n + k - 1) // k, 1, 1)[: case.n].contiguous()


def path_labels(case, sms):
    return pr.path_labels(case.m, case_boxes(case), case.h, case.w, case.thr, sms)


@functools.lru_cache(maxsize=None)
def _inputs(name):
    case = BY_NAME[name]
    return case_masks(case), torch.from_numpy(case_boxes(case))


def check_against_reference(got, masks, boxes, case):
    """Every decidable pixel equals the float64 decision; returns (undecided pixels, pixels inside the rectangles)."""
    got = got.numpy().astype(np.int64)
    h, w, thr = case.h, case.w, case.thr
    zb = pr.outside_byte(thr)
    mk, bx = masks.numpy(), boxes.numpy()
    undecided, inside, memo = 0, 0, {}
    for k in range(len(bx)):
        key = (mk[k].tobytes(), bx[k].tobytes())
        if key not in memo:
            P = pr.Paste(mk[k], bx[k], h, w)
            want, dec, lo, hi = pr.decide(P.v, P.b, thr)
            memo[key] = (P, want, dec, lo, hi, pr.rect_pixels(pr.paste_rect(bx[k], case.m, h, w)[0]))
        P, want, dec, lo, hi, npix = memo[key]
        g = got[k]
        win = g[P.r0:P.r1, P.c0:P.c1]
        rest = g.copy()
        rest[P.r0:P.r1, P.c0:P.c1] = zb
        assert (rest == zb).all(), (case.name, k, "a pixel beyond the support is not the outside value", np.argwhere(rest != zb)[:4])
        bad = dec & (win != want)
        assert not bad.any(), (case.name, k, np.argwhere(bad)[:4] + [P.r0, P.c0], P.v[bad][:4], P.b[bad][:4])
        assert ((win >= lo) & (win <= hi)).all(), (case.name, k, "outside the bound")
        undecided += int((~dec).sum())
        inside += npix
    return undecided, inside


@pytest.mark.parametrize("name", ids)
def test_paste_path_case(name):
    import detectron2_b200.layers as L

    case = BY_NAME[name]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert case.labels <= path_labels(case, sms)
    masks, boxes = _inputs(name)
    hw = (case.h, case.w)
    got = L.paste_masks_in_image(masks.to(DEV), boxes.to(DEV), hw, case.thr)
    assert got.dtype == (torch.bool if case.thr >= 0 else torch.uint8) and got.shape == (case.n, case.h, case.w)
    got = got.cpu()
    assert torch.equal(got, orc.paste_masks(masks, boxes, hw, case.thr)), name
    undecided, inside = check_against_reference(got.to(torch.uint8), masks, boxes, case)
    # not vacuous: the bound decides nearly every pixel the kernel evaluates (uint8 steps are 1/255 apart: a wider margin)
    assert undecided <= (0.02 if case.thr < 0 else 0.002) * max(inside, 1), (undecided, inside)
    if case.thr >= 0:
        packed = L.paste_masks_in_image_packed(masks.to(DEV), boxes.to(DEV), hw, case.thr)
        assert torch.equal(L.unpack_mask_bits(packed, case.w).cpu(), got), name


def test_plane_is_independent_of_the_launch():
    """A mask's plane, pasted alone (balanced launch, head aligned), at index 0 and 1 of a 9-mask balanced batch (aligned
    and unaligned head), and at indices 300 and 301 of a 600-mask uniform batch: the same bytes."""
    import detectron2_b200.layers as L

    h, w = 61, 83
    masks, boxes = _inputs("balanced_borders")
    others_m, others_b = _inputs("uniform_tab_40x72")
    for thr in (0.5, -1.0):
        for k in range(len(boxes)):
            m, b = masks[k:k + 1], boxes[k:k + 1]
            alone = L.paste_masks_in_image(m.to(DEV), b.to(DEV), (h, w), thr)[0]
            planes = []
            for pos, n in ((0, 9), (1, 9), (300, 600), (301, 600)):
                bm, bb = others_m[:n].clone(), others_b[:n].clone()
                bm[pos], bb[pos] = m[0], b[0]
                planes.append(L.paste_masks_in_image(bm.to(DEV), bb.to(DEV), (h, w), thr)[pos])
            for pos, p in zip((0, 1, 300, 301), planes):
                assert torch.equal(p, alone), (thr, k, pos)


class _Boxes:
    """The one attribute of detectron2.structures.Boxes the wrapper reads."""

    def __init__(self, t):
        self.tensor = t


def test_wrapper_surface():
    """fp16 / bf16 inputs paste as their fp32 up-casts; (N, 1, M, M) masks and Boxes are accepted; M = 65 is refused."""
    import detectron2_b200.layers as L

    masks, boxes = _inputs("balanced_borders")
    hw = (61, 83)
    for dt in (torch.float16, torch.bfloat16):
        mh, bh = masks.to(dt).to(DEV), boxes.to(dt).to(DEV)
        for thr in (0.5, -1.0):
            assert torch.equal(L.paste_masks_in_image(mh, bh, hw, thr), L.paste_masks_in_image(mh.float(), bh.float(), hw, thr))
        assert torch.equal(L.paste_masks_in_image_packed(mh, bh, hw, 0.5), L.paste_masks_in_image_packed(mh.float(), bh.float(), hw, 0.5))
    ref = L.paste_masks_in_image(masks.to(DEV), boxes.to(DEV), hw, 0.5)
    assert torch.equal(L.paste_masks_in_image(masks[:, None].to(DEV), _Boxes(boxes.to(DEV)), hw, 0.5), ref)
    assert torch.equal(L.paste_masks_in_image_packed(masks[:, None].to(DEV), _Boxes(boxes.to(DEV)), hw, 0.5),
                       L.paste_masks_in_image_packed(masks.to(DEV), boxes.to(DEV), hw, 0.5))
    big = torch.rand(2, 65, 65, device=DEV)
    with pytest.raises(RuntimeError):
        L.paste_masks_in_image(big, boxes[:2].to(DEV), hw, 0.5)
    with pytest.raises(RuntimeError):
        L.paste_masks_in_image_packed(big, boxes[:2].to(DEV), hw, 0.5)
