"""CPU checks of tests/paste_masks_ref.py: the float64 reference against the golden fixture (the reference's own paste) and
against the fp32 oracle within the derived bound; known answers for constant masks; every case of
tests/test_paste_masks_paths_gpu.py reaching the kernel paths it declares on an H100 SXM (132 SMs) and PCIe (114 SMs); the
path model's limits against the library's own refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import paste_masks_ref as pr
from oracle import oracle as orc
from test_paste_masks_paths_gpu import CASES, path_labels

# every path label of the model: launches, tables, rectangles, plane geometry, thresholds, mask sides, the packed form
ALL_LABELS = {
    "byte_balanced", "byte_uniform", "tab", "notab_narrow", "notab_large", "uniform_gx_capped", "mask_multi_cta",
    "rect_narrowed", "rect_full_narrow", "rect_full_degenerate", "rect_full_nonfinite", "rect_full_huge", "rect_empty",
    "rect_clipped", "head_unaligned", "ragged_tail", "spill_prev_row", "spill_next_row", "chunk_wrap_active", "thr_zero",
    "u8", "M1", "M64", "packed", "packed_partial_word", "packed_word_at_cx1", "packed_gx_capped", "n_over_65535",
}


def _within(got, v, b, what):
    got = np.asarray(got, dtype=np.float64)
    bad = np.abs(got - v) > b
    assert not bad.any(), (what, np.argwhere(bad)[:4], got[bad][:4], v[bad][:4], b[bad][:4])


def test_reference_matches_the_golden_fixture(golden):
    """The fixture's soft values come from the reference's own _do_paste_mask (grid_sample on the CPU, fp32): every finite
    one is within the bound of the float64 reference."""
    d = golden("paste_masks")
    h, w = [int(x) for x in d["hw"]]
    v, b = pr.soft(d["masks"], d["boxes"], h, w)
    s = np.asarray(d["soft"], dtype=np.float64).reshape(v.shape)
    fin = np.isfinite(s)
    assert fin.mean() > 0.5
    _within(s[fin], v[fin], b[fin], "golden soft")


@pytest.mark.parametrize("m", [1, 7, 28, 64])
def test_reference_matches_the_fp32_oracle(m):
    """orc.paste_masks restates the kernel's fp32 arithmetic: its soft value is within the bound everywhere, on boxes from
    sub-pixel to 1e8 wide, partly or wholly off the image, degenerate and non-finite."""
    rng = np.random.default_rng(m)
    h, w = 45, 70
    ctr = rng.random((40, 2)) * [w * 1.4, h * 1.4] - [w * 0.2, h * 0.2]
    wh = np.exp(rng.uniform(np.log(0.2), np.log(200), (40, 2)))
    boxes = np.concatenate([ctr - wh / 2, ctr + wh / 2], 1)
    boxes[:8] = [(30.3, 20.35, 30.6, 20.65), (10.1, 5.2, 10.35, 40.7), (-1e8, 3.0, 1e8, 40.0), (5.0, -3e8, 60.0, 2e8),
                 (30.0, 10.0, 30.0, 30.0), (40.0, 10.0, 20.0, 30.0), (np.nan, 1.0, 20.0, 20.0), (5.0, 5.0, np.inf, 30.0)]
    boxes = boxes.astype(np.float32)
    masks = rng.random((40, m, m)).astype(np.float32)
    masks[-1] = 1.0
    _, s = orc.paste_masks(torch.from_numpy(masks), torch.from_numpy(boxes), (h, w), 0.5, return_soft=True)
    v, b = pr.soft(masks, boxes, h, w)
    _within(s.numpy(), v, b, "oracle soft")


def test_known_answers_for_constant_masks():
    """A constant mask c pastes as c tri(ix) tri(iy); a box of exactly M x M pixels at the origin samples the mask centres
    (ix = px): v = c on the whole box, 0 beyond its one-pixel bilinear border."""
    for m, box, (h, w) in ((28, (0.0, 0.0, 28.0, 28.0), (30, 31)), (7, (3.5, -2.25, 40.0, 17.5), (20, 45)),
                           (1, (2.0, 2.0, 9.0, 5.0), (8, 12)), (64, (-10.5, 4.0, 70.0, 30.0), (40, 64))):
        c = 0.625
        p = pr.Paste(np.full((m, m), c, np.float32), box, h, w)
        want = pr.known_constant(c, box, m, h, w)
        assert np.allclose(p.full("v"), want, rtol=0, atol=1e-12), (m, box)
    p = pr.Paste(np.full((28, 28), 0.625, np.float32), (0.0, 0.0, 28.0, 28.0), 30, 31)
    v = p.full("v")
    assert (v[:28, :28] == 0.625).all() and (v[28:] == 0).all() and (v[:, 28:] == 0).all()
    assert not pr.Paste(np.ones((28, 28), np.float32), (np.nan, 0.0, 10.0, 10.0), 12, 12).full("v").any()
    assert not pr.Paste(np.ones((28, 28), np.float32), (5.0, 0.0, 5.0, 10.0), 12, 12).full("v").any()


def test_decisions():
    v, b = np.array([0.5, 0.5, 0.49, 0.0, 1.0]), np.array([0.0, 1e-6, 1e-6, 0.0, 0.0])
    want, dec, _, _ = pr.decide(v, b, 0.5)
    assert want.tolist()[:3] == [1, 0, 0] and dec.tolist() == [True, False, True, True, True]
    want, dec, lo, hi = pr.decide(np.array([0.0, 0.5, 2 / 255, 0.3]), np.array([0.0, 0.0, 1e-5, 1e-6]), -1.0)
    assert want[0] == 0 and want[1] == 127 and not dec[2] and lo[2] == 1 and hi[2] == 2 and dec[3] and want[3] == 76
    assert pr.outside_byte(0.0) == 1 and pr.outside_byte(0.5) == 0 and pr.outside_byte(-1.0) == 0


# ------------------------------------------------------------------------------------------- path coverage
@pytest.mark.parametrize("sms", [132, 114])
def test_every_case_reaches_its_paths(sms):
    for case in CASES:
        got = path_labels(case, sms)
        assert case.labels <= got, (case.name, sms, sorted(case.labels - got))


def test_every_path_label_is_declared():
    declared = set().union(*(c.labels for c in CASES))
    assert declared == ALL_LABELS, (sorted(ALL_LABELS - declared), sorted(declared - ALL_LABELS))


def test_launch_examples():
    assert pr.launch(9, 28, 61, 83, 132)["balanced"] and pr.launch(528, 28, 61, 83, 132)["balanced"]
    assert not pr.launch(529, 28, 61, 83, 132)["balanced"] and not pr.launch(457, 28, 61, 83, 114)["balanced"]
    u = pr.launch(600, 28, 100, 100, 132)
    assert u["gx"] == 2 and u["capped"] and u["launches"] == 1
    assert pr.launch(65600, 4, 5, 7, 132)["launches"] == 2 and pr.launch_packed(65600, 5, 7, 132)["launches"] == 2
    assert pr.launch(3, 28, 3, 7675, 132)["tab"] and not pr.launch(3, 28, 3, 7676, 132)["tab"]
    assert not pr.launch(3, 28, 100, 31, 132)["tab"]
    counts = pr.cta_counts([pr.paste_rect(b, 28, 61, 83)[0] for b in CASES[0].boxes], 61, 83, 132)
    assert sum(counts) == 8 * 132 and min(counts) >= 1
    assert pr.paste_rect((20.0, 10.0, 48.0, 38.0), 28, 61, 83) == ((17, 51, 7, 41), "narrowed")
    assert pr.paste_rect((-60.2, 10.3, -20.7, 50.1), 28, 61, 83)[0][1] < 0
    assert pr.head_of(1, 61 * 83) == 9 and pr.head_of(16, 61 * 83) == 0


def test_limits_agree_with_the_library():
    """The model's refusals against the library's, with non-null dummy pointers: each is refused before any launch."""
    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL, EUNSUPPORTED = -1, -3
    code = {"einval": EINVAL, "unsupported": EUNSUPPORTED}
    dummy = C.c_void_p(256)
    for n, m, h, w, thr in ((1, 65, 10, 10, 0.5), (3, 128, 10, 10, -1.0), (1, 28, 1 << 15, 1 << 15, 0.5),
                            (2, 64, 1 << 20, 1 << 10, 0.5), (1, 0, 10, 10, 0.5), (-1, 28, 10, 10, 0.5)):
        want = code[pr.status(n, m, h, w, thr)]
        assert lib.d2b_paste_masks(dummy, dummy, n, m, h, w, thr, dummy, None) == want, (n, m, h, w)
        if thr >= 0:
            want = code[pr.status(n, m, h, w, thr, packed=True)]
            assert lib.d2b_paste_masks_packed(dummy, dummy, n, m, h, w, thr, dummy, None) == want, (n, m, h, w)
    assert pr.status(1, 65, 10, 10) == "unsupported" and pr.status(1, 28, 1 << 15, 1 << 15) == "unsupported"
    assert pr.status(70000, 64, (1 << 15) - 1, 1 << 15) == "ok"  # any number of masks; M = 64 and H * W < 2^30 are taken
    assert lib.d2b_paste_masks_packed(dummy, dummy, 3, 28, 10, 10, float("nan"), dummy, None) == EINVAL
    assert pr.status(3, 28, 10, 10, float("nan"), packed=True) == "einval"
