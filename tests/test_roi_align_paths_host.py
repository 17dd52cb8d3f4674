"""CPU checks of tests/roi_align_ref.py: the float64 reference pinned to the reference's known answers, the fp32 oracle and
torchvision; every case of tests/test_roi_align_paths_gpu.py reaching the kernel paths it declares on an H100 SXM (132 SMs)
and PCIe (114 SMs); the path model's launch arithmetic against the library's own shape limits."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import roi_align_ref as ra
from oracle import oracle as orc
from test_roi_align_column_walk import sample_pos
from test_roi_align_paths_gpu import CASES, image_rois, levels_of, path_labels

# every path label of the model: channels-last forward, channels-last backward, NCHW kernel, launches, boundaries
ALL_LABELS = {
    "walk_ry1", "walk_ry2", "walk_ry3", "walk_ry4", "walk_ry5", "walk_ry6", "walk_carry_in", "walk_empty_row",
    "refuse_three_bins", "refuse_colcap", "refuse_nymax", "refuse_profit", "refuse_pw7",
    "bin42", "bin42_padded", "bin81", "bin81_padded", "bin_empty_row", "fwd_onfly_pooled", "fwd_onfly_overflow",
    "fwd_nchunks1", "fwd_nchunks_even", "fwd_nchunks_ragged", "slab_partial", "slab_full", "slab_multi", "slab_ragged",
    "slab_many", "fwd_out_f16", "fwd_out_bf16",
    "bwd_separable", "bwd_general", "bwd_per_sample_pooled", "bwd_per_sample_wide", "bwd_bands1", "bwd_bands2",
    "bwd_bands3", "bwd_band_edge_in_bin_row", "bwd_rows_split", "bwd_rows_split_ragged", "bwd_empty", "bwd_go_f16",
    "bwd_go_bf16",
    "v3_staged_1band", "v3_staged_bands", "v3_direct_rowoff", "v3_direct_sparse", "v3_onfly", "v3_empty",
    "v3_groups_split", "v3_groups_whole", "v3_ragged_group",
    "unaligned_clamp", "pos_-1", "pos_0", "pos_H-1", "pos_H", "sr0", "sr1", "sr2", "sr3", "sr4", "pyramid",
}


# ------------------------------------------------------------------------------------------- reference pins
def _fwd(x, rois, scale, ph, pw, sr, aligned):
    return ra.forward([x], np.asarray(rois, dtype=np.float32), [scale], [0] * len(rois), ph, pw, sr, aligned)


def test_reference_known_answers():
    # the reference's tables (detectron2 tests/layers/test_roi_align.py), as in test_gpu_parity.test_roi_align_reference_kats
    img = np.arange(25, dtype=np.float64).reshape(1, 1, 5, 5)
    old = [[7.5, 8, 8.5, 9], [10, 10.5, 11, 11.5], [12.5, 13, 13.5, 14], [15, 15.5, 16, 16.5]]
    new = [[4.5, 5.0, 5.5, 6.0], [7.0, 7.5, 8.0, 8.5], [9.5, 10.0, 10.5, 11.0], [12.0, 12.5, 13.0, 13.5]]
    assert np.array_equal(_fwd(img, [[0, 1, 1, 3, 3]], 1.0, 4, 4, 0, False)[0][0, 0], old)
    assert np.array_equal(_fwd(img, [[0, 1, 1, 3, 3]], 1.0, 4, 4, 0, True)[0][0, 0], new)
    # an empty box with aligned=True samples nothing: zero output, zero gradient
    y = _fwd(np.random.default_rng(0).random((1, 1, 5, 5)), [[0, 3, 4, 5, 4]], 1.0, 7, 7, 0, True)[0]
    assert (y == 0).all()
    (g, _, _), = ra.backward(np.ones((1, 1, 7, 7)), [(1, 1, 5, 5)], np.array([[0, 3, 4, 5, 4]], np.float32), [1.0], [0], 7, 7,
                             0, True)
    assert (g == 0).all()


@pytest.mark.parametrize("sr,aligned", [(0, True), (2, False), (3, True)])
def test_reference_matches_fp32_oracle(sr, aligned):
    rng = np.random.default_rng(sr)
    x = rng.standard_normal((2, 5, 30, 41)).astype(np.float32)
    k = 40
    ctr = rng.random((k, 2)) * [164, 120]
    wh = 2 + rng.random((k, 2)) * 120
    rois = np.concatenate([rng.integers(0, 2, (k, 1)), ctr - wh / 2, ctr + wh / 2], 1).astype(np.float32)
    rois[0] = [0, -60, -40, -10, -5]  # outside the map
    # the oracle computes the sample positions in fp32 in the same order, then sums 4 taps per sample (two roundings per
    # term in the backward's scatter): its terms per output are bounded with the largest sampling grid of the set
    spb = max(ra.geom(r, 0.25, 7, 6, sr, aligned).count for r in rois)
    ref, a, _ = _fwd(x, rois, 0.25, 7, 6, sr, aligned)
    got = orc.roi_align_forward(torch.from_numpy(x), torch.from_numpy(rois), 0.25, 7, 6, sr, aligned).numpy()
    ra.check(got, ref, a, 4 * spb + 4, what="oracle forward")
    go = rng.standard_normal((k, 5, 7, 6)).astype(np.float32)
    (g, ga, gm), = ra.backward(go, [x.shape], rois, [0.25], [0] * k, 7, 6, sr, aligned)
    got = orc.roi_align_backward(torch.from_numpy(go), torch.from_numpy(rois), 0.25, 7, 6, 2, 5, 30, 41, sr, aligned).numpy()
    ra.check(got, g, ga, 3 * spb * gm + 4, what="oracle backward")


def test_reference_matches_torchvision_float64():
    tv = pytest.importorskip("torchvision")
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, 3, 24, 30))
    # dyadic boxes at 8x8 (the last one below a pixel, clamped when aligned=False): every sample position is exact in fp32,
    # so the fp32 positions equal torchvision's float64 ones
    rois = np.array([[0, 2, 3, 30, 17], [1, -3, -2, 11, 26], [0, 4.5, 1.25, 46.5, 57.25], [1, 60, 40, 116, 96],
                     [0, 10, 10, 10.5, 10.5]], dtype=np.float32)
    for sr, aligned in [(0, True), (2, True), (0, False), (4, False)]:
        ref = _fwd(x, rois, 0.5, 8, 8, sr, aligned)[0]
        got = tv.ops.roi_align(torch.from_numpy(x), torch.from_numpy(rois.astype(np.float64)), (8, 8), 0.5, sr, aligned)
        np.testing.assert_allclose(ref, got.numpy(), rtol=1e-14, atol=1e-14)


def test_case_positions_are_exact_in_fp32():
    """The dyadic geometry of the GPU cases: the fp32 sample positions equal the exact rational ones."""
    for case in CASES:
        rois = image_rois(case)
        for r, l in zip(rois, levels_of(case, rois)):
            s = Fraction(case.levels[l][2])
            off = Fraction(1, 2) if case.aligned else 0
            g = ra.geom(r, float(s), case.ph, case.pw, case.sr, case.aligned)
            for start, side, n, grid, fp in ((r[2], r[4] - r[2], case.ph, g.gh, g.start_h), (r[1], r[3] - r[1], case.pw, g.gw, g.start_w)):
                side = Fraction(float(side)) * s
                if not case.aligned:
                    side = max(side, Fraction(1))
                b = side / n
                for p in range(n):
                    for i in range(grid):
                        exact = Fraction(float(start)) * s - off + p * b + (2 * i + 1) * b / (2 * grid)
                        assert Fraction(sample_pos(fp, float(b), grid, p, i, True)) == exact, (case.name, p, i)


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
    assert ra.launch_fwd_nhwc(100, 128, 14, 14, 132) == (10, 21)  # 9 chunks of 21 bins and a last one of 7
    assert ra.launch_fwd_nhwc(1100, 4, 7, 7, 132) == (1, 49)
    assert [ra.launch_bwd_nhwc(k, 8, 10, 10, 132) for k in (263, 264, 527, 528)] == [3, 5, 5, 10]
    assert [ra.launch_bwd_nhwc(k, 8, 8, 8, 132) for k in (527, 528)] == [4, 8]
    assert ra.launch_bwd_nhwc(100, 256, 14, 14, 132) == 4
    assert ra.launch_fwd(24, 256, 132) == 8 and ra.launch_fwd(4000, 256, 132) == 64
    assert ra.slabs(132) == [(0, 128), (128, 4)]


def test_backward_pooled_sizes_agree_with_the_library():
    """nhwc_bwd_supported restates nhwc_supported's backward branch; d2b_roi_pooler_nhwc_supported is the library's."""
    from detectron2_b200 import _C, ops

    for ph in range(1, 41):
        for pw in range(1, 41):
            lib = ops._nhwc_supported(8, ((64, 64),), ph, pw, _C.ROI_BACKWARD)
            assert lib == ra.nhwc_bwd_supported(ph, pw), (ph, pw)
