"""CPU checks of tests/roi_align_rotated_ref.py: the float64 reference against the fp32 oracle (within the derived bound on
random rotated boxes, to the (m + 5) bound alone at angle 0 on dyadic geometry); every case of
tests/test_roi_align_rotated_paths_gpu.py reaching the kernel paths it declares on an H100 SXM (132 SMs) and PCIe (114 SMs);
no case with a sample within its position error of the map edge, except the angle-0 lattice case; the path model's
pooled-size limit against the library's own."""
import numpy as np
import pytest
import torch

import roi_align_rotated_ref as rr
from oracle import oracle as orc
from test_roi_align_rotated_paths_gpu import CASES, roi_objects, path_labels

# every path label of the model: table / on the fly in both kernels, launches and layouts, angles, positions, box shapes
ALL_LABELS = {
    "nchw_table", "nchw_table_1024", "nchw_onfly", "nhwc_table", "nhwc_table_1024", "nhwc_onfly", "empty_grid",
    "cpc_whole", "cpc_split", "cpc_ragged", "c_not_4", "nhwc_refused", "nhwc_largest_pooled", "non_square",
    "slab_partial", "slab_full", "slab_multi", "slab_ragged",
    "angle0", "angle90", "angle-90", "angle180", "angle-180", "angle45", "angle_other",
    "inside", "outside_partial", "outside_whole", "mirrored", "sub_pixel", "batch1",
    "pos_-1", "pos_0", "pos_H-1", "pos_H", "sr0", "sr1", "sr2", "sr3",
    "f16_layer_upcast", "out_f16", "go_f16", "out_bf16", "go_bf16", "pyramid", "dead_level", "level_boundary",
}


def _random_rois(rng, k, h, w, scale):
    ctr = rng.random((k, 2)) * [w / scale, h / scale] + rng.random((k, 2)) * 40 - 20
    wh = 4 + rng.random((k, 2)) * 60
    ang = 180 - rng.random((k, 1)) * 360
    ang[:6, 0] = [90, -90, 180, -180, 45, 0.5]
    return np.concatenate([rng.integers(0, 2, (k, 1)), ctr, wh, ang], 1).astype(np.float32)


def _oracle_both(x, rois, scale, ph, pw, sr, go):
    n, c, h, w = x.shape
    y = orc.roi_align_rotated_forward(torch.from_numpy(x), torch.from_numpy(rois), scale, ph, pw, sr).numpy()
    g = orc.roi_align_rotated_backward(torch.from_numpy(go), torch.from_numpy(rois), scale, ph, pw, n, c, h, w, sr).numpy()
    return y, g


@pytest.mark.parametrize("sr,ph,pw", [(0, 7, 7), (2, 5, 9), (1, 13, 4)])
def test_reference_matches_fp32_oracle(sr, ph, pw):
    """The oracle computes the same fp32 geometry with cosf / sinf and without contraction, then sums the taps in fp32: its
    positions are within delta_s of the float64 ones, so the reference's bound holds for it as for the kernels.  The first
    channel is all ones: its output is (in-map samples) / count, which pins the sampling grid of every RoI."""
    rng = np.random.default_rng(10 * sr + ph)
    x = rng.standard_normal((2, 5, 30, 41)).astype(np.float32)
    x[:, 0] = 1.0
    scale = 0.25
    rois = _random_rois(rng, 40, 30, 41, scale)
    rois[6] = [1, 60, 50, 0, 30, 20]  # zero width
    rois[7] = [0, 70, 40, -20, 30, -30]  # negative width
    for r in rois:
        assert rr.Roi(r, scale, ph, pw, sr, 30, 41).ambiguous == 0, r
    go = rng.standard_normal((len(rois), 5, ph, pw)).astype(np.float32)
    ref = rr.forward([x], rois, [scale], [0] * len(rois), ph, pw, sr)
    (gref, ga, gm, gp), = rr.backward(go, [x.shape], rois, [scale], [0] * len(rois), ph, pw, sr)
    y, g = _oracle_both(x, rois, scale, ph, pw, sr, go)
    rr.check(y, *ref, what="oracle forward")
    rr.check(g, gref, ga, gm, gp, what="oracle backward")


def test_reference_matches_fp32_oracle_exactly_at_angle_0():
    """Angle 0 on dyadic geometry: every fp32 position is exact, P = 0, and the (m + 5) bound alone holds."""
    rng = np.random.default_rng(3)
    x = rng.standard_normal((1, 4, 20, 24)).astype(np.float32)
    scale = 0.5
    rois = np.array([[0, 9, 9, 14, 14, 0], [0, 21, 5, 7, 3.5, 0], [0, 3, 37, 28, 10.5, 0], [0, 40, 30, 5.25, 7, 0],
                     [0, -3, -3, 7, 10.5, 0]], dtype=np.float32)
    for sr in (0, 1, 2):
        for r in rois:
            assert not rr.Roi(r, scale, 7, 7, sr, 20, 24).delta.any(), (r, sr)
        go = rng.standard_normal((len(rois), 4, 7, 7)).astype(np.float32)
        y, a, m, p = rr.forward([x], rois, [scale], [0] * len(rois), 7, 7, sr)
        (gref, ga, gm, gp), = rr.backward(go, [x.shape], rois, [scale], [0] * len(rois), 7, 7, sr)
        assert not p.any() and not gp.any()
        yo, go_ = _oracle_both(x, rois, scale, 7, 7, sr, go)
        rr.check(yo, y, a, m, p, what="oracle forward sr=%d" % sr)
        rr.check(go_, gref, ga, gm, gp, what="oracle backward sr=%d" % sr)


def test_empty_and_dead_grids():
    """Zero or negative sides at sampling_ratio 0, and a RoI without a level: no sample, zero output, no gradient."""
    for r in ([0, 40, 40, 0, 12, 10], [0, 40, 40, 12, 0, 10], [0, 40, 40, -12, 12, 10], [0, 40, 40, -1, -1, 10]):
        R = rr.Roi(np.float32(r), 0.25, 7, 7, 0, 20, 20)
        assert R.samples == 0 and R.W.nnz == 0, r
    R = rr.Roi(np.float32([0, 40, 40, 30, 30, 10]), 0.25, 7, 7, 2, 20, 20, dead=True)
    assert R.samples == 0 and R.W.nnz == 0
    R = rr.Roi(np.float32([0, 40, 40, -12, 12, 10]), 0.25, 7, 7, 2, 20, 20)  # sr > 0: the mirrored grid is sampled
    assert R.samples == 4 and R.W.nnz > 0


# ------------------------------------------------------------------------------------------- path coverage
@pytest.mark.parametrize("sms", [132, 114])
def test_every_case_reaches_its_paths(sms):
    for case in CASES:
        got = path_labels(case, sms)
        assert case.labels <= got, (case.name, sms, sorted(case.labels - got))


def test_every_path_label_is_declared():
    declared = set().union(*(c.labels for c in CASES))
    assert declared == ALL_LABELS, (sorted(ALL_LABELS - declared), sorted(declared - ALL_LABELS))


def test_no_case_has_an_ambiguous_sample():
    """No sample within delta_s of y = -1, y = H, x = -1 or x = W, where the kernel and the reference may take different
    branches -- except at angle 0, where the positions are exact and the lattice hits are what the case is for."""
    for case in CASES:
        for r, _, R in roi_objects(case):
            if float(r[5]) == 0.0 and not R.delta.any():
                continue
            assert R.ambiguous == 0, (case.name, r)


def test_launch_examples():
    assert rr.pick_c_per_cta(4, 200, 132) == 13 and rr.pick_c_per_cta(4, 200, 114) == 13  # 16 slabs, the last of 5
    assert rr.pick_c_per_cta(600, 32, 132) == 32 and rr.pick_c_per_cta(8, 128, 132) == 16
    assert rr.slabs(132) == [(0, 128), (128, 4)]
    assert rr.nhwc_supported(16, [(48, 56)], 13, 23) and not rr.nhwc_supported(16, [(48, 56)], 20, 15)


def test_rotated_pooled_sizes_agree_with_the_library():
    """nhwc_supported restates nhwc_supported's D2B_ROI_ROTATED branch; d2b_roi_pooler_nhwc_supported is the library's."""
    from detectron2_b200 import _C, ops

    for ph in range(1, 41):
        for pw in range(1, 41):
            for flags in (_C.ROI_ROTATED, _C.ROI_ROTATED | _C.ROI_BACKWARD):
                lib = ops._nhwc_supported(8, ((64, 64),), ph, pw, flags)
                assert lib == rr.nhwc_supported(8, [(64, 64)], ph, pw), (ph, pw, flags)
    assert not ops._nhwc_supported(6, ((64, 64),), 7, 7, _C.ROI_ROTATED) and not rr.nhwc_supported(6, [(64, 64)], 7, 7)
    for setting, cl, want in (("nchw", True, "nchw"), ("nhwc", False, "xpose"), ("nhwc", True, "cl")):
        assert rr.pick_layout(setting, 8, [(64, 64)], 7, 7, cl) == want
    assert rr.pick_layout("nhwc", 8, [(64, 64)], 20, 15, True) == "nchw"
