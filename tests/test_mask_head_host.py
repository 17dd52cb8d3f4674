"""CPU checks of tests/mask_loss_ref.py and of the case table of tests/test_mask_head_gpu.py: the float64 reference pinned to
known answers and to the real BitMasks.crop_and_resize (tests/golden/postprocessing.npz); every case reaching the edges it
declares, with dyadic geometry; ground-truth masks of every dtype read as BitMasks reads them on the CPU host path."""
import numpy as np
import torch

import mask_loss_ref as mr
from test_host_logic_cpu import _OracleROIAlign
from test_mask_head_gpu import CASES, _inputs, dtype_case, edge_labels, encodings
from test_roi_align_column_walk import sample_pos

ALL_LABELS = {
    "passes1", "bins256", "passes4_ragged", "passes4_full", "inside", "cut_left", "cut_top", "cut_right", "cut_bottom",
    "outside", "zero_size", "grid_negative", "subpixel", "grid9", "large_offmap", "mask_h1", "mask_w1", "pos_-1", "pos_0",
    "pos_H-1", "pos_H", "half", "below_half", "odd_hw", "image_sizes", "empty_image_middle", "shared_mask",
    "per_proposal_masks", "C1", "C80", "C1203", "class0", "classC-1", "logit_30", "logit_88",
}


def test_cases_reach_their_edges():
    reached = set()
    for case in CASES:
        got = edge_labels(case)
        assert case.labels <= got, (case.name, case.labels - got)
        assert {"logit_30", "logit_88"} <= got, case.name
        reached |= got
    assert reached == ALL_LABELS, reached ^ ALL_LABELS


def test_case_geometry_is_dyadic():
    """Every sample position of every case is the same in fp32 and in float64, on a 1/16-pixel lattice, and the sampling
    grid has at most 4096 samples: the weight products are multiples of 2^-8 and every fp32 partial sum is exact."""
    for case in CASES:
        for ref in _inputs(case.name)[5]:
            for R in ref.rois:
                g = R.g
                assert g.count <= 4096
                for start, size, grid in ((g.start_h, g.bin_h, g.gh), (g.start_w, g.bin_w, g.gw)):
                    for p in range(case.s):
                        for i in range(grid):
                            v = sample_pos(start, size, grid, p, i, True)
                            assert v == sample_pos(start, size, grid, p, i) and v * 16 == int(v * 16), (case.name, v)


def test_reference_known_answers():
    # one 1 x 1 bin, one sample at (y, x) = (1.5, 1.125): rows 1, 2 weigh 1/2 each, columns 1, 2 weigh 7/8 and 1/8
    gt = np.zeros((3, 4, 4), np.uint8)
    gt[0, 1, 1] = 1                 # 7/16: one weight step (1/16) below 0.5 -> 0
    gt[1, 1, 1] = gt[1, 1, 2] = 1   # exactly 0.5 -> 1
    gt[2, 2, 1] = gt[2, 2, 2] = 1   # exactly 0.5 from the other row
    box = [[1.125, 1.5, 2.125, 2.5]] * 4
    r = mr.targets(gt, box, [0, 1, 2, 3], 1)
    assert r.v[:3, 0, 0].tolist() == [7 / 16, 0.5, 0.5] and r.t[:, 0, 0].tolist() == [False, True, True, False]
    # a 2 x 2 sampling grid (bin 2) on integer positions: count 4; a float mask with 0.25 and 255 entries reads as 0 / 1
    big = np.zeros((1, 8, 8))
    big[0, 2, 2:4] = 0.25
    big[0, 4, 4] = 255
    r = mr.targets(big, [[2.0, 2.0, 6.0, 6.0]], None, 2)
    assert r.v[0].tolist() == [[0.5, 0.0], [0.0, 0.25]] and r.t[0].tolist() == [[True, False], [False, False]]
    # loss and gradient: x = 0 gives log 2 per bin and (1/2 - t) scale; +-88 stay finite (terms of about e^-88)
    t = np.array([[[1.0, 0.0], [1.0, 0.0]]])
    lg = np.zeros((1, 2, 2, 2))
    lg[0, 1] = [[0.0, 0.0], [88.0, -88.0]]
    loss, tol = mr.loss_per_roi(lg, t, [1])
    assert np.isclose(loss[0], 2 * np.log(2), rtol=1e-15, atol=0)
    assert tol[0] == (1 + 5 + 8 + 8) * mr.EPS32 * (loss[0] + 4)
    g, gtol = mr.grad(lg, t, [1], 0.25)
    assert (g[0, 0] == 0).all() and g[0, 1, 0].tolist() == [-0.125, 0.125] and abs(g[0, 1, 1, 0]) <= 1e-38
    assert np.isclose(g[0, 1, 1, 1], 0.25 * np.exp(-88.0), rtol=1e-14, atol=0)
    assert gtol[0] == mr.EPS32
    # a class outside [0, C) contributes nothing
    assert mr.loss_per_roi(lg, t, [2])[0][0] == 0 and (mr.grad(lg, t, [-1], 0.25)[0] == 0).all()


def test_reference_reproduces_bitmasks_crop_and_resize(golden):
    """The fixture's crops were made by the reference's BitMasks.crop_and_resize (torchvision roi_align on the CPU) on
    non-dyadic boxes: the float64 targets equal them except at bins within the bound of 0.5."""
    d = golden("postprocessing")
    ref = mr.targets(d["bit_masks"], d["crop_boxes"], None, int(d["mask_size"]))
    crops = d["crops"]
    assert crops.shape == ref.t.shape
    assert not ((crops != ref.t) & ~ref.near).any()
    assert ref.near.sum() <= 4 and ref.t.any() and not ref.t.all()


def test_crop_and_resize_reads_gt_as_bitmasks_host(monkeypatch):
    """crop_and_resize on CPU tensors (the oracle's RoIAlign): bool, uint8 {0, 1, 255} and float {0, 0.25, 0.5, 1} ground
    truth give the reference's targets."""
    from detectron2_b200 import postprocessing as pp

    monkeypatch.setattr(pp, "ROIAlign", _OracleROIAlign)
    g, gt, b, mi, t_ref = dtype_case()
    for name, m in encodings(gt, g).items():
        assert np.array_equal(pp.crop_and_resize(m[mi], b, 14).numpy(), t_ref), name
