"""Rotated RRPN proposal selection and rotated Fast R-CNN inference, on CPU: the oracle restatements and the product's host
logic against the fixtures from the REAL reference functions (tests/golden/make_golden_rotated.py), the training failure
mode and thresholds that IoU 0 passes."""
import pytest
import torch

import rotated_inference_ref as rref
from oracle import oracle as orc

T = torch.from_numpy


def oracle_nms_fixed_rotated(boxes, scores, idxs, iou_threshold, rotated, apply_offsets=True, max_segment=0):
    """Same contract as detectron2_b200.ops.nms_fixed for the rotated calls (padded keep buffer + count), computed by the
    CPU oracle: D2B_NMS_NO_OFFSET, idxs are pure segment ids, -1 = ignored."""
    assert rotated and not apply_offsets
    boxes, scores = boxes.float().contiguous(), scores.float().contiguous()
    m = boxes.shape[0]
    parts = []
    for c in torch.unique(idxs):
        if c < 0:
            continue
        ii = torch.nonzero(idxs == c, as_tuple=True)[0]
        assert max_segment <= 0 or len(ii) <= max_segment, "caller's max_segment bound violated"
        parts.append(ii[orc.nms_rotated(boxes[ii], scores[ii], iou_threshold)])
    kept = torch.cat(parts).sort().values if parts else torch.zeros(0, dtype=torch.int64)
    kept = kept[torch.sort(scores[kept], descending=True, stable=True).indices]  # score order, lower index first on ties
    keep = torch.zeros(m, dtype=torch.int64)
    keep[: kept.numel()] = kept
    return keep, torch.tensor([kept.numel()], dtype=torch.int64)


@pytest.fixture()
def cpu_nms(monkeypatch):
    from detectron2_b200 import ops

    monkeypatch.setattr(ops, "nms_fixed", oracle_nms_fixed_rotated)


def rrpn_fixture(golden):
    d = golden("rrpn_proposals")
    thr, pre, post, mbs = float(d["cfg"][0]), int(d["cfg"][1]), int(d["cfg"][2]), float(d["cfg"][3])
    sizes = [tuple(int(v) for v in r) for r in d["sizes"]]
    nl = len(d["per_level"])
    props = [T(d[f"props{l}"]) for l in range(nl)]
    logits = [T(d[f"logits{l}"]) for l in range(nl)]
    return d, props, logits, sizes, thr, pre, post, mbs


def frcnn_fixture(golden):
    d = golden("rotated_fast_rcnn_inference")
    thr, nms_thr, topk = float(d["cfg"][0]), float(d["cfg"][1]), int(d["cfg"][2])
    shapes = [tuple(int(v) for v in r) for r in d["shapes"]]
    return d, thr, nms_thr, topk, shapes


def check_frcnn(d, i, tag, boxes, scores, classes, rows):
    assert torch.equal(boxes.cpu(), T(d[f"out_boxes{i}{tag}"])), (i, tag)
    assert torch.equal(scores.cpu(), T(d[f"out_scores{i}{tag}"])), (i, tag)
    assert torch.equal(classes.cpu(), T(d[f"out_classes{i}{tag}"])), (i, tag)
    assert torch.equal(rows.cpu(), T(d[f"out_rows{i}{tag}"])), (i, tag)


def test_fixture_inputs_cover_the_edge_cases(golden):
    d, props, logits, sizes, thr, pre, post, mbs = rrpn_fixture(golden)
    assert len(props) >= 3 and len(sizes) == 2
    assert not torch.isfinite(props[0]).all() and not torch.isfinite(logits[1]).all()
    out = torch.cat([T(d["boxes_img0"]), T(d["boxes_img1"])])
    for a in (1.0, -1.0, 179.5, -90.0, 170.0, -180.0, 180.0):  # 270 -> -90, -190 -> 170, 540 -> -180, -180.00002 -> 180
        assert (out[:, 4] == a).any(), a
    assert (out[:, 4].abs() == 180.0).any() and (out[:, :2] < 0).any()
    f, *_ = frcnn_fixture(golden)
    assert f["out_boxes2"].shape[0] == 0 and f["boxes1"].shape[1] == 5 and f["boxes0"].shape[1] == 30


def test_rrpn_oracle_restatement_matches_reference(golden):
    d, props, logits, sizes, thr, pre, post, mbs = rrpn_fixture(golden)
    res = rref.find_top_rrpn_proposals(props, logits, sizes, thr, pre, post, mbs, False)
    for i, (b, s) in enumerate(res):
        assert torch.equal(b, T(d[f"boxes_img{i}"])), i
        assert torch.equal(s, T(d[f"scores_img{i}"])), i


def test_rotated_fast_rcnn_oracle_restatement_matches_reference(golden):
    d, thr, nms_thr, topk, shapes = frcnn_fixture(golden)
    for i in range(3):
        for tk, tag in ((topk, ""), (-1, "_all")):
            out = rref.fast_rcnn_inference_single_image_rotated(T(d[f"boxes{i}"]), T(d[f"scores{i}"]), shapes[i], thr,
                                                                nms_thr, tk)
            check_frcnn(d, i, tag, *out)


def test_rrpn_host_logic(golden, cpu_nms):
    from detectron2_b200.rrpn import find_top_rrpn_proposals

    d, props, logits, sizes, thr, pre, post, mbs = rrpn_fixture(golden)
    res = find_top_rrpn_proposals(props, logits, sizes, thr, pre, post, mbs, False)
    for i, r in enumerate(res):
        assert r.image_size == sizes[i]
        assert torch.equal(r.proposal_boxes.tensor, T(d[f"boxes_img{i}"])), i
        assert torch.equal(r.objectness_logits, T(d[f"scores_img{i}"])), i
    with pytest.raises(FloatingPointError):
        find_top_rrpn_proposals(props, logits, sizes, thr, pre, post, mbs, True)
    with pytest.raises(FloatingPointError):
        rref.find_top_rrpn_proposals(props, logits, sizes, thr, pre, post, mbs, True)


def test_rotated_fast_rcnn_host_logic(golden, cpu_nms):
    from detectron2_b200 import rotated_fast_rcnn as rfr

    d, thr, nms_thr, topk, shapes = frcnn_fixture(golden)
    for tk, tag in ((topk, ""), (-1, "_all")):
        # class-specific images in one call (image 0 twice, image 2 has no candidate), class-agnostic alone
        res, rows = rfr.fast_rcnn_inference_rotated([T(d["boxes0"]), T(d["boxes2"]), T(d["boxes0"])],
                                                    [T(d["scores0"]), T(d["scores2"]), T(d["scores0"])],
                                                    [shapes[0], shapes[2], shapes[0]], thr, nms_thr, tk)
        for j, i in enumerate([0, 2, 0]):
            check_frcnn(d, i, tag, res[j].pred_boxes, res[j].scores, res[j].pred_classes, rows[j])
        det, rows1 = rfr.fast_rcnn_inference_single_image_rotated(T(d["boxes1"]), T(d["scores1"]), shapes[1], thr, nms_thr, tk)
        check_frcnn(d, 1, tag, det.pred_boxes, det.scores, det.pred_classes, rows1)


@pytest.mark.parametrize("nms_thr", [0.0, -0.5])
def test_thresholds_that_iou_zero_passes(golden, cpu_nms, nms_thr):
    """thr <= 0: the reference's single NMS over the offset boxes suppresses across levels / classes too."""
    from detectron2_b200 import rotated_fast_rcnn as rfr
    from detectron2_b200.rrpn import find_top_rrpn_proposals

    d, props, logits, sizes, _, pre, post, mbs = rrpn_fixture(golden)
    ref = rref.find_top_rrpn_proposals(props, logits, sizes, nms_thr, pre, post, mbs, False)
    res = find_top_rrpn_proposals(props, logits, sizes, nms_thr, pre, post, mbs, False)
    for r, (b, s) in zip(res, ref):
        assert torch.equal(r.proposal_boxes.tensor, b) and torch.equal(r.objectness_logits, s)
    f, thr, _, topk, shapes = frcnn_fixture(golden)
    res, rows = rfr.fast_rcnn_inference_rotated([T(f["boxes0"]), T(f["boxes2"])], [T(f["scores0"]), T(f["scores2"])],
                                                [shapes[0], shapes[2]], thr, nms_thr, -1)
    ref = rref.fast_rcnn_inference_rotated([T(f["boxes0"]), T(f["boxes2"])], [T(f["scores0"]), T(f["scores2"])],
                                           [shapes[0], shapes[2]], thr, nms_thr, -1)
    for j, (b, s, c, rw) in enumerate(ref):
        assert len(b) == (1 if j == 0 else 0)  # every candidate of the image meets the first with IoU >= 0
        assert torch.equal(res[j].pred_boxes, b) and torch.equal(res[j].scores, s)
        assert torch.equal(res[j].pred_classes, c) and torch.equal(rows[j], rw)


def test_clip_rotated_matches_reference_clip():
    from detectron2_b200.rrpn import clip_rotated

    g = torch.Generator().manual_seed(3)
    b = torch.cat([torch.rand(4000, 2, generator=g) * 300 - 50, torch.rand(4000, 2, generator=g) * 80,
                   (torch.rand(4000, 1, generator=g) - 0.5) * 1500], 1)
    b[:8, 4] = torch.tensor([1.0, -1.0, 1.0001, -180.00002, 179.99998, 540.0, -540.0, -0.0])
    b[8:2000, 4] = (torch.rand(1992, generator=g) - 0.5) * 4
    ref = rref.clip_(b.clone(), (150, 200))
    assert torch.equal(clip_rotated(b, 150.0, 200.0), ref)
    assert ref[3, 4] == 180.0  # -180.00002 normalises to +180
