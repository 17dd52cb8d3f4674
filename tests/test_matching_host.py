"""Anchor / proposal matching on CPU: the host restatement (detectron2_b200.matching) against the fixture from the REAL
reference functions (tests/golden/make_golden_matching.py), including the sampled indices under the same CPU seed, the
reference's AssertionError on invalid IoUs, the fixture's edge-case coverage and the argument checks of d2b_match_boxes
(no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import oracle as orc

T = torch.from_numpy
RPN_CFG = ([0.3, 0.7], [0, -1, 1], True)
RETINA_CFG = ([0.4, 0.5], [0, -1, 1], True)
ROI_CFG = ([0.5], [0, 1], False)
NIMG = 4  # images of the fixture


@pytest.fixture()
def cpu_rotated_iou(monkeypatch):
    from detectron2_b200 import ops

    monkeypatch.setattr(ops, "box_iou_rotated_op", orc.box_iou_rotated)


def load(golden):
    d = golden("matching")
    sizes = [tuple(int(v) for v in r) for r in d["sizes"]]
    gts = [T(d[f"gt{i}"]) for i in range(NIMG)]
    cls = [T(d[f"cls{i}"]) for i in range(NIMG)]
    rgts = [T(d[f"rgt{i}"]) for i in range(NIMG)]
    rcls = [T(d[f"rcls{i}"]) for i in range(NIMG)]
    return d, sizes, gts, cls, rgts, rcls


def eq(a, b, what):
    a, b = a.cpu(), torch.as_tensor(b)
    assert a.dtype == b.dtype and torch.equal(a, b), what


def check_deterministic(d, device):
    """The outputs that do not depend on the RNG, computed on `device`: Matcher (both configs), RetinaNet, cascade (three
    stages), and the matched boxes of RPN / RRPN."""
    from detectron2_b200 import matching as mt

    _, sizes, gts, cls, rgts, rcls = load(lambda n: d)
    dv = lambda ts: [t.to(device) for t in ts]  # noqa: E731
    anchors = T(d["anchors"]).to(device)
    for tag, cfg in (("rpn", RPN_CFG), ("roi", ROI_CFG)):
        for i, g in enumerate(dv(gts)):
            m, lab = mt.Matcher(*cfg)(mt.pairwise_iou(g, anchors))
            eq(m, T(d[f"matcher_{tag}_matches{i}"]), (tag, i))
            eq(lab, T(d[f"matcher_{tag}_labels{i}"]), (tag, i))
    labels, boxes = mt.retinanet_label_anchors([anchors], dv(gts), dv(cls), mt.Matcher(*RETINA_CFG), 5)
    for i in range(NIMG):
        eq(labels[i], T(d[f"retina_labels{i}"]), ("retina", i))
        eq(boxes[i], T(d[f"retina_boxes{i}"]), ("retina boxes", i))
    props = dv([T(d[f"props{i}"]) for i in range(NIMG)])
    for stage, t in enumerate((0.5, 0.6, 0.7)):
        res = mt.cascade_match_and_label_boxes(props, dv(gts), dv(cls), mt.Matcher([t], [0, 1], False), 5)
        for i, (c, b) in enumerate(res):
            eq(c, T(d[f"cascade{stage}_classes{i}"]), ("cascade", stage, i))
            eq(b, T(d[f"cascade{stage}_boxes{i}"]), ("cascade boxes", stage, i))


def mutated_labels(iou, thresholds, labels, double=False, ties=True):
    """Matcher labels from an IoU matrix, with the threshold compares in fp32 (the rule) or in double, and the low-quality
    matches with ties (the rule) or with the first prediction per GT only."""
    vals = iou.max(dim=0).values
    vals = vals.double() if double else vals
    out = torch.ones(vals.shape, dtype=torch.int8)
    th = [-float("inf")] + list(thresholds) + [float("inf")]
    for l, lo, hi in zip(labels, th[:-1], th[1:]):
        out[(vals >= lo) & (vals < hi)] = l
    best = iou.max(dim=1).values
    idx = torch.nonzero(iou == best[:, None], as_tuple=True)[1] if ties else iou.argmax(dim=1)
    out[idx] = 1
    return out


def test_fixture_inputs_cover_the_edge_cases(golden):
    d, sizes, gts, cls, rgts, rcls = load(golden)
    iou = T(d["matcher_rpn_iou0"])
    fixture = T(d["matcher_rpn_labels0"])
    # duplicate GT boxes: argmax ties go to the first
    assert torch.equal(gts[0][1], gts[0][2]) and torch.equal(rgts[0][0], rgts[0][1])
    assert torch.equal(iou[1], iou[2]) and (iou[1] > 0).any()
    assert not (T(d["matcher_rpn_matches0"]) == 2).any() and (T(d["matcher_rpn_matches0"]) == 1).any()
    # image 0 is not saturated by the all-positive quirk: every GT overlaps something, and each label value occurs
    assert (iou.max(dim=1).values > 0).all()
    assert all((fixture == v).any() for v in (-1, 0, 1))
    # a GT whose maximum IoU > 0 is shared by two predictions: both get the low-quality match
    best = iou.max(dim=1).values
    tied = (iou == best[:, None]).sum(dim=1)
    assert ((tied >= 2) & (best > 0)).any()
    # IoUs at float32(thr) and one ulp either side, for every threshold
    vals = set(iou[0].numpy().tolist())
    for t in (0.3, 0.4, 0.5, 0.6, 0.7):
        t32 = np.float32(t)
        for v in (np.nextafter(t32, np.float32(-1)), t32, np.nextafter(t32, np.float32(2))):
            assert float(v) in vals, (t, v)
    # the labels pin the two rules: fp32 threshold compares (float32(0.7) < 0.7 in double) and low-quality ties
    assert torch.equal(mutated_labels(iou, *RPN_CFG[:2]), fixture)
    assert not torch.equal(mutated_labels(iou, *RPN_CFG[:2], double=True), fixture)
    assert not torch.equal(mutated_labels(iou, *RPN_CFG[:2], ties=False), fixture)
    # a zero-area GT overlaps nothing: its maximum is 0, so every prediction at IoU 0 to it is positive (image 3)
    z = gts[3][(gts[3][:, 2] - gts[3][:, 0]) * (gts[3][:, 3] - gts[3][:, 1]) == 0]
    assert len(z) and (T(d["matcher_rpn_labels3"]) == 1).all()
    assert (rgts[3][:, 2] * rgts[3][:, 3] == 0).any() and not (rgts[0][:, 2] * rgts[0][:, 3] == 0).any()
    # an image without GT, and the boundary rule changing labels
    assert len(gts[2]) == 0 and len(rgts[2]) == 0
    assert not torch.equal(T(d["rpn_b0_labels1"]), T(d["rpn_b1_labels1"]))
    assert d["bad_xyxy_inf_raised"] == 1 and d["bad_rot_nan_raised"] == 1
    assert d["bad_rot_negative_iou_raised"] == 1 and (T(d["bad_rot_negative_iou_iou"]) < 0).any()


def test_host_restatement_matches_reference(golden, cpu_rotated_iou):
    d = golden("matching")
    check_deterministic(d, "cpu")


def test_host_sampling_matches_reference_under_the_same_seed(golden, cpu_rotated_iou):
    from detectron2_b200 import matching as mt

    d, sizes, gts, cls, rgts, rcls = load(golden)
    anchors = T(d["anchors"])
    for bt in (-1, 0):
        torch.manual_seed(7)
        labels, boxes = mt.rpn_label_and_sample_anchors([anchors[:400], anchors[400:]], gts, sizes, mt.Matcher(*RPN_CFG),
                                                        bt, 64, 0.5)
        for i in range(NIMG):
            eq(labels[i], T(d[f"rpn_b{bt + 1}_labels{i}"]), ("rpn", bt, i))
            eq(boxes[i], T(d[f"rpn_b{bt + 1}_boxes{i}"]), ("rpn boxes", bt, i))
    torch.manual_seed(13)
    labels, boxes = mt.rpn_label_and_sample_anchors(T(d["ranchors"]), rgts, sizes, mt.Matcher(*RPN_CFG), -1, 64, 0.5)
    for i in range(NIMG):
        eq(labels[i], T(d[f"rrpn_labels{i}"]), ("rrpn", i))
        eq(boxes[i], T(d[f"rrpn_boxes{i}"]), ("rrpn boxes", i))
    for seed, pk, gk, ck, tag in ((11, "props", gts, cls, "roi"), (17, "rprops", rgts, rcls, "rroi")):
        props = [T(d[f"{pk}{i}"]) for i in range(NIMG)]
        torch.manual_seed(seed)
        res = mt.label_and_sample_proposals(props, gk, ck, mt.Matcher(*ROI_CFG), 5, 64, 0.25)
        check_sampled_proposals(d, tag, props, gk, res)


def check_sampled_proposals(d, tag, props, gts, res):
    for i, (idx, c, m) in enumerate(res):
        allb = torch.cat([props[i], gts[i].to(props[i].dtype)])
        eq(allb[idx.cpu()], T(d[f"{tag}_props{i}"]), (tag, i))
        eq(c, T(d[f"{tag}_classes{i}"]), (tag, "classes", i))
        if len(gts[i]):
            eq(gts[i][m.cpu()], T(d[f"{tag}_gtboxes{i}"]), (tag, "gt boxes", i))


def test_invalid_iou_raises_assertion_error(golden, cpu_rotated_iou):
    from detectron2_b200 import matching as mt

    d = golden("matching")
    for k in ("xyxy_inf", "rot_nan", "rot_negative", "rot_negative_iou"):
        gt, pred = T(d[f"bad_{k}_gt"]), T(d[f"bad_{k}_pred"])
        raised = 0
        try:
            mt.Matcher(*RPN_CFG)(mt._iou(gt, pred))
        except AssertionError:
            raised = 1
        assert raised == int(d[f"bad_{k}_raised"]), k
        if raised:
            with pytest.raises(AssertionError):
                mt.retinanet_label_anchors(pred, [gt], [torch.zeros(1, dtype=torch.int64)], mt.Matcher(*RETINA_CFG), 3)


def test_rrpn_refuses_the_boundary_rule(cpu_rotated_iou):
    """RRPN.__init__ raises for anchor_boundary_thresh >= 0 (proposal_generator/rrpn.py:139-142)."""
    from detectron2_b200 import matching as mt

    anchors = torch.tensor([[10.0, 10.0, 4.0, 4.0, 0.0]])
    with pytest.raises(NotImplementedError):
        mt.rpn_label_and_sample_anchors(anchors, [anchors], [(20, 20)], mt.Matcher(*RPN_CFG), 0, 8, 0.5)


def test_matcher_constructor_assertions():
    from detectron2_b200 import matching as mt

    for thr, lab in (([0.0], [0, 1]), ([0.7, 0.3], [0, -1, 1]), ([0.5], [0, 2]), ([0.5], [0, 1, 1])):
        with pytest.raises(AssertionError):
            mt.Matcher(thr, lab)


def test_match_boxes_rejects_bad_arguments():
    """Every argument is checked before the first CUDA call: these return D2B_EINVAL without a GPU."""
    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL = -1
    p = C.c_void_p(16)  # never dereferenced: the checks fail first
    ws = 1 << 20
    names = ["gt", "gt_count", "N", "Gmax", "pred", "stride", "pred_count", "Pmax", "thr", "nthr", "lab", "flags", "hw",
             "bthr", "gt_classes", "num_classes", "matches", "labels", "boxes", "classes", "status", "ws", "ws_bytes",
             "stream"]
    thr2 = (C.c_double * 2)(0.3, 0.7)
    lab3 = (C.c_int * 3)(0, -1, 1)
    good = [p, p, 2, 5, p, 0, None, 100, thr2, 2, lab3, _C.MATCH_LOW_QUALITY, None, -1.0, None, 0, p, p, p, None, p, p, ws,
            None]

    def call(**over):
        a = list(good)
        for k, v in over.items():
            a[names.index(k)] = v
        return lib.d2b_match_boxes(*a)

    assert lib.d2b_match_workspace_bytes(2, 5, 100) <= ws
    bad = [dict(nthr=0), dict(nthr=9), dict(thr=None), dict(lab=None), dict(thr=(C.c_double * 2)(0.0, 0.7)),
           dict(thr=(C.c_double * 2)(0.7, 0.3)), dict(thr=(C.c_double * 2)(float("nan"), 0.7)),
           dict(lab=(C.c_int * 3)(0, 2, 1)), dict(lab=(C.c_int * 3)(0, -2, 1)), dict(flags=8), dict(N=-1),
           dict(N=65536), dict(Gmax=-1), dict(Pmax=-1), dict(stride=50), dict(bthr=0.0),
           dict(bthr=0.0, flags=_C.MATCH_ROTATED), dict(gt_count=None), dict(matches=None), dict(labels=None),
           dict(status=None), dict(ws=None), dict(gt=None), dict(pred=None), dict(classes=p), dict(ws_bytes=16)]
    for over in bad:
        assert call(**over) == EINVAL, over
