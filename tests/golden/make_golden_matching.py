"""Generate tests/golden/matching.npz from the REAL reference functions: Matcher (modeling/matcher.py), pairwise_iou
(structures/boxes.py), RPN.label_and_sample_anchors (proposal_generator/rpn.py:307-363), RetinaNet.label_anchors
(meta_arch/retinanet.py:213-255), ROIHeads.label_and_sample_proposals (roi_heads/roi_heads.py:220-302),
CascadeROIHeads._match_and_label_boxes (roi_heads/cascade_rcnn.py:209-256), RRPN.label_and_sample_anchors
(proposal_generator/rrpn.py:151-195) and RROIHeads.label_and_sample_proposals (roi_heads/rotated_fast_rcnn.py:218-270).

Run in the authoring container only (needs /root/reference and oracle/_ref, like make_golden.py):
    python tests/golden/make_golden_matching.py
It writes only this file.  The modules are imported with the stubs of make_golden_rotated.py plus permissive stubs for their
unrelated dependencies; the methods run on a stand-in `self` that carries the attributes they read.  The rotated IoU is the
reference CPU csrc compiled in oracle/_ref.  Sampling uses the reference's subsample_labels with a seeded CPU RNG.
"""
import functools
import math
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402
import make_golden_rotated as mgr  # noqa: E402

REF = "/root/reference/detectron2"


class _Auto(types.ModuleType):
    """A module whose every missing attribute is a do-nothing class (usable as a base class, a Registry, a decorator)."""

    def __getattr__(self, k):
        if k.startswith("__"):
            raise AttributeError(k)
        v = type(k, (), {"__init__": lambda self, *a, **kw: None, "register": lambda *a, **kw: (lambda o: o)})
        setattr(self, k, v)
        return v


def _auto(name):
    m = _Auto(name)
    m.__path__ = []
    sys.modules[name] = m
    return m


class _Storage:
    def put_scalar(self, *a, **k):
        pass


def import_reference():
    mgr._import_reference_rotated()  # fast_rcnn stubs, structures, rrpn + rotated_fast_rcnn modules
    sys.modules["detectron2.utils.events"].get_event_storage = lambda: _Storage()
    sys.modules["fvcore.nn"].sigmoid_focal_loss_jit = None
    for name in ("detectron2.utils.registry", "detectron2.modeling.anchor_generator", "detectron2.modeling.backbone",
                 "detectron2.modeling.backbone.resnet", "detectron2.modeling.meta_arch.build",
                 "detectron2.modeling.meta_arch.dense_detector", "detectron2.modeling.roi_heads.keypoint_head",
                 "detectron2.modeling.roi_heads.mask_head", "detectron2.modeling.poolers"):
        _auto(name)
    ma = _auto("detectron2.modeling.meta_arch")
    ma.__path__ = []
    sys.modules["detectron2.modeling.box_regression"]._dense_box_regression_loss = None
    sys.modules["detectron2.modeling.roi_heads.fast_rcnn"].fast_rcnn_inference = None
    matcher = mgr._load("detectron2.modeling.matcher", REF + "/modeling/matcher.py")
    sampling = mgr._load("detectron2.modeling.sampling", REF + "/modeling/sampling.py")
    pu = mgr._load("detectron2.modeling.proposal_generator.proposal_utils",
                   REF + "/modeling/proposal_generator/proposal_utils.py")
    rpn = mgr._load("detectron2.modeling.proposal_generator.rpn", REF + "/modeling/proposal_generator/rpn.py")
    ret = mgr._load("detectron2.modeling.meta_arch.retinanet", REF + "/modeling/meta_arch/retinanet.py")
    rh = mgr._load("detectron2.modeling.roi_heads.roi_heads", REF + "/modeling/roi_heads/roi_heads.py")
    casc = mgr._load("detectron2.modeling.roi_heads.cascade_rcnn", REF + "/modeling/roi_heads/cascade_rcnn.py")
    rrpn = mgr._load("detectron2.modeling.proposal_generator.rrpn", REF + "/modeling/proposal_generator/rrpn.py")
    rfr = mgr._load("detectron2.modeling.roi_heads.rotated_fast_rcnn", REF + "/modeling/roi_heads/rotated_fast_rcnn.py")
    assert rh.add_ground_truth_to_proposals is pu.add_ground_truth_to_proposals
    return types.SimpleNamespace(Matcher=matcher.Matcher, sampling=sampling, rpn=rpn, ret=ret, rh=rh, casc=casc, rrpn=rrpn,
                                 rfr=rfr)


def _self(**attrs):
    return types.SimpleNamespace(**attrs)


def probe_boxes(ref_iou, thresholds):
    """Anchors (0, 0, w, h) against the GT (0, 0, 10, 10) whose reference IoU is float32(t) and one ulp below and above
    it, for every threshold t.  Several heights h (inside the GT and a little taller) give several roundings of the
    intersection and the union, so that every neighbour is hit."""
    gt = torch.tensor([[0.0, 0.0, 10.0, 10.0]])
    out = []
    for t in thresholds:
        t32 = np.float32(t)
        want = [np.nextafter(t32, np.float32(-1)), t32, np.nextafter(t32, np.float32(2))]
        found = {}
        for h in (10.0, 9.5, 9.0, 8.5, 8.0, 7.5, 7.0, 6.5, 10.5, 11.0, 11.5):
            base = np.float32(100 * t / h if h <= 10 else 100 * t / (10 + 10 * t - t * h))
            cand = torch.tensor([float(base + np.float32(k) * np.spacing(base)) for k in range(-300, 301)],
                                dtype=torch.float32)
            a = torch.stack([torch.zeros_like(cand), torch.zeros_like(cand), cand, torch.full_like(cand, h)], 1)
            iou = ref_iou(gt, a)[0].numpy()
            for j, w_ in enumerate(want):
                hit = np.nonzero(iou == w_)[0]
                if j not in found and len(hit):
                    found[j] = [0.0, 0.0, float(cand[hit[0]]), h]
        assert len(found) == 3, (t, found)
        out += [found[j] for j in range(3)]
    return torch.tensor(out)


# Regions kept free of random boxes: the threshold probes around the GT (0, 0, 10, 10), and the GT (100, 80, 120, 100)
# whose maximum IoU (320 / 480) is shared by two translated anchors.
ZONES = torch.tensor([[0.0, 0.0, 12.0, 12.0], [88.0, 70.0, 132.0, 110.0]])


def outside_zones(b):
    z = ZONES
    apart = ((b[:, None, 2] <= z[:, 0]) | (b[:, None, 0] >= z[:, 2]) | (b[:, None, 3] <= z[:, 1]) | (b[:, None, 1] >= z[:, 3]))
    return b[apart.all(dim=1)]


def xyxy_scene(g, n_rand, size):
    h, w = size
    ctr = torch.rand(n_rand, 2, generator=g) * torch.tensor([w + 40.0, h + 40.0]) - 20
    wh = torch.rand(n_rand, 2, generator=g) * 60 + 2
    return outside_zones(torch.cat([ctr - wh / 2, ctr + wh / 2], 1))


def main():
    torch.set_num_threads(1)
    R = import_reference()
    from detectron2.structures import Boxes, Instances, RotatedBoxes, pairwise_iou  # the reference's

    ref_iou = lambda a, b: pairwise_iou(Boxes(a), Boxes(b))  # noqa: E731
    out = {}
    g = torch.Generator().manual_seed(2024)
    size = (120, 160)
    probes = probe_boxes(ref_iou, [0.3, 0.4, 0.5, 0.6, 0.7])
    # anchors: random boxes, the threshold probes and a copy of their GT (IoU 1: the probe GT's low-quality match is not
    # a probe), the two tied anchors of the tie GT, boxes crossing the image border
    special = torch.tensor([[0.0, 0.0, 10.0, 10.0], [96.0, 80.0, 116.0, 100.0], [104.0, 80.0, 124.0, 100.0],
                            [-0.5, 5.0, 30.0, 40.0], [140.0, 60.0, 160.0, 69.0], [140.0, 60.0, 160.5, 69.0]])
    anchors = torch.cat([xyxy_scene(g, 900, size), probes, special])
    # image 0: the probe GT, a duplicated GT (argmax ties), the tie GT (low-quality ties), random GT
    gt0 = torch.cat([torch.tensor([[0.0, 0.0, 10.0, 10.0], [40.0, 30.0, 80.0, 70.0], [40.0, 30.0, 80.0, 70.0],
                                   [100.0, 80.0, 120.0, 100.0]]), xyxy_scene(g, 8, size)[:5]])
    gt1 = xyxy_scene(g, 3, size)
    gt2 = torch.zeros((0, 4))  # no GT
    gt3 = torch.cat([torch.tensor([[100.0, 20.0, 100.0, 50.0]]), xyxy_scene(g, 3, size)[:1]])  # zero-area GT: the quirk
    gts = [gt0, gt1, gt2, gt3]
    for b in (gt0, gt1):  # no GT of these images overlaps nothing, so their labels are not saturated by the quirk
        assert (ref_iou(b, anchors).max(dim=1).values > 0).all()
    cls = [torch.randint(0, 5, (len(x),), generator=g) for x in gts]
    sizes = [size, (100, 150), size, size]
    out.update(anchors=anchors, sizes=np.asarray(sizes), probes=probes)
    for i, (b, c) in enumerate(zip(gts, cls)):
        out[f"gt{i}"], out[f"cls{i}"] = b, c

    # Matcher with both configs, on the real pairwise_iou
    for tag, m in (("rpn", R.Matcher([0.3, 0.7], [0, -1, 1], True)), ("roi", R.Matcher([0.5], [0, 1], False))):
        for i, b in enumerate(gts):
            mq = ref_iou(b, anchors)
            mi, ml = m(mq)
            out[f"matcher_{tag}_iou{i}"] = mq if i == 0 else np.zeros(0)
            out[f"matcher_{tag}_matches{i}"], out[f"matcher_{tag}_labels{i}"] = mi, ml

    # RPN, with and without the boundary rule (seeded sampling)
    inst = [Instances(sz, gt_boxes=Boxes(b.clone()), gt_classes=c) for sz, b, c in zip(sizes, gts, cls)]
    for bt in (-1, 0):
        s = _self(anchor_matcher=R.Matcher([0.3, 0.7], [0, -1, 1], True), anchor_boundary_thresh=bt,
                  batch_size_per_image=64, positive_fraction=0.5)
        s._subsample_labels = functools.partial(R.rpn.RPN._subsample_labels, s)
        torch.manual_seed(7)
        labels, boxes = R.rpn.RPN.label_and_sample_anchors(s, [Boxes(anchors[:400]), Boxes(anchors[400:])], inst)
        for i in range(len(gts)):
            out[f"rpn_b{bt + 1}_labels{i}"], out[f"rpn_b{bt + 1}_boxes{i}"] = labels[i], boxes[i]

    # RetinaNet (deterministic)
    s = _self(anchor_matcher=R.Matcher([0.4, 0.5], [0, -1, 1], True), num_classes=5)
    labels, boxes = R.ret.RetinaNet.label_anchors(s, [Boxes(anchors)], inst)
    for i in range(len(gts)):
        out[f"retina_labels{i}"], out[f"retina_boxes{i}"] = labels[i], boxes[i]

    # ROI heads with proposal_append_gt (seeded sampling); proposals are anchors[:300] jittered per image
    props = [anchors[:300] + torch.randn(300, 4, generator=g) * 2 for _ in gts]
    for i, p in enumerate(props):
        out[f"props{i}"] = p
    s = _self(proposal_append_gt=True, proposal_matcher=R.Matcher([0.5], [0, 1], False), num_classes=5,
              batch_size_per_image=64, positive_fraction=0.25)
    s._sample_proposals = functools.partial(R.rh.ROIHeads._sample_proposals, s)
    pin = [Instances(sz, proposal_boxes=Boxes(p.clone()), objectness_logits=torch.arange(len(p), dtype=torch.float32))
           for sz, p in zip(sizes, props)]
    torch.manual_seed(11)
    res = R.rh.ROIHeads.label_and_sample_proposals(s, pin, inst)
    for i, r in enumerate(res):
        out[f"roi_props{i}"], out[f"roi_classes{i}"] = r.proposal_boxes.tensor, r.gt_classes
        out[f"roi_gtboxes{i}"] = r.gt_boxes.tensor if r.has("gt_boxes") else np.zeros((0, 4), np.float32)

    # Cascade, three stages (deterministic)
    s = _self(proposal_matchers=[R.Matcher([t], [0, 1], False) for t in (0.5, 0.6, 0.7)], num_classes=5)
    for stage in range(3):
        pin = [Instances(sz, proposal_boxes=Boxes(p.clone())) for sz, p in zip(sizes, props)]
        res = R.casc.CascadeROIHeads._match_and_label_boxes(s, pin, stage, inst)
        for i, r in enumerate(res):
            out[f"cascade{stage}_classes{i}"], out[f"cascade{stage}_boxes{i}"] = r.gt_classes, r.gt_boxes.tensor

    # rotated: RRPN anchors and RROI heads
    def rot(n):
        return mgr._rand_rotated(g, (n,), (-10.0, -10.0), (170.0, 130.0), 50.0)

    ranchors = torch.cat([rot(500), torch.tensor([[30.0, 30.0, 20.0, 10.0, 0.0], [30.0, 30.0, 20.0, 10.0, 90.0],
                                                  [30.0, 30.0, 20.0, 10.0, 45.0]])])
    rgt0 = torch.cat([torch.tensor([[30.0, 30.0, 20.0, 10.0, 0.0], [30.0, 30.0, 20.0, 10.0, 0.0]]), rot(4)])  # duplicate
    rgt3 = torch.cat([torch.tensor([[150.0, 10.0, 0.0, 8.0, 30.0]]), rot(1)])  # zero-area
    rgts = [rgt0, rot(2), torch.zeros((0, 5)), rgt3]
    rinst = [Instances(sz, gt_boxes=RotatedBoxes(b.clone()), gt_classes=c[: len(b)] if len(c) >= len(b) else
                       torch.randint(0, 5, (len(b),), generator=g)) for sz, b, c in zip(sizes, rgts, cls)]
    out["ranchors"] = ranchors
    for i, r in enumerate(rinst):
        out[f"rgt{i}"], out[f"rcls{i}"] = r.gt_boxes.tensor, r.gt_classes
    s = _self(anchor_matcher=R.Matcher([0.3, 0.7], [0, -1, 1], True), batch_size_per_image=64, positive_fraction=0.5)
    s._subsample_labels = functools.partial(R.rpn.RPN._subsample_labels, s)
    torch.manual_seed(13)
    labels, boxes = R.rrpn.RRPN.label_and_sample_anchors(s, [RotatedBoxes(ranchors)], rinst)
    for i in range(len(gts)):
        out[f"rrpn_labels{i}"], out[f"rrpn_boxes{i}"] = labels[i], boxes[i]
    rprops = [ranchors[:200] + torch.randn(200, 5, generator=g) * torch.tensor([2.0, 2.0, 1.0, 1.0, 3.0]) for _ in rgts]
    for p in rprops:
        p[:, 2:4] = p[:, 2:4].abs() + 0.5
    for i, p in enumerate(rprops):
        out[f"rprops{i}"] = p
    s = _self(proposal_append_gt=True, proposal_matcher=R.Matcher([0.5], [0, 1], False), num_classes=5,
              batch_size_per_image=64, positive_fraction=0.25)
    s._sample_proposals = functools.partial(R.rh.ROIHeads._sample_proposals, s)
    pin = [Instances(sz, proposal_boxes=RotatedBoxes(p.clone()), objectness_logits=torch.arange(len(p), dtype=torch.float32))
           for sz, p in zip(sizes, rprops)]
    torch.manual_seed(17)
    res = R.rfr.RROIHeads.label_and_sample_proposals(s, pin, rinst)
    for i, r in enumerate(res):
        out[f"rroi_props{i}"], out[f"rroi_classes{i}"] = r.proposal_boxes.tensor, r.gt_classes
        out[f"rroi_gtboxes{i}"] = r.gt_boxes.tensor if r.has("gt_boxes") else np.zeros((0, 5), np.float32)

    # invalid IoUs: the reference's assertion (1 = AssertionError)
    bad = {"xyxy_inf": (torch.tensor([[0.0, 0.0, math.inf, 10.0]]), torch.tensor([[0.0, 0.0, math.inf, 10.0], [0, 0, 5, 5.0]])),
           "rot_nan": (torch.tensor([[10.0, 10.0, math.nan, 5.0, 0.0]]), torch.tensor([[10.0, 10.0, 4.0, 5.0, 0.0]])),
           "rot_negative": (torch.tensor([[10.0, 10.0, -4.0, -5.0, 0.0]]), torch.tensor([[10.0, 10.0, 4.0, 5.0, 0.0],
                                                                                        [10.0, 10.0, -4.0, -5.0, 0.0]])),
           # a tiny box and a thin one: the reference's 1e-5 edge tolerance takes the thin box's far vertices as inside the
           # tiny one, the intersection polygon outgrows both areas and the IoU is negative
           "rot_negative_iou": (torch.tensor([[0.0, 0.0, 1e-3, 1e-3, 0.0]]),
                                torch.tensor([[0.0, 0.0, 0.015, 1e-4, 0.0], [5.0, 5.0, 2.0, 2.0, 0.0]]))}
    for k, (b1, b2) in bad.items():
        mq = ref_iou(b1, b2) if b1.shape[1] == 4 else R.rrpn.pairwise_iou_rotated(RotatedBoxes(b1), RotatedBoxes(b2))
        try:
            R.Matcher([0.3, 0.7], [0, -1, 1], True)(mq)
            raised = 0
        except AssertionError:
            raised = 1
        out[f"bad_{k}_gt"], out[f"bad_{k}_pred"], out[f"bad_{k}_raised"] = b1, b2, raised
        out[f"bad_{k}_iou"] = mq
    mg.save("matching", **out)


if __name__ == "__main__":
    main()
