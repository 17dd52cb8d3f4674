"""Generate tests/golden/rrpn_proposals.npz and tests/golden/rotated_fast_rcnn_inference.npz from the REAL reference
functions find_top_rrpn_proposals (detectron2/modeling/proposal_generator/rrpn.py:20-127) and
fast_rcnn_inference_rotated (modeling/roi_heads/rotated_fast_rcnn.py:46-132).

Run in the authoring container only (needs /root/reference and oracle/_ref, like make_golden.py):
    python tests/golden/make_golden_rotated.py
It writes only these two files.  The modules are imported with stubs for their unrelated dependencies (.rpn, .build,
box_regression, box_head, roi_heads, ...); rotated NMS is the reference CPU csrc compiled in oracle/_ref.

The reference's CPU rotated NMS orders equal scores with a non-stable sort (nms_rotated_cpu.cpp:26), so the tied scores in
these inputs are placed where the result does not depend on their order (identical boxes of one category, where either of the
tied boxes gives the same output, or tied boxes that a higher-scoring box suppresses); the stable tie order itself is pinned in tests/test_oracle_pins.py.
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (stubs, save(), reference CPU csrc)

ANGLES = [1.0, -1.0, 1.0001, 179.5, 270.0, -190.0, 540.0, -180.00002]


def _stub(name, **attrs):
    m = types.ModuleType(name)
    m.__dict__.update(attrs)
    sys.modules[name] = m
    return m


class _Registry:
    def register(self, *a, **k):
        return lambda obj: obj


def _load(name, path):
    spec = importlib.util.spec_from_file_location(name, path)
    m = importlib.util.module_from_spec(spec)
    sys.modules[name] = m
    spec.loader.exec_module(m)
    return m


def _import_reference_rotated():
    mg._import_reference_fast_rcnn()  # fvcore / pycocotools / config / events / data stubs, detectron2.layers + structures
    sys.modules["detectron2.modeling.box_regression"].Box2BoxTransformRotated = object
    _stub("detectron2.utils.memory", retry_if_cuda_oom=lambda f: f)
    pg = _stub("detectron2.modeling.proposal_generator")
    pg.__path__ = []
    _stub("detectron2.modeling.proposal_generator.build", PROPOSAL_GENERATOR_REGISTRY=_Registry())
    _stub("detectron2.modeling.proposal_generator.rpn", RPN=object)
    _stub("detectron2.modeling.proposal_generator.proposal_utils", _is_tracing=lambda: False,
          add_ground_truth_to_proposals=None)
    _stub("detectron2.modeling.poolers", ROIPooler=None)
    rh = _stub("detectron2.modeling.roi_heads")
    rh.__path__ = []
    _stub("detectron2.modeling.roi_heads.box_head", build_box_head=None)
    _stub("detectron2.modeling.roi_heads.fast_rcnn", FastRCNNOutputLayers=object)
    _stub("detectron2.modeling.roi_heads.roi_heads", ROI_HEADS_REGISTRY=_Registry(), StandardROIHeads=object)
    rrpn = _load("detectron2.modeling.proposal_generator.rrpn",
                 "/root/reference/detectron2/modeling/proposal_generator/rrpn.py")
    rfr = _load("detectron2.modeling.roi_heads.rotated_fast_rcnn",
                "/root/reference/detectron2/modeling/roi_heads/rotated_fast_rcnn.py")
    return rrpn, rfr


def _rand_rotated(g, shape, lo_xy, hi_xy, wmax, horizontal_frac=0.5):
    ctr = torch.rand(*shape, 2, generator=g) * (torch.tensor(hi_xy) - torch.tensor(lo_xy)) + torch.tensor(lo_xy)
    wh = torch.rand(*shape, 2, generator=g) * wmax + 0.5
    a = (torch.rand(*shape, 1, generator=g) - 0.5) * 720
    near = torch.rand(*shape, 1, generator=g) < horizontal_frac
    a = torch.where(near, (torch.rand(*shape, 1, generator=g) - 0.5) * 4, a)  # within +-2 degrees: about half clipped
    return torch.cat([ctr, wh, a], -1)


def gen_rrpn_proposals(ref):
    g = torch.Generator().manual_seed(505)
    n, sizes = 2, [(120, 160), (100, 200)]
    per_level = [500, 250, 80]
    thr, pre, post, mbs = 0.7, 200, 80, 2.0
    props, logits = [], []
    for a in per_level:
        props.append(_rand_rotated(g, (n, a), (-15.0, -15.0), (215.0, 135.0), 60.0))
        logits.append(torch.randn(n, a, generator=g))
    p0, l0 = props[0], logits[0]
    # the special boxes carry high logits so that they pass the per-level top-k
    for i, ang in enumerate(ANGLES):  # angle normalisation and the clip threshold, both images
        for img in range(n):
            p0[img, 20 + i] = torch.tensor([-4.0 + 25 * i, 60.0, 30.0, 14.0, ang])  # straddles x = 0 for i = 0
            l0[img, 20 + i] = 4.0 + 0.01 * i + 0.003 * img
    p0[0, 3] = torch.tensor([50.0, 50.0, float("nan"), 10.0, 0.0])   # non-finite box
    l0[0, 3] = 5.0
    logits[1][1, 5] = float("inf")                                    # non-finite score
    p0[1, 40] = torch.tensor([-5.0, 40.0, 12.0, 30.0, 0.5])           # clipped to width 1 < min_box_size
    l0[1, 40] = 4.5
    p0[0, 41] = torch.tensor([158.0, 118.0, 20.0, 10.0, -0.7])        # straddles the far corner
    l0[0, 41] = 4.6
    p0[1, 42] = torch.tensor([-20.0, -12.0, 30.0, 18.0, 45.0])       # negative centre, not clipped
    l0[1, 42] = 4.7
    p0[0, 50:53] = torch.tensor([70.0, 70.0, 20.0, 20.0, 10.0])      # identical boxes with tied scores
    l0[0, 50:53] = 3.9
    logits[2][0, 10:12] = 3.8                                         # tied scores on identical boxes, another level
    props[2][0, 10:12] = torch.tensor([20.0, 20.0, 8.0, 8.0, 30.0])
    out = {"sizes": np.asarray(sizes), "per_level": np.asarray(per_level), "cfg": np.asarray([thr, pre, post, mbs])}
    for l in range(len(per_level)):
        out[f"props{l}"] = props[l]
        out[f"logits{l}"] = logits[l]
    res = ref.find_top_rrpn_proposals([p.clone() for p in props], [x.clone() for x in logits], sizes, thr, pre, post, mbs,
                                      False)
    for i, r in enumerate(res):
        out[f"boxes_img{i}"] = r.proposal_boxes.tensor
        out[f"scores_img{i}"] = r.objectness_logits
    mg.save("rrpn_proposals", **out)


def gen_rotated_fast_rcnn_inference(ref):
    g = torch.Generator().manual_seed(61)
    score_thresh, nms_thresh, topk = 0.05, 0.5, 25
    shapes = [(120, 160), (90, 200), (100, 100)]
    out = {"cfg": np.asarray([score_thresh, nms_thresh, topk]), "shapes": np.asarray(shapes)}
    # image 0: class-specific boxes, image 1: class-agnostic, image 2: class-specific without any candidate
    for i, (r, k, agnostic) in enumerate([(80, 6, False), (50, 6, True), (30, 6, False)]):
        base = _rand_rotated(g, (12,), (-10.0, -10.0), (170.0, 110.0), 50.0)
        pick = torch.randint(0, 12, (r,), generator=g)
        nb = 1 if agnostic else k
        jitter = torch.randn(r, nb, 5, generator=g) * torch.tensor([3.0, 3.0, 2.0, 2.0, 4.0])
        boxes = (base[pick][:, None, :] + jitter)
        boxes[..., 2:4] = boxes[..., 2:4].abs() + 0.5
        boxes = boxes.reshape(r, nb * 5)
        scores = torch.softmax(torch.randn(r, k + 1, generator=g) * 2.5, dim=1)
        if i == 0:
            boxes[7, 2] = float("inf")       # invalid row (dropped before everything else)
            scores[9] = float("nan")
            for j, ang in enumerate(ANGLES):
                boxes[30 + j, 4::5] = ang     # every class column of the row
            boxes[40, 0:5] = torch.tensor([2.0, 50.0, 30.0, 20.0, 0.2])  # straddles x = 0
            scores[40, 0] = 0.9
            boxes[41, 5:10] = torch.tensor([-30.0, -20.0, 10.0, 10.0, 33.0])  # negative centre
            scores[41, 1] = 0.85
            # tie: two candidates of class 2 on identical boxes, both below a stronger duplicate (both suppressed)
            boxes[42:45, 10:15] = torch.tensor([90.0, 60.0, 20.0, 12.0, 5.0])
            scores[42, 2] = 0.95
            scores[43:45, 2] = 0.6
        if i == 1:
            # tie between rows 3 and 4 on the box of row 5, which scores higher: both suppressed
            boxes[3:6] = torch.tensor([10.0, 10.0, 6.0, 6.0, 0.0])
            scores[3:6] = 0.0
            scores[3:5, 0] = 0.7
            scores[5, 0] = 0.8
        if i == 2:
            scores = torch.full((r, k + 1), 0.01)
            scores[:, k] = 1.0 - 0.01 * k
        out.update({f"boxes{i}": boxes, f"scores{i}": scores})
        for tk, tag in ((topk, ""), (-1, "_all")):
            res, rows = ref.fast_rcnn_inference_rotated([boxes.clone()], [scores.clone()], [shapes[i]], score_thresh,
                                                        nms_thresh, tk)
            out.update({f"out_boxes{i}{tag}": res[0].pred_boxes.tensor, f"out_scores{i}{tag}": res[0].scores,
                        f"out_classes{i}{tag}": res[0].pred_classes, f"out_rows{i}{tag}": rows[0]})
    mg.save("rotated_fast_rcnn_inference", **out)


if __name__ == "__main__":
    torch.set_num_threads(1)
    rrpn, rfr = _import_reference_rotated()
    gen_rrpn_proposals(rrpn)
    gen_rotated_fast_rcnn_inference(rfr)
