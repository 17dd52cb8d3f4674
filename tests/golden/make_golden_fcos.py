"""Generate tests/golden/fcos.npz from the REAL reference FCOS methods: FCOS._match_anchors / label_anchors, losses,
compute_ctrness_targets and inference_single_image (modeling/meta_arch/fcos.py:97-301) on Box2BoxTransformLinear
(modeling/box_regression.py:230-307) and the real DenseDetector decode (meta_arch/dense_detector.py:186-258).

Run in the authoring container only (needs /root/reference and oracle/_ref, like the other generators):
    python tests/golden/make_golden_fcos.py
It writes only this file.  The modules are imported with the stubs of make_golden_matching.py / make_golden_losses.py
(fvcore formulas of fvcore 0.1.5); the methods run on a stand-in `self` carrying the attributes they read, with
DenseDetector._ema_update and the _decode_* methods taken from dense_detector.py.  NMS is the reference's batched_nms on CPU.

Points: DefaultAnchorGenerator's boxes for strides 8, 16, 32, 64 on a 128 x 128 image (dyadic coordinates, so the strict
comparisons at the edges are exact).  Scenes: images with 14, 1 and 0 GT boxes, where image 0 holds a GT edge through a
point centre, a centre distance of exactly radius * size, a maximum distance of exactly 4 * size and 8 * size, and two
boxes of areas 100 and 97 that tie in 1e8 - area (the first wins); a second batch with a GT box with an infinite coordinate
and one with a NaN coordinate, which take every point of their image.  Losses: fp32 predictions over two calls (the EMA),
fp16 predictions (their fp32 values enter the reference), and a NaN delta on a positive row (the reference asserts).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_losses as mgl  # noqa: E402
import make_golden_rotated as mgr  # noqa: E402

REF = mgl.REF
STRIDES = (8, 16, 32, 64)
SIZE = 128
K = 6


def import_reference():
    R = mgl.import_reference()
    bmod = sys.modules["detectron2.modeling.box_regression"]
    bmod.Box2BoxTransformLinear = R.br.Box2BoxTransformLinear
    bmod._dense_box_regression_loss = R.br._dense_box_regression_loss
    sys.modules["detectron2.modeling.postprocessing"] = types.ModuleType("detectron2.modeling.postprocessing")
    sys.modules["detectron2.modeling.postprocessing"].detector_postprocess = None
    sys.modules["detectron2.data.detection_utils"].convert_image_to_rgb = None
    sys.modules["detectron2.modeling"].Backbone = object
    spec = importlib.util.spec_from_file_location("detectron2.modeling.meta_arch.dense_detector_real",
                                                  REF + "/modeling/meta_arch/dense_detector.py")
    dd = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(dd)
    fcos = mgr._load("detectron2.modeling.meta_arch.fcos", REF + "/modeling/meta_arch/fcos.py")
    fcos.sigmoid_focal_loss_jit = mgl.sigmoid_focal_loss
    fcos.get_event_storage = lambda: R.storage
    return R, dd, fcos


def points():
    """DefaultAnchorGenerator(sizes=[[s] for s in strides], aspect_ratios=[1.0], strides, offset 0)."""
    out = []
    for s in STRIDES:
        n = SIZE // s
        ys, xs = torch.meshgrid(torch.arange(n, dtype=torch.float32) * s, torch.arange(n, dtype=torch.float32) * s,
                                indexing="ij")
        c = torch.stack([xs.reshape(-1), ys.reshape(-1)], 1)
        out.append(torch.cat([c - s / 2, c + s / 2], 1))
    return out


def scene0(g):
    """14 GT boxes with the edge cases of the module docstring."""
    special = torch.tensor([
        [16.0, 8.0, 40.0, 32.0],      # left edge x0 = 16 through the level-0 points at x = 16: l = 0, not inside
        [40.0, 40.0, 76.0, 64.0],     # centre (58, 52): the level-0 point (70, 52) is exactly 1.5 * 8 = 12 away
        [0.0, 0.0, 64.0, 128.0],      # level-1 point (32, 64): max distance 64 = 4 * 16 (not > lower)
        [64.0, 0.0, 128.0, 128.0],    # level-2 point (96, 64): max distance 64 (not > 4 * 32 = 128 either: level 1 takes it)
        [83.5, 83.0, 96.0, 91.0],     # area 12.5 * 8 = 100 ...
        [83.875, 83.0, 96.0, 91.0],   # ... and 12.125 * 8 = 97: 1e8 - area ties in fp32, the first wins
        [0.0, 32.0, 16.0, 160.0],     # level-3 point (0, 64)... a tall box reaching past the image
    ])
    xy = torch.randint(0, 24, (7, 2), generator=g).float() * 4
    wh = torch.randint(2, 20, (7, 2), generator=g).float() * 4
    rand = torch.cat([xy, xy + wh], 1)
    return torch.cat([special, rand])


def run_label(fcos, anchors, gts, classes, radius=1.5):
    from detectron2.structures import Boxes, Instances

    self = types.SimpleNamespace(center_sampling_radius=float(radius), num_classes=K)
    self._match_anchors = types.MethodType(fcos.FCOS._match_anchors, self)
    inst = [Instances((SIZE, SIZE), gt_boxes=Boxes(b.clone()), gt_classes=c.clone()) for b, c in zip(gts, classes)]
    labels, boxes = fcos.FCOS.label_anchors(self, [Boxes(a) for a in anchors], inst)
    quality = [self._match_anchors(Boxes(b), [Boxes(a) for a in anchors]) if len(b) else torch.zeros(0, sum(map(len, anchors)))
               for b in gts]
    return labels, boxes, quality


def leaves(ts):
    # fp16 predictions enter as their fp32 values: the reference's fvcore giou_loss cannot index_put fp32 intersections
    # into the fp16 tensor of a half-precision decode, and the kernels read fp16 in place with fp32 arithmetic
    return [t.detach().float().clone().requires_grad_(True) for t in ts]


def run_loss(R, fcos, out, case, anchors, labels, boxes, g, dtype=torch.float32, calls=1, nan_delta=False):
    from detectron2.structures import Boxes

    n, r = len(labels), sum(len(a) for a in anchors)
    logits = [(torch.randn(n, len(a), K, generator=g) * 2).to(dtype) for a in anchors]
    deltas = [(torch.randn(n, len(a), 4, generator=g) + 0.5).to(dtype) for a in anchors]
    ctr = [torch.randn(n, len(a), 1, generator=g).to(dtype) for a in anchors]
    deltas[0][0, :6, 1] = 0.0  # zero deltas: relu's gradient is 0 there
    if nan_delta:
        pos = torch.nonzero((labels[0] >= 0) & (labels[0] < K))[:, 0]
        lvl0 = pos[pos < len(anchors[0])]
        deltas[0][0, int(lvl0[0]), 2] = float("nan")
    self = types.SimpleNamespace(num_classes=K, focal_loss_alpha=0.25, focal_loss_gamma=2.0,
                                 box2box_transform=R.br.Box2BoxTransformLinear(normalize_by_size=True))
    self.compute_ctrness_targets = types.MethodType(fcos.FCOS.compute_ctrness_targets, self)

    def _ema_update(name, value, initial_value, momentum=0.9):
        old = getattr(self, name) if hasattr(self, name) else initial_value
        new = old * momentum + value * (1 - momentum)
        setattr(self, name, new)
        return new

    self._ema_update = _ema_update
    box_anchors = [Boxes(a) for a in anchors]
    mgl.put(case, logits=logits, deltas=deltas, ctr=ctr, calls=calls)
    for c in range(calls):
        lx, ld, lc = leaves(logits), leaves(deltas), leaves(ctr)
        try:
            losses = fcos.FCOS.losses(self, box_anchors, lx, [x.clone() for x in labels], ld, boxes, lc)
        except AssertionError:
            mgl.put(case, raises=1)
            return
        sum(losses.values()).backward()
        mgl.put(case + "_call%d" % c, loss_fcos_cls=losses["loss_fcos_cls"], loss_fcos_loc=losses["loss_fcos_loc"],
                loss_fcos_ctr=losses["loss_fcos_ctr"], normalizer=self.loss_normalizer, grad_logits=[x.grad for x in lx],
                grad_deltas=[x.grad for x in ld], grad_ctr=[x.grad for x in lc])
    pos = sum(int(((lb >= 0) & (lb < K)).sum()) for lb in labels)
    mgl.put(case, raises=0, num_pos=pos, ctr_targets=self.compute_ctrness_targets(box_anchors, boxes))


def run_inference(dd, fcos, out, anchors, g):
    from detectron2.layers import batched_nms  # noqa: F401  (the module fcos.py imported)
    from detectron2.structures import Boxes

    n = 2
    logits = [torch.randn(n, len(a), K, generator=g) * 1.5 - 1.5 for a in anchors]
    ctr = [torch.randn(n, len(a), 1, generator=g) for a in anchors]
    deltas = [torch.randn(n, len(a), 4, generator=g) * 0.5 + 0.3 for a in anchors]
    logits[3][1] = -20.0  # a level without any candidate for image 1
    self = types.SimpleNamespace(box2box_transform=None, test_score_thresh=0.2, test_topk_candidates=1000,
                                 test_nms_thresh=0.6, max_detections_per_image=100)
    import detectron2.modeling.box_regression as brm

    self.box2box_transform = brm.Box2BoxTransformLinear(normalize_by_size=True)
    self._decode_per_level_predictions = types.MethodType(dd.DenseDetector._decode_per_level_predictions, self)
    self._decode_multi_level_predictions = types.MethodType(dd.DenseDetector._decode_multi_level_predictions, self)
    mgl.put("inf", logits=logits, ctr=ctr, deltas=deltas)
    for i in range(n):
        scores = [torch.sqrt(x[i].clone().sigmoid_() * y[i].clone().sigmoid_()) for x, y in zip(logits, ctr)]  # fcos.py:269
        res = fcos.FCOS.inference_single_image(self, [Boxes(a) for a in anchors], scores, [x[i] for x in deltas],
                                               (SIZE, SIZE))
        mgl.put("inf%d" % i, boxes=res.pred_boxes.tensor, scores=res.scores, classes=res.pred_classes)


def main():
    torch.set_num_threads(1)
    R, dd, fcos = import_reference()
    g = torch.Generator().manual_seed(1234)
    anchors = points()
    mgl.put("pts", anchors=anchors)
    gts = [scene0(g), torch.tensor([[30.0, 20.0, 90.0, 100.0]]), torch.zeros((0, 4))]
    classes = [torch.randint(0, K, (len(b),), generator=g) for b in gts]
    labels, boxes, quality = run_label(fcos, anchors, gts, classes)
    mgl.put("a", gt=gts, cls=classes, labels=labels, boxes=boxes, quality=quality)
    # non-finite GT boxes: NaN quality at every point of their image
    nf = [torch.tensor([[10.0, 10.0, 50.0, 50.0], [0.0, 0.0, float("inf"), 40.0], [60.0, 60.0, 100.0, 90.0]]),
          torch.tensor([[20.0, 20.0, 60.0, 60.0], [float("nan"), 5.0, 30.0, 30.0]])]
    nf_cls = [torch.tensor([1, 2, 3]), torch.tensor([4, 5])]
    labels_nf, boxes_nf, quality_nf = run_label(fcos, anchors, nf, nf_cls)
    mgl.put("nf", gt=nf, cls=nf_cls, labels=labels_nf, boxes=boxes_nf, quality=quality_nf)

    run_loss(R, fcos, mgl.OUT, "loss_f32", anchors, labels, boxes, g, calls=2)
    run_loss(R, fcos, mgl.OUT, "loss_f16", anchors, labels, boxes, g, dtype=torch.float16)
    run_loss(R, fcos, mgl.OUT, "loss_nan_delta", anchors, labels, boxes, g, nan_delta=True)
    run_inference(dd, fcos, mgl.OUT, anchors, g)
    np.savez_compressed(os.path.join(HERE, "fcos.npz"), **mgl.OUT)
    print("fcos", len(mgl.OUT), "arrays")


if __name__ == "__main__":
    main()
