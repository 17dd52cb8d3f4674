"""Generate tests/golden/losses.npz from the REAL reference functions: RPN.losses (proposal_generator/rpn.py:366-429, also
RRPN's), RetinaNet.losses (meta_arch/retinanet.py:160-210), FastRCNNOutputLayers.losses / box_reg_loss /
_log_classification_stats (roi_heads/fast_rcnn.py:88-115, 307-352, 424-463), _dense_box_regression_loss and both
get_deltas / apply_deltas (modeling/box_regression.py), and diou_loss / ciou_loss (layers/losses.py).

Run in the authoring container only (needs /root/reference, like the other generators):
    python tests/golden/make_golden_losses.py
It writes only this file.  The modules are imported with the stubs of make_golden_matching.py.  fvcore is not installed, so
the fvcore.nn stub carries its three formulas (smooth_l1_loss, giou_loss, sigmoid_focal_loss), written from fvcore 0.1.5.
The methods run on a stand-in `self` carrying the attributes they read; RetinaNet's `_ema_update` is DenseDetector's
(dense_detector.py:160-182).  Stored per case: inputs, the loss dict, counts, the get_deltas targets and autograd's
gradients of the summed losses.  Assertion cases store whether the reference raised.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_matching as mgm  # noqa: E402
import make_golden_rotated as mgr  # noqa: E402

REF = mgm.REF


# ---- fvcore 0.1.5 formulas (fvcore/nn/smooth_l1_loss.py, giou_loss.py, focal_loss.py) --------------------------------
def smooth_l1_loss(input, target, beta, reduction="none"):
    if beta < 1e-5:
        loss = torch.abs(input - target)
    else:
        n = torch.abs(input - target)
        cond = n < beta
        loss = torch.where(cond, 0.5 * n ** 2 / beta, n - 0.5 * beta)
    return loss.mean() if reduction == "mean" else (loss.sum() if reduction == "sum" else loss)


def giou_loss(boxes1, boxes2, reduction="none", eps=1e-7):
    x1, y1, x2, y2 = boxes1.unbind(dim=-1)
    x1g, y1g, x2g, y2g = boxes2.unbind(dim=-1)
    assert (x2 >= x1).all(), "bad box: x1 larger than x2"
    assert (y2 >= y1).all(), "bad box: y1 larger than y2"
    xkis1, ykis1 = torch.max(x1, x1g), torch.max(y1, y1g)
    xkis2, ykis2 = torch.min(x2, x2g), torch.min(y2, y2g)
    intsctk = torch.zeros_like(x1)
    mask = (ykis2 > ykis1) & (xkis2 > xkis1)
    intsctk[mask] = (xkis2[mask] - xkis1[mask]) * (ykis2[mask] - ykis1[mask])
    unionk = (x2 - x1) * (y2 - y1) + (x2g - x1g) * (y2g - y1g) - intsctk
    iouk = intsctk / (unionk + eps)
    xc1, yc1 = torch.min(x1, x1g), torch.min(y1, y1g)
    xc2, yc2 = torch.max(x2, x2g), torch.max(y2, y2g)
    area_c = (xc2 - xc1) * (yc2 - yc1)
    miouk = iouk - ((area_c - unionk) / (area_c + eps))
    loss = 1 - miouk
    return loss.mean() if reduction == "mean" else (loss.sum() if reduction == "sum" else loss)


def sigmoid_focal_loss(inputs, targets, alpha=-1, gamma=2, reduction="none"):
    inputs, targets = inputs.float(), targets.float()
    p = torch.sigmoid(inputs)
    ce_loss = torch.nn.functional.binary_cross_entropy_with_logits(inputs, targets, reduction="none")
    p_t = p * targets + (1 - p) * (1 - targets)
    loss = ce_loss * ((1 - p_t) ** gamma)
    if alpha >= 0:
        loss = (alpha * targets + (1 - alpha) * (1 - targets)) * loss
    return loss.mean() if reduction == "mean" else (loss.sum() if reduction == "sum" else loss)


class _Storage:
    def __init__(self):
        self.scalars = {}

    def put_scalar(self, k, v, *a, **kw):
        self.scalars[k] = float(v)


def import_reference():
    ns = mgm.import_reference()
    fv = sys.modules["fvcore.nn"]
    fv.smooth_l1_loss, fv.giou_loss, fv.sigmoid_focal_loss_jit = smooth_l1_loss, giou_loss, sigmoid_focal_loss
    import detectron2.layers as dl

    br = mgr._load("detectron2.modeling.box_regression_real", REF + "/modeling/box_regression.py")
    frc = mgr._load("detectron2.modeling.roi_heads.fast_rcnn_real", REF + "/modeling/roi_heads/fast_rcnn.py")
    for m in (ns.rpn, ns.ret, frc):
        m._dense_box_regression_loss = br._dense_box_regression_loss
    ns.ret.sigmoid_focal_loss_jit = sigmoid_focal_loss
    storage = _Storage()
    frc.get_event_storage = lambda: storage
    ns.rpn.get_event_storage = ns.ret.get_event_storage = lambda: storage
    return types.SimpleNamespace(br=br, rpn=ns.rpn, ret=ns.ret, frc=frc, storage=storage, layers=dl)


OUT = {}


def put(case, **arrs):
    for k, v in arrs.items():
        if isinstance(v, (list, tuple)):
            for i, t in enumerate(v):
                OUT["%s__%s%d" % (case, k, i)] = t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)
        else:
            OUT["%s__%s" % (case, k)] = v.detach().cpu().numpy() if isinstance(v, torch.Tensor) else np.asarray(v)


def boxes(n, g, rotated=False):
    xy = torch.rand(n, 2, generator=g) * 200
    wh = 4 + torch.rand(n, 2, generator=g) * 60
    if rotated:
        return torch.cat([xy, wh, (torch.rand(n, 1, generator=g) - 0.5) * 360], 1)
    return torch.cat([xy, xy + wh], 1)


def near(b, g, rotated=False):
    """GT boxes near the given boxes (positive rows regress to something close)."""
    j = (torch.rand(b.shape, generator=g) - 0.5) * 6
    if rotated:
        out = b + j
        out[:, 2:4] = b[:, 2:4].abs() + 1 + j[:, 2:4].abs()
        return out
    out = b + j
    out[:, 2:] = torch.maximum(out[:, 2:], out[:, :2] + 1)
    return out


def leaves(ts):
    return [t.detach().clone().requires_grad_(True) for t in ts]


def run_rpn(R, case, g, rotated=False, beta=0.0, no_gt_image=False, zero_width=False, loss_type="smooth_l1"):
    levels, n = (30, 12), 2
    d = 5 if rotated else 4
    anchors = [boxes(rl, g, rotated) for rl in levels]
    cat_a = torch.cat(anchors)
    if zero_width:
        anchors[1][3, 2] = anchors[1][3, 0] if not rotated else 0.0
        cat_a = torch.cat(anchors)
    labels = [torch.randint(-1, 2, (sum(levels),), generator=g).to(torch.int8) for _ in range(n)]
    gt = [near(cat_a, g, rotated) for _ in range(n)]
    if no_gt_image:
        labels[1][labels[1] == 1] = 0
        gt[1] = torch.zeros_like(cat_a)
    logits = [torch.randn(n, rl, generator=g) for rl in levels]
    deltas = [torch.randn(n, rl, d, generator=g) * 0.3 for rl in levels]
    w = (1.0,) * d
    B = R.br.Box2BoxTransformRotated(w) if rotated else R.br.Box2BoxTransform(w)
    self = types.SimpleNamespace(box2box_transform=B, box_reg_loss_type=loss_type, smooth_l1_beta=beta,
                                 batch_size_per_image=64, loss_weight={"loss_rpn_cls": 1.0, "loss_rpn_loc": 2.0})
    lx, ld = leaves(logits), leaves(deltas)
    put(case, anchors=anchors, labels=labels, gt=gt, logits=logits, deltas=deltas, beta=beta, weights=np.asarray(w))
    try:
        losses = R.rpn.RPN.losses(self, anchors, lx, labels, ld, gt)
    except AssertionError:
        put(case, raises=1)
        return
    sum(losses.values()).backward()
    put(case, raises=0, loss_rpn_cls=losses["loss_rpn_cls"], loss_rpn_loc=losses["loss_rpn_loc"],
        num_pos=sum(int((lb == 1).sum()) for lb in labels), num_neg=sum(int((lb == 0).sum()) for lb in labels),
        targets=torch.stack([B.get_deltas(cat_a, k) for k in gt]) if not no_gt_image else torch.zeros(0),
        grad_logits=[x.grad for x in lx], grad_deltas=[x.grad for x in ld])


def run_retina(R, case, g, beta=0.1, loss_type="smooth_l1", no_pos=False, nan_ignored=False, calls=1, nan_box=False):
    levels, n, k = (40, 16), 2, 5
    anchors = [boxes(rl, g) for rl in levels]
    cat_a = torch.cat(anchors)
    labels = [torch.randint(-1, k + 1, (sum(levels),), generator=g) for _ in range(n)]
    if no_pos:
        labels = [torch.where(lb >= 0, torch.full_like(lb, k), lb) for lb in labels]
    gt = [near(cat_a, g) for _ in range(n)]
    logits = [torch.randn(n, rl, k, generator=g) for rl in levels]
    deltas = [torch.randn(n, rl, 4, generator=g) * 0.3 for rl in levels]
    if nan_ignored:
        ign = torch.nonzero(labels[0][: levels[0]] == -1)[:, 0]
        logits[0][0, ign] = float("nan")
    if nan_box:
        pos = torch.nonzero((labels[0] >= 0) & (labels[0] < k))[:, 0]
        deltas[0][0, int(pos[pos < levels[0]][0]), 0] = float("nan")
    B = R.br.Box2BoxTransform((1.0, 1.0, 1.0, 1.0))
    self = types.SimpleNamespace(num_classes=k, focal_loss_alpha=0.25, focal_loss_gamma=2.0, box2box_transform=B,
                                 box_reg_loss_type=loss_type, smooth_l1_beta=beta)

    def _ema_update(name, value, initial_value, momentum=0.9):
        old = getattr(self, name) if hasattr(self, name) else initial_value
        new = old * momentum + value * (1 - momentum)
        setattr(self, name, new)
        return new

    self._ema_update = _ema_update
    put(case, anchors=anchors, labels=labels, gt=gt, logits=logits, deltas=deltas, beta=beta, calls=calls)
    for c in range(calls):
        lx, ld = leaves(logits), leaves(deltas)
        try:
            losses = R.ret.RetinaNet.losses(self, anchors, lx, labels, ld, gt)
        except AssertionError:
            put(case, raises=1)
            return
        sum(losses.values()).backward()
        put(case + "_call%d" % c, loss_cls=losses["loss_cls"], loss_box_reg=losses["loss_box_reg"],
            normalizer=self.loss_normalizer, grad_logits=[x.grad for x in lx], grad_deltas=[x.grad for x in ld])
    pos = sum(int(((lb >= 0) & (lb < k)).sum()) for lb in labels)
    put(case, raises=0, num_pos=pos, targets=torch.stack([B.get_deltas(cat_a, q) for q in gt]))


def run_frcnn(R, case, g, rotated=False, agnostic=False, beta=0.0, loss_type="smooth_l1", weights=(10.0, 10.0, 5.0, 5.0),
              sizes=(24, 17), zero_width=False):
    from detectron2.structures import Boxes, Instances, RotatedBoxes

    k, d = 6, 5 if rotated else 4
    r = sum(sizes)
    props = boxes(r, g, rotated)
    gtb = near(props, g, rotated)
    cls = torch.randint(0, k + 1, (r,), generator=g)
    if zero_width:
        fg = int(torch.nonzero(cls < k)[0])
        props[fg, 2] = props[fg, 0] if not rotated else 0.0
    scores = torch.randn(r, k + 1, generator=g)
    if r:
        scores[0] = 0.0  # argmax tie
    deltas = torch.randn(r, d if agnostic else k * d, generator=g) * 0.3
    B = R.br.Box2BoxTransformRotated(weights) if rotated else R.br.Box2BoxTransform(weights)
    BoxT = RotatedBoxes if rotated else Boxes
    proposals, s0 = [], 0
    for sz in sizes:
        inst = Instances((300, 300))
        inst.proposal_boxes = BoxT(props[s0:s0 + sz])
        inst.gt_boxes = BoxT(gtb[s0:s0 + sz])
        inst.gt_classes = cls[s0:s0 + sz]
        proposals.append(inst)
        s0 += sz
    cls_t = R.frc.FastRCNNOutputLayers
    self = types.SimpleNamespace(use_sigmoid_ce=False, num_classes=k, box2box_transform=B, box_reg_loss_type=loss_type,
                                 smooth_l1_beta=beta, loss_weight={"loss_cls": 1.0, "loss_box_reg": 0.5})
    self.box_reg_loss = types.MethodType(cls_t.box_reg_loss, self)
    s, dd = leaves([scores, deltas])
    put(case, scores=scores, deltas=deltas, props=props, gt=gtb, classes=cls, beta=beta, weights=np.asarray(weights))
    R.storage.scalars.clear()
    try:
        losses = cls_t.losses(self, (s, dd), proposals)
    except AssertionError:
        put(case, raises=1)
        return
    sum(losses.values()).backward()
    st = R.storage.scalars
    fg = (cls >= 0) & (cls < k)
    put(case, raises=0, loss_cls=losses["loss_cls"], loss_box_reg=losses["loss_box_reg"], grad_scores=s.grad,
        grad_deltas=dd.grad, targets=B.get_deltas(props[fg], gtb[fg]) if loss_type == "smooth_l1" else torch.zeros(0),
        cls_accuracy=st.get("fast_rcnn/cls_accuracy", -1.0), fg_cls_accuracy=st.get("fast_rcnn/fg_cls_accuracy", -1.0),
        false_negative=st.get("fast_rcnn/false_negative", -1.0))


def main():
    R = import_reference()
    g = torch.Generator().manual_seed(11)
    cases = []

    def case(fn, name, **kw):
        fn(R, name, g, **kw)
        cases.append(name)

    case(run_rpn, "rpn_b0")
    case(run_rpn, "rpn_b01", beta=0.1)
    case(run_rpn, "rpn_nogt", no_gt_image=True)
    case(run_rpn, "rrpn", rotated=True)
    case(run_rpn, "rpn_giou", loss_type="giou")
    case(run_rpn, "rpn_zero_width", zero_width=True)
    case(run_retina, "retina_ema", calls=2)
    case(run_retina, "retina_b0", beta=0.0)
    case(run_retina, "retina_giou", loss_type="giou")
    case(run_retina, "retina_diou", loss_type="diou")
    case(run_retina, "retina_ciou", loss_type="ciou")
    case(run_retina, "retina_nopos", no_pos=True)
    case(run_retina, "retina_nan_ignored", nan_ignored=True)
    case(run_retina, "retina_giou_nan_box", loss_type="giou", nan_box=True)
    case(run_frcnn, "frcnn_specific")
    case(run_frcnn, "frcnn_agnostic", agnostic=True)
    case(run_frcnn, "frcnn_b01_cascade", beta=0.1, weights=(20.0, 20.0, 10.0, 10.0))
    case(run_frcnn, "frcnn_giou", loss_type="giou")
    case(run_frcnn, "frcnn_rotated", rotated=True, weights=(10.0, 10.0, 5.0, 5.0, 1.0))
    case(run_frcnn, "frcnn_empty", sizes=(0,))
    case(run_frcnn, "frcnn_zero_width", zero_width=True)
    OUT["cases"] = np.asarray(cases)
    np.savez_compressed(os.path.join(HERE, "losses.npz"), **OUT)
    print("losses", len(OUT), "arrays", cases)


if __name__ == "__main__":
    main()
