"""Box-branch training losses without a GPU: the fvcore formulas of the torch restatement against torchvision's
implementations of the same losses, the CPU path of the reference-shaped wrappers, and argument validation of the new
C entry points (every check runs before the first CUDA call)."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch
from torch.nn import functional as F


def _boxes(n, g, scale=100.0):
    xy = torch.rand(n, 2, generator=g) * scale
    wh = 1 + torch.rand(n, 2, generator=g) * scale
    return torch.cat([xy, xy + wh], dim=1)


def test_focal_formula_matches_torchvision():
    from torchvision.ops import sigmoid_focal_loss

    from detectron2_b200 import losses as L

    g = torch.Generator().manual_seed(0)
    x = torch.randn(4000, generator=g) * 4
    t = (torch.rand(4000, generator=g) < 0.2).float()
    for alpha, gamma in ((0.25, 2.0), (-1.0, 0.0), (0.5, 1.5), (-1.0, 2.0)):
        ours = L._sigmoid_focal_loss(x, t, alpha, gamma)
        ref = sigmoid_focal_loss(x, t, alpha=alpha, gamma=gamma, reduction="sum")
        assert torch.allclose(ours, ref, rtol=1e-6, atol=0), (alpha, gamma)
    # gamma = 0 without alpha is binary_cross_entropy_with_logits: the RPN objectness loss
    assert torch.allclose(L._sigmoid_focal_loss(x, t, -1.0, 0.0),
                          F.binary_cross_entropy_with_logits(x, t, reduction="sum"), rtol=1e-6)


def test_giou_formula_matches_torchvision():
    from torchvision.ops import generalized_box_iou_loss

    from detectron2_b200 import losses as L

    g = torch.Generator().manual_seed(1)
    a, b = _boxes(3000, g), _boxes(3000, g)
    ref = generalized_box_iou_loss(a, b, reduction="sum", eps=1e-7)
    assert torch.allclose(L._giou_loss(a, b), ref, rtol=1e-6)
    bad = a.clone()
    bad[3, 2] = bad[3, 0] - 1  # x2 < x1: fvcore's assertion
    with pytest.raises(AssertionError):
        L._giou_loss(bad, b)


def test_smooth_l1_formula():
    from detectron2_b200 import losses as L

    d = torch.tensor([-2.0, -0.05, 0.0, 0.05, 0.3])
    z = torch.zeros_like(d)
    assert torch.equal(L._smooth_l1_loss(d, z, 0.0), d.abs().sum())
    expect = sum(0.5 * v * v / 0.1 if abs(v) < 0.1 else abs(v) - 0.05 for v in d.tolist())
    assert math.isclose(float(L._smooth_l1_loss(d, z, 0.1)), expect, rel_tol=1e-6)


def test_get_deltas_round_trip_and_assertion():
    from detectron2_b200 import losses as L

    g = torch.Generator().manual_seed(2)
    src, tgt = _boxes(500, g), _boxes(500, g)
    w = (10.0, 10.0, 5.0, 5.0)
    back = L._apply_deltas(L._get_deltas(src, tgt, w), src, w, 1e9)
    assert torch.allclose(back, tgt, rtol=1e-5, atol=1e-3)
    src[7, 2] = src[7, 0]  # zero width
    with pytest.raises(AssertionError):
        L._get_deltas(src, tgt, w)
    # rotated: the angle difference wraps into [-180, 180) with torch.remainder, then degrees -> radians * wa
    rs = torch.tensor([[10.0, 10.0, 4.0, 2.0, 170.0]])
    rt = torch.tensor([[12.0, 9.0, 8.0, 1.0, -170.0]])
    d = L._get_deltas(rs, rt, (1.0, 1.0, 1.0, 1.0, 1.0))
    assert torch.allclose(d[0], torch.tensor([0.5, -0.5, math.log(2.0), math.log(0.5), math.radians(20.0)]), atol=1e-6)


def _dense_case(g, n=2, levels=(40, 12), k=5, d=4):
    r = sum(levels)
    anchors = [_boxes(rl, g) for rl in levels]
    logits = [torch.randn(n, rl, k, generator=g) for rl in levels]
    deltas = [torch.randn(n, rl, d, generator=g) * 0.3 for rl in levels]
    gt = [_boxes(r, g) for _ in range(n)]
    return anchors, logits, deltas, gt, r


def test_wrappers_run_the_restatement_on_cpu():
    from detectron2_b200 import losses as L

    g = torch.Generator().manual_seed(3)
    anchors, logits, deltas, gt, r = _dense_case(g)
    labels = [torch.randint(-1, 6, (r,), generator=g) for _ in range(2)]  # 5 = background
    losses, num_pos, new_norm = L.retinanet_losses(anchors, logits, labels, deltas, gt, num_classes=5)
    pos = sum(int(((lb >= 0) & (lb < 5)).sum()) for lb in labels)
    assert num_pos == pos and new_norm == 100.0 * 0.9 + max(pos, 1) * (1 - 0.9)
    assert set(losses) == {"loss_cls", "loss_box_reg"} and all(torch.isfinite(v) for v in losses.values())
    rpn_labels = [torch.randint(-1, 2, (r,), generator=g).to(torch.int8) for _ in range(2)]
    obj = [x[..., 0] for x in logits]
    losses, counts = L.rpn_losses(anchors, obj, rpn_labels, deltas, gt, batch_size_per_image=256)
    assert counts["num_pos_anchors"] == sum(int((lb == 1).sum()) for lb in rpn_labels)
    assert counts["num_neg_anchors"] == sum(int((lb == 0).sum()) for lb in rpn_labels)
    _, _ = L.rpn_losses(anchors, obj, rpn_labels, deltas, gt, batch_size_per_image=256, box_reg_loss_type="giou")
    _, _ = L.rpn_losses(anchors, obj, rpn_labels, deltas, gt, batch_size_per_image=256, box_reg_loss_type="diou")
    with pytest.raises(ValueError):
        L.rpn_losses(anchors, obj, rpn_labels, deltas, gt, batch_size_per_image=256, box_reg_loss_type="iou")
    # Fast R-CNN: the counts of _log_classification_stats; no rows give zero losses
    scores = torch.randn(30, 6, generator=g)
    cls = torch.randint(0, 6, (30,), generator=g)
    props, gtb = _boxes(30, g), _boxes(30, g)
    losses, stats = L.fast_rcnn_losses(scores, torch.randn(30, 20, generator=g), props, gtb, cls)
    pred = scores.argmax(1)
    fg = cls < 5
    assert stats == {"num_fg": int(fg.sum()), "num_accurate": int((pred == cls).sum()),
                     "fg_num_accurate": int((pred[fg] == cls[fg]).sum()), "num_false_negative": int((pred[fg] == 5).sum())}
    losses, _ = L.fast_rcnn_losses(scores[:0], torch.zeros(0, 20), props[:0], gtb[:0], cls[:0])
    assert float(losses["loss_cls"]) == 0.0 and float(losses["loss_box_reg"]) == 0.0


# The box-branch loss entry points.  Each row is one fault in an otherwise valid call whose pointers are dummy addresses,
# never dereferenced: (entry points, fault, arguments that differ, expected status or a function of the call's kind giving
# it, None where the row does not apply).  The kinds are every loss type and label kind an entry point takes; a dense call
# has K = 1 with int8 labels and K = 80 with int64 ones, and one centerness level table (ctr, grad_ctr) with LINEAR_GIOU.
# The valid forward calls pass a workspace of 0 bytes, so a call that passes every argument check returns D2B_EWORKSPACE;
# the valid backward calls have rows, so a row must end before their launch (None where it would not).
EINVAL, EWORKSPACE = -1, -2
SL1, GIOU, LIN = 0, 1, 2  # D2B_LOSS_SMOOTH_L1 / _GIOU / _LINEAR_GIOU
I8, I64 = 0, 1            # D2B_LABELS_I8 / _I64
DF, DB = "d2b_dense_loss_forward", "d2b_dense_loss_backward"
FF, FB = "d2b_frcnn_loss_forward", "d2b_frcnn_loss_backward"
DENSE, FRCNN = (DF, DB), (FF, FB)
_LOSS_KINDS = {  # (loss type, int8 labels) of every call each entry point takes
    DF: ((SL1, True), (SL1, False), (GIOU, True), (GIOU, False), (LIN, False)),
    DB: ((SL1, True), (SL1, False), (GIOU, True), (GIOU, False), (LIN, False)),
    FF: ((SL1, False), (GIOU, False)),
    FB: ((SL1, False), (GIOU, False)),
}
_P = 0x1000  # a 16-byte aligned dummy address
_MISALIGNED = 0x1004
_W = (1.0, 1.0, 1.0, 1.0, 1.0)
_DENSE_IN = dict(lv=None, N=2, K=80, box_dim=4, dtype=0, anchors=_P, gt_boxes=_P, labels=_P, label_kind=I64, gamma=2.0,
                 alpha=0.25, beta=0.1, loss_type=SL1, scale_clamp=4.135, weights=_W)
_FRCNN_IN = dict(scores=_P, deltas=_P, R=10, K=80, kreg=80, box_dim=4, dtype=0, proposals=_P, gt_boxes=_P, gt_classes=_P,
                 beta=0.0, loss_type=SL1, scale_clamp=4.135, weights=_W)
_LOSS_PARAMS = {  # every parameter in order, with its value in a valid call (lv: the levels built by _loss_call)
    DF: dict(_DENSE_IN, sums=_P, counts=_P, status=_P, workspace=_P, workspace_bytes=0),
    DB: dict(_DENSE_IN, grad_sums=_P),
    FF: dict(_FRCNN_IN, sums=_P, counts=_P, status=_P, workspace=_P, workspace_bytes=0),
    FB: dict(_FRCNN_IN, grad_sums=_P, grad_scores=_P, grad_deltas=_P),
}
_PASSES = lambda k: None if k.bwd else EWORKSPACE  # noqa: E731  (every check passed: the backward would launch)
_BWD_ONLY = lambda want: lambda k: want if k.bwd else _PASSES(k)  # noqa: E731  (the forward does not read it)
_LIN_ONLY = lambda k: _PASSES(k) if k.lt == LIN else EINVAL  # noqa: E731
_NOT_LIN = lambda k: EINVAL if k.lt == LIN else _PASSES(k)  # noqa: E731
_NO_ROWS = lambda want: lambda k: want if k.bwd else None  # noqa: E731  (the forward would launch its finish)
_LOSS_FAULTS = [
    (DENSE, "N < 0", dict(N=-1), EINVAL),
    (DENSE, "no class", dict(K=0), EINVAL),
    (DENSE, "box_dim 3", dict(box_dim=3), EINVAL),
    (DENSE, "rotated boxes: smooth-L1 only", dict(box_dim=5), lambda k: EINVAL if k.lt != SL1 else _PASSES(k)),
    (DENSE, "no such dtype", dict(dtype=3), EINVAL),
    (DENSE, "weights NULL: LINEAR_GIOU reads none", dict(weights=None), _LIN_ONLY),
    (DENSE, "weights NULL, no rows", dict(weights=None, N=0), _NO_ROWS(None)),
    (DB, "weights NULL, no rows", dict(weights=None, N=0), lambda k: 0 if k.lt == LIN else EINVAL),
    (DENSE, "no such label kind", dict(label_kind=2), EINVAL),
    (DENSE, "int8 labels need K = 1", dict(label_kind=I8, K=80), EINVAL),
    (DENSE, "gamma < 0", dict(gamma=-1.0), EINVAL),
    (DENSE, "gamma NaN", dict(gamma=math.nan), EINVAL),
    (DENSE, "beta < 0", dict(beta=-0.1), EINVAL),
    (DENSE, "beta NaN", dict(beta=math.nan), EINVAL),
    (DENSE, "alpha NaN", dict(alpha=math.nan), EINVAL),
    (DENSE, "no such loss type", dict(loss_type=3), EINVAL),
    (DENSE, "negative loss type", dict(loss_type=-1), EINVAL),
    (DENSE, "LINEAR_GIOU on rotated boxes", dict(loss_type=LIN, box_dim=5, ctr=[_P], grad_ctr=[_P]), EINVAL),
    (DENSE, "LINEAR_GIOU with int8 labels", dict(loss_type=LIN, label_kind=I8, K=1, ctr=[_P], grad_ctr=[_P]), EINVAL),
    (DENSE, "no level struct", dict(lv=None), EINVAL),
    (DENSE, "no level", dict(num_levels=0), EINVAL),
    (DENSE, "9 levels", dict(num_levels=9), EINVAL),
    (DENSE, "R < 0", dict(R=[-1]), EINVAL),
    (DENSE, "R > INT_MAX", dict(num_levels=2, R=[2 ** 30] * 2), EINVAL),
    (DENSE, "logits NULL", dict(logits=[None]), EINVAL),
    (DENSE, "deltas NULL", dict(deltas=[None]), EINVAL),
    (DENSE, "logits misaligned", dict(logits=[_MISALIGNED]), EINVAL),
    (DENSE, "a level without rows needs no pointer", dict(num_levels=2, R=[10, 0], logits=[_P, None], deltas=[_P, None],
                                                         grad_logits=[_P, None], grad_deltas=[_P, None]), _PASSES),
    (DENSE, "grad_logits NULL", dict(grad_logits=[None]), _BWD_ONLY(EINVAL)),
    (DENSE, "grad_deltas NULL", dict(grad_deltas=[None]), _BWD_ONLY(EINVAL)),
    (DENSE, "grad_logits misaligned", dict(grad_logits=[_MISALIGNED]), _BWD_ONLY(EINVAL)),
    (DENSE, "ctr NULL", dict(ctr=[None]), lambda k: EINVAL if k.lt == LIN else _PASSES(k)),
    (DENSE, "ctr set", dict(ctr=[_P]), _LIN_ONLY),
    (DENSE, "grad_ctr NULL", dict(grad_ctr=[None]), lambda k: _BWD_ONLY(EINVAL)(k) if k.lt == LIN else _PASSES(k)),
    (DENSE, "grad_ctr set", dict(grad_ctr=[_P]), _LIN_ONLY),
    (DENSE, "ctr NULL on a level without rows", dict(num_levels=2, R=[10, 0], ctr=[_P, None], grad_ctr=[_P, None]),
     _LIN_ONLY),
    (DENSE, "anchors NULL", dict(anchors=None), EINVAL),
    (DENSE, "gt_boxes NULL", dict(gt_boxes=None), EINVAL),
    (DENSE, "labels NULL", dict(labels=None), EINVAL),
    (DENSE, "inputs NULL without rows", dict(N=0, anchors=None, gt_boxes=None, labels=None), _NO_ROWS(0)),
    (DENSE, "more than INT_MAX CTAs", dict(N=2 ** 30, R=[2 ** 14]), EINVAL),
    (DF, "sums NULL", dict(sums=None), EINVAL),
    (DF, "counts NULL", dict(counts=None), EINVAL),
    (DF, "status NULL", dict(status=None), EINVAL),
    (DF, "workspace NULL", dict(workspace=None), EINVAL),
    (DF, "workspace misaligned", dict(workspace=_MISALIGNED), EINVAL),
    (DF, "valid call: the workspace is too small", dict(), EWORKSPACE),
    (DB, "grad_sums NULL", dict(grad_sums=None), EINVAL),
    (DB, "grad_sums NULL without rows", dict(grad_sums=None, N=0), EINVAL),
    (DB, "no rows: nothing to do", dict(N=0, grad_logits=[None], grad_deltas=[None], grad_ctr=[None]), 0),
    (FRCNN, "R < 0", dict(R=-1), EINVAL),
    (FRCNN, "no class", dict(K=0), EINVAL),
    (FRCNN, "kreg neither 1 nor K", dict(kreg=3), EINVAL),
    (FRCNN, "class-agnostic deltas", dict(kreg=1), _PASSES),
    (FRCNN, "box_dim 6", dict(box_dim=6), EINVAL),
    (FRCNN, "rotated boxes: smooth-L1 only", dict(box_dim=5), lambda k: EINVAL if k.lt != SL1 else _PASSES(k)),
    (FRCNN, "no such dtype", dict(dtype=9), EINVAL),
    (FRCNN, "weights NULL", dict(weights=None), EINVAL),
    (FRCNN, "beta < 0", dict(beta=-0.1), EINVAL),
    (FRCNN, "beta NaN", dict(beta=math.nan), EINVAL),
    (FRCNN, "kreg * box_dim > INT_MAX / 2", dict(K=2 ** 30, kreg=2 ** 30), EINVAL),
    (FRCNN, "LINEAR_GIOU is dense only", dict(loss_type=LIN), EINVAL),
    (FRCNN, "no such loss type", dict(loss_type=3), EINVAL),
] + [(FRCNN, name + " NULL", {name: None}, EINVAL)
     for name in ("scores", "deltas", "proposals", "gt_boxes", "gt_classes")] + [
    (FRCNN, "inputs NULL without rows", dict(R=0, scores=None, deltas=None, proposals=None, gt_boxes=None, gt_classes=None),
     _NO_ROWS(0)),
    (FF, "sums NULL", dict(sums=None), EINVAL),
    (FF, "counts NULL", dict(counts=None), EINVAL),
    (FF, "status NULL", dict(status=None), EINVAL),
    (FF, "workspace NULL", dict(workspace=None), EINVAL),
    (FF, "workspace misaligned", dict(workspace=_MISALIGNED), EINVAL),
    (FF, "valid call: the workspace is too small", dict(), EWORKSPACE),
    (FB, "no rows: D2B_OK before the gradient pointers", dict(R=0, grad_sums=None, grad_scores=None), 0),
    (FB, "grad_sums NULL", dict(grad_sums=None), EINVAL),
    (FB, "grad_scores NULL", dict(grad_scores=None), EINVAL),
    (FB, "grad_deltas NULL", dict(grad_deltas=None), EINVAL),
]


def _loss_call(lib, entry, kind, **over):
    from detectron2_b200 import _C

    args = dict(_LOSS_PARAMS[entry], loss_type=kind.lt)
    if "lv" in args:  # levels of 10 anchors each
        args.update(label_kind=I8 if kind.i8 else I64, K=1 if kind.i8 else 80)
        lv = _C.DenseLossLevels()
        lv.num_levels = over.pop("num_levels", 1)
        for name, _ in lv._fields_[1:]:
            default = 10 if name == "R" else None if name in ("ctr", "grad_ctr") and kind.lt != LIN else _P
            for l, v in enumerate(over.pop(name, [default] * _C.MAX_LEVELS)):
                getattr(lv, name)[l] = v
        args["lv"] = C.byref(lv)
    args.update(over)
    if args["weights"] is not None:
        args["weights"] = (C.c_float * 5)(*args["weights"])
    return getattr(lib, entry)(*args.values(), None)


def test_loss_entry_points_validate_arguments_without_a_gpu():
    """Every fault of the four box-branch loss entry points gets its status before anything is launched, for each loss type
    and label kind the entry point takes.  Without a GPU a launch attempt returns a positive CUDA error, so a status <= 0
    here also shows that nothing was launched or written (not even the forward's finish).  The workspace queries make no
    CUDA call."""
    import types

    from detectron2_b200 import _C

    lib = _C.lib()
    assert (_C.LOSS_TYPES["smooth_l1"], _C.LOSS_TYPES["giou"], _C.LOSS_LINEAR_GIOU) == (SL1, GIOU, LIN)
    assert (_C.LABELS_I8, _C.LABELS_I64) == (I8, I64)
    for entry, kinds in _LOSS_KINDS.items():
        for lt, i8 in kinds:
            kind = types.SimpleNamespace(bwd=entry in (DB, FB), lt=lt, i8=i8)
            for entries, what, args, want in _LOSS_FAULTS:
                w = want(kind) if callable(want) else want
                if entry in entries and w is not None:
                    got = _loss_call(lib, entry, kind, **args)
                    assert got == w, (entry, what, lt, i8, got)
    lv = _C.DenseLossLevels()
    lv.num_levels, lv.R[0], lv.logits[0], lv.deltas[0] = 1, 10, _P, _P
    size = lib.d2b_dense_loss_workspace_bytes(C.byref(lv), 2, 80, 0)
    assert size > 0 and size % 16 == 0
    lv.ctr[0] = _P  # the query reads no centerness
    assert lib.d2b_dense_loss_workspace_bytes(C.byref(lv), 2, 80, 0) == size
    assert lib.d2b_dense_loss_workspace_bytes(None, 2, 80, 0) == 0
    for n, k, dt in ((-1, 80, 0), (2, 0, 0), (2, 80, 3)):
        assert lib.d2b_dense_loss_workspace_bytes(C.byref(lv), n, k, dt) == 0
    lv.logits[0] = _MISALIGNED
    assert lib.d2b_dense_loss_workspace_bytes(C.byref(lv), 2, 80, 0) == 0
    assert lib.d2b_frcnn_loss_workspace_bytes(0) == lib.d2b_frcnn_loss_workspace_bytes(-1) == 0
    assert lib.d2b_frcnn_loss_workspace_bytes(10) > 0


# ---- the fixture taken from the real reference functions (tests/golden/make_golden_losses.py) ------------------------
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "losses.npz")


def _golden():
    return np.load(GOLDEN)


def _arr(z, key, device):
    return torch.from_numpy(z[key]).to(device)


def _list(z, case, key, device):
    out, i = [], 0
    while "%s__%s%d" % (case, key, i) in z:
        out.append(_arr(z, "%s__%s%d" % (case, key, i), device))
        i += 1
    return out


def _close(a, b, tol):
    a, b = a.detach().cpu().double(), torch.as_tensor(b).double()
    if b.numel() == 0:
        return a.numel() == 0
    return float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-12)


def run_golden_case(z, case, device, tol=1e-6):
    """Runs one fixture case through the reference-shaped wrappers on `device` (CPU: the torch restatement; CUDA: the
    kernels) and checks losses, counts, gradients and assertions against the reference's."""
    from detectron2_b200 import losses as L

    kind = "rpn" if case.startswith("rpn") or case.startswith("rrpn") else case.split("_")[0]
    loss_type = next((t for t in ("giou", "diou", "ciou") if t in case), "smooth_l1")
    raises = int(z[case + "__raises"])
    if kind in ("rpn", "retina"):
        anchors = _list(z, case, "anchors", device)
        labels = _list(z, case, "labels", device)
        gt = _list(z, case, "gt", device)
        logits = [t.requires_grad_(True) for t in _list(z, case, "logits", device)]
        deltas = [t.requires_grad_(True) for t in _list(z, case, "deltas", device)]
        beta = float(z[case + "__beta"])
    if kind == "rpn":
        w = tuple(z[case + "__weights"].tolist())
        call = lambda: L.rpn_losses(anchors, logits, labels, deltas, gt, batch_size_per_image=64, box2box_weights=w,
                                    smooth_l1_beta=beta, box_reg_loss_type=loss_type,
                                    loss_weight={"loss_rpn_cls": 1.0, "loss_rpn_loc": 2.0})
        if raises:
            with pytest.raises(AssertionError):
                call()
            return
        losses, counts = call()
        assert counts == {"num_pos_anchors": int(z[case + "__num_pos"]), "num_neg_anchors": int(z[case + "__num_neg"])}
        for k in ("loss_rpn_cls", "loss_rpn_loc"):
            assert _close(losses[k], z[case + "__" + k], tol), k
        sum(losses.values()).backward()
        for a, b in zip(logits + deltas, _list(z, case, "grad_logits", "cpu") + _list(z, case, "grad_deltas", "cpu")):
            assert _close(a.grad, b, tol)
        return
    if kind == "retina":
        norm = None
        for c in range(int(z[case + "__calls"])):
            for t in logits + deltas:
                t.grad = None
            call = lambda: L.retinanet_losses(anchors, logits, labels, deltas, gt, num_classes=5, loss_normalizer=norm,
                                              smooth_l1_beta=beta, box_reg_loss_type=loss_type)
            if raises:
                with pytest.raises(AssertionError):
                    call()
                return
            losses, num_pos, norm = call()
            pre = "%s_call%d__" % (case, c)
            assert num_pos == int(z[case + "__num_pos"]) and norm == float(z[pre + "normalizer"])
            for k in ("loss_cls", "loss_box_reg"):
                assert _close(losses[k], z[pre + k], tol), k
            sum(losses.values()).backward()
            for a, b in zip(logits + deltas, _list(z, case + "_call%d" % c, "grad_logits", "cpu")
                            + _list(z, case + "_call%d" % c, "grad_deltas", "cpu")):
                assert _close(a.grad, b, tol)
        return
    scores = _arr(z, case + "__scores", device).requires_grad_(True)
    deltas = _arr(z, case + "__deltas", device).requires_grad_(True)
    props, gtb, cls = (_arr(z, case + "__" + k, device) for k in ("props", "gt", "classes"))
    call = lambda: L.fast_rcnn_losses(scores, deltas, props, gtb, cls, box2box_weights=tuple(z[case + "__weights"].tolist()),
                                      smooth_l1_beta=float(z[case + "__beta"]), box_reg_loss_type=loss_type,
                                      loss_weight={"loss_cls": 1.0, "loss_box_reg": 0.5})
    if raises:
        with pytest.raises(AssertionError):
            call()
        return
    losses, st = call()
    for k in ("loss_cls", "loss_box_reg"):
        assert _close(losses[k], z[case + "__" + k], tol), k
    r = cls.numel()
    if r:
        assert st["num_accurate"] / r == float(z[case + "__cls_accuracy"])
        if st["num_fg"]:
            assert st["fg_num_accurate"] / st["num_fg"] == float(z[case + "__fg_cls_accuracy"])
            assert st["num_false_negative"] / st["num_fg"] == float(z[case + "__false_negative"])
    sum(losses.values()).backward()
    assert _close(scores.grad, z[case + "__grad_scores"], tol) and _close(deltas.grad, z[case + "__grad_deltas"], tol)


def golden_case_names():
    return [str(c) for c in _golden()["cases"]]


@pytest.mark.parametrize("case", golden_case_names())
def test_restatement_reproduces_reference_fixture(case):
    run_golden_case(_golden(), case, "cpu")


def test_get_deltas_targets_equal_reference_fixture():
    """Box2BoxTransform[Rotated].get_deltas of the reference, bit for bit."""
    from detectron2_b200 import losses as L

    z = _golden()
    checked = 0
    for case in golden_case_names():
        key = case + "__targets"
        if key not in z or z[key].size == 0:
            continue
        if case.startswith("frcnn"):
            cls = torch.from_numpy(z[case + "__classes"])
            fg = (cls >= 0) & (cls < 6)
            src, tgts = torch.from_numpy(z[case + "__props"])[fg], [torch.from_numpy(z[case + "__gt"])[fg]]
        else:
            src = torch.cat(_list(z, case, "anchors", "cpu"))
            tgts = _list(z, case, "gt", "cpu")
        w = tuple(z[case + "__weights"].tolist()) if case + "__weights" in z else (1.0,) * src.shape[1]
        ours = torch.stack([L._get_deltas(src, t, w) for t in tgts])
        assert torch.equal(ours.reshape(z[key].shape), torch.from_numpy(z[key])), case
        checked += 1
    assert checked >= 8
