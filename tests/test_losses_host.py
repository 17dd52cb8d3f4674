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


def test_new_entry_points_validate_arguments_without_a_gpu():
    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL = -1
    w = (C.c_float * 5)(1, 1, 1, 1, 1)
    lv = _C.DenseLossLevels()
    lv.num_levels = 1
    lv.R[0] = 10
    dummy = C.c_void_p(16)  # never dereferenced: every call below fails its checks first
    lv.logits[0] = lv.deltas[0] = 16
    args = dict(N=2, K=80, D=4, dt=0, kind=_C.LABELS_I64, gamma=2.0, alpha=0.25, beta=0.1, lt=0)

    def fwd(lvp=C.byref(lv), **kw):
        a = dict(args, **kw)
        return lib.d2b_dense_loss_forward(lvp, a["N"], a["K"], a["D"], a["dt"], dummy, dummy, dummy, a["kind"], a["gamma"],
                                          a["alpha"], a["beta"], a["lt"], 4.135, w, dummy, dummy, dummy, dummy, dummy, dummy, 0, None)

    assert fwd(lvp=None) == EINVAL
    assert fwd(D=3) == EINVAL
    assert fwd(dt=3) == EINVAL
    assert fwd(kind=_C.LABELS_I8) == EINVAL  # int8 labels need K = 1
    assert fwd(gamma=-1.0) == EINVAL
    assert fwd(beta=float("nan")) == EINVAL
    assert fwd(K=0) == EINVAL
    assert fwd(lt=2) == EINVAL  # no such loss type
    assert fwd(lt=1, D=5) == EINVAL  # GIoU is axis-aligned only
    assert fwd(lt=1) == -2
    assert fwd() == -2  # workspace too small (checked after the arguments)
    lv.logits[0] = 8  # logits must be 16-byte aligned
    assert fwd() == EINVAL
    lv.logits[0] = 16
    lv.num_levels = _C.MAX_LEVELS + 1
    assert fwd() == EINVAL
    lv.num_levels = 1
    assert lib.d2b_dense_loss_workspace_bytes(C.byref(lv), 2, 80, 0) > 0
    assert lib.d2b_dense_loss_backward(C.byref(lv), 2, 80, 4, 0, dummy, dummy, dummy, _C.LABELS_I64, 2.0, 0.25, 0.1, 0,
                                       4.135, w,
                                       dummy, dummy, None) == EINVAL  # no gradient buffers
    assert lib.d2b_frcnn_loss_workspace_bytes(0) == 0
    frc = lambda R, K, kreg, D, dt, lt=0: lib.d2b_frcnn_loss_forward(dummy, dummy, R, K, kreg, D, dt, dummy, dummy, dummy,
                                                                     0.0, lt, 4.135, w, *([dummy] * 7), dummy, 0, None)
    assert frc(-1, 80, 80, 4, 0) == EINVAL
    assert frc(10, 80, 3, 4, 0) == EINVAL  # kreg must be 1 or K
    assert frc(10, 80, 80, 6, 0) == EINVAL
    assert frc(10, 80, 80, 4, 9) == EINVAL
    assert frc(10, 80, 80, 5, 0, lt=1) == EINVAL
    assert frc(10, 80, 80, 4, 0) == -2
    assert lib.d2b_frcnn_loss_backward(dummy, dummy, 10, 80, 80, 4, 0, dummy, dummy, dummy, 0.0, 0, 4.135, w, dummy,
                                       dummy, None, None, None) == EINVAL


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
