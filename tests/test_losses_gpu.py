"""Box-branch loss kernels on the GPU against the torch restatement (the reference's operations) run on the same CUDA
tensors under autograd, at the training sizes of the model zoo: RetinaNet 2 x 201 600 anchors x 80 classes, RPN 2 x 268 569
anchors with the reference's sampling, Fast R-CNN 2 x 512 x 81 class-specific, cascade weights, RRPN and rotated ROI heads."""
import math

import pytest
import torch

import test_losses_host as H

pytestmark = pytest.mark.gpu

DEV = "cuda"


def grid_anchors(image_hw, strides, sizes, ratios):
    """Per-level [H_l * W_l * A, 4] anchors centred on the stride grid (DefaultAnchorGenerator's layout)."""
    out = []
    for s, sz in zip(strides, sizes):
        h, w = math.ceil(image_hw[0] / s), math.ceil(image_hw[1] / s)
        base = []
        for size in sz:
            for r in ratios:
                ww = math.sqrt(size * size / r)
                hh = r * ww
                base.append([-ww / 2, -hh / 2, ww / 2, hh / 2])
        yy, xx = torch.meshgrid(torch.arange(h) * float(s), torch.arange(w) * float(s), indexing="ij")
        shifts = torch.stack([xx, yy, xx, yy], dim=-1).reshape(-1, 1, 4)
        out.append((shifts + torch.tensor(base)).reshape(-1, 4).to(DEV))
    return out


def retina_anchors():
    sizes = [[x, x * 2 ** (1 / 3), x * 2 ** (2 / 3)] for x in (32, 64, 128, 256, 512)]
    return grid_anchors((800, 1344), (8, 16, 32, 64, 128), sizes, (0.5, 1.0, 2.0))


def rpn_anchors():
    return grid_anchors((800, 1344), (4, 8, 16, 32, 64), [[32], [64], [128], [256], [512]], (0.5, 1.0, 2.0))


def gt_scene(n, g, counts=(14, 9), rotated=False):
    out = []
    for i in range(n):
        k = counts[i % len(counts)]
        xy = torch.rand(k, 2, generator=g) * torch.tensor([1100.0, 600.0])
        wh = 20 + torch.rand(k, 2, generator=g) * 300
        if rotated:
            out.append(torch.cat([xy + wh / 2, wh, (torch.rand(k, 1, generator=g) - 0.5) * 180], 1).to(DEV))
        else:
            out.append(torch.cat([xy, xy + wh], 1).to(DEV))
    return out


def leaves(ts):
    return [t.detach().clone().requires_grad_(True) for t in ts]


def rel(a, b):
    a, b = a.detach(), b.detach()
    return float((a - b).abs().max()) / max(float(b.abs().max()), 1e-30)


def retina_inputs(seed=0, dtype=torch.float32, counts=(14, 9)):
    from detectron2_b200 import matching

    g = torch.Generator().manual_seed(seed)
    anchors = retina_anchors()
    gts = gt_scene(2, g, counts)
    classes = [torch.randint(0, 80, (len(b),), generator=g).to(DEV) for b in gts]
    matcher = matching.Matcher([0.4, 0.5], [0, -1, 1], allow_low_quality_matches=True)
    labels, matched = matching.retinanet_label_anchors(anchors, gts, classes, matcher, 80)
    logits = [(torch.randn(2, a.shape[0], 80, generator=g) * 2 - 3).to(DEV, dtype) for a in anchors]
    deltas = [(torch.randn(2, a.shape[0], 4, generator=g) * 0.5).to(DEV, dtype) for a in anchors]
    return anchors, logits, deltas, labels, matched


def test_retinanet_losses_match_restatement():
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = retina_inputs()
    assert sum(a.shape[0] for a in anchors) == 201600
    lx, ld = leaves(logits), leaves(deltas)
    ours, num_pos, norm = L.retinanet_losses(anchors, lx, labels, ld, matched, num_classes=80, loss_normalizer=250.0)
    sum(ours.values()).backward()
    rx, rd = leaves(logits), leaves(deltas)
    ref, ref_pos, ref_norm = L._retinanet_losses_host(torch.cat(anchors), rx, labels, rd, matched, 80, 250.0, 0.25, 2.0,
                                                      (1.0, 1.0, 1.0, 1.0), L._SCALE_CLAMP, "smooth_l1", 0.1)
    sum(ref.values()).backward()
    assert num_pos == ref_pos > 0 and norm == ref_norm
    for k in ref:
        assert rel(ours[k], ref[k]) <= 1e-5, k
    for a, b in zip(lx, rx):
        assert float((a.grad - b.grad).abs().max()) <= 1e-5 * float(b.grad.abs().max())
    for a, b in zip(ld, rd):
        assert rel(a.grad, b.grad) <= 1e-6


def rpn_inputs(seed=1, rotated=False, dtype=torch.float32):
    from detectron2_b200 import matching

    g = torch.Generator().manual_seed(seed)
    if rotated:  # RRPN: rotated anchors at three angles on a coarser grid
        base = rpn_anchors()[2:]
        anchors = []
        for a in base:
            c = torch.cat([(a[:, :2] + a[:, 2:]) / 2, a[:, 2:] - a[:, :2]], 1)
            anchors.append(torch.cat([torch.cat([c, torch.full_like(c[:, :1], ang)], 1) for ang in (-60.0, 0.0, 60.0)]))
    else:
        anchors = rpn_anchors()
    gts = gt_scene(2, g, rotated=rotated)
    matcher = matching.Matcher([0.3, 0.7], [0, -1, 1], allow_low_quality_matches=True)
    torch.manual_seed(seed)
    labels, matched = matching.rpn_label_and_sample_anchors(anchors, gts, [(800, 1344)] * 2, matcher, -1, 256, 0.5)
    d = 5 if rotated else 4
    logits = [torch.randn(2, a.shape[0], generator=g).to(DEV, dtype) for a in anchors]
    deltas = [(torch.randn(2, a.shape[0], d, generator=g) * 0.5).to(DEV, dtype) for a in anchors]
    return anchors, logits, deltas, labels, matched


@pytest.mark.parametrize("rotated,beta", [(False, 0.0), (False, 0.1), (True, 0.0)])
def test_rpn_losses_match_restatement(rotated, beta):
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = rpn_inputs(rotated=rotated)
    if not rotated:
        assert sum(a.shape[0] for a in anchors) == 268569
    w = (1.0, 1.0, 1.0, 1.0, 1.0) if rotated else (1.0, 1.0, 1.0, 1.0)
    lw = {"loss_rpn_cls": 1.0, "loss_rpn_loc": 2.0}
    lx, ld = leaves(logits), leaves(deltas)
    ours, counts = L.rpn_losses(anchors, lx, labels, ld, matched, batch_size_per_image=256, box2box_weights=w,
                                smooth_l1_beta=beta, loss_weight=lw)
    sum(ours.values()).backward()
    rx, rd = leaves(logits), leaves(deltas)
    ref, ref_counts = L._rpn_losses_host(torch.cat(anchors), rx, labels, rd, matched, 256, w, L._SCALE_CLAMP, "smooth_l1",
                                         beta, lw)
    sum(ref.values()).backward()
    assert counts == ref_counts and counts["num_pos_anchors"] > 0
    for k in ref:
        assert rel(ours[k], ref[k]) <= 1e-5, k
    for a, b in zip(lx, rx):
        assert float((a.grad - b.grad).abs().max()) <= 1e-5 * float(b.grad.abs().max())
    for a, b in zip(ld, rd):
        if beta == 0.0:
            assert torch.equal(a.grad, b.grad)  # sign(d) times the same scalar
        else:
            assert rel(a.grad, b.grad) <= 1e-6


def frcnn_inputs(seed=2, r=1024, k=80, rotated=False, agnostic=False, dtype=torch.float32):
    g = torch.Generator().manual_seed(seed)
    d = 5 if rotated else 4
    xy = torch.rand(r, 2, generator=g) * 1000
    wh = 8 + torch.rand(r, 2, generator=g) * 300
    jit = 1 + (torch.rand(r, 2, generator=g) - 0.5) * 0.4
    if rotated:
        props = torch.cat([xy, wh, (torch.rand(r, 1, generator=g) - 0.5) * 360], 1)
        gt = torch.cat([xy + wh * 0.1, wh * jit, props[:, 4:] + 30 * (torch.rand(r, 1, generator=g) - 0.5)], 1)
    else:
        props = torch.cat([xy, xy + wh], 1)
        gt = torch.cat([xy + wh * 0.05, xy + wh * jit], 1)
    cls = torch.randint(0, k, (r,), generator=g)
    cls[torch.rand(r, generator=g) < 0.75] = k  # background
    scores = torch.randn(r, k + 1, generator=g) * 2
    scores[:7] = 0.0  # argmax ties: the first index wins
    deltas = torch.randn(r, d if agnostic else k * d, generator=g) * 0.3
    return [t.to(DEV) for t in (scores.to(dtype), deltas.to(dtype), props, gt, cls)]


@pytest.mark.parametrize("rotated,agnostic,beta,weights", [
    (False, False, 0.0, (10.0, 10.0, 5.0, 5.0)),
    (False, True, 0.0, (10.0, 10.0, 5.0, 5.0)),
    (False, False, 0.1, (20.0, 20.0, 10.0, 10.0)),
    (False, False, 0.0, (30.0, 30.0, 15.0, 15.0)),
    (True, False, 0.0, (10.0, 10.0, 5.0, 5.0, 1.0)),
])
def test_fast_rcnn_losses_match_restatement(rotated, agnostic, beta, weights):
    from detectron2_b200 import losses as L

    scores, deltas, props, gt, cls = frcnn_inputs(rotated=rotated, agnostic=agnostic)
    lw = {"loss_cls": 1.0, "loss_box_reg": 0.5}
    s1, d1 = leaves([scores, deltas])
    ours, stats = L.fast_rcnn_losses(s1, d1, props, gt, cls, box2box_weights=weights, smooth_l1_beta=beta, loss_weight=lw)
    sum(ours.values()).backward()
    s2, d2 = leaves([scores, deltas])
    ref, ref_stats = L._fast_rcnn_losses_host(s2, d2, props, gt, cls, weights, L._SCALE_CLAMP, "smooth_l1", beta, lw)
    sum(ref.values()).backward()
    assert stats == ref_stats and stats["num_fg"] > 0
    for k in ref:
        assert rel(ours[k], ref[k]) <= 1e-5, k
    assert float((s1.grad - s2.grad).abs().max()) <= 1e-5 * float(s2.grad.abs().max())
    if beta == 0.0:
        assert torch.equal(d1.grad, d2.grad)
    else:
        assert rel(d1.grad, d2.grad) <= 1e-6


def test_fast_rcnn_no_rows_and_assertions():
    from detectron2_b200 import losses as L

    scores, deltas, props, gt, cls = frcnn_inputs(r=64)
    s, d = leaves([scores[:0], deltas[:0]])
    losses, stats = L.fast_rcnn_losses(s, d, props[:0], gt[:0], cls[:0])
    assert float(losses["loss_cls"]) == 0.0 and float(losses["loss_box_reg"]) == 0.0 and stats["num_fg"] == 0
    sum(losses.values()).backward()
    assert s.grad.shape == s.shape
    bad = props.clone()
    fg = int(torch.nonzero(cls < 80)[0])
    bad[fg, 2] = bad[fg, 0]  # a zero-width foreground proposal: get_deltas' assertion
    with pytest.raises(AssertionError):
        L.fast_rcnn_losses(scores, deltas, bad, gt, cls)
    bg = int(torch.nonzero(cls == 80)[0])
    bad = props.clone()
    bad[bg, 2] = bad[bg, 0]  # background proposals are not regressed: no assertion
    L.fast_rcnn_losses(scores, deltas, bad, gt, cls)


def test_dense_edge_cases():
    """Ignored rows holding NaN logits, an image without GT, a batch without positives, a zero-width anchor."""
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = retina_inputs(seed=5, counts=(6, 0))
    assert int(((labels[1] >= 0) & (labels[1] < 80)).sum()) == 0  # the second image has no GT: all background
    ign = torch.nonzero(labels[0] == -1)[:, 0]
    assert ign.numel() > 0
    logits[0][0, ign[ign < logits[0].shape[1]]] = float("nan")
    lx, ld = leaves(logits), leaves(deltas)
    ours, num_pos, _ = L.retinanet_losses(anchors, lx, labels, ld, matched, num_classes=80)
    sum(ours.values()).backward()
    assert all(bool(torch.isfinite(v)) for v in ours.values()) and all(bool(torch.isfinite(x.grad).all()) for x in lx)
    rx, rd = leaves(logits), leaves(deltas)
    ref, ref_pos, _ = L._retinanet_losses_host(torch.cat(anchors), rx, labels, rd, matched, 80, 100.0, 0.25, 2.0,
                                               (1.0,) * 4, L._SCALE_CLAMP, "smooth_l1", 0.1)
    assert num_pos == ref_pos and all(rel(ours[k], ref[k]) <= 1e-5 for k in ref)
    # a batch without positives: regression loss 0, normaliser max(0, 1)
    bg = [torch.where(lb >= 0, torch.full_like(lb, 80), lb) for lb in labels]
    ours, num_pos, norm = L.retinanet_losses(anchors, logits, bg, deltas, matched, num_classes=80)
    assert num_pos == 0 and float(ours["loss_box_reg"]) == 0.0 and norm == 100.0 * 0.9 + 1 * (1 - 0.9)
    # a zero-width anchor anywhere (positive or not) trips get_deltas' assertion
    bad = [a.clone() for a in anchors]
    bad[4][3, 2] = bad[4][3, 0]
    with pytest.raises(AssertionError):
        L.retinanet_losses(bad, logits, labels, deltas, matched, num_classes=80)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_half_precision_inputs_read_in_place(dtype):
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = retina_inputs(seed=3, dtype=dtype)
    lx, ld = leaves(logits), leaves(deltas)
    ours, _, _ = L.retinanet_losses(anchors, lx, labels, ld, matched, num_classes=80)
    sum(ours.values()).backward()
    fx, fd = leaves([x.float() for x in logits]), leaves([d.float() for d in deltas])
    ref, _, _ = L.retinanet_losses(anchors, fx, labels, fd, matched, num_classes=80)
    sum(ref.values()).backward()
    for k in ref:
        assert rel(ours[k], ref[k]) <= 1e-5, k
    for a, b in zip(lx + ld, fx + fd):
        assert a.grad.dtype == dtype
        assert torch.equal(a.grad, b.grad.to(dtype))  # the fp32 gradient rounded once
    scores, deltas_f, props, gt, cls = frcnn_inputs(dtype=dtype)
    s1, d1 = leaves([scores, deltas_f])
    ours, _ = L.fast_rcnn_losses(s1, d1, props, gt, cls)
    sum(ours.values()).backward()
    s2, d2 = leaves([scores.float(), deltas_f.float()])
    ref, _ = L.fast_rcnn_losses(s2, d2, props, gt, cls)
    sum(ref.values()).backward()
    assert all(rel(ours[k], ref[k]) <= 1e-5 for k in ref)
    assert s1.grad.dtype == dtype and torch.equal(s1.grad, s2.grad.to(dtype)) and torch.equal(d1.grad, d2.grad.to(dtype))


def test_runs_are_bitwise_reproducible():
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = retina_inputs(seed=4)
    outs = []
    for _ in range(2):
        lx, ld = leaves(logits), leaves(deltas)
        losses, _, _ = L.retinanet_losses(anchors, lx, labels, ld, matched, num_classes=80)
        sum(losses.values()).backward()
        outs.append([losses["loss_cls"], losses["loss_box_reg"]] + [x.grad for x in lx + ld])
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_fixed_forms_capture_in_a_cuda_graph():
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = retina_inputs(seed=6)
    lab, gtb = torch.stack(labels), torch.stack(matched)
    ra, rl, rd, rlab, rgt = rpn_inputs(seed=7)
    rlab, rgt = torch.stack(rlab), torch.stack(rgt)
    fr = frcnn_inputs(seed=8)
    ema = torch.full((1,), 100.0, dtype=torch.float64, device=DEV)

    def step():
        a, pos, _ = L.retinanet_losses_fixed(anchors, logits, lab, deltas, gtb, ema, num_classes=80)
        b, _, _, _ = L.rpn_losses_fixed(ra, rl, rlab, rd, rgt, batch_size_per_image=256)
        c, counts, _ = L.fast_rcnn_losses_fixed(*fr)
        return torch.stack(list(a.values()) + list(b.values()) + list(c.values())), pos, counts

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        eager, pos, counts = step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out, gpos, gcounts = step()
    ema.fill_(100.0)
    expect = 100.0
    p = int(pos)
    for _ in range(3):
        graph.replay()
        expect = expect * 0.9 + max(p, 1) * (1 - 0.9)
    torch.cuda.synchronize()
    assert float(ema.item()) == expect
    assert torch.equal(gpos, pos) and torch.equal(gcounts, counts)
    # the last replay normalises by the third EMA value; the RPN and Fast R-CNN losses are the eager ones
    assert torch.equal(out[2:], eager[2:])
    ema_first = 100.0 * 0.9 + max(p, 1) * (1 - 0.9)
    assert rel(out[:2] * float(torch.tensor(expect, dtype=torch.float32)),
               eager[:2] * float(torch.tensor(ema_first, dtype=torch.float32))) <= 1e-6


@pytest.mark.parametrize("case", H.golden_case_names())
def test_kernels_reproduce_reference_fixture(case):
    tol = 1e-4 if "giou" in case else 1e-5
    H.run_golden_case(H._golden(), case, DEV, tol=tol)


def test_giou_losses_match_restatement():
    """GIoU regression through the decode at RetinaNet and Fast R-CNN sizes: losses within 1e-5, gradients within 1e-4."""
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = retina_inputs(seed=9)
    lx, ld = leaves(logits), leaves(deltas)
    ours, _, _ = L.retinanet_losses(anchors, lx, labels, ld, matched, num_classes=80, box_reg_loss_type="giou")
    sum(ours.values()).backward()
    rx, rd = leaves(logits), leaves(deltas)
    ref, _, _ = L._retinanet_losses_host(torch.cat(anchors), rx, labels, rd, matched, 80, 100.0, 0.25, 2.0, (1.0,) * 4,
                                         L._SCALE_CLAMP, "giou", 0.1)
    sum(ref.values()).backward()
    for k in ref:
        assert rel(ours[k], ref[k]) <= 1e-5, k
    for a, b in zip(ld, rd):
        assert rel(a.grad, b.grad) <= 1e-4
    # Fast R-CNN, class-specific, with some dw / dh above the clamp (no gradient there) and one exactly at it (passes)
    scores, fdeltas, props, gt, cls = frcnn_inputs(seed=10)
    fg = torch.nonzero(cls < 80)[:, 0]
    c0, c1 = int(cls[fg[0]]), int(cls[fg[1]])
    fdeltas[fg[0], c0 * 4 + 2] = 5.0 * 6.0
    fdeltas[fg[1], c1 * 4 + 3] = torch.tensor(L._SCALE_CLAMP, dtype=torch.float32) * 5.0
    s1, d1 = leaves([scores, fdeltas])
    ours, _ = L.fast_rcnn_losses(s1, d1, props, gt, cls, box_reg_loss_type="giou")
    sum(ours.values()).backward()
    s2, d2 = leaves([scores, fdeltas])
    ref, _ = L._fast_rcnn_losses_host(s2, d2, props, gt, cls, (10.0, 10.0, 5.0, 5.0), L._SCALE_CLAMP, "giou", 0.0, None)
    sum(ref.values()).backward()
    for k in ref:
        assert rel(ours[k], ref[k]) <= 1e-5, k
    assert rel(d1.grad, d2.grad) <= 1e-4
    assert float(d1.grad[fg[0], c0 * 4 + 2]) == 0.0 and float(d2.grad[fg[0], c0 * 4 + 2]) == 0.0


def test_out_of_range_labels_raise():
    from detectron2_b200 import losses as L

    anchors, logits, deltas, labels, matched = retina_inputs(seed=11)
    bad = [lb.clone() for lb in labels]
    bad[1][5] = 81  # F.one_hot(num_classes=81) rejects it
    with pytest.raises(RuntimeError):
        L.retinanet_losses(anchors, logits, bad, deltas, matched, num_classes=80)
    scores, fdeltas, props, gt, cls = frcnn_inputs(seed=12, r=64)
    cls = cls.clone()
    cls[3] = 81
    with pytest.raises(RuntimeError):
        L.fast_rcnn_losses(scores, fdeltas, props, gt, cls)
