"""GPU tests of the FCOS kernels: d2b_fcos_assign, d2b_dense_loss_* (D2B_LOSS_LINEAR_GIOU) and d2b_dense_prepare
(D2B_SELECT_LINEAR) against the fixture taken from the real reference methods and against the torch restatement on the
same CUDA tensors."""
import pytest
import torch

import fcos_ref as R

pytestmark = pytest.mark.gpu

DEV = "cuda"
NUM_CLASSES = 80


def _points(h=800, w=1344, strides=(8, 16, 32, 64, 128)):
    """DefaultAnchorGenerator's point boxes of P3-P7 (22 400 points at 800 x 1344)."""
    out = []
    for s in strides:
        gh, gw = -(-h // s), -(-w // s)
        ys, xs = torch.meshgrid(torch.arange(gh, dtype=torch.float32) * s, torch.arange(gw, dtype=torch.float32) * s,
                                indexing="ij")
        c = torch.stack([xs.reshape(-1), ys.reshape(-1)], 1)
        out.append(torch.cat([c - s / 2, c + s / 2], 1).to(DEV))
    return out


def _gt(g, n, h=800, w=1344):
    xy = torch.rand(n, 2, generator=g) * torch.tensor([w * 0.9, h * 0.9])
    wh = 8 + torch.rand(n, 2, generator=g) ** 2 * torch.tensor([w * 0.6, h * 0.6])
    return torch.cat([xy, xy + wh], 1).to(DEV)


def _scene(G, seed=0):
    g = torch.Generator().manual_seed(seed)
    anchors = _points()
    gts = [_gt(g, G), _gt(g, G // 2)]  # uneven counts per image
    cls = [torch.randint(0, NUM_CLASSES, (len(b),), generator=g).to(DEV) for b in gts]
    return g, anchors, gts, cls


def _preds(g, anchors, n=2, dtype=torch.float32):
    logits = [(torch.randn(n, len(a), NUM_CLASSES, generator=g) * 2 - 2).to(DEV, dtype) for a in anchors]
    deltas = [(torch.randn(n, len(a), 4, generator=g) + 0.5).to(DEV, dtype) for a in anchors]
    ctr = [torch.randn(n, len(a), 1, generator=g).to(DEV, dtype) for a in anchors]
    return logits, deltas, ctr


def _leaves(ts):
    return [t.detach().clone().requires_grad_(True) for t in ts]


def test_kernels_reproduce_fixture():
    from detectron2_b200 import fcos as F

    z = R.load()
    an = R.anchors(z, DEV)
    for case in ("a", "nf"):
        labels, boxes = F.fcos_label_anchors(an, [t.to(DEV) for t in R.lst(z, case, "gt")],
                                             [t.to(DEV) for t in R.lst(z, case, "cls")], num_classes=R.K)
        R.check_labels(z, case, labels, boxes)
    R.run_loss_case(z, "loss_f32", DEV, 1e-5, 1e-4)
    R.run_loss_case(z, "loss_nan_delta", DEV, 1e-5, 1e-4)
    R.run_loss_case(z, "loss_f16", DEV, 1e-5, 2e-3)  # fp16 predictions read in place; fp16 gradients


@pytest.mark.parametrize("G", [0, 14, 100, 1000])
def test_assign_loss_backward_match_restatement(G):
    from detectron2_b200 import fcos as F

    g, anchors, gts, cls = _scene(G, seed=G)
    an = torch.cat(anchors)
    counts = [len(a) for a in anchors]
    labels, boxes = F.fcos_label_anchors(anchors, gts, cls, num_classes=NUM_CLASSES)
    want_l, want_b, want_m = F._fcos_label_anchors_host(an, counts, gts, cls, NUM_CLASSES)
    for i in range(2):
        assert torch.equal(labels[i], want_l[i]) and torch.equal(boxes[i], want_b[i])
    gt_pad = torch.zeros((2, max(G, 1), 4), device=DEV)
    cls_pad = torch.zeros((2, max(G, 1)), dtype=torch.int64, device=DEV)
    for i, (b, c) in enumerate(zip(gts, cls)):
        gt_pad[i, :len(b)], cls_pad[i, :len(c)] = b, c
    cnt = torch.tensor([len(b) for b in gts], device=DEV)
    _, _, matches = F.fcos_label_anchors_fixed(anchors, gt_pad, cnt, cls_pad, num_classes=NUM_CLASSES)
    assert torch.equal(matches, torch.stack(want_m))

    logits, deltas, ctr = _preds(g, anchors)
    lx, ld, lc = _leaves(logits), _leaves(deltas), _leaves(ctr)
    got, pos, norm = F.fcos_losses(anchors, lx, labels, ld, boxes, lc, num_classes=NUM_CLASSES)
    hx, hd, hc = _leaves(logits), _leaves(deltas), _leaves(ctr)
    want, hpos, hnorm = F._fcos_losses_host(an, hx, want_l, hd, want_b, hc, NUM_CLASSES, 300.0, 0.25, 2.0)
    assert pos == hpos and norm == hnorm
    for k in want:
        assert R.close(got[k], want[k], 1e-5), (k, float(got[k]), float(want[k]))
    sum(got.values()).backward()
    sum(want.values()).backward()
    for a, b in zip(lx + ld + lc, hx + hd + hc):
        assert R.close(a.grad, b.grad, 1e-4)
    if G == 0:
        assert pos == 0 and float(got["loss_fcos_loc"].detach()) == 0.0 and float(got["loss_fcos_ctr"].detach()) == 0.0


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_half_inputs_are_read_in_place(dtype):
    from detectron2_b200 import fcos as F

    g, anchors, gts, cls = _scene(100, seed=5)
    labels, boxes = F.fcos_label_anchors(anchors, gts, cls, num_classes=NUM_CLASSES)
    logits, deltas, ctr = _preds(g, anchors, dtype=dtype)
    lx, ld, lc = _leaves(logits), _leaves(deltas), _leaves(ctr)
    got, _, _ = F.fcos_losses(anchors, lx, labels, ld, boxes, lc, num_classes=NUM_CLASSES)
    fx, fd, fc = _leaves([t.float() for t in logits]), _leaves([t.float() for t in deltas]), _leaves([t.float() for t in ctr])
    want, _, _ = F.fcos_losses(anchors, fx, labels, fd, boxes, fc, num_classes=NUM_CLASSES)
    for k in want:
        assert R.close(got[k], want[k], 1e-5), k
    sum(got.values()).backward()
    sum(want.values()).backward()
    for a, b in zip(lx + ld + lc, fx + fd + fc):
        assert a.grad.dtype == dtype and a.grad.shape == a.shape
        assert torch.equal(a.grad, b.grad.to(dtype))


def test_repeated_runs_are_bitwise_identical():
    from detectron2_b200 import fcos as F

    g, anchors, gts, cls = _scene(100, seed=9)
    logits, deltas, ctr = _preds(g, anchors)
    runs = []
    for _ in range(3):
        labels, boxes = F.fcos_label_anchors(anchors, gts, cls, num_classes=NUM_CLASSES)
        lx, ld, lc = _leaves(logits), _leaves(deltas), _leaves(ctr)
        losses, _, _ = F.fcos_losses(anchors, lx, labels, ld, boxes, lc, num_classes=NUM_CLASSES)
        sum(losses.values()).backward()
        runs.append([torch.stack(labels), torch.stack(boxes)] + [v.detach() for v in losses.values()] +
                    [t.grad for t in lx + ld + lc])
    for r in runs[1:]:
        assert all(torch.equal(a, b) for a, b in zip(runs[0], r))


def test_graph_capture_replays_on_new_gt_boxes():
    from detectron2_b200 import fcos as F

    g, anchors, gts, cls = _scene(100, seed=13)
    an = torch.cat(anchors)
    counts = [len(a) for a in anchors]
    logits, deltas, ctr = _preds(g, anchors)
    lx, ld, lc = _leaves(logits), _leaves(deltas), _leaves(ctr)
    gmax = 128
    s_gt = torch.zeros((2, gmax, 4), device=DEV)
    s_cls = torch.zeros((2, gmax), dtype=torch.int64, device=DEV)
    s_cnt = torch.zeros((2,), dtype=torch.int64, device=DEV)
    ema = torch.full((1,), 300.0, dtype=torch.float64, device=DEV)

    def load(gts_, cls_):
        s_gt.zero_()
        s_cls.zero_()
        for i, (b, c) in enumerate(zip(gts_, cls_)):
            s_gt[i, :len(b)], s_cls[i, :len(c)] = b, c
        s_cnt.copy_(torch.tensor([len(b) for b in gts_]))

    def step():
        labels, boxes, _ = F.fcos_label_anchors_fixed(an, s_gt, s_cnt, s_cls, num_classes=NUM_CLASSES,
                                                      level_counts=counts)
        losses, num_pos, status = F.fcos_losses_fixed(an, lx, labels, ld, boxes, lc, ema, num_classes=NUM_CLASSES)
        total = sum(losses.values())
        grads = torch.autograd.grad(total, lx + ld + lc)
        return [labels, boxes, total.detach(), num_pos] + list(grads)

    load(gts, cls)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static_out = step()
    g2 = torch.Generator().manual_seed(99)
    new_gts = [_gt(g2, 60), _gt(g2, 17)]
    new_cls = [torch.randint(0, NUM_CLASSES, (len(b),), generator=g2).to(DEV) for b in new_gts]
    load(new_gts, new_cls)
    ema.fill_(300.0)
    graph.replay()
    torch.cuda.synchronize()
    replayed = [t.clone() for t in static_out]
    ema.fill_(300.0)
    eager = step()
    assert all(torch.equal(a, b) for a, b in zip(replayed, eager))
    want_l, _, _ = F._fcos_label_anchors_host(an, counts, new_gts, new_cls, NUM_CLASSES)
    assert torch.equal(replayed[0], torch.stack(want_l))


def test_inference_matches_host_path_and_fixture():
    from detectron2_b200 import fcos as F
    from detectron2_b200.dense_inference import _dense_detector_inference_host

    z = R.load()
    an = R.anchors(z, DEV)
    logits, ctr, deltas = R.lst(z, "inf", "logits", DEV), R.lst(z, "inf", "ctr", DEV), R.lst(z, "inf", "deltas", DEV)
    sizes = [(128, 128)] * 2
    dets = F.fcos_inference(an, logits, deltas, ctr, sizes)
    host = _dense_detector_inference_host(an, F._scores(logits, ctr), deltas, sizes, 0.2, 1000, 0.6, 100,
                                          transform="linear")
    for i, (d, h) in enumerate(zip(dets, host)):
        assert torch.equal(d.pred_boxes, h.pred_boxes) and torch.equal(d.scores, h.scores)
        assert torch.equal(d.pred_classes, h.pred_classes)
        # the fixture was taken on the CPU, whose vectorised sigmoid / sqrt may differ from CUDA's in the last bit
        assert R.same(d.pred_boxes, R.arr(z, "inf%d__boxes" % i))
        assert R.close(d.scores, R.arr(z, "inf%d__scores" % i), 1e-6)
        assert R.same(d.pred_classes, R.arr(z, "inf%d__classes" % i))
    assert len(dets[0].scores) > 0
    # the same scores on the same device: bit for bit
    ours = F._scores(logits, ctr)
    for x, y, o in zip(logits, ctr, ours):
        assert torch.equal(o[0], torch.sqrt(x[0].clone().sigmoid_() * y[0].clone().sigmoid_()))
