"""d2b_match_boxes on the GPU: bit-exact against the fixture from the REAL reference functions, against the torch
restatement run on CUDA at full training size (axis-aligned and rotated), sampling under the same CUDA seed,
proposal_append_gt fed by find_top_rpn_proposals_fixed's device counts, the status flag and CUDA-graph replay."""
import pytest
import torch

import test_matching_host as H

pytestmark = pytest.mark.gpu
T = torch.from_numpy
DEV = torch.device("cuda:0")


def rand_xyxy(g, n, h=800.0, w=1344.0, smax=400.0):
    ctr = torch.rand(n, 2, generator=g, device=DEV) * torch.tensor([w, h], device=DEV)
    wh = torch.rand(n, 2, generator=g, device=DEV) * smax + 4
    return torch.cat([ctr - wh / 2, ctr + wh / 2], 1)


def rpn_anchors(g, n=268569):  # p2-p6 of 800 x 1344, 3 per location
    return rand_xyxy(g, n, smax=600.0)


def reference_loop(anchors, gts, matcher, sizes=None, boundary=-1, classes=None, num_classes=None):
    """The reference's per-image loop on CUDA with the torch restatement: matches, labels (+ boundary), boxes, classes."""
    from detectron2_b200 import matching as mt

    out = []
    for i, g in enumerate(gts):
        m, lab = matcher(mt._iou(g, anchors))
        if boundary >= 0:
            lab[~mt.inside_box(anchors, sizes[i], boundary)] = -1
        boxes = g[m] if len(g) else torch.zeros_like(anchors)
        c = mt._class_targets(m, lab, classes[i], num_classes) if classes is not None else None
        out.append((m, lab, boxes, c))
    return out


def fused(anchors, gts, matcher, **kw):
    from detectron2_b200 import matching as mt

    gt, cnt = mt._pad(gts, anchors.shape[-1], DEV)
    return mt.match_boxes_fixed(gt, cnt, anchors, matcher, **kw)


def test_fixture_bit_exact():
    from detectron2_b200 import matching as mt

    d = H.load(lambda n: __import__("numpy").load(__file__.rsplit("/", 1)[0] + "/golden/matching.npz"))[0]
    H.check_deterministic(d, DEV)  # RetinaNet and cascade wrappers run the fused kernels on CUDA
    _, sizes, gts, cls, rgts, rcls = H.load(lambda n: d)
    anchors = T(d["anchors"]).to(DEV)
    for tag, cfg in (("rpn", H.RPN_CFG), ("roi", H.ROI_CFG)):
        m, lab, _, _, st = fused(anchors, [g.to(DEV) for g in gts], mt.Matcher(*cfg))
        assert not st.any()
        for i in range(H.NIMG):
            H.eq(m[i], T(d[f"matcher_{tag}_matches{i}"]), (tag, i))
            H.eq(lab[i], T(d[f"matcher_{tag}_labels{i}"]), (tag, i))
    for bt in (-1, 0):
        _, boxes = mt.rpn_label_and_sample_anchors(anchors, [g.to(DEV) for g in gts], sizes, mt.Matcher(*H.RPN_CFG), bt, 64,
                                                   0.5)
        for i in range(H.NIMG):
            H.eq(boxes[i], T(d[f"rpn_b{bt + 1}_boxes{i}"]), ("rpn boxes", bt, i))
    _, boxes = mt.rpn_label_and_sample_anchors(T(d["ranchors"]).to(DEV), [g.to(DEV) for g in rgts], sizes,
                                               mt.Matcher(*H.RPN_CFG), -1, 64, 0.5)
    for i in range(H.NIMG):
        H.eq(boxes[i], T(d[f"rrpn_boxes{i}"]), ("rrpn boxes", i))


@pytest.mark.parametrize("G", [0, 1, 7, 100, 2000])
def test_rpn_full_size_against_torch_restatement(G):
    from detectron2_b200 import matching as mt

    g = torch.Generator(device=DEV).manual_seed(G)
    anchors = rpn_anchors(g)
    gts = [rand_xyxy(g, G), rand_xyxy(g, max(G // 2, 0))]
    if G >= 7:
        gts[0][3] = gts[0][1]  # duplicate GT
        gts[0][4] = anchors[1000]  # a GT equal to an anchor: IoU exactly 1
    sizes = [(800, 1344), (800, 1200)]
    matcher = mt.Matcher(*H.RPN_CFG)
    for bt in (-1, 0):
        m, lab, boxes, _, st = fused(anchors, gts, matcher, image_hw=sizes, boundary_thresh=bt)
        assert not st.any()
        for i, (rm, rl, rb, _) in enumerate(reference_loop(anchors, gts, matcher, sizes, bt)):
            assert torch.equal(m[i], rm) and torch.equal(lab[i], rl) and torch.equal(boxes[i], rb), (G, bt, i)


def test_rpn_65_images_full_size():
    """65 images (one more than D2B_MAX_IMAGES of the inference kernels) at the full 268 569 anchors, with the boundary rule
    and the class gather."""
    from detectron2_b200 import matching as mt

    g = torch.Generator(device=DEV).manual_seed(65)
    anchors = rpn_anchors(g)
    gts = [rand_xyxy(g, int(k)) for k in torch.randint(0, 30, (65,), generator=g, device=DEV).tolist()]
    cls = [torch.randint(0, 80, (len(x),), generator=g, device=DEV) for x in gts]
    sizes = [(800, 1344) if i % 2 else (704, 1216) for i in range(65)]
    matcher = mt.Matcher(*H.RPN_CFG)
    m, lab, boxes, c, st = fused(anchors, gts, matcher, image_hw=sizes, boundary_thresh=0,
                                 gt_classes=mt._pad_classes(cls, DEV), num_classes=80)
    assert not st.any()
    ref = reference_loop(anchors, gts, matcher, sizes, 0, classes=cls, num_classes=80)
    for i, (rm, rl, rb, rc) in enumerate(ref):
        assert torch.equal(m[i], rm) and torch.equal(lab[i], rl) and torch.equal(boxes[i], rb), i
        assert torch.equal(c[i], rc), i


def test_retinanet_full_size():
    from detectron2_b200 import matching as mt

    g = torch.Generator(device=DEV).manual_seed(3)
    anchors = rand_xyxy(g, 201600, smax=500.0)
    gts = [rand_xyxy(g, 40), rand_xyxy(g, 0)]
    cls = [torch.randint(0, 80, (len(x),), generator=g, device=DEV) for x in gts]
    matcher = mt.Matcher(*H.RETINA_CFG)
    labels, boxes = mt.retinanet_label_anchors(anchors, gts, cls, matcher, 80)
    for i, (rm, rl, rb, rc) in enumerate(reference_loop(anchors, gts, matcher, classes=cls, num_classes=80)):
        assert torch.equal(labels[i], rc) and torch.equal(boxes[i], rb), i


def rand_rot(g, n, smax=300.0):
    c = torch.rand(n, 2, generator=g, device=DEV) * torch.tensor([1344.0, 800.0], device=DEV)
    wh = torch.rand(n, 2, generator=g, device=DEV) * smax + 4
    a = (torch.rand(n, 1, generator=g, device=DEV) - 0.5) * 180
    return torch.cat([c, wh, a], 1)


def test_rrpn_full_size_against_box_iou_rotated():
    from detectron2_b200 import matching as mt

    g = torch.Generator(device=DEV).manual_seed(5)
    anchors = rand_rot(g, 805707)
    gts = [rand_rot(g, 20), rand_rot(g, 3)]
    gts[0][1] = gts[0][0]
    gts[0][2] = anchors[77]
    matcher = mt.Matcher(*H.RPN_CFG)
    m, lab, boxes, _, st = fused(anchors, gts, matcher)
    assert not st.any()
    for i, (rm, rl, rb, _) in enumerate(reference_loop(anchors, gts, matcher)):
        assert torch.equal(m[i], rm) and torch.equal(lab[i], rl) and torch.equal(boxes[i], rb), i


def test_sampling_matches_restatement_under_the_same_cuda_seed():
    from detectron2_b200 import matching as mt

    g = torch.Generator(device=DEV).manual_seed(9)
    anchors = rpn_anchors(g, 100000)
    gts = [rand_xyxy(g, 12), rand_xyxy(g, 0), rand_xyxy(g, 5)]
    sizes = [(800, 1344)] * 3
    for rotated in (False, True):
        a = rand_rot(g, 100000) if rotated else anchors
        gg = [rand_rot(g, len(x)) for x in gts] if rotated else gts
        torch.manual_seed(21)
        labels, boxes = mt.rpn_label_and_sample_anchors(a, gg, sizes, mt.Matcher(*H.RPN_CFG), -1 if rotated else 0, 256,
                                                        0.5)
        torch.manual_seed(21)
        for i, (rm, rl, rb, _) in enumerate(reference_loop(a, gg, mt.Matcher(*H.RPN_CFG), sizes, -1 if rotated else 0)):
            assert torch.equal(labels[i], mt._rpn_subsample(rl, 256, 0.5)) and torch.equal(boxes[i], rb), (rotated, i)
        props = [rand_rot(g, 2000) if rotated else rand_xyxy(g, 2000) for _ in gg]
        cls = [torch.randint(0, 80, (len(x),), generator=g, device=DEV) for x in gg]
        torch.manual_seed(22)
        res = mt.label_and_sample_proposals(props, gg, cls, mt.Matcher(*H.ROI_CFG), 80, 512, 0.25)
        torch.manual_seed(22)
        for i, (p, x, c) in enumerate(zip(props, gg, cls)):
            pa = torch.cat([p, x])
            m, lab = mt.Matcher(*H.ROI_CFG)(mt._iou(x, pa))
            rc = mt._class_targets(m, lab, c, 80)
            fg, bg = mt.subsample_labels(rc, 512, 0.25, 80)
            idx = torch.cat([fg, bg])
            assert torch.equal(res[i][0], idx) and torch.equal(res[i][1], rc[idx]) and torch.equal(res[i][2], m[idx])


def test_append_gt_fed_by_rpn_device_counts():
    from detectron2_b200 import matching as mt
    from detectron2_b200.proposal_utils import find_top_rpn_proposals_fixed

    g = torch.Generator(device=DEV).manual_seed(13)
    sizes = [(800, 1344), (640, 960)]
    props = [rand_xyxy(g, 2 * a).reshape(2, a, 4) for a in (3000, 800)]
    logits = [torch.randn(2, p.shape[1], generator=g, device=DEV) for p in props]
    boxes, _, counts, _ = find_top_rpn_proposals_fixed(props, logits, sizes, 0.7, 1000, 500, 0.0)
    gts = [rand_xyxy(g, 9), rand_xyxy(g, 4)]
    cls = [torch.randint(0, 80, (len(x),), generator=g, device=DEV) for x in gts]
    gt, gc = mt._pad(gts, 4, DEV)
    matcher = mt.Matcher(*H.ROI_CFG)
    m, lab, mb, c, st = mt.match_boxes_fixed(gt, gc, boxes, matcher, pred_count=counts, append_gt=True,
                                             gt_classes=mt._pad_classes(cls, DEV), num_classes=80)
    assert not st.any()
    for i, k in enumerate(counts.tolist()):
        pa = torch.cat([boxes[i, :k], gts[i]])
        rm, rl = matcher(mt._iou(gts[i], pa))
        v = pa.shape[0]
        assert torch.equal(m[i, :v], rm) and torch.equal(lab[i, :v], rl) and torch.equal(mb[i, :v], gts[i][rm])
        assert torch.equal(c[i, :v], mt._class_targets(rm, rl, cls[i], 80))
        assert (lab[i, v:] == -1).all() and (m[i, v:] == 0).all() and (c[i, v:] == -1).all()


def test_status_flag():
    from detectron2_b200 import matching as mt

    d = __import__("numpy").load(__file__.rsplit("/", 1)[0] + "/golden/matching.npz")
    good = torch.tensor([[1.0, 1.0, 5.0, 5.0]], device=DEV)
    for k in ("xyxy_inf", "rot_nan", "rot_negative_iou"):
        gt, pred = T(d[f"bad_{k}_gt"]).to(DEV), T(d[f"bad_{k}_pred"]).to(DEV)
        ok = torch.tensor([[5.0, 5.0, 4.0, 4.0, 0.0]], device=DEV) if gt.shape[1] == 5 else good
        _, _, _, _, st = fused(pred, [gt, ok], mt.Matcher(*H.RPN_CFG))
        assert st.tolist() == [1, 0], k
        with pytest.raises(AssertionError):
            mt.rpn_label_and_sample_anchors(pred, [gt], [(100, 100)], mt.Matcher(*H.RPN_CFG), -1, 8, 0.5)


def test_cuda_graph_replay_on_new_gt():
    from detectron2_b200 import matching as mt

    g = torch.Generator(device=DEV).manual_seed(17)
    anchors = rpn_anchors(g, 60000)
    matcher = mt.Matcher(*H.RPN_CFG)
    gt = torch.zeros((2, 50, 4), device=DEV)
    cnt = torch.zeros((2,), dtype=torch.int64, device=DEV)
    hw = torch.tensor([[800.0, 1344.0], [800.0, 1344.0]], device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        mt.match_boxes_fixed(gt, cnt, anchors, matcher, image_hw=hw, boundary_thresh=0)  # warm-up
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            out = mt.match_boxes_fixed(gt, cnt, anchors, matcher, image_hw=hw, boundary_thresh=0)
    torch.cuda.current_stream().wait_stream(s)
    for k0, k1 in ((7, 50), (0, 3), (31, 0)):
        gts = [rand_xyxy(g, k0), rand_xyxy(g, k1)]
        gt.zero_()
        gt[0, :k0], gt[1, :k1] = gts[0], gts[1]
        cnt.copy_(torch.tensor([k0, k1]))
        graph.replay()
        torch.cuda.synchronize()
        m, lab, boxes, _, st = out
        assert not st.any()
        for i, (rm, rl, rb, _) in enumerate(reference_loop(anchors, gts, matcher, [(800, 1344)] * 2, 0)):
            assert torch.equal(m[i], rm) and torch.equal(lab[i], rl) and torch.equal(boxes[i], rb), (k0, k1, i)
