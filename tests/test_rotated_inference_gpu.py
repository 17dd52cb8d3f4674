"""Rotated RRPN proposal selection and rotated Fast R-CNN inference on the GPU kernels: bit-exact against the fixtures from
the real reference functions, against the CPU oracle restatements at realistic sizes, against the host restatements (GPU NMS
on both sides), in a CUDA graph, for thresholds that IoU 0 passes, and across the D2B_MAX_IMAGES chunking."""
import pytest
import torch

import rotated_inference_ref as rref
from test_rotated_inference_host import check_frcnn, frcnn_fixture, rrpn_fixture

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
T = torch.from_numpy


def rand_rotated(g, shape, hi_xy, wmax, lo_xy=(-20.0, -20.0)):
    lo = torch.tensor(lo_xy)
    ctr = torch.rand(*shape, 2, generator=g) * (torch.tensor(hi_xy) - lo) + lo
    wh = torch.rand(*shape, 2, generator=g) * wmax + 1.0
    a = (torch.rand(*shape, 1, generator=g) - 0.5) * 400
    a = torch.where(torch.rand(*shape, 1, generator=g) < 0.4, (torch.rand(*shape, 1, generator=g) - 0.5) * 3, a)
    return torch.cat([ctr, wh, a], -1)


def check_rrpn(res, ref):
    assert len(res) == len(ref)
    for r, (b, s) in zip(res, ref):
        assert torch.equal(r.proposal_boxes.tensor.cpu(), b.cpu()) and torch.equal(r.objectness_logits.cpu(), s.cpu())


def check_dets(res, rows, ref):
    assert len(res) == len(ref)
    for det, rw, (b, s, c, r) in zip(res, rows, ref):
        assert torch.equal(det.pred_boxes.cpu(), b.cpu()) and torch.equal(det.scores.cpu(), s.cpu())
        assert torch.equal(det.pred_classes.cpu(), c.cpu()) and torch.equal(rw.cpu(), r.cpu())


# ------------------------------------------------------------------------------------------------------------ fixtures
def test_rrpn_golden(golden):
    from detectron2_b200.rrpn import find_top_rrpn_proposals

    d, props, logits, sizes, thr, pre, post, mbs = rrpn_fixture(golden)
    res = find_top_rrpn_proposals([p.to(DEV) for p in props], [x.to(DEV) for x in logits], sizes, thr, pre, post, mbs, False)
    check_rrpn(res, [(T(d[f"boxes_img{i}"]), T(d[f"scores_img{i}"])) for i in range(2)])
    with pytest.raises(FloatingPointError):
        find_top_rrpn_proposals([p.to(DEV) for p in props], [x.to(DEV) for x in logits], sizes, thr, pre, post, mbs, True)
    # the same image twice, and an image whose every candidate is removed (non-finite scores)
    idx = [0, 0, 1]
    lg = [x[idx].clone() for x in logits]
    for x in lg:
        x[2] = float("nan")
    res = find_top_rrpn_proposals([p[idx].to(DEV) for p in props], [x.to(DEV) for x in lg], [sizes[0]] * 2 + [sizes[1]], thr,
                                  pre, post, mbs, False)
    check_rrpn(res, [(T(d["boxes_img0"]), T(d["scores_img0"]))] * 2 + [(torch.zeros(0, 5), torch.zeros(0))])


def test_rotated_fast_rcnn_golden(golden):
    from detectron2_b200 import rotated_fast_rcnn as rfr

    d, thr, nms_thr, topk, shapes = frcnn_fixture(golden)
    for tk, tag in ((topk, ""), (-1, "_all")):
        # image 0 twice and image 2 (no candidate) in one call; the class-agnostic image alone
        res, rows = rfr.fast_rcnn_inference_rotated([T(d[f"boxes{i}"]).to(DEV) for i in (0, 2, 0)],
                                                    [T(d[f"scores{i}"]).to(DEV) for i in (0, 2, 0)],
                                                    [shapes[0], shapes[2], shapes[0]], thr, nms_thr, tk)
        for j, i in enumerate([0, 2, 0]):
            check_frcnn(d, i, tag, res[j].pred_boxes, res[j].scores, res[j].pred_classes, rows[j])
        det, rows1 = rfr.fast_rcnn_inference_single_image_rotated(T(d["boxes1"]).to(DEV), T(d["scores1"]).to(DEV), shapes[1],
                                                                  thr, nms_thr, tk)
        check_frcnn(d, 1, tag, det.pred_boxes, det.scores, det.pred_classes, rows1)


# ------------------------------------------------------------------------------------------- realistic sizes vs oracle
def _rrpn_inputs(seed, n=2, per_level=(6000, 3000, 1500, 800, 400), sizes=((800, 1333), (750, 1200))):
    g = torch.Generator().manual_seed(seed)
    props = [rand_rotated(g, (n, a), (1400.0, 850.0), 300.0) for a in per_level]
    logits = [torch.randn(n, a, generator=g) for a in per_level]
    return props, logits, [tuple(s) for s in sizes[:n]]


@pytest.mark.parametrize("pre", [1000, 2000])
def test_rrpn_fpn_size_vs_oracle(pre):
    from detectron2_b200.rrpn import find_top_rrpn_proposals

    props, logits, sizes = _rrpn_inputs(40 + pre)
    ref = rref.find_top_rrpn_proposals(props, logits, sizes, 0.7, pre, 1000, 0.0, False)
    res = find_top_rrpn_proposals([p.to(DEV) for p in props], [x.to(DEV) for x in logits], sizes, 0.7, pre, 1000, 0.0, False)
    assert min(len(r) for r in res) > 500
    check_rrpn(res, ref)


def _frcnn_inputs(seed, n=4, r=1000, k=15, agnostic=False):
    g = torch.Generator().manual_seed(seed)
    boxes, scores = [], []
    for _ in range(n):
        base = rand_rotated(g, (60,), (1300.0, 780.0), 250.0)
        nb = 1 if agnostic else k
        b = base[torch.randint(0, 60, (r,), generator=g)][:, None, :] + torch.randn(r, nb, 5, generator=g) * torch.tensor(
            [6.0, 6.0, 4.0, 4.0, 5.0])
        b[..., 2:4] = b[..., 2:4].abs() + 1.0
        boxes.append(b.reshape(r, nb * 5))
        scores.append(torch.softmax(torch.randn(r, k + 1, generator=g) * 2.0, dim=1))
    boxes[0][3, 1] = float("nan")
    scores[1][7] = float("inf")
    return boxes, scores, [(800, 1333), (750, 1200), (800, 1100), (640, 1333)][:n]


@pytest.mark.parametrize("agnostic", [False, True])
def test_rotated_fast_rcnn_size_vs_oracle(agnostic):
    from detectron2_b200 import rotated_fast_rcnn as rfr

    boxes, scores, shapes = _frcnn_inputs(7 + int(agnostic), agnostic=agnostic)
    ref = rref.fast_rcnn_inference_rotated(boxes, scores, shapes, 0.05, 0.5, 100)
    res, rows = rfr.fast_rcnn_inference_rotated([b.to(DEV) for b in boxes], [s.to(DEV) for s in scores], shapes, 0.05, 0.5,
                                                100)
    assert sum(len(r) for r in res) > 300
    check_dets(res, rows, ref)


# ------------------------------------------------------------------------------------ kernels vs the host restatements
def test_kernels_match_host_restatements_with_gpu_nms():
    from detectron2_b200 import rotated_fast_rcnn as rfr
    from detectron2_b200 import rrpn

    props, logits, sizes = _rrpn_inputs(5, n=3, per_level=(3000, 800, 200), sizes=((800, 1333), (750, 1200), (600, 900)))
    args = ([p.to(DEV) for p in props], [x.to(DEV) for x in logits], sizes, 0.7, 1000, 700, 1.0, False)
    res, ref = rrpn.find_top_rrpn_proposals(*args), rrpn._find_top_rrpn_proposals_host(*args)
    check_rrpn(res, [(r.proposal_boxes.tensor, r.objectness_logits) for r in ref])
    # image 1 overflows the candidate slots (every one of its 700 x 15 pairs passes the threshold): redone exactly
    boxes, scores, shapes = _frcnn_inputs(11, n=3, r=700)
    scores[1] = torch.full_like(scores[1], 0.5)
    scores[1][:, :-1] += torch.randperm(700 * 15, generator=torch.Generator().manual_seed(0)).reshape(700, 15) * 1e-5
    bd, sd = [b.to(DEV) for b in boxes], [s.to(DEV) for s in scores]
    for tk in (100, -1):
        res, rows = rfr.fast_rcnn_inference_rotated(bd, sd, shapes, 0.05, 0.5, tk)
        hres, hrows = rfr._fast_rcnn_inference_rotated_host(bd, sd, shapes, 0.05, 0.5, tk)
        check_dets(res, rows, [(h.pred_boxes, h.scores, h.pred_classes, r) for h, r in zip(hres, hrows)])
    out = rfr.fast_rcnn_inference_rotated_fixed(bd, sd, shapes, 0.05, 0.5, 100)
    assert out["n_cand"][1].item() > out["cap"] >= out["n_cand"][0].item()


def test_candidate_cap_overflow_vs_oracle():
    # the image whose 700 x 15 pairs all pass the threshold is redone on the exact path: same results as the reference loop
    from detectron2_b200 import rotated_fast_rcnn as rfr

    boxes, scores, shapes = _frcnn_inputs(11, n=3, r=700)
    scores[1] = torch.full_like(scores[1], 0.5)
    scores[1][:, :-1] += torch.randperm(700 * 15, generator=torch.Generator().manual_seed(0)).reshape(700, 15) * 1e-5
    res, rows = rfr.fast_rcnn_inference_rotated([b.to(DEV) for b in boxes], [s.to(DEV) for s in scores], shapes, 0.05, 0.5,
                                                100)
    ref = rref.fast_rcnn_inference_single_image_rotated(boxes[1], scores[1], shapes[1], 0.05, 0.5, 100)
    check_dets([res[1]], [rows[1]], [ref])


# ---------------------------------------------------------------------------------------------------------- CUDA graphs
def test_fixed_forms_replay_in_cuda_graph():
    from detectron2_b200 import rotated_fast_rcnn as rfr
    from detectron2_b200 import rrpn

    props, logits, sizes = _rrpn_inputs(77, per_level=(2000, 600, 150))
    pd, ld = [p.to(DEV) for p in props], [x.to(DEV) for x in logits]
    hw = torch.tensor([[float(h), float(w)] for (h, w) in sizes], device=DEV)
    boxes, scores, shapes = _frcnn_inputs(78, n=3, r=400)
    bd, sd = [b.to(DEV) for b in boxes], [s.to(DEV) for s in scores]
    fhw = torch.tensor([[float(h), float(w)] for (h, w) in shapes], device=DEV)
    rrpn.find_top_rrpn_proposals_fixed(pd, ld, hw, 0.7, 1000, 500, 0.0)  # warm-up outside the capture
    rfr.fast_rcnn_inference_rotated_fixed(bd, sd, fhw, 0.05, 0.5, 100)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            ob, osc, cnt, _ = rrpn.find_top_rrpn_proposals_fixed(pd, ld, hw, 0.7, 1000, 500, 0.0)
            out = rfr.fast_rcnn_inference_rotated_fixed(bd, sd, fhw, 0.05, 0.5, 100)
    for rep in range(2):
        if rep == 1:  # new inputs in the captured buffers: reversed image order
            for t in pd + ld + bd + sd:
                t.copy_(t.flip(0).clone())
            hw.copy_(hw.flip(0).clone())
            fhw.copy_(fhw.flip(0).clone())
        graph.replay()
        torch.cuda.synchronize()
        szs = sizes if rep == 0 else list(reversed(sizes))
        ref = rrpn.find_top_rrpn_proposals([p.clone() for p in pd], [x.clone() for x in ld], szs, 0.7, 1000, 500, 0.0, False)
        for i, r in enumerate(ref):
            c = int(cnt[i])
            assert c == len(r) > 0 and torch.equal(ob[i, :c], r.proposal_boxes.tensor)
            assert torch.equal(osc[i, :c], r.objectness_logits) and (ob[i, c:] == 0).all()
        shp = shapes if rep == 0 else list(reversed(shapes))
        res, rows = rfr.fast_rcnn_inference_rotated([b.clone() for b in bd], [s.clone() for s in sd], shp, 0.05, 0.5, 100)
        for i in range(3):
            c = int(out["counts"][i])
            assert c == len(res[i]) > 0
            assert torch.equal(out["boxes"][i, :c], res[i].pred_boxes) and torch.equal(out["scores"][i, :c], res[i].scores)
            assert torch.equal(out["classes"][i, :c], res[i].pred_classes) and torch.equal(out["rows"][i, :c], rows[i])


# ------------------------------------------------------------------------------------ thr <= 0, and 65 images (chunks)
@pytest.mark.parametrize("nms_thr", [0.0, -0.1])
def test_thresholds_that_iou_zero_passes(nms_thr):
    from detectron2_b200 import rotated_fast_rcnn as rfr
    from detectron2_b200.rrpn import find_top_rrpn_proposals

    props, logits, sizes = _rrpn_inputs(3, per_level=(900, 300, 100))
    ref = rref.find_top_rrpn_proposals(props, logits, sizes, nms_thr, 400, 100, 0.0, False)
    res = find_top_rrpn_proposals([p.to(DEV) for p in props], [x.to(DEV) for x in logits], sizes, nms_thr, 400, 100, 0.0,
                                  False)
    check_rrpn(res, ref)
    boxes, scores, shapes = _frcnn_inputs(4, n=2, r=300)
    ref = rref.fast_rcnn_inference_rotated(boxes, scores, shapes, 0.05, nms_thr, -1)
    res, rows = rfr.fast_rcnn_inference_rotated([b.to(DEV) for b in boxes], [s.to(DEV) for s in scores], shapes, 0.05, nms_thr,
                                                -1)
    check_dets(res, rows, ref)


def test_65_images_in_chunks():
    from detectron2_b200 import rotated_fast_rcnn as rfr
    from detectron2_b200.rrpn import find_top_rrpn_proposals

    boxes, scores, shapes = _frcnn_inputs(21, n=4, r=120, k=5)
    idx = [i % 4 for i in range(65)]
    res, rows = rfr.fast_rcnn_inference_rotated([boxes[i].to(DEV) for i in idx], [scores[i].to(DEV) for i in idx],
                                                [shapes[i] for i in idx], 0.05, 0.5, 50)
    ref = rref.fast_rcnn_inference_rotated(boxes, scores, shapes, 0.05, 0.5, 50)
    check_dets(res, rows, [ref[i] for i in idx])
    props, logits, sizes = _rrpn_inputs(22, n=2, per_level=(500, 120))
    idx = [i % 2 for i in range(65)]
    ref = rref.find_top_rrpn_proposals(props, logits, sizes, 0.7, 200, 100, 0.0, False)
    res = find_top_rrpn_proposals([p[idx].to(DEV) for p in props], [x[idx].to(DEV) for x in logits], [sizes[i] for i in idx],
                                  0.7, 200, 100, 0.0, False)
    check_rrpn(res, [ref[i] for i in idx])
