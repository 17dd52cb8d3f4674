"""Per-op micro-benchmarks at the BASELINE.json / SURVEY 8(d) shapes, next to the reference's GPU kernels where the
image has them (torchvision CUDA ops = the reference's backend for roi_align / nms / deform_conv2d).

    python tools/bench_ops.py [--out profiles/r1_ops.md]

Timing: CUDA events around REP back-to-back launches after warm-up; inputs rotate over NBUF copies (> L2) for the
bandwidth-bound ops.  Reported: our time, reference-GPU time (tv), algorithmic bytes / flops and achieved fraction of
the measured peaks (MEASURED_PEAKS.json).
"""
import argparse
import json
import math
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
import detectron2_b200.layers as L  # noqa: E402
from detectron2_b200.poolers import ROIPooler  # noqa: E402

DEV = "cuda"


def timeit(fn, rep=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(rep):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / rep * 1e3  # us


def ref_pooler_grad(fg, b, out, scales, tv):
    sizes = torch.sqrt((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1]))
    lv = torch.floor(4 + torch.log2(sizes / 224 + 1e-8)).clamp(2, 5).to(torch.int64) - 2
    r5 = torch.cat([torch.zeros(len(b), 1, device=DEV), b], 1)
    res = torch.zeros(len(b), fg[0].shape[1], out, out, device=DEV)
    for l, s in enumerate(scales):
        inds = torch.nonzero(lv == l, as_tuple=True)[0]
        res = res.index_put((inds,), tv.roi_align(fg[l], r5[inds], (out, out), s, 0, True))
    return res


def per_level_rotated_pooler(feats, rois, scales, out):
    """This library's multi-level rotated ROIPooler before the fused kernels: the reference's per-level loop
    (poolers.py:245-263) over the single-level ROIAlignRotated layer."""
    sizes = torch.sqrt(rois[:, 3] * rois[:, 4])
    lv = torch.floor(4 + torch.log2(sizes / 224 + 1e-8)).clamp(2, 5).to(torch.int64) - 2
    res = feats[0].new_zeros((rois.shape[0], feats[0].shape[1], out, out))
    for l, s in enumerate(scales):
        inds = torch.nonzero(lv == l, as_tuple=True)[0]
        res.index_put_((inds,), L.ROIAlignRotated((out, out), s, 0)(feats[l], rois[inds]))
    return res


def bench_rotated_pooler(add, refgpu):
    """Rotated ROIPooler, 2 images x 512 RoIs, 7x7, p2..p5 at 256 channels: the fused op, this library's former per-level loop
    and (tools/bench_ref_gpu.py) the same loop over the reference's CUDA roi_align_rotated kernels."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    from bench_ref_gpu import rotated_pooler_inputs

    feats, boxes, scales = rotated_pooler_inputs()
    rois = torch.cat([torch.cat([torch.full((len(b), 1), float(i), device=DEV), b], 1) for i, b in enumerate(boxes)])
    pooler = ROIPooler(7, scales, 0, "ROIAlignRotated")
    name = "ROIPooler ROIAlignRotated %s 7x7 K=2x512 (p2..p5)"
    t = timeit(lambda: pooler(feats, boxes))
    add(name % "fwd", t, refgpu.get(name % "fwd"), "fused; ref = per-level loop over reference csrc CUDA")
    t = timeit(lambda: per_level_rotated_pooler(feats, rois, scales, 7))
    add(name % "fwd" + " former loop", t, refgpu.get(name % "fwd"), "per-level loop over our ROIAlignRotated")
    fg = [f.clone().requires_grad_(True) for f in feats]
    y = pooler(fg, boxes)
    go = torch.randn_like(y)
    t = timeit(lambda: torch.autograd.grad(y, fg, go, retain_graph=True))
    add(name % "bwd", t, refgpu.get(name % "bwd"), "fused; ref = per-level reference csrc CUDA backward")
    y2 = per_level_rotated_pooler(fg, rois, scales, 7)
    t = timeit(lambda: torch.autograd.grad(y2, fg, go, retain_graph=True))
    add(name % "bwd" + " former loop", t, refgpu.get(name % "bwd"), "autograd of the per-level loop over our ROIAlignRotated")


def _clip_rotated_ref(b, h, w):
    """RotatedBoxes.clip as the reference writes it (structures/rotated_boxes.py:279-303): torch.where(...)[0] + indexing."""
    b = b.clone()
    b[:, 4] = (b[:, 4] + 180.0) % 360.0 - 180.0
    idx = torch.where(torch.abs(b[:, 4]) <= 1.0)[0]
    x1, y1 = (b[idx, 0] - b[idx, 2] / 2.0).clamp(0, w), (b[idx, 1] - b[idx, 3] / 2.0).clamp(0, h)
    x2, y2 = (b[idx, 0] + b[idx, 2] / 2.0).clamp(0, w), (b[idx, 1] + b[idx, 3] / 2.0).clamp(0, h)
    b[idx, 0], b[idx, 1] = (x1 + x2) / 2.0, (y1 + y2) / 2.0
    b[idx, 2], b[idx, 3] = torch.min(b[idx, 2], x2 - x1), torch.min(b[idx, 3], y2 - y1)
    return b


def bench_rotated_inference(add):
    """find_top_rrpn_proposals and fast_rcnn_inference_rotated against the reference's per-image loops (rrpn.py:90-126,
    rotated_fast_rcnn.py:98-132) on the same GPU over this library's batched_nms_rotated."""
    from detectron2_b200.rotated_fast_rcnn import fast_rcnn_inference_rotated
    from detectron2_b200.rrpn import find_top_rrpn_proposals

    gb = torch.Generator().manual_seed(13)
    # p2..p6 of an 800 x 1344 input, 9 anchors per location (3 ratios x 3 angles)
    per_level = [9 * h * w for h, w in ((200, 336), (100, 168), (50, 84), (25, 42), (13, 21))]
    pp, ll = [], []
    for a in per_level:
        ctr = torch.rand(2, a, 2, generator=gb) * torch.tensor([1400.0, 850.0]) - 20
        wh = torch.exp(torch.rand(2, a, 2, generator=gb) * 5.0) + 0.5
        ang = (torch.randint(0, 3, (2, a, 1), generator=gb).float() - 1) * 60 + torch.randn(2, a, 1, generator=gb) * 5
        pp.append(torch.cat([ctr, wh, ang], 2).to(DEV))
        ll.append(torch.randn(2, a, generator=gb).to(DEV))
    szs = [(800, 1344), (800, 1344)]

    def ref_rrpn(pre, post):
        bi = torch.arange(2, device=DEV)
        ts, tp, lv = [], [], []
        for lid, (p_i, l_i) in enumerate(zip(pp, ll)):
            k = min(l_i.shape[1], pre)
            s_i, idx = l_i.topk(k, dim=1)
            tp.append(p_i[bi[:, None], idx]); ts.append(s_i); lv.append(torch.full((k,), lid, dtype=torch.int64, device=DEV))
        ts, tp, lv = torch.cat(ts, 1), torch.cat(tp, 1), torch.cat(lv, 0)
        outs = []
        for n_, (h_, w_) in enumerate(szs):
            b_, s_, l_ = tp[n_], ts[n_], lv
            v_ = torch.isfinite(b_).all(1) & torch.isfinite(s_)
            if not v_.all():
                b_, s_, l_ = b_[v_], s_[v_], l_[v_]
            b_ = _clip_rotated_ref(b_, h_, w_)
            kp = (b_[:, 2] > 0) & (b_[:, 3] > 0)
            if kp.sum().item() != len(b_):
                b_, s_, l_ = b_[kp], s_[kp], l_[kp]
            kk_ = L.batched_nms_rotated(b_, s_, l_, 0.7)[:post]
            outs.append((b_[kk_], s_[kk_]))
        return outs

    for pre, post, tag in ((2000, 2000, "train"), (1000, 1000, "test")):
        t = timeit(lambda: find_top_rrpn_proposals(pp, ll, szs, 0.7, pre, post, 0.0, tag == "train"), rep=10)
        tr = timeit(lambda: ref_rrpn(pre, post), rep=10)
        add("find_top_rrpn_proposals 2 img x p2-p6 800x1344 x 9 anchors, top %d/%d (%s)" % (pre, post, tag), t, tr,
            "ref = reference per-image loop over our batched_nms_rotated")
    k_cls, r = 15, 1000
    boxes, scores = [], []
    for _ in range(2):
        base = torch.cat([torch.rand(80, 2, generator=gb) * torch.tensor([1300.0, 780.0]),
                          8 + torch.rand(80, 2, generator=gb) * 250, (torch.rand(80, 1, generator=gb) - 0.5) * 180], 1)
        b = base[torch.randint(0, 80, (r,), generator=gb)][:, None, :] + torch.randn(r, k_cls, 5, generator=gb) * torch.tensor(
            [6.0, 6.0, 4.0, 4.0, 3.0])
        boxes.append(b.reshape(r, k_cls * 5).to(DEV))
        scores.append(torch.softmax(torch.randn(r, k_cls + 1, generator=gb) * 2.0, dim=1).to(DEV))
    shapes = [(800, 1344), (800, 1344)]

    def ref_frcnn():
        res = []
        for b_, s_, (h_, w_) in zip(boxes, scores, shapes):
            v_ = torch.isfinite(b_).all(1) & torch.isfinite(s_).all(1)
            if not v_.all():
                b_, s_ = b_[v_], s_[v_]
            s_ = s_[:, :-1]
            bb = _clip_rotated_ref(b_.reshape(-1, 5), h_, w_).view(-1, k_cls, 5)
            fm = s_ > 0.05
            fi = fm.nonzero()
            bb, sc = bb[fm], s_[fm]
            kk_ = L.batched_nms_rotated(bb, sc, fi[:, 1], 0.5)[:100]
            res.append((bb[kk_], sc[kk_], fi[kk_, 1], fi[kk_, 0]))
        return res

    t = timeit(lambda: fast_rcnn_inference_rotated(boxes, scores, shapes, 0.05, 0.5, 100), rep=10)
    tr = timeit(ref_frcnn, rep=10)
    add("fast_rcnn_inference_rotated 2 img x 1000 rows x 15 classes", t, tr,
        "ref = reference per-image loop over our batched_nms_rotated")


def bench_matching(add):
    """Fused matching (d2b_match_boxes through detectron2_b200.matching) against the reference's per-image loop of torch
    ops on the same GPU (pairwise_iou + Matcher + inside_box + the box / class gathers; the rotated IoU of that loop is
    this library's d2b_box_iou_rotated).  Both sides stop before the sampling, which is the same torch code on both."""
    from detectron2_b200 import matching as mt

    g = torch.Generator(device=DEV).manual_seed(0)

    def xyxy(n, smax):
        c = torch.rand(n, 2, generator=g, device=DEV) * torch.tensor([1344.0, 800.0], device=DEV)
        wh = torch.rand(n, 2, generator=g, device=DEV) * smax + 4
        return torch.cat([c - wh / 2, c + wh / 2], 1)

    def rot(n, smax):
        c = torch.rand(n, 2, generator=g, device=DEV) * torch.tensor([1344.0, 800.0], device=DEV)
        wh = torch.rand(n, 2, generator=g, device=DEV) * smax + 4
        return torch.cat([c, wh, (torch.rand(n, 1, generator=g, device=DEV) - 0.5) * 180], 1)

    def ref_loop(preds, gts, matcher, sizes=None, bt=-1, cls=None, num_classes=80):
        out = []
        for i, gt in enumerate(gts):
            p = preds[i] if isinstance(preds, list) else preds
            m, lab = matcher(mt._iou(gt, p))
            if bt >= 0:
                lab[~mt.inside_box(p, sizes[i], bt)] = -1
            c = mt._class_targets(m, lab, cls[i], num_classes) if cls is not None else None
            out.append((m, lab, gt[m], c))
        return out

    def fused(preds, gts, matcher, **kw):
        gt, cnt = mt._pad(gts, gts[0].shape[-1], DEV)
        if isinstance(preds, list):
            pr, pc = mt._pad(preds, preds[0].shape[-1], DEV)
            return mt.match_boxes_fixed(gt, cnt, pr, matcher, pred_count=pc, **kw)
        return mt.match_boxes_fixed(gt, cnt, preds, matcher, **kw)

    sizes = [(800, 1344), (800, 1344)]
    anchors = xyxy(268569, 600.0)
    for G in (7, 100):
        gts = [xyxy(G, 400.0), xyxy(G, 400.0)]
        m = mt.Matcher([0.3, 0.7], [0, -1, 1], True)
        t = timeit(lambda: fused(anchors, gts, m, image_hw=sizes, boundary_thresh=0), rep=10)
        tr = timeit(lambda: ref_loop(anchors, gts, m, sizes, 0), rep=10)
        add("match RPN 2 img x 268569 anchors, G = %d" % G, t, tr, "labels + boxes, boundary 0")
    ret_anchors = xyxy(201600, 500.0)
    gts = [xyxy(40, 400.0), xyxy(40, 400.0)]
    cls = [torch.randint(0, 80, (40,), generator=g, device=DEV) for _ in gts]
    m = mt.Matcher([0.4, 0.5], [0, -1, 1], True)
    gcls = mt._pad_classes(cls, DEV)
    t = timeit(lambda: fused(ret_anchors, gts, m, gt_classes=gcls, num_classes=80), rep=10)
    tr = timeit(lambda: ref_loop(ret_anchors, gts, m, cls=cls), rep=10)
    add("match RetinaNet 2 img x 201600 anchors, G = 40", t, tr, "labels + boxes + classes")
    props = [xyxy(2000, 400.0), xyxy(2000, 400.0)]
    m = mt.Matcher([0.5], [0, 1], False)
    t = timeit(lambda: fused(props, gts, m, append_gt=True, gt_classes=gcls, num_classes=80), rep=10)
    tr = timeit(lambda: ref_loop([torch.cat([p, x]) for p, x in zip(props, gts)], gts, m, cls=cls), rep=10)
    add("match ROI heads 2 img x (2000 + 40) proposals", t, tr, "proposal_append_gt, classes")
    ms = [mt.Matcher([th], [0, 1], False) for th in (0.5, 0.6, 0.7)]
    t = timeit(lambda: [fused(props, gts, mm, gt_classes=gcls, num_classes=80) for mm in ms], rep=10)
    tr = timeit(lambda: [ref_loop(props, gts, mm, cls=cls) for mm in ms], rep=10)
    add("match cascade 3 stages x 2 img x 2000 proposals", t, tr, "classes + boxes")
    ranchors = rot(805707, 500.0)
    rgts = [rot(20, 300.0), rot(20, 300.0)]
    m = mt.Matcher([0.3, 0.7], [0, -1, 1], True)
    t = timeit(lambda: fused(ranchors, rgts, m), rep=5, warm=1)
    tr = timeit(lambda: ref_loop(ranchors, rgts, m), rep=5, warm=1)
    add("match RRPN 2 img x 805707 anchors, G = 20", t, tr,
        "%.2f G rotated IoU pairs/s (fused)" % (2 * 805707 * 20 / t * 1e-3))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "r2_ops.md"))
    ap.add_argument("--rotated-inference-only", action="store_true", help="only the rotated RRPN / Fast R-CNN inference rows")
    ap.add_argument("--matching-only", action="store_true", help="only the anchor / proposal matching rows")
    args = ap.parse_args()
    if args.rotated_inference_only or args.matching_only:
        def show(name, ours_us, ref_us, note=""):
            print("%-58s ours %9.1f us   ref-gpu %9.1f us   %s" % (name, ours_us, ref_us, note), flush=True)

        print(torch.cuda.get_device_name(0), flush=True)
        (bench_matching if args.matching_only else bench_rotated_inference)(show)
        return
    try:
        import torchvision
        tv = torchvision.ops
    except Exception:
        tv = None
    peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    hbm = peaks.get("hbm_gbs", 6650.0)
    rows = []
    # the reference's own CUDA kernels (rotated ops, deform conv, paste): timed in a separate process (tools/bench_ref_gpu.py)
    import subprocess
    refgpu = {}
    try:
        subprocess.run([sys.executable, os.path.join(ROOT, "tools", "bench_ref_gpu.py")], timeout=600, capture_output=True)
        refgpu = json.load(open(os.path.join(ROOT, "gpurun_out", "ref_gpu.json")))
    except Exception as e:
        print("reference GPU kernels not timed:", e)

    def add(name, ours_us, ref_us, note=""):
        rows.append((name, ours_us, ref_us, note))
        print("%-58s ours %9.1f us   ref-gpu %s   %s" % (name, ours_us, ("%9.1f us" % ref_us) if ref_us else "      n/a", note), flush=True)

    g = torch.Generator().manual_seed(0)
    # ---- cfg1: single-level RoIAlign 512 boxes over 1x256x200x304
    x = torch.rand(1, 256, 200, 304, generator=g).to(DEV)
    k = 512
    cx, cy = torch.rand(k, generator=g) * 1216, torch.rand(k, generator=g) * 800
    w, h = 16 + torch.rand(k, generator=g) * 300, 16 + torch.rand(k, generator=g) * 300
    rois = torch.stack([torch.zeros(k), (cx - w / 2).clamp(0, 1216), (cy - h / 2).clamp(0, 800), (cx + w / 2).clamp(0, 1216),
                        (cy + h / 2).clamp(0, 800)], 1).to(DEV)
    for sr in (0, 2):
        op = L.ROIAlign((7, 7), 0.25, sr, True)
        t = timeit(lambda: op(x, rois))
        tr = timeit(lambda: tv.roi_align(x, rois, (7, 7), 0.25, sr, True)) if tv else None
        add("roi_align fwd cfg1 (512 boxes, 1x256x200x304, sr=%d)" % sr, t, tr, "alg 87.96 MB -> %.0f GB/s" % (87.96e6 / t / 1e3))
        xg = x.clone().requires_grad_(True)
        y = op(xg, rois)
        go = torch.randn_like(y)
        t = timeit(lambda: torch.autograd.grad(y, xg, go, retain_graph=True))
        if tv:
            y2 = tv.roi_align(xg, rois, (7, 7), 0.25, sr, True)
            tr = timeit(lambda: torch.autograd.grad(y2, xg, go, retain_graph=True))
        add("roi_align bwd cfg1 (sr=%d)" % sr, t, tr if tv else None)
    # ---- cfg2/3 poolers (fused multi-level) fwd + bwd
    d = bench.make_image_inputs(1)
    feats = [f.to(DEV) for f in d["feats"]]
    props = d["proposals"].to(DEV)
    scales = [s for (_, _, s) in bench.LEVELS]
    for out, kk in ((7, 1000), (14, 100)):
        pooler = ROIPooler(out, scales, 0, "ROIAlignV2")
        b = props[:kk].contiguous()
        t = timeit(lambda: pooler(feats, [b]))

        def ref_pooler():
            sizes = torch.sqrt((b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1]))
            lv = torch.floor(4 + torch.log2(sizes / 224 + 1e-8)).clamp(2, 5).to(torch.int64) - 2
            r5 = torch.cat([torch.zeros(len(b), 1, device=DEV), b], 1)
            res = torch.zeros(len(b), 256, out, out, device=DEV)
            for l, s in enumerate(scales):
                inds = torch.nonzero(lv == l, as_tuple=True)[0]
                res.index_put_((inds,), tv.roi_align(feats[l], r5[inds], (out, out), s, 0, True))
            return res

        tr = timeit(ref_pooler) if tv else None
        add("ROIPooler fwd %dx%d K=%d (p2..p5)" % (out, out, kk), t, tr, "ref = per-level loop over tv.roi_align")
        fg = [f.clone().requires_grad_(True) for f in feats]
        y = pooler(fg, [b])
        go = torch.randn_like(y)
        t = timeit(lambda: torch.autograd.grad(y, fg, go, retain_graph=True))
        trb = None
        if tv:
            yr_ = ref_pooler_grad(fg, b, out, scales, tv)
            trb = timeit(lambda: torch.autograd.grad(yr_, fg, go, retain_graph=True, allow_unused=True))
        add("ROIPooler bwd %dx%d K=%d" % (out, out, kk), t, trb, "ref = autograd of the per-level tv.roi_align loop")
    # ---- NMS
    for m, ncls, thr, tag in ((4819, 5, 0.7, "RPN test"), (8819, 5, 0.7, "RPN train"), (5000, 80, 0.5, "RetinaNet/FastRCNN"),
                              (25000, 80, 0.5, "stress")):
        gb = torch.Generator().manual_seed(m)
        boxes = bench.synth_boxes(gb, m, 16, 500).to(DEV)
        scores = torch.rand(m, generator=gb).to(DEV)
        idxs = torch.randint(0, ncls, (m,), generator=gb).to(DEV)
        t = timeit(lambda: L.batched_nms(boxes, scores, idxs, thr))
        tr = timeit(lambda: tv.boxes.batched_nms(boxes, scores, idxs, thr)) if tv else None
        add("batched_nms M=%d classes=%d (%s)" % (m, ncls, tag), t, tr, "%.1f Mpairs/s" % (m * (m - 1) / 2 / t))
    # ---- batched RPN proposal selection (2 images, 5 FPN levels, pre-NMS top 1000 per level)
    from detectron2_b200.proposal_utils import find_top_rpn_proposals
    gb = torch.Generator().manual_seed(9)
    per_level = [3 * 200 * 336, 3 * 100 * 168, 3 * 50 * 84, 3 * 25 * 42, 3 * 13 * 21]
    pp, ll = [], []
    for a in per_level:
        ctr = torch.rand(2, a, 2, generator=gb) * torch.tensor([1400.0, 850.0]) - 20
        wh = torch.exp(torch.rand(2, a, 2, generator=gb) * 5.0) + 0.5
        pp.append(torch.cat([ctr - wh / 2, ctr + wh / 2], 2).to(DEV))
        ll.append(torch.randn(2, a, generator=gb).to(DEV))
    szs = [(800, 1333), (800, 1333)]
    t = timeit(lambda: find_top_rpn_proposals(pp, ll, szs, 0.7, 1000, 1000, 0.0, False), rep=10)

    def ref_rpn():  # the reference's structure on the GPU: per-image loop, boolean filtering, tv batched_nms
        bi = torch.arange(2, device=DEV)
        ts, tp, lv = [], [], []
        for lid, (p_i, l_i) in enumerate(zip(pp, ll)):
            k = min(l_i.shape[1], 1000)
            s_i, idx = l_i.topk(k, dim=1)
            tp.append(p_i[bi[:, None], idx]); ts.append(s_i); lv.append(torch.full((k,), lid, dtype=torch.int64, device=DEV))
        ts, tp, lv = torch.cat(ts, 1), torch.cat(tp, 1), torch.cat(lv, 0)
        outs = []
        for n_, (h_, w_) in enumerate(szs):
            b_, s_, l_ = tp[n_].clone(), ts[n_], lv
            v_ = torch.isfinite(b_).all(1) & torch.isfinite(s_)
            if not v_.all():
                b_, s_, l_ = b_[v_], s_[v_], l_[v_]
            b_[:, 0::2].clamp_(0, w_); b_[:, 1::2].clamp_(0, h_)
            kp = ((b_[:, 2] - b_[:, 0]) > 0) & ((b_[:, 3] - b_[:, 1]) > 0)
            if kp.sum().item() != len(b_):
                b_, s_, l_ = b_[kp], s_[kp], l_[kp]
            kk_ = tv.boxes.batched_nms(b_, s_, l_, 0.7)[:1000]
            outs.append((b_[kk_], s_[kk_]))
        return outs

    tr = timeit(ref_rpn, rep=10) if tv else None
    add("find_top_rpn_proposals 2 img x 5 levels (242k anchors/img)", t, tr, "ref = reference loop structure with tv CUDA nms")
    # ---- rotated
    gb = torch.Generator().manual_seed(5)
    rb = torch.cat([torch.rand(1000, 2, generator=gb) * 300, 1 + torch.rand(1000, 2, generator=gb) * 120,
                    (torch.rand(1000, 1, generator=gb) - 0.5) * 360], 1).to(DEV)
    t = timeit(lambda: L.pairwise_iou_rotated(rb, rb))
    add("box_iou_rotated 1000x1000", t, refgpu.get("box_iou_rotated 1000x1000"), "%.1f Mpairs/s; ref = reference csrc CUDA" % (1e6 / t))
    sc = torch.rand(1000, generator=gb).to(DEV)
    t = timeit(lambda: L.nms_rotated(rb, sc, 0.5))
    add("nms_rotated M=1000", t, refgpu.get("nms_rotated M=1000"), "ref = reference csrc CUDA (mask on GPU, scan on host)")
    xr = torch.rand(2, 256, 50, 84, generator=gb).to(DEV)
    rr = torch.cat([torch.randint(0, 2, (512, 1), generator=gb).float(), torch.rand(512, 2, generator=gb) * 800,
                    16 + torch.rand(512, 2, generator=gb) * 300, (torch.rand(512, 1, generator=gb) - 0.5) * 360], 1).to(DEV)
    opr = L.ROIAlignRotated((7, 7), 1 / 16, 0)
    t = timeit(lambda: opr(xr, rr))
    add("roi_align_rotated fwd 512 boxes, 2x256x50x84", t, refgpu.get("roi_align_rotated fwd 512 boxes, 2x256x50x84"), "ref = reference csrc CUDA")
    xrg = xr.clone().requires_grad_(True)
    yr = opr(xrg, rr)
    gor = torch.randn_like(yr)
    t = timeit(lambda: torch.autograd.grad(yr, xrg, gor, retain_graph=True))
    add("roi_align_rotated bwd 512 boxes, 2x256x50x84", t, refgpu.get("roi_align_rotated bwd 512 boxes, 2x256x50x84"), "ref = reference csrc CUDA")
    bench_rotated_pooler(add, refgpu)
    bench_rotated_inference(add)
    # ---- paste
    masks, det = d["masks"].to(DEV), d["det_boxes"][:100].to(DEV)
    t = timeit(lambda: L.paste_masks_in_image(masks, det, (800, 1333), 0.5))
    add("paste_masks 100 x 28x28 -> 800x1333", t, refgpu.get("paste_masks 100 x 28x28 -> 800x1333"), "ref = GPU branch of the reference function (grid_sample); alg 106.96 MB -> %.0f GB/s (%.2f of HBM peak)" % (106.96e6 / t / 1e3, 106.96e6 / t / 1e3 / hbm))
    # ---- deformable conv layer sweep (SURVEY 8d cfg5), N=2, k=3, pad=1
    for cin, hh, ww, grp in ((128, 100, 168, 1), (256, 50, 84, 1), (512, 25, 42, 1), (512, 100, 168, 32), (1024, 50, 84, 32),
                             (2048, 25, 42, 32)):
        n = 2
        xx = torch.randn(n, cin, hh, ww, device=DEV)
        off = torch.randn(n, 18, hh, ww, device=DEV) * 2
        wt = torch.randn(cin, cin // grp, 3, 3, device=DEV) * 0.05
        flops = 2.0 * n * cin * (cin // grp) * 9 * hh * ww
        from detectron2_b200 import ops as _ops
        tr = timeit(lambda: tv.deform_conv2d(xx, off, wt, None, 1, 1, 1), rep=5, warm=1) if (tv and True) else None
        for prec, tag in ((0, "fp32 FFMA"), (1, "bf16x3 wgmma"), (2, "bf16 wgmma")):
            try:
                t = timeit(lambda: _ops.deform_conv_op(xx, off, None, wt, None, [1, 1], [1, 1], [1, 1], grp, 1, prec), rep=10, warm=2)
            except RuntimeError:
                continue
            rc = refgpu.get("deform_conv fwd C=%d %dx%d g=%d" % (cin, hh, ww, grp))
            add("deform_conv fwd C=%d %dx%d g=%d (%s)" % (cin, hh, ww, grp, tag), t, tr,
                "%.2f TFLOP/s; reference csrc CUDA: %s us" % (flops / t / 1e6, ("%.1f" % rc) if rc else "n/a"))
        try:  # the training forward: also lays x out channels-last once and keeps its sampled columns for the backward
            t = timeit(lambda: _ops.deform_conv_train_op(xx, off, None, wt, None, [1, 1], [1, 1], [1, 1], grp, 1, 1), rep=10, warm=2)
            add("deform_conv fwd C=%d %dx%d g=%d (bf16x3 wgmma, training: saves columns)" % (cin, hh, ww, grp), t, tr,
                "%.2f TFLOP/s" % (flops / t / 1e6))
        except RuntimeError:
            pass
        xg, og, wg = xx.clone().requires_grad_(True), off.clone().requires_grad_(True), wt.clone().requires_grad_(True)
        y = L.deform_conv(xg, og, wg, 1, 1, 1, grp, 1)
        go = torch.randn_like(y)
        t = timeit(lambda: torch.autograd.grad(y, (xg, og, wg), go, retain_graph=True), rep=3, warm=1)
        if tv:
            y2 = tv.deform_conv2d(xg, og, wg, None, 1, 1, 1)
            tr = timeit(lambda: torch.autograd.grad(y2, (xg, og, wg), go, retain_graph=True), rep=3, warm=1)
        rc = refgpu.get("deform_conv bwd C=%d %dx%d g=%d" % (cin, hh, ww, grp))
        add("deform_conv bwd C=%d %dx%d g=%d (auto: bf16x3 wgmma)" % (cin, hh, ww, grp), t, tr if tv else None,
            "%.2f TFLOP/s; reference csrc CUDA: %s us" % (2 * flops / t / 1e6, ("%.1f" % rc) if rc else "n/a"))

    with open(args.out, "w") as f:
        f.write("# Per-op timings on H100 (tools/bench_ops.py) — ours vs the reference's GPU kernels (torchvision %s CUDA ops)\n\n" %
                (getattr(__import__('torchvision'), '__version__', '?') if tv else 'n/a'))
        f.write("Eager launches incl. Python op dispatch (both sides); CUDA events, mean of back-to-back launches.\n\n")
        f.write("| op / shape | ours (us) | reference GPU (us) | speed-up | note |\n|---|---:|---:|---:|---|\n")
        for name, a, b, note in rows:
            f.write("| %s | %.1f | %s | %s | %s |\n" % (name, a, ("%.1f" % b) if b else "n/a", ("%.2fx" % (b / a)) if b else "", note))
    print("wrote", args.out)


if __name__ == "__main__":
    main()
