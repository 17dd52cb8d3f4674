"""Time the FCOS training-target and loss step and FCOS inference with CUDA events:

  * assign + loss forward + backward at 2 images x 22 400 points (P3-P7 of 800 x 1344) x 80 classes, G = 14 and G = 100 GT
    boxes per image (the second image gets half): the reference-shaped per-image path (the torch restatement of
    FCOS.label_anchors + FCOS.losses in detectron2_b200/fcos.py, on CUDA tensors), the fused eager path
    (fcos_label_anchors_fixed + fcos_losses_fixed + autograd) and the same step replayed as one CUDA graph;
  * inference for 2 images (fcos_inference: scores, per-level top-k, linear decode, one NMS) against the host restatement of
    the selection on the same CUDA tensors.

    python tools/bench_fcos.py [--iters 30] [--out tools/results/bench_fcos_h100.json]

The card's name, power limit and max SM clock are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectron2_b200 import fcos as F  # noqa: E402
from detectron2_b200.dense_inference import _dense_detector_inference_host  # noqa: E402

K = 80


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not available"
    return name, q


def time_ms(fn, iters, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def points(h=800, w=1344, strides=(8, 16, 32, 64, 128)):
    out = []
    for s in strides:
        gh, gw = -(-h // s), -(-w // s)
        ys, xs = torch.meshgrid(torch.arange(gh, dtype=torch.float32) * s, torch.arange(gw, dtype=torch.float32) * s,
                                indexing="ij")
        c = torch.stack([xs.reshape(-1), ys.reshape(-1)], 1)
        out.append(torch.cat([c - s / 2, c + s / 2], 1).cuda())
    return out


def gt_boxes(g, n):
    xy = torch.rand(n, 2, generator=g) * torch.tensor([1200.0, 720.0])
    wh = 8 + torch.rand(n, 2, generator=g) ** 2 * torch.tensor([800.0, 480.0])
    return torch.cat([xy, xy + wh], 1).cuda()


def train_case(G, g, iters):
    anchors = points()
    an = torch.cat(anchors)
    counts = [len(a) for a in anchors]
    gts = [gt_boxes(g, G), gt_boxes(g, G // 2)]
    cls = [torch.randint(0, K, (len(b),), generator=g).cuda() for b in gts]
    logits = [(torch.randn(2, len(a), K, generator=g) - 2).cuda().requires_grad_(True) for a in anchors]
    deltas = [(torch.randn(2, len(a), 4, generator=g) + 0.5).cuda().requires_grad_(True) for a in anchors]
    ctr = [torch.randn(2, len(a), 1, generator=g).cuda().requires_grad_(True) for a in anchors]
    leaves = logits + deltas + ctr
    s_gt = torch.zeros((2, G, 4), device="cuda")
    s_cls = torch.zeros((2, G), dtype=torch.int64, device="cuda")
    for i, (b, c) in enumerate(zip(gts, cls)):
        s_gt[i, :len(b)], s_cls[i, :len(c)] = b, c
    s_cnt = torch.tensor([len(b) for b in gts], device="cuda")
    ema = torch.full((1,), 300.0, dtype=torch.float64, device="cuda")

    def reference():
        labels, boxes, _ = F._fcos_label_anchors_host(an, counts, gts, cls, K)
        losses = F._fcos_losses_host(an, logits, labels, deltas, boxes, ctr, K, 300.0, 0.25, 2.0)[0]
        return torch.autograd.grad(sum(losses.values()), leaves)

    def fused():
        labels, boxes, _ = F.fcos_label_anchors_fixed(an, s_gt, s_cnt, s_cls, num_classes=K, level_counts=counts)
        losses = F.fcos_losses_fixed(an, logits, labels, deltas, boxes, ctr, ema, num_classes=K)[0]
        return torch.autograd.grad(sum(losses.values()), leaves)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fused()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fused()
    ref_ms = time_ms(reference, max(iters // 3, 3))
    fused_ms = time_ms(fused, iters)
    graph_ms = time_ms(graph.replay, iters)
    return {"workload": "assign+loss fwd+bwd", "images": 2, "points": int(an.shape[0]), "classes": K, "G": [G, G // 2],
            "reference_ms": round(ref_ms, 3), "fused_eager_ms": round(fused_ms, 3), "graph_replay_ms": round(graph_ms, 3),
            "speedup_eager": round(ref_ms / fused_ms, 2), "speedup_graph": round(ref_ms / graph_ms, 2)}


def inference_case(g, iters):
    anchors = points()
    logits = [(torch.randn(2, len(a), K, generator=g) * 1.5 - 3).cuda() for a in anchors]
    ctr = [torch.randn(2, len(a), 1, generator=g).cuda() for a in anchors]
    deltas = [(torch.randn(2, len(a), 4, generator=g) * 0.5 + 0.5).cuda() for a in anchors]
    sizes = [(800, 1344)] * 2
    ours = lambda: F.fcos_inference(anchors, logits, deltas, ctr, sizes)  # noqa: E731
    host = lambda: _dense_detector_inference_host(anchors, F._scores(logits, ctr), deltas, sizes, 0.2, 1000, 0.6, 100,  # noqa: E731
                                                  transform="linear")
    k_ms = time_ms(ours, iters)
    h_ms = time_ms(host, max(iters // 3, 3))
    return {"workload": "inference", "images": 2, "points": sum(len(a) for a in anchors), "classes": K,
            "fused_ms": round(k_ms, 3), "host_restatement_ms": round(h_ms, 3), "speedup": round(h_ms / k_ms, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_fcos: needs a CUDA device")
    name, limits = card()
    print("device: %s | power.limit, clocks.max.sm: %s" % (name, limits))
    g = torch.Generator().manual_seed(0)
    rows = [train_case(14, g, args.iters), train_case(100, g, args.iters), inference_case(g, args.iters)]
    for r in rows:
        r.update(device=name, limits=limits)
        print(json.dumps(r))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"device": name, "power_limit_and_max_sm_clock": limits, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
