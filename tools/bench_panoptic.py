"""Time Panoptic FPN post-processing with CUDA events, per batch of COCO-like scenes (C = 54 semantic classes, 100
detections per image with masks pasted from random boxes, default thresholds, logits [N, 54, 800, 1344]):

  * the reference-shaped per-image path on CUDA tensors: sem_seg_postprocess(...).argmax(0) with the C x H x W map, and
    the torch restatement of combine_semantic_and_instance_outputs with its host reads (detectron2_b200/panoptic.py);
  * the fused eager path: sem_seg_labels + combine_semantic_and_instance_outputs_fixed;
  * the same two calls replayed as one CUDA graph.

It also times each kernel pair on its own and reports the achieved bytes/s against the bytes the algorithm needs, computed
from the shapes (`algorithmic_bytes`).

    python tools/bench_panoptic.py [--iters 20] [--out tools/results/bench_panoptic_h100.json]

The card's name, power limit and max SM clock are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.nn import functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectron2_b200 import panoptic as P  # noqa: E402
from detectron2_b200.layers import paste_masks_in_image  # noqa: E402

C = 54
R = 100
THR = (0.5, 4096.0, 0.5)  # PanopticFPN's defaults: combine.overlap_thresh, stuff_area_thresh, instances_score_thresh


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


def scene(g, h, w):
    ctr = torch.rand(R, 2, generator=g) * torch.tensor([w, h])
    wh = 16 + torch.rand(R, 2, generator=g) ** 2 * torch.tensor([w, h]) * 0.5
    boxes = torch.cat([ctr - wh / 2, ctr + wh / 2], 1).cuda()
    masks = paste_masks_in_image(torch.rand(R, 28, 28, generator=g).cuda(), boxes, (h, w), 0.5)
    scores = torch.rand(R, generator=g).cuda()
    classes = torch.randint(0, 80, (R,), generator=g).cuda()
    return scores, classes, masks


def algorithmic_bytes(logits, crops, outs, elem):
    """Least traffic: the cropped logits read once (a down-scale reads each element about once; an up-scale fewer), int64
    labels written; the combine reads each mask byte and label once and writes each panoptic pixel once."""
    sem = sum(C * min(h * w, oh * ow) * elem + oh * ow * 8 for (h, w), (oh, ow) in zip(crops, outs))
    comb = sum(R * oh * ow + oh * ow * 8 + oh * ow * 4 for oh, ow in outs)
    return sem, comb


def case(out_size, n, g, iters):
    oh, ow = out_size
    crop = (800, int(round(800 * ow / oh))) if ow / oh < 1.68 else (int(round(1333 * oh / ow)), 1333)
    crop = (min(crop[0], 800), min(crop[1], 1344))
    logits = torch.randn(n, C, 800, 1344, generator=g).cuda()
    crops, outs = [crop] * n, [out_size] * n
    parts = [scene(g, oh, ow) for _ in range(n)]
    scores, classes, masks = [list(x) for x in zip(*parts)]

    def reference():
        res = []
        for i in range(n):
            lab = F.interpolate(logits[i, :, :crop[0], :crop[1]][None], size=out_size, mode="bilinear",
                                align_corners=False)[0].argmax(0)
            res.append(P._combine_host(scores[i], classes[i], masks[i], lab, *THR))
        return res

    def fused():
        labels = P.sem_seg_labels(logits, crops, outs)
        return P.combine_semantic_and_instance_outputs_fixed(scores, classes, masks, labels, C, *THR)

    labels = P.sem_seg_labels(logits, crops, outs)
    sem_only = lambda: P.sem_seg_labels(logits, crops, outs)  # noqa: E731
    comb_only = lambda: P.combine_semantic_and_instance_outputs_fixed(scores, classes, masks, labels, C, *THR)  # noqa: E731
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            fused()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        fused()
    ref_ms = time_ms(reference, max(iters // 4, 2), warmup=1)
    fused_ms = time_ms(fused, iters)
    graph_ms = time_ms(graph.replay, iters)
    sem_ms = time_ms(sem_only, iters)
    comb_ms = time_ms(comb_only, iters)
    sem_b, comb_b = algorithmic_bytes(logits, crops, outs, 4)
    return {"images": n, "output_size": list(out_size), "crop": list(crop), "logits": [n, C, 800, 1344],
            "detections_per_image": R, "reference_ms": round(ref_ms, 3), "fused_eager_ms": round(fused_ms, 3),
            "graph_replay_ms": round(graph_ms, 3), "speedup_eager": round(ref_ms / fused_ms, 2),
            "speedup_graph": round(ref_ms / graph_ms, 2), "sem_seg_labels_ms": round(sem_ms, 3),
            "sem_seg_labels_algorithmic_GBps": round(sem_b / sem_ms / 1e6, 1), "combine_ms": round(comb_ms, 3),
            "combine_algorithmic_GBps": round(comb_b / comb_ms / 1e6, 1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_panoptic: needs a CUDA device")
    name, limits = card()
    print("device: %s | power.limit, clocks.max.sm: %s" % (name, limits))
    g = torch.Generator().manual_seed(0)
    rows = [case(size, n, g, args.iters) for size in ((480, 640), (800, 1333)) for n in (1, 4)]
    for r in rows:
        r.update(device=name, limits=limits)
        print(json.dumps(r))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"device": name, "power_limit_and_max_sm_clock": limits, "results": rows}, f, indent=1)


if __name__ == "__main__":
    main()
