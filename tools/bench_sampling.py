"""Time the sampling of the training labels: the reference-shaped per-image path (matching.subsample_labels, the
reference's own code, looped over the images as RPN._subsample_labels and ROIHeads._sample_proposals do) against
subsample_labels_fixed (one d2b_sample_labels for the batch), eager and replayed from a CUDA graph, with CUDA events.

    python tools/bench_sampling.py [--iters 50] [--out FILE]

Workloads (2 images per batch, labels drawn with fixed proportions, the same tensors for every arm):
  RPN        2 x 268 569 int8 labels (0.1 % positive, 10 % ignored), 256 per image, half positive, RPN label-map output;
  ROI heads  2 x (2 000 + 40) int64 classes over 80 classes (5 % foreground), 512 per image, a quarter foreground.
The reference arm includes its host syncs (two nonzero per image), as a training step pays them.  Prints one JSON line with
the card's name, power limit and max SM clock read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectron2_b200 import matching as mt  # noqa: E402
from detectron2_b200 import sampling  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not available"
    return name, q


def time_us(fn, iters, warmup=5):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters * 1000.0


def graphed(fn):
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(3):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        fn()
    return g.replay


def labels_of(n, p, dtype, pos, ign, bg, num_classes, g):
    u = torch.rand(n, p, generator=g)
    fg = torch.randint(0, num_classes, (n, p), generator=g) if dtype == torch.int64 else torch.ones(n, p, dtype=torch.int64)
    lab = torch.where(u < pos, fg, torch.where(u < pos + ign, torch.full_like(fg, -1), torch.full_like(fg, bg)))
    return lab.to(dtype).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_sampling needs a CUDA device"
    g = torch.Generator().manual_seed(0)
    rpn = labels_of(2, 268569, torch.int8, 0.001, 0.1, 0, 1, g)
    roi = labels_of(2, 2040, torch.int64, 0.05, 0.0, 80, 80, g)

    def ref_rpn():
        return [mt._rpn_subsample(rpn[i].clone(), 256, 0.5) for i in range(rpn.shape[0])]

    def ref_roi():
        out = []
        for i in range(roi.shape[0]):
            fg, bg = mt.subsample_labels(roi[i], 512, 0.25, 80)
            out.append(torch.cat([fg, bg]))
        return out

    def fixed_rpn():
        return sampling.sample_labels(rpn, 256, 0.5, 0, rpn_labels=True)

    def fixed_roi():
        return sampling.subsample_labels_fixed(roi, 512, 0.25, 80)

    name, limits = card()
    res = {"device": name, "power_limit_and_max_sm_clock": limits, "iters": args.iters, "unit": "us per batch of 2"}
    for label, ref, fixed in (("rpn_2x268569", ref_rpn, fixed_rpn), ("roi_2x2040", ref_roi, fixed_roi)):
        res[label] = {"reference_per_image": round(time_us(ref, args.iters), 1),
                      "fixed_eager": round(time_us(fixed, args.iters), 1),
                      "fixed_graph": round(time_us(graphed(fixed), args.iters), 1)}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
