"""Time heatmaps_to_keypoints: the native kernel (d2b_keypoints_from_heatmaps) against the reference-shaped per-detection
loop (the torch restatement of structures/keypoints.py:164-235 on the same CUDA tensors), with CUDA events.

    python tools/bench_keypoints.py [--iters 50] [--loop-iters 5] [--out FILE]

Workload: 1 and 2 images x 100 detections, K = 17, S = 56 (the COCO keypoint head), box sides log-uniform in 16-600 px
inside an 800 x 1333 image, and one full-image 800 x 1333 box per batch (the worst case for a one-CTA-per-map design).
Work = K * sum over boxes of ceil(h) * ceil(w) bicubic evaluations; both arms do the same work.  The card's name and power
limit are read in the same run and printed with the numbers.
"""
import argparse
import json
import math
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectron2_b200 import keypoint_head as kh  # noqa: E402

K, S = 17, 56


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "power limit not available"
    return name, q


def scene(images, seed):
    g = torch.Generator().manual_seed(seed)
    r = 100 * images
    side = torch.exp(torch.empty(r, 2).uniform_(math.log(16.0), math.log(600.0), generator=g))
    lo = torch.rand(r, 2, generator=g) * (torch.tensor([1333.0, 800.0]) - side).clamp(min=0)
    rois = torch.cat([lo, lo + side], dim=1)
    rois[0] = torch.tensor([0.0, 0.0, 1333.0, 800.0])
    maps = torch.randn((r, K, S, S), generator=g) * 3
    return maps.cuda(), rois.cuda()


def evaluations(rois):
    w = (rois[:, 2] - rois[:, 0]).clamp(min=1).ceil()
    h = (rois[:, 3] - rois[:, 1]).clamp(min=1).ceil()
    return int(K * (w.double() * h.double()).sum().item())


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--loop-iters", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_keypoints: needs a CUDA device")
    name, limits = card()
    print("device: %s | power.limit, clocks.max.sm: %s" % (name, limits))
    print("%-8s %-6s %-14s %-12s %-12s %-16s %-16s %-8s" % ("images", "rois", "evaluations", "kernel_ms", "loop_ms",
                                                             "kernel_eval/s", "loop_eval/s", "speedup"))
    rows = []
    for images in (1, 2):
        maps, rois = scene(images, seed=images)
        ev = evaluations(rois)
        ours = kh.heatmaps_to_keypoints(maps, rois)
        ref = kh._heatmaps_to_keypoints_host(maps, rois)
        xy_mismatches = int((ours[..., :2] != ref[..., :2]).any(dim=-1).sum())  # argmax near-ties, if any
        k_ms = time_ms(lambda: kh.heatmaps_to_keypoints(maps, rois), args.iters)
        l_ms = time_ms(lambda: kh._heatmaps_to_keypoints_host(maps, rois), args.loop_iters, warmup=1)
        row = {"images": images, "rois": int(rois.shape[0]), "evaluations": ev, "kernel_ms": round(k_ms, 4),
               "loop_ms": round(l_ms, 3), "kernel_eval_per_s": ev / (k_ms * 1e-3), "loop_eval_per_s": ev / (l_ms * 1e-3),
               "speedup": round(l_ms / k_ms, 2), "xy_mismatches": xy_mismatches, "device": name, "limits": limits}
        rows.append(row)
        print("%-8d %-6d %-14d %-12.4f %-12.3f %-16.3e %-16.3e %-8.2f" % (images, row["rois"], ev, k_ms, l_ms,
                                                                          row["kernel_eval_per_s"],
                                                                          row["loop_eval_per_s"], row["speedup"]))
    print(json.dumps(rows))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
