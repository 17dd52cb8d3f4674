"""Time the polygon mask paths with CUDA events at the Mask R-CNN training size: 2 images x 128 foreground RoIs, S = 28,
C = 80, about 7 ground-truth instances per image of 1-3 star polygons with 10-300 vertices, on 800 x 1333 images.

  * mask_rcnn_loss forward + backward on the packed polygons (one fused forward launch, one backward launch), next to the
    bitmask fused loss at the same shapes (gt_masks as [G, 800, 1333] bitmasks of the same instances);
  * polygons_to_bitmask of all the batch's instances at 800 x 1333;
  * crop_and_resize alone.

The reference's host path (pycocotools in a Python loop, after copying the boxes to the host) cannot run without
pycocotools and is reported as "not measured".

    python tools/bench_polygon_masks.py [--iters 50] [--out tools/results/bench_polygon_masks_h100.json]

The card's name and power limit are read in the same run and written beside the numbers.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectron2_b200 import mask_head, polygon_masks as pm  # noqa: E402


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = ""
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


def star(rng, n, cx, cy, r0, r1):
    a = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = rng.uniform(r0, r1, n)
    return np.stack([cx + r * np.cos(a), cy + r * np.sin(a)], 1).reshape(-1)


def batch(seed=0, images=2, k=128, n_inst=7, h=800, w=1333, c=80, s=28):
    rng = np.random.default_rng(seed)
    imgs, boxes, midx, cls = [], [], [], []
    for _ in range(images):
        inst = []
        for _ in range(n_inst):
            cx, cy, rad = rng.uniform(0, w), rng.uniform(0, h), rng.uniform(20, 300)
            inst.append([star(rng, int(rng.integers(10, 301)), cx + rng.uniform(-rad, rad) / 2,
                              cy + rng.uniform(-rad, rad) / 2, rad * 0.3, rad) for _ in range(int(rng.integers(1, 4)))])
        mi = rng.integers(0, n_inst, k)
        b = []
        for g in mi:
            xy = np.concatenate(inst[g]).reshape(-1, 2)
            lo, hi = xy.min(0), xy.max(0)
            ctr = (lo + hi) / 2 + rng.normal(0, 10, 2)
            half = (hi - lo) / 2 * rng.uniform(0.7, 1.3, 2)
            b.append([ctr[0] - half[0], ctr[1] - half[1], ctr[0] + half[0], ctr[1] + half[1]])
        imgs.append(inst)
        boxes.append(torch.tensor(np.array(b), dtype=torch.float32, device="cuda"))
        midx.append(torch.from_numpy(mi).cuda())
        cls.append(torch.from_numpy(rng.integers(0, c, k)).cuda())
    x = torch.randn(images * k, c, s, s, device="cuda") * 4
    return imgs, boxes, midx, cls, x


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default="tools/results/bench_polygon_masks_h100.json")
    a = ap.parse_args()
    name, q = card()
    imgs, boxes, midx, cls, x = batch()
    packed = pm.pack_polygons(imgs, "cuda")
    bitmasks = [pm.polygons_to_bitmask(pm.pack_polygons([inst], "cuda"), 800, 1333) for inst in imgs]
    xg = x.clone().requires_grad_(True)

    def poly_step():
        xg.grad = None
        loss, _ = mask_head.mask_rcnn_loss(xg, packed, boxes, cls, midx)
        loss.backward()

    def bitmask_step():
        xg.grad = None
        loss, _ = mask_head.mask_rcnn_loss(xg, bitmasks, boxes, cls, midx)
        loss.backward()

    allb, allm = torch.cat(boxes), pm.batch_mask_index(packed, [len(b) for b in boxes], midx, "cuda")
    res = {
        "card": name,
        "power_limit_and_max_sm_clock": q,
        "iters": a.iters,
        "shape": {"images": 2, "rois_per_image": 128, "S": 28, "C": 80, "instances_per_image": 7,
                  "polygons_per_instance": "1-3", "vertices_per_polygon": "10-300", "image": [800, 1333],
                  "vertices_total": int(packed.coords.shape[0]), "polygons_total": int(packed.poly_start.shape[0] - 1)},
        "reference_host_path_ms": "not measured (the reference path needs pycocotools)",
        "polygon_loss_fwd_bwd_ms": time_ms(poly_step, a.iters),
        "bitmask_loss_fwd_bwd_ms": time_ms(bitmask_step, a.iters),
        "polygons_crop_and_resize_ms": time_ms(lambda: pm.polygons_crop_and_resize(packed, allb, 28, allm), a.iters),
        "polygons_to_bitmask_800x1333_ms": time_ms(lambda: pm.polygons_to_bitmask(packed, 800, 1333), a.iters),
    }
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
