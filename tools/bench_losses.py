"""Time the box-branch training losses, forward + backward: the native kernels (d2b_dense_loss_*, d2b_frcnn_loss_*) against
the reference-shaped torch expressions (the restatement of RPN.losses, RetinaNet.losses and FastRCNNOutputLayers.losses in
detectron2_b200/losses.py) on the same CUDA tensors, with CUDA events.  FCOS, the dense loss with D2B_LOSS_LINEAR_GIOU, is
timed by tools/bench_fcos.py.

    python tools/bench_losses.py [--iters 30] [--out FILE]

Workloads (800 x 1344 images, 2 per batch):
  RetinaNet  201 600 anchors (p3-p7, 9 per location) x 80 classes, fp32 and bf16 logits / deltas;
  RPN        268 569 anchors (p2-p6, 3 per location), 256 sampled per image;
  Fast R-CNN 2 x 512 proposals x 81 classes, class-specific deltas.
Labels are drawn with fixed proportions (RetinaNet: 0.1 % positive, 1 % ignored; Fast R-CNN: 25 % foreground); both arms
get the same tensors.  The algorithmic bytes of the native path (logits read once forward, read + gradient written once
backward) are printed with the achieved rate.  The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from detectron2_b200 import losses as L  # noqa: E402


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


def boxes(n, g, d=4):
    xy = torch.rand(n, 2, generator=g) * 1200
    wh = 16 + torch.rand(n, 2, generator=g) * 400
    return torch.cat([xy, xy + wh], 1)


def dense_case(levels, k, dtype, g, pos, ign, rpn):
    n, r = 2, sum(levels)
    anchors = [boxes(rl, g).cuda() for rl in levels]
    gt = torch.stack([boxes(r, g) for _ in range(n)]).cuda()
    u = torch.rand(n, r, generator=g)
    if rpn:
        labels = torch.full((n, r), -1, dtype=torch.int8)
        labels[u < 256 / r] = 0
        labels[u < 128 / r * 0.3] = 1
        logits = [torch.randn(n, rl, generator=g).to("cuda", dtype) for rl in levels]
    else:
        labels = torch.full((n, r), k, dtype=torch.int64)
        labels[u < pos] = torch.randint(0, k, (n, r), generator=g)[u < pos]
        labels[(u >= pos) & (u < pos + ign)] = -1
        logits = [(torch.randn(n, rl, k, generator=g) - 3).to("cuda", dtype) for rl in levels]
    deltas = [(torch.randn(n, rl, 4, generator=g) * 0.5).to("cuda", dtype) for rl in levels]
    return anchors, logits, deltas, labels.cuda(), gt


def fwd_bwd(fn, ts):
    leaves = [t.detach().requires_grad_(True) for t in ts]
    out = fn(leaves)
    sum(out.values()).backward()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_losses: needs a CUDA device")
    name, limits = card()
    print("device: %s | power.limit, clocks.max.sm: %s" % (name, limits))
    g = torch.Generator().manual_seed(0)
    retina_levels = [100 * 168 * 9, 50 * 84 * 9, 25 * 42 * 9, 13 * 21 * 9, 7 * 11 * 9]
    rpn_levels = [200 * 336 * 3, 100 * 168 * 3, 50 * 84 * 3, 25 * 42 * 3, 13 * 21 * 3]
    rows = []
    for what, dtype in (("retinanet", torch.float32), ("retinanet", torch.bfloat16), ("rpn", torch.float32)):
        rpn = what == "rpn"
        anchors, logits, deltas, labels, gt = dense_case(rpn_levels if rpn else retina_levels, 1 if rpn else 80, dtype, g,
                                                         1e-3, 1e-2, rpn)
        nl = len(logits)
        cat_a = torch.cat(anchors)
        if rpn:
            ours = lambda ts: L.rpn_losses_fixed(anchors, ts[:nl], labels, ts[nl:], gt, batch_size_per_image=256)[0]
            ref = lambda ts: L._rpn_losses_host(cat_a, ts[:nl], list(labels), ts[nl:], list(gt), 256, (1.0,) * 4,
                                                L._SCALE_CLAMP, "smooth_l1", 0.0, None)[0]
        else:
            ema = torch.full((1,), 100.0, dtype=torch.float64, device="cuda")
            ours = lambda ts: L.retinanet_losses_fixed(anchors, ts[:nl], labels, ts[nl:], gt, ema, num_classes=80)[0]
            ref = lambda ts: L._retinanet_losses_host(cat_a, ts[:nl], list(labels), ts[nl:], list(gt), 80, 100.0, 0.25, 2.0,
                                                      (1.0,) * 4, L._SCALE_CLAMP, "smooth_l1", 0.1)[0]
        ts = logits + deltas
        k_ms = time_ms(lambda: fwd_bwd(ours, ts), args.iters)
        r_ms = time_ms(lambda: fwd_bwd(ref, ts), max(args.iters // 3, 3))
        elem = sum(x.numel() for x in logits)
        nbytes = 3 * elem * logits[0].element_size()  # forward read, backward read + gradient write
        rows.append({"loss": what, "dtype": str(dtype).replace("torch.", ""), "logits": elem, "kernel_ms": round(k_ms, 4),
                     "reference_ms": round(r_ms, 3), "speedup": round(r_ms / k_ms, 2), "logit_bytes": nbytes,
                     "logit_GBps": round(nbytes / (k_ms * 1e-3) / 1e9, 1), "device": name, "limits": limits})
        print(rows[-1])
    # Fast R-CNN, 2 x 512 proposals, 81 classes, class-specific deltas
    r, k = 1024, 80
    scores = torch.randn(r, k + 1, generator=g).cuda()
    pdeltas = (torch.randn(r, k * 4, generator=g) * 0.3).cuda()
    props = boxes(r, g).cuda()
    gtb = (props + torch.randn(r, 4, generator=g).cuda() * 5)
    gtb[:, 2:] = torch.maximum(gtb[:, 2:], gtb[:, :2] + 1)
    cls = torch.full((r,), k, dtype=torch.int64)
    fg = torch.rand(r, generator=g) < 0.25
    cls[fg] = torch.randint(0, k, (r,), generator=g)[fg]
    cls = cls.cuda()
    ours = lambda ts: L.fast_rcnn_losses_fixed(ts[0], ts[1], props, gtb, cls)[0]
    ref = lambda ts: L._fast_rcnn_losses_host(ts[0], ts[1], props, gtb, cls, (10.0, 10.0, 5.0, 5.0), L._SCALE_CLAMP,
                                              "smooth_l1", 0.0, None)[0]
    k_ms = time_ms(lambda: fwd_bwd(ours, [scores, pdeltas]), args.iters)
    r_ms = time_ms(lambda: fwd_bwd(ref, [scores, pdeltas]), args.iters)
    rows.append({"loss": "fast_rcnn", "dtype": "float32", "rows": r, "kernel_ms": round(k_ms, 4),
                 "reference_ms": round(r_ms, 3), "speedup": round(r_ms / k_ms, 2), "device": name, "limits": limits})
    print(rows[-1])
    print(json.dumps(rows))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
