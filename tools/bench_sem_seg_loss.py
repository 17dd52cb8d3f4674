"""Time the semantic segmentation training loss (forward + backward) with CUDA events at the Panoptic FPN size
(2 x 54 x 200 x 336 logits, stride 4, cross-entropy mean) and the Panoptic-DeepLab Cityscapes size (4 x 19 x 256 x 512,
stride 4, DeepLabCE top-k 0.2 with per-pixel weights), for three paths:

  * the reference composition on CUDA: logits.float(), F.interpolate(bilinear), F.cross_entropy / DeepLabCE (torch.topk);
  * the fused eager path: sem_seg_loss_fixed + autograd backward;
  * the same forward + backward replayed as one CUDA graph.

Each path's torch.cuda.max_memory_allocated above the inputs is recorded.  The fused forward and backward are also timed on
their own and reported against the bytes and exp evaluations the algorithm needs, computed from the shapes
(`algorithmic`): bytes/s against 3.35 TB/s of HBM3, exp/s against the SFU rate of the card (16 per SM per clock at the
max SM clock).

    python tools/bench_sem_seg_loss.py [--iters 20] [--out tools/results/bench_sem_seg_loss_h100.json]

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
from detectron2_b200 import semantic_seg as S  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
SFU_PER_SM_PER_CLK = 16

# name: (N, C, Hp, Wp, stride, top_k, weights)
SIZES = {
    "panoptic_fpn_coco": (2, 54, 200, 336, 4, None, False),
    "panoptic_deeplab_cityscapes": (4, 19, 256, 512, 4, 0.2, True),
}


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


def inputs(n, c, hp, wp, s, with_w):
    g = torch.Generator(device="cuda").manual_seed(0)
    h, w = hp * s, wp * s
    logits = torch.randn((n, c, hp, wp), generator=g, device="cuda") * 3.0
    targets = torch.randint(0, c, (n, h, w), generator=g, device="cuda")
    targets[torch.rand((n, h, w), generator=g, device="cuda") < 0.1] = 255
    weights = 0.5 + 2.5 * torch.rand((n, h, w), generator=g, device="cuda") if with_w else None
    return logits.requires_grad_(True), targets, weights


def reference(logits, targets, s, top_k, weights):
    """SemSegFPNHead.losses / PanopticDeepLabSemSegHead.losses with DeepLabCE, as the reference runs them."""
    up = F.interpolate(logits.float(), scale_factor=s, mode="bilinear", align_corners=False)
    if top_k is None:
        return F.cross_entropy(up, targets, reduction="mean", ignore_index=255)
    pixel = F.cross_entropy(up, targets, reduction="none", ignore_index=255)
    if weights is not None:
        pixel = pixel * weights
    pixel = pixel.contiguous().view(-1)
    return torch.topk(pixel, int(top_k * pixel.numel()))[0].mean()


def algorithmic(n, c, hp, wp, s, top_k, with_w):
    p = n * hp * s * wp * s
    logits = n * c * hp * wp * 4
    fwd = logits + 8 * p + 4 * p  # logits, targets, lse
    bwd = logits + 8 * p + 4 * p + logits  # logits, targets, lse, grad_logits
    if with_w:
        fwd += 4 * p
        bwd += 4 * p
    if top_k is not None and top_k != 1.0:
        fwd += 4 * p * 2 + p  # per-pixel losses written and read back, selected written
        bwd += p  # selected
    return {"fwd_bytes": fwd, "bwd_bytes": bwd, "exp_per_direction": n * c * hp * s * wp * s}


def bench(name, iters, sfu_rate):
    n, c, hp, wp, s, top_k, with_w = SIZES[name]
    logits, targets, weights = inputs(n, c, hp, wp, s, with_w)
    base = torch.cuda.memory_allocated()
    out = {"shape": {"N": n, "C": c, "Hp": hp, "Wp": wp, "stride": s, "top_k_percent_pixels": top_k,
                     "weights": with_w}}

    def ref_step():
        logits.grad = None
        reference(logits, targets, s, top_k, weights).backward()

    def fused_step():
        logits.grad = None
        S.sem_seg_loss_fixed(logits, targets, s, 255, top_k, weights)[0].backward()

    for key, fn in (("reference_ms", ref_step), ("fused_eager_ms", fused_step)):
        fn()
        torch.cuda.synchronize()
        logits.grad = None
        torch.cuda.reset_peak_memory_stats()
        out[key] = time_ms(fn, iters)
        out[key.replace("_ms", "_peak_bytes")] = torch.cuda.max_memory_allocated() - base
    logits.grad = None

    static = logits.detach().clone().requires_grad_(True)

    def graph_body():
        loss = S.sem_seg_loss_fixed(static, targets, s, 255, top_k, weights)[0]
        return torch.autograd.grad(loss, static)[0]

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            graph_body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graph_body()
    out["fused_graph_ms"] = time_ms(graph.replay, iters)
    out["fused_graph_peak_bytes"] = torch.cuda.max_memory_allocated() - base
    del graph

    # the fused directions on their own
    ld = logits.detach()
    res = S.sem_seg_loss_op(ld, targets, s, 255, top_k, weights)
    gs = torch.ones((), device="cuda")
    fwd_ms = time_ms(lambda: S.sem_seg_loss_op(ld, targets, s, 255, top_k, weights), iters)
    bwd_ms = time_ms(lambda: S.sem_seg_loss_backward_op(ld, targets, s, 255, weights, res[4], res[3], gs), iters)
    alg = algorithmic(n, c, hp, wp, s, top_k, with_w)
    out["algorithmic"] = alg
    for d, ms in (("fwd", fwd_ms), ("bwd", bwd_ms)):
        bps, eps = alg[d + "_bytes"] / (ms * 1e-3), alg["exp_per_direction"] / (ms * 1e-3)
        out[d] = {"ms": ms, "bytes_per_s": bps, "share_of_hbm": bps / HBM_BYTES_PER_S, "exp_per_s": eps,
                  "share_of_sfu": eps / sfu_rate,
                  "nearer_roof": "HBM" if bps / HBM_BYTES_PER_S >= eps / sfu_rate else "SFU (exp rate)"}
    out["speedup_eager"] = out["reference_ms"] / out["fused_eager_ms"]
    out["speedup_graph"] = out["reference_ms"] / out["fused_graph_ms"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sem_seg_loss: needs a CUDA device")
    name, q = card()
    props = torch.cuda.get_device_properties(0)
    try:
        max_mhz = float(q.split(",")[1].split()[0])
    except (IndexError, ValueError):
        max_mhz = float("nan")
    sfu_rate = props.multi_processor_count * SFU_PER_SM_PER_CLK * max_mhz * 1e6
    res = {"card": name, "power_limit_and_max_sm_clock": q, "sm_count": props.multi_processor_count,
           "sfu_exp_per_s_at_max_clock": sfu_rate, "hbm_bytes_per_s_datasheet": HBM_BYTES_PER_S, "iters": args.iters,
           "cases": {k: bench(k, args.iters, sfu_rate) for k in SIZES}}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
