"""Timings of the REFERENCE's own GPU kernels on the box (the kernel-to-beat for the ops torchvision does not cover).

Loads oracle/_ref/d2_ref_cuda.so -- the reference's csrc (CPU + CUDA) compiled for sm_90a by oracle/build.py
(build_ref_cuda; SURVEY.md Appendix B.2) -- in a process that never imports detectron2_b200, so the two `detectron2::`
op registrations cannot collide.  Writes gpurun_out/ref_gpu.json: {name: microseconds}.  Shapes match tools/bench_ops.py.
"""
import importlib.machinery
import importlib.util
import json
import math
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "oracle", "_ref", "d2_ref_cuda.so")
DEV = "cuda"


def timeit(fn, rep=10, warm=2):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(rep):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / rep * 1e3


def paste_gpu_branch(masks, boxes, img_h, img_w, threshold=0.5):
    """The GPU branch of the reference's paste_masks_in_image (detectron2/layers/mask_ops.py:17-69,120-141) restated:
    every mask sampled over the whole image with grid_sample, chunked to <= 1 GB of fp32 grid."""
    n = masks.shape[0]
    chunks = int(math.ceil(n * img_h * img_w * 4 / (1024 ** 3)))
    out = torch.empty((n, img_h, img_w), dtype=torch.bool, device=masks.device)
    for inds in torch.chunk(torch.arange(n, device=masks.device), chunks):
        b = boxes[inds]
        x0, y0, x1, y1 = torch.split(b, 1, dim=1)
        img_y = torch.arange(0, img_h, device=masks.device, dtype=torch.float32) + 0.5
        img_x = torch.arange(0, img_w, device=masks.device, dtype=torch.float32) + 0.5
        img_y = (img_y - y0) / (y1 - y0) * 2 - 1
        img_x = (img_x - x0) / (x1 - x0) * 2 - 1
        gx = img_x[:, None, :].expand(len(inds), img_h, img_w)
        gy = img_y[:, :, None].expand(len(inds), img_h, img_w)
        grid = torch.stack([gx, gy], dim=3)
        img = F.grid_sample(masks[inds][:, None], grid, align_corners=False)
        out[inds] = img[:, 0] >= threshold
    return out


def rotated_pooler_inputs(device=DEV):
    """Rotated ROIPooler bench shape (also used by tools/bench_ops.py): 2 images x 512 rotated RoIs, p2..p5 of an 800x1344
    image at 256 channels, sizes log-uniform in [16, 800], angles uniform in (-180, 180]."""
    g = torch.Generator().manual_seed(31)
    feats = [torch.randn(2, 256, 200 // 2 ** l, 336 // 2 ** l, generator=g).to(device) for l in range(4)]
    boxes = []
    for _ in range(2):
        s = torch.exp(torch.rand(512, generator=g) * (math.log(800) - math.log(16)) + math.log(16))
        ar = torch.exp((torch.rand(512, generator=g) - 0.5) * 1.4)
        ctr = torch.rand(512, 2, generator=g) * torch.tensor([1344.0, 800.0])
        ang = 180.0 - torch.rand(512, generator=g) * 360.0
        boxes.append(torch.cat([ctr, (s * ar.sqrt())[:, None], (s / ar.sqrt())[:, None], ang[:, None]], 1).to(device))
    return feats, boxes, [1 / 4, 1 / 8, 1 / 16, 1 / 32]


def time_rotated_pooler(D, res):
    """The reference's ROIPooler(pooler_type="ROIAlignRotated") structure (poolers.py:245-263): level assignment, then per level
    nonzero / gather / roi_align_rotated_forward / index_put_; the backward as its autograd does it (per level: gather of the
    output gradient rows, zero-filled gradient map, roi_align_rotated_backward)."""
    feats, boxes, scales = rotated_pooler_inputs()
    rois = torch.cat([torch.cat([torch.full((len(b), 1), float(i), device=DEV), b], 1) for i, b in enumerate(boxes)])

    def levels():
        sizes = torch.sqrt(rois[:, 3] * rois[:, 4])
        return torch.floor(4 + torch.log2(sizes / 224 + 1e-8)).clamp(2, 5).to(torch.int64) - 2

    def fwd():
        lv = levels()
        out = torch.zeros(len(rois), 256, 7, 7, device=DEV)
        for l, s in enumerate(scales):
            inds = torch.nonzero(lv == l, as_tuple=True)[0]
            out.index_put_((inds,), D.roi_align_rotated_forward(feats[l], rois[inds], s, 7, 7, 0))
        return out

    go = torch.randn(len(rois), 256, 7, 7, device=DEV)

    def bwd():
        lv = levels()
        grads = []
        for l, s in enumerate(scales):
            inds = torch.nonzero(lv == l, as_tuple=True)[0]
            n, c, h, w = feats[l].shape
            grads.append(D.roi_align_rotated_backward(go[inds], rois[inds], s, 7, 7, n, c, h, w, 0))
        return grads

    res["ROIPooler ROIAlignRotated fwd 7x7 K=2x512 (p2..p5)"] = timeit(fwd)
    res["ROIPooler ROIAlignRotated bwd 7x7 K=2x512 (p2..p5)"] = timeit(bwd)


def main():
    res = {}
    torch.ops.load_library(SO)
    D = torch.ops.detectron2
    time_rotated_pooler(D, res)
    spec = importlib.util.spec_from_loader("d2_ref_cuda", importlib.machinery.ExtensionFileLoader("d2_ref_cuda", SO))
    ref = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(ref)

    gb = torch.Generator().manual_seed(5)
    rb = torch.cat([torch.rand(1000, 2, generator=gb) * 300, 1 + torch.rand(1000, 2, generator=gb) * 120,
                    (torch.rand(1000, 1, generator=gb) - 0.5) * 360], 1).to(DEV)
    res["box_iou_rotated 1000x1000"] = timeit(lambda: D.box_iou_rotated(rb, rb))
    sc = torch.rand(1000, generator=gb).to(DEV)
    res["nms_rotated M=1000"] = timeit(lambda: D.nms_rotated(rb, sc, 0.5))
    xr = torch.rand(2, 256, 50, 84, generator=gb).to(DEV)
    rr = torch.cat([torch.randint(0, 2, (512, 1), generator=gb).float(), torch.rand(512, 2, generator=gb) * 800,
                    16 + torch.rand(512, 2, generator=gb) * 300, (torch.rand(512, 1, generator=gb) - 0.5) * 360], 1).to(DEV)
    res["roi_align_rotated fwd 512 boxes, 2x256x50x84"] = timeit(lambda: D.roi_align_rotated_forward(xr, rr, 1 / 16, 7, 7, 0))
    go = torch.randn(512, 256, 7, 7, device=DEV)
    res["roi_align_rotated bwd 512 boxes, 2x256x50x84"] = timeit(
        lambda: D.roi_align_rotated_backward(go, rr, 1 / 16, 7, 7, 2, 256, 50, 84, 0))
    # paste (torch GPU branch of the reference function)
    g2 = torch.Generator().manual_seed(1)
    masks = torch.rand(100, 28, 28, generator=g2).to(DEV)
    ctr = torch.rand(100, 2, generator=g2) * torch.tensor([1333.0, 800.0])
    wh = 20 + torch.rand(100, 2, generator=g2) * 300
    boxes = torch.cat([ctr - wh / 2, ctr + wh / 2], 1).to(DEV)
    res["paste_masks 100 x 28x28 -> 800x1333"] = timeit(lambda: paste_gpu_branch(masks, boxes, 800, 1333), rep=5, warm=1)
    # deformable conv: the reference's own CUDA path (deform_conv.py:43-141 calling _C.deform_conv_*), N=2
    for cin, hh, ww, grp in ((128, 100, 168, 1), (256, 50, 84, 1), (512, 25, 42, 1), (512, 100, 168, 32), (1024, 50, 84, 32),
                             (2048, 25, 42, 32)):
        n = 2
        x = torch.randn(n, cin, hh, ww, device=DEV)
        off = torch.randn(n, 18, hh, ww, device=DEV) * 2
        wt = torch.randn(cin, cin // grp, 3, 3, device=DEV) * 0.05
        gout = torch.randn(n, cin, hh, ww, device=DEV)
        bufs = [x.new_empty(0), x.new_empty(0)]
        step = 2  # im2col_step = min(N, 64)

        def fwd():
            out = x.new_empty(n, cin, hh, ww)
            ref.deform_conv_forward(x, wt, off, out, bufs[0], bufs[1], 3, 3, 1, 1, 1, 1, 1, 1, grp, 1, step)
            return out

        def bwd():
            gi, goff, gw = torch.zeros_like(x), torch.zeros_like(off), torch.zeros_like(wt)
            ref.deform_conv_backward_input(x, off, gout, gi, goff, wt, bufs[0], 3, 3, 1, 1, 1, 1, 1, 1, grp, 1, step)
            ref.deform_conv_backward_filter(x, off, gout, gw, bufs[0], bufs[1], 3, 3, 1, 1, 1, 1, 1, 1, grp, 1, 1.0, step)
            return gi, goff, gw

        try:
            res["deform_conv fwd C=%d %dx%d g=%d" % (cin, hh, ww, grp)] = timeit(fwd, rep=5, warm=1)
            res["deform_conv bwd C=%d %dx%d g=%d" % (cin, hh, ww, grp)] = timeit(bwd, rep=3, warm=1)
        except Exception as e:
            res["deform_conv C=%d g=%d error" % (cin, grp)] = str(e)[:200]
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(res, open(os.path.join(ROOT, "gpurun_out", "ref_gpu.json"), "w"), indent=1)
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    sys.exit(main())
