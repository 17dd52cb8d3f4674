"""Fused multi-level ROIPooler(pooler_type="ROIAlignRotated") on the GPU: against the reference's per-level loop on the CPU
oracle, against this library's own single-level ROIAlignRotated, in fp16 / bf16, and captured in a CUDA graph."""
import math

import numpy as np
import pytest
import torch

import roi_align_rotated_ref as rr
from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda"
SCALES = [1 / 4, 1 / 8, 1 / 16, 1 / 32]


def rel_close(a, b, rtol=1e-4, atol=1e-5):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return torch.allclose(a, b, rtol=rtol, atol=atol), (a - b).abs().max().item()


def _rot_boxes(g, k, img_w=672.0, img_h=400.0):
    """k rotated boxes (cx, cy, w, h, angle): sizes log-uniform in [8, 700], aspect ratios up to ~2, angles in (-180, 180]."""
    s = torch.exp(torch.rand(k, generator=g) * (math.log(700) - math.log(8)) + math.log(8))
    ar = torch.exp((torch.rand(k, generator=g) - 0.5) * 1.4)
    ctr = torch.rand(k, 2, generator=g) * torch.tensor([img_w, img_h])
    ang = 180.0 - torch.rand(k, generator=g) * 360.0
    return torch.cat([ctr, (s * ar.sqrt())[:, None], (s / ar.sqrt())[:, None], ang[:, None]], 1)


def _case(seed, c, k=60):
    g = torch.Generator().manual_seed(seed)
    feats = [torch.randn(2, c, 100 // 2 ** i, 168 // 2 ** i, generator=g) for i in range(4)]
    per_img = [_rot_boxes(g, k), _rot_boxes(g, k)]
    # exactly on level boundaries: sqrt(w*h) = 112, 224, 448 (the 56 x 224 box as well)
    per_img[0][:4, 2:4] = torch.tensor([[112.0, 112.0], [224.0, 224.0], [448.0, 448.0], [56.0, 224.0]])
    per_img[1][0, 2:4] = torch.tensor([-30.0, 40.0])  # negative area: NaN level, matches no level in the reference's loop
    per_img[1][1] = torch.tensor([330.0, 200.0, 900.0, 700.0, 30.0])  # larger than the image
    per_img[1][2, 2:4] = 0.0                                           # empty box
    rois = torch.cat([torch.cat([torch.full((k, 1), float(i)), b], 1) for i, b in enumerate(per_img)])
    return g, feats, per_img, rois, k  # row k of rois is the negative-area box


def _oracle_levels(rois):
    # detectron2/modeling/poolers.py:23-59 with RotatedBoxes.area() = w * h
    sizes = torch.sqrt(rois[:, 3] * rois[:, 4])
    return torch.floor(4 + torch.log2(sizes / 224 + 1e-8)).clamp(2, 5).to(torch.int64) - 2


def _rot_bin_f64(feat, roi, scale, ph_n, pw_n, sr, c, ph, pw):
    """One output element of ROIAlignRotated in float64 (tests/roi_align_rotated_ref.py), to tell which of two fp32
    evaluations is off when they disagree."""
    R = rr.Roi(roi.numpy().astype(np.float32), scale, ph_n, pw_n, sr, feat.shape[2], feat.shape[3])
    return float(R.forward(feat[R.g.b, c:c + 1])[0][0, ph, pw])


def _set_layout(layout, feats, monkeypatch):
    from detectron2_b200 import ops

    if layout == "cl":
        return [f.to(DEV).contiguous(memory_format=torch.channels_last) for f in feats]
    monkeypatch.setattr(ops, "POOLER_LAYOUT", layout)
    return [f.to(DEV) for f in feats]


@pytest.mark.parametrize("layout", ["nchw", "nhwc", "cl"])
@pytest.mark.parametrize("c", [32, 132, 6])
@pytest.mark.parametrize("out,sr", [(7, 0), (7, 2), (14, 0), (14, 2)])
def test_fused_rotated_pooler_vs_reference_loop(layout, c, out, sr, monkeypatch):
    from detectron2_b200.poolers import ROIPooler, assign_boxes_to_levels

    g, feats, per_img, rois, neg = _case(c + out + sr, c)
    lv = _oracle_levels(rois)
    assert not (0 <= lv[neg] < 4)
    ref = torch.zeros(len(rois), c, out, out)
    for l, s in enumerate(SCALES):
        inds = torch.nonzero(lv == l, as_tuple=True)[0]
        ref[inds] = orc.roi_align_rotated_forward(feats[l], rois[inds], s, out, out, sr)
    fd = [f.requires_grad_(True) for f in _set_layout(layout, feats, monkeypatch)]
    boxes = [b.to(DEV) for b in per_img]
    assert torch.equal(assign_boxes_to_levels(boxes, 2, 5, 224, 4).cpu()[lv != lv[neg]], lv[lv != lv[neg]])
    y = ROIPooler(out, SCALES, sr, "ROIAlignRotated")(fd, boxes)
    # Within rtol 1e-4 / atol 5e-5 of the oracle.  Where the two fp32 evaluations differ by more (sample coordinates rotated
    # with sincosf / FMA here and cosf / sinf without FMA in the oracle land on slightly different points of a steep bilinear
    # patch of the randn maps), the output must be within the same tolerance of the float64 evaluation of that element.
    yc = y.detach().cpu()
    off = ((yc - ref).abs() > 5e-5 + 1e-4 * ref.abs()).nonzero().tolist()
    assert len(off) <= 8, len(off)
    for k, ch, i, j in off:
        l = int(lv[k])
        v64 = _rot_bin_f64(feats[l], rois[k], SCALES[l], out, out, sr, ch, i, j)
        ours, theirs = yc[k, ch, i, j].item(), ref[k, ch, i, j].item()
        assert abs(ours - v64) <= 5e-5 + 1e-4 * abs(v64), (k, ch, i, j, ours, theirs, v64)
    assert (y[neg] == 0).all()
    go = torch.randn(y.shape, generator=g)
    go_no_neg = go.clone()
    go_no_neg[neg] = 0
    y.backward(go.to(DEV))
    for l, s in enumerate(SCALES):
        inds = torch.nonzero(lv == l, as_tuple=True)[0]
        gref = orc.roi_align_rotated_backward(go[inds], rois[inds], s, out, out, 2, c, feats[l].shape[2], feats[l].shape[3], sr)
        if layout == "cl" and c % 4 == 0:
            assert fd[l].grad.is_contiguous(memory_format=torch.channels_last)
        ok, err = rel_close(fd[l].grad, gref, atol=3e-4)
        assert ok, (l, err)
    # the negative-area box contributes no gradient: the same backward without its grad_out row gives the same maps
    fd2 = [f.detach().clone().requires_grad_(True) for f in fd]
    ROIPooler(out, SCALES, sr, "ROIAlignRotated")(fd2, boxes).backward(go_no_neg.to(DEV))
    for a, b in zip(fd, fd2):
        ok, err = rel_close(a.grad, b.grad, rtol=1e-5, atol=1e-5)
        assert ok, err


@pytest.mark.parametrize("layout", ["nchw", "nhwc", "cl"])
def test_fused_rotated_pooler_equals_single_level_layer(layout, monkeypatch):
    # same kernel arithmetic per RoI as the library's own ROIAlignRotated applied level by level with the same layout
    import detectron2_b200.layers as L
    from detectron2_b200.poolers import ROIPooler

    g, feats, per_img, rois, neg = _case(7, 64, k=150)
    lv = _oracle_levels(rois)
    fd = [f.requires_grad_(True) for f in _set_layout(layout, feats, monkeypatch)]
    y = ROIPooler(7, SCALES, 0, "ROIAlignRotated")(fd, [b.to(DEV) for b in per_img])
    go = torch.randn(y.shape, generator=g).to(DEV)
    y.backward(go)
    rd = rois.to(DEV)
    for l, s in enumerate(SCALES):
        inds = torch.nonzero(lv == l, as_tuple=True)[0].to(DEV)
        xl = fd[l].detach().clone() if layout != "cl" else fd[l].detach().clone(memory_format=torch.channels_last)
        xl.requires_grad_(True)
        yl = L.ROIAlignRotated((7, 7), s, 0)(xl, rd[inds])
        assert torch.equal(y[inds], yl), l
        yl.backward(go[inds])
        ok, err = rel_close(fd[l].grad, xl.grad, rtol=1e-5, atol=1e-5)  # only the order of the atomic adds differs
        assert ok, (l, err)
    assert (y[neg] == 0).all()


@pytest.mark.parametrize("layout", ["auto", "nhwc", "cl"])
@pytest.mark.parametrize("dt", [torch.float16, torch.bfloat16])
def test_fused_rotated_pooler_half_precision(dt, layout, monkeypatch):
    # fp32 arithmetic on the stored half values: the output is the fp32 result rounded once to the feature dtype, and the
    # gradients come back in the feature dtype
    from detectron2_b200.poolers import ROIPooler

    eps = 2.0 ** -8 if dt == torch.bfloat16 else 2.0 ** -11
    g, feats, per_img, rois, neg = _case(5, 128, k=100)
    feats = [f.to(dt) for f in feats]
    boxes = [b.to(DEV) for b in per_img]
    fd = [f.requires_grad_(True) for f in _set_layout(layout, feats, monkeypatch)]
    f32 = [f.detach().float().requires_grad_(True) for f in fd]  # preserves the memory format
    y = ROIPooler(7, SCALES, 0, "ROIAlignRotated")(fd, boxes)
    y32 = ROIPooler(7, SCALES, 0, "ROIAlignRotated")(f32, boxes)
    assert y.dtype == dt
    assert torch.equal(y, y32.to(dt))
    go = torch.randn(y.shape, generator=g).to(dt).to(DEV)
    y.backward(go)
    y32.backward(go.float())
    for a, b in zip(fd, f32):
        assert a.grad.dtype == dt
        ok, err = rel_close(a.grad, b.grad.to(dt), rtol=2 * eps, atol=2 * eps * max(b.grad.abs().max().item(), 1.0))
        assert ok, err


def test_rotated_pooler_forward_backward_in_cuda_graph():
    # the public pooler, forward + autograd backward over 4 levels, captured once and replayed on new features and boxes
    from detectron2_b200.poolers import ROIPooler

    g, feats, per_img, rois, neg = _case(17, 48, k=80)
    pooler = ROIPooler(7, SCALES, 0, "ROIAlignRotated")
    fs = [f.to(DEV).requires_grad_(True) for f in feats]
    bs = [b.to(DEV) for b in per_img]
    go = torch.randn(len(rois), 48, 7, 7, generator=g).to(DEV)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):  # warm-up (allocations, shared-memory opt-in) outside the capture
        for _ in range(2):
            for f in fs:
                f.grad = None
            pooler(fs, bs).backward(go)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    for f in fs:
        f.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        y = pooler(fs, bs)
        y.backward(go)
    for rep in range(2):
        if rep == 1:  # new values in the captured buffers
            _, feats2, per_img2, _, _ = _case(18, 48, k=80)
            with torch.no_grad():
                for f, f2 in zip(fs, feats2):
                    f.copy_(f2)
                for b, b2 in zip(bs, per_img2):
                    b.copy_(b2)
        graph.replay()
        torch.cuda.synchronize()
        fe = [f.detach().clone().requires_grad_(True) for f in fs]
        ye = pooler(fe, [b.clone() for b in bs])
        ye.backward(go)
        assert torch.equal(y, ye), rep
        for a, b in zip(fs, fe):
            ok, err = rel_close(a.grad, b.grad, rtol=1e-5, atol=1e-5)
            assert ok, (rep, err)
