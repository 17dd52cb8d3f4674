"""Keypoint head kernels on the GPU against the torch restatement run on the same CUDA tensors (the reference's own
operations: F.interpolate bicubic, max / argmax, cross_entropy), and detector_postprocess against the reference fixture."""
import math

import pytest
import torch
from torch.nn import functional as F

pytestmark = pytest.mark.gpu

K, S = 17, 56
DEV = "cuda"


def scene(images, per_image=100, seed=0):
    """Detections of `images` 800 x 1333 images: box sides log-uniform in 16-600 px, plus one full-image box."""
    g = torch.Generator().manual_seed(seed)
    r = images * per_image
    side = torch.exp(torch.empty(r, 2).uniform_(math.log(16.0), math.log(600.0), generator=g))
    ctr = torch.rand(r, 2, generator=g) * torch.tensor([1333.0, 800.0])
    rois = torch.cat([ctr - side / 2, ctr + side / 2], dim=1)
    rois[0] = torch.tensor([0.0, 0.0, 1333.0, 800.0])
    maps = torch.randn((r, K, S, S), generator=g) * 3
    return maps.to(DEV), rois.to(DEV)


def top2(maps, rois):
    """Largest and second-largest value of every resized map (the reference's own interpolation)."""
    w = (rois[:, 2] - rois[:, 0]).clamp(min=1).ceil()
    h = (rois[:, 3] - rois[:, 1]).clamp(min=1).ceil()
    out = []
    for i, (hi, wi) in enumerate(torch.stack([h, w], 1).tolist()):
        m = F.interpolate(maps[[i]], size=(int(hi), int(wi)), mode="bicubic", align_corners=False)[0]
        out.append(m.reshape(maps.shape[1], -1).topk(2, dim=1).values)
    return torch.stack(out)


@pytest.mark.parametrize("images", [1, 2])
def test_keypoints_from_heatmaps_matches_reference(images):
    from detectron2_b200 import keypoint_head as kh

    maps, rois = scene(images, seed=images)
    ref = kh._heatmaps_to_keypoints_host(maps, rois)
    out = kh.heatmaps_to_keypoints(maps, rois)
    torch.cuda.synchronize()
    t2 = top2(maps, rois)
    clear = (t2[..., 0] - t2[..., 1]) > 1e-6 * t2[..., 0].abs()
    same_xy = (out[..., :2] == ref[..., :2]).all(dim=-1)
    assert bool(same_xy[clear].all()), int((~same_xy[clear]).sum())
    near_ties = int((~clear).sum())
    assert int((~same_xy[~clear]).sum()) <= max(near_ties, 0) and near_ties <= 0.01 * clear.numel()
    assert torch.equal(out[..., 2], ref[..., 2]), float((out[..., 2] - ref[..., 2]).abs().max())
    assert bool(((out[..., 3] - ref[..., 3]).abs() <= 1e-5 * ref[..., 3].abs()).all())


def test_argmax_ties_and_nan_follow_torch():
    from detectron2_b200 import keypoint_head as kh

    rois = torch.tensor([[10.0, 20.0, 110.0, 70.5], [3.0, 4.0, 60.0, 61.0], [0.0, 0.0, 56.0, 56.0]], device=DEV)
    maps = torch.randn((3, K, S, S), generator=torch.Generator().manual_seed(5)).to(DEV)
    maps[0] = 0.0  # constant: every resized pixel is exactly 0, all tie and the first wins
    maps[1, 2, 30, 17] = float("nan")  # a NaN spreads over a 4 x 4 footprint of the resized map: the first NaN wins
    maps[2, 4, 7, 9] = float("nan")  # same-size map (PyTorch copies): the NaN pixel itself
    maps[2, 5] = -maps[2, 5].abs() - 1.0
    maps[2, 5, 0, 1] = -0.0
    maps[2, 5, 0, 3] = 0.0  # maximum 0 as -0 at (0, 1) and as +0 at (0, 3): equal values, (0, 1) wins
    out = kh.heatmaps_to_keypoints(maps, rois)
    ref = kh._heatmaps_to_keypoints_host(maps, rois)
    assert bool((out[0, :, 0] == 10.5).all()) and torch.equal(out[0, :, :3], ref[0, :, :3])
    for i, k in ((1, 2), (2, 4)):
        assert torch.equal(out[i, k, :2], ref[i, k, :2]), (i, k)
        assert math.isnan(float(out[i, k, 2])) and math.isnan(float(out[i, k, 3]))
    assert float(out[2, 4, 0]) == 9.5 and float(out[2, 4, 1]) == 7.5
    assert torch.equal(out[2, 5, :3], ref[2, 5, :3]) and float(out[2, 5, 0]) == 1.5 and float(out[2, 5, 1]) == 0.5
    assert math.copysign(1.0, float(out[2, 5, 2])) < 0
    keep = torch.ones((3, K), dtype=torch.bool, device=DEV)
    keep[1, 2] = keep[2, 4] = False
    assert torch.equal(out[..., :3][keep], ref[..., :3][keep])


def test_keypoints_from_heatmaps_edge_shapes():
    from detectron2_b200 import keypoint_head as kh

    assert kh.heatmaps_to_keypoints(torch.zeros(0, K, S, S, device=DEV), torch.zeros(0, 4, device=DEV)).shape == (0, K, 4)
    # non-finite boxes and a box of more than 2^32 pixels: NaN rows, the other rows untouched
    rois = torch.tensor([[0.0, 0.0, 30.0, 20.0], [float("nan"), 0.0, 5.0, 5.0], [0.0, 0.0, float("inf"), 9.0],
                         [0.0, 0.0, 70000.0, 70000.0], [1.0, 2.0, 9.0, 40.0]], device=DEV)
    maps = torch.randn((5, 3, 20, 20), generator=torch.Generator().manual_seed(9)).to(DEV)
    out = kh.heatmaps_to_keypoints(maps, rois)
    assert bool(torch.isnan(out[1:4]).all())
    ref = kh._heatmaps_to_keypoints_host(maps[[0, 4]], rois[[0, 4]])
    assert torch.equal(out[[0, 4], :, :3], ref[..., :3])
    # half-precision maps are read as their fp32 up-cast
    hm = maps[[0, 4]].half()
    assert torch.equal(kh.heatmaps_to_keypoints(hm, rois[[0, 4]]), kh.heatmaps_to_keypoints(hm.float(), rois[[0, 4]]))


def test_keypoints_from_heatmaps_graph_capture():
    from detectron2_b200 import keypoint_head as kh

    maps, rois = scene(2, seed=3)
    eager = kh.heatmaps_to_keypoints(maps, rois)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        kh.heatmaps_to_keypoints(maps, rois)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static = kh.heatmaps_to_keypoints(maps, rois)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, eager)
    res = kh.keypoint_rcnn_inference(maps, [rois[:100], rois[100:]])
    assert torch.equal(torch.cat([r[0] for r in res]), eager[:, :, [0, 1, 3]])


# ---- loss -----------------------------------------------------------------------------------------------------------
def loss_scene(seed=0, images=2, per_image=64):
    g = torch.Generator().manual_seed(seed)
    boxes, kps = [], []
    for _ in range(images):
        side = 4 + torch.rand(per_image, 2, generator=g) * 200
        x1y1 = torch.rand(per_image, 2, generator=g) * 600
        b = torch.cat([x1y1, x1y1 + side], dim=1)
        b[0] = b[0].round()
        b[1, 2] = b[1, 0]  # zero width
        kp = torch.empty(per_image, K, 3)
        kp[..., :2] = b[:, None, :2] + (torch.rand(per_image, K, 2, generator=g) * 1.3 - 0.15) * side[:, None]
        kp[..., 2] = torch.randint(0, 3, (per_image, K), generator=g).float()
        kp[:, 0, 0], kp[:, 1, 1] = b[:, 2], b[:, 3]  # on x2 / y2
        kp[:, :2, 2] = 2.0
        boxes.append(b.to(DEV))
        kps.append(kp.to(DEV))
    logits = (torch.randn((images * per_image, K, S, S), generator=g) * 2).to(DEV)
    return logits, kps, boxes


def reference_loss(logits, kps, boxes, normalizer):
    """keypoint_rcnn_loss written out with the reference's operations (autograd through cross_entropy)."""
    from detectron2_b200 import keypoint_head as kh

    t, v = kh._keypoints_to_heatmap_host(torch.cat(kps), torch.cat(boxes), S)
    rows = torch.nonzero(v.view(-1)).squeeze(1)
    flat = logits.view(-1, S * S)
    loss = F.cross_entropy(flat[rows].float(), t.view(-1)[rows], reduction="sum")
    return loss / (rows.numel() if normalizer is None else normalizer)


def test_loss_targets_bit_exact():
    from detectron2_b200 import keypoint_head as kh

    logits, kps, boxes = loss_scene(1)
    kp, bx = torch.cat(kps), torch.cat(boxes)
    t_ref, v_ref = kh._keypoints_to_heatmap_host(kp, bx, S)
    t, v = kh.keypoints_to_heatmap(kp, bx, S)
    assert torch.equal(t, t_ref) and torch.equal(v, v_ref)
    _, t2, v2, nv = kh.keypoint_loss_op(logits, kp, bx)
    assert torch.equal(t2, t_ref) and torch.equal(v2.long(), v_ref) and int(nv) == int(v_ref.sum())
    assert 0 < int(nv) < v_ref.numel()


@pytest.mark.parametrize("normalizer", [None, 96.0])
def test_loss_and_gradient_match_reference(normalizer):
    from detectron2_b200 import keypoint_head as kh

    logits, kps, boxes = loss_scene(2)
    a = logits.clone().requires_grad_(True)
    b = logits.clone().requires_grad_(True)
    loss = kh.keypoint_rcnn_loss(a, kps, boxes, normalizer)
    ref = reference_loss(b, kps, boxes, normalizer)
    lv, rv = loss.detach().item(), ref.detach().item()
    assert abs(lv - rv) <= 1e-5 * abs(rv)
    loss.backward()
    ref.backward()
    assert float((a.grad - b.grad).abs().max()) <= 1e-4 * float(b.grad.abs().max())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_loss_half_precision_reads_the_upcast(dtype):
    from detectron2_b200 import keypoint_head as kh

    logits, kps, boxes = loss_scene(3)
    lh = logits.to(dtype).requires_grad_(True)
    lf = logits.to(dtype).float().requires_grad_(True)
    loss_h = kh.keypoint_rcnn_loss(lh, kps, boxes)
    loss_f = kh.keypoint_rcnn_loss(lf, kps, boxes)
    assert loss_h.dtype == torch.float32 and torch.equal(loss_h, loss_f)
    loss_h.backward()
    loss_f.backward()
    assert lh.grad.dtype == dtype and torch.equal(lh.grad, lf.grad.to(dtype))


def test_loss_without_valid_keypoints_is_zero():
    from detectron2_b200 import keypoint_head as kh

    logits, kps, boxes = loss_scene(4)
    for kp in kps:
        kp[..., 2] = 0.0
    a = logits.clone().requires_grad_(True)
    for normalizer in (None, 8.0):
        loss, nv = kh.keypoint_rcnn_loss_fixed(a, kps, boxes, normalizer)
        assert int(nv) == 0 and loss.detach().item() == 0.0
        loss.backward()
        assert a.grad is not None and not bool(a.grad.any())


def test_loss_fixed_graph_capture():
    from detectron2_b200 import keypoint_head as kh

    logits, kps, boxes = loss_scene(5)
    eager, nv = kh.keypoint_rcnn_loss_fixed(logits, kps, boxes)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        kh.keypoint_rcnn_loss_fixed(logits, kps, boxes)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        static, static_nv = kh.keypoint_rcnn_loss_fixed(logits, kps, boxes)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, eager) and torch.equal(static_nv, nv)


def test_detector_postprocess_keypoints_on_cuda(golden):
    from detectron2_b200.fast_rcnn_inference import Detections
    from detectron2_b200.postprocessing import detector_postprocess

    d = golden("keypoints")
    T = lambda k: torch.from_numpy(d[k]).to(DEV)  # noqa: E731
    h, w, oh, ow = (int(v) for v in d["pp_hw"])
    res = detector_postprocess(Detections((h, w), T("pp_boxes"), T("pp_scores"), T("pp_classes")), oh, ow,
                               pred_keypoints=T("pp_keypoints"))
    assert torch.equal(res.pred_boxes, T("pp_out_boxes")) and torch.equal(res.pred_keypoints, T("pp_out_keypoints"))
