"""Keypoint head on CPU: the torch restatement (detectron2_b200.keypoint_head) against the fixture from the REAL reference
functions (tests/golden/make_golden_keypoints.py), the argument checks of the native entry points and the fake kernels
(no GPU needed)."""
import ctypes as C

import numpy as np
import pytest
import torch

T = torch.from_numpy


def heatmaps(d):
    """The fixture's maps, regenerated from its seed as make_golden_keypoints.heatmaps() does."""
    k, s, r = int(d["K"]), int(d["S"]), len(d["rois"])
    maps = torch.randn((r, k, s, s), generator=torch.Generator().manual_seed(int(d["maps_seed"])))
    maps[int(d["const_roi"])] = float(d["const_value"])
    return maps


def loss_logits(d, n):
    k, s = int(d["K"]), int(d["S"])
    return torch.randn((n, k, s, s), generator=torch.Generator().manual_seed(int(d["logits_seed"])))


def loss_inputs(d):
    boxes = [T(d[f"boxes{i}"]) for i in range(3)]
    kps = [T(d[f"kps{i}"]) for i in range(3)]
    return boxes, kps, loss_logits(d, sum(len(b) for b in boxes))


def rel_close(a, b, tol):
    a, b = torch.as_tensor(a, dtype=torch.float64), torch.as_tensor(b, dtype=torch.float64)
    return bool(((a - b).abs() <= tol * b.abs()).all())


def test_fixture_inputs_cover_the_edge_cases(golden):
    d = golden("keypoints")
    rois = T(d["rois"])
    w, h = rois[:, 2] - rois[:, 0], rois[:, 3] - rois[:, 1]
    assert ((w < 1) & (h > 1)).any() and ((w < 1) & (h < 1)).any()  # narrower than 1 px
    assert ((rois == rois.round()).all(dim=1)).any() and (rois != rois.round()).any()  # integer and sub-pixel edges
    assert ((w.clamp(min=1).ceil() == int(d["S"])) & (h.clamp(min=1).ceil() == int(d["S"]))).any()  # same-size copy
    assert (w > 10 * int(d["S"])).any()  # larger than the map
    xy = T(d["xy_preds"])
    c = int(d["const_roi"])
    # the constant maps: every keypoint at the first pixel
    assert torch.equal(xy[c, :, 0], torch.full_like(xy[c, :, 0], float((0.5 * (w[c] / w[c].ceil())) + rois[c, 0])))
    boxes, kps, _ = loss_inputs(d)
    kp0, b0 = kps[0], boxes[0]
    assert (kp0[:, :, 0] == b0[:, 2:3]).any() and (kp0[:, :, 1] == b0[:, 3:4]).any()  # on x2 / y2
    assert set(kp0[:, :, 2].unique().tolist()) == {0.0, 1.0, 2.0}
    assert ((kp0[:, :, 0] < b0[:, 0:1]) | (kp0[:, :, 0] > b0[:, 2:3])).any()  # outside the box
    assert T(d["valid0"]).any() and not T(d["valid2"]).any() and len(boxes[1]) == 0  # an image without valid keypoints
    assert float(d["loss_no_valid"]) == 0.0


def test_heatmaps_to_keypoints_restatement_matches_reference(golden):
    from detectron2_b200 import keypoint_head as kh

    d = golden("keypoints")
    ref = T(d["xy_preds"])
    out = kh.heatmaps_to_keypoints(heatmaps(d), T(d["rois"]))
    assert torch.equal(out[..., :3], ref[..., :3])  # positions and logits: the same torch CPU ops
    assert rel_close(out[..., 3], ref[..., 3], 1e-6)


def test_inference_split_per_image(golden):
    from detectron2_b200 import keypoint_head as kh

    d = golden("keypoints")
    maps, rois = heatmaps(d), T(d["rois"])
    res = kh.keypoint_rcnn_inference(maps, [rois[:6], rois[6:6], rois[6:]])
    assert [r[0].shape[0] for r in res] == [6, 0, len(rois) - 6]
    ref = T(d["xy_preds"])[:, :, [0, 1, 3]]
    assert torch.equal(torch.cat([r[0] for r in res])[..., :2], ref[..., :2])
    assert torch.equal(torch.cat([r[1] for r in res]), maps)


def test_targets_restatement_matches_reference(golden):
    from detectron2_b200 import keypoint_head as kh

    d = golden("keypoints")
    boxes, kps, _ = loss_inputs(d)
    for i in (0, 2):
        t, v = kh.keypoints_to_heatmap(kps[i], boxes[i], int(d["S"]))
        assert torch.equal(t, T(d[f"target{i}"])) and torch.equal(v, T(d[f"valid{i}"])), i


def test_loss_restatement_matches_reference(golden):
    from detectron2_b200 import keypoint_head as kh

    d = golden("keypoints")
    boxes, kps, logits = loss_inputs(d)
    assert rel_close(kh.keypoint_rcnn_loss(logits, kps, boxes, None), T(d["loss_none"]), 1e-6)
    assert rel_close(kh.keypoint_rcnn_loss(logits, kps, boxes, 7.5), T(d["loss_norm"]), 1e-6)
    n2 = len(boxes[2])
    zero = kh.keypoint_rcnn_loss(logits[-n2:].requires_grad_(True), [kps[2]], [boxes[2]], None)
    assert zero.requires_grad and float(zero.detach()) == float(d["loss_no_valid"]) == 0.0


def test_detector_postprocess_keypoints_match_reference(golden):
    from detectron2_b200.fast_rcnn_inference import Detections
    from detectron2_b200.postprocessing import detector_postprocess

    d = golden("keypoints")
    h, w, oh, ow = (int(v) for v in d["pp_hw"])
    det = Detections((h, w), T(d["pp_boxes"]), T(d["pp_scores"]), T(d["pp_classes"]))
    kp = T(d["pp_keypoints"])
    kp_in = kp.clone()
    res = detector_postprocess(det, oh, ow, pred_keypoints=kp)
    assert torch.equal(kp, kp_in)  # the caller's tensor is not modified
    assert torch.equal(res.pred_boxes, T(d["pp_out_boxes"]))
    assert torch.equal(res.pred_keypoints, T(d["pp_out_keypoints"]))
    assert detector_postprocess(det, oh, ow).pred_keypoints is None


def test_keypoint_entry_points_reject_bad_arguments():
    """Argument checks run before the first CUDA call: D2B_EINVAL / D2B_EWORKSPACE without a GPU."""
    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL, EWORKSPACE = -1, -2
    p = C.c_void_p(16)  # never dereferenced: the checks fail first
    ws = lib.d2b_keypoints_workspace_bytes(10, 17)
    assert ws >= 10 * 17 * 8 and lib.d2b_keypoints_workspace_bytes(0, 17) == 0
    good = dict(maps=p, R=10, K=17, S=56, rois=p, out=p, ws=p, ws_bytes=ws, stream=None)

    def heat(**over):
        a = dict(good, **over)
        return lib.d2b_keypoints_from_heatmaps(*a.values())

    for over in (dict(R=-1), dict(K=0), dict(S=0), dict(S=242), dict(maps=None), dict(rois=None), dict(out=None),
                 dict(ws=None), dict(out=C.c_void_p(20)), dict(ws=C.c_void_p(20))):
        assert heat(**over) == EINVAL, over
    assert heat(ws_bytes=ws - 1) == EWORKSPACE
    assert heat(R=0, maps=None, rois=None, out=None, ws=None) == 0  # nothing to do, nothing launched

    fwd = dict(logits=p, dtype=0, N=4, K=17, S=56, kps=p, boxes=p, target=p, valid=p, loss=p, num_valid=p, stream=None)

    def loss_fwd(**over):
        a = dict(fwd, **over)
        return lib.d2b_keypoint_loss_forward(*a.values())

    for over in (dict(N=-1), dict(K=0), dict(S=0), dict(S=50000), dict(dtype=3), dict(num_valid=None), dict(loss=None),
                 dict(logits=None), dict(kps=None), dict(boxes=None), dict(target=None), dict(valid=None)):
        assert loss_fwd(**over) == EINVAL, over

    bwd = dict(logits=p, dtype=0, N=4, K=17, S=56, target=p, valid=p, gs=p, grad=p, stream=None)

    def loss_bwd(**over):
        a = dict(bwd, **over)
        return lib.d2b_keypoint_loss_backward(*a.values())

    for over in (dict(N=-1), dict(K=0), dict(S=-3), dict(dtype=-1), dict(logits=None), dict(target=None), dict(valid=None),
                 dict(gs=None), dict(grad=None)):
        assert loss_bwd(**over) == EINVAL, over
    assert loss_bwd(N=0, logits=None, target=None, valid=None, gs=None, grad=None) == 0


def test_fake_kernels_trace_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    from detectron2_b200 import keypoint_head as kh

    with FakeTensorMode():
        maps = torch.empty(7, 17, 56, 56, device="cuda")
        assert kh.keypoints_from_heatmaps_op(maps, torch.empty(7, 4, device="cuda")).shape == (7, 17, 4)
        for dt in (torch.float32, torch.float16, torch.bfloat16):
            logits = torch.empty(5, 17, 56, 56, device="cuda", dtype=dt)
            loss, target, valid, nv = kh.keypoint_loss_op(logits, torch.empty(5, 17, 3, device="cuda"),
                                                          torch.empty(5, 4, device="cuda"))
            assert loss.shape == (5, 17) and loss.dtype == torch.float32
            assert target.shape == (5, 17) and target.dtype == torch.int64
            assert valid.shape == (5, 17) and valid.dtype == torch.uint8 and nv.shape == () and nv.dtype == torch.int64
            g = kh.keypoint_loss_backward_op(logits, target, valid, loss)
            assert g.shape == logits.shape and g.dtype == dt


@pytest.mark.parametrize("n", [0, 3])
def test_restatement_shapes_without_rois(n):
    from detectron2_b200 import keypoint_head as kh

    maps = torch.randn(n, 5, 8, 8)
    rois = torch.tensor([[0.0, 0.0, 4.0, 4.0]]).repeat(n, 1)
    assert kh.heatmaps_to_keypoints(maps, rois).shape == (n, 5, 4)
    assert np.all(np.isfinite(kh.heatmaps_to_keypoints(maps, rois).numpy()))
