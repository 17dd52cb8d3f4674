"""CPU-side checks of the multi-level rotated pooler: the layout chooser, the rotated level rule of assign_boxes_to_levels,
and the fake kernels.  (The argument checks of the pooler entry points are in test_abi_and_host.py.)"""
import torch


def test_layout_chooser_sends_large_rotated_pooled_sizes_to_nchw(monkeypatch):
    """The one RoIAlign layout chooser, for rotated pyramids: shapes beyond the channels-last kernels' shared-memory tile
    (d2b_roi_pooler_nhwc_supported) go to the NCHW kernels whatever D2B_POOLER_LAYOUT says."""
    from detectron2_b200 import ops

    monkeypatch.setattr(ops, "POOLER_LAYOUT", "nhwc")
    shapes = [(2, 256, 200 // 2 ** l, 336 // 2 ** l) for l in range(4)]
    assert ops._pick_layout(shapes, 10, (7, 7), rotated=True, backward=False, channels_last=False) == "xpose"
    assert ops._pick_layout(shapes, 10, (14, 14), rotated=True, backward=True, channels_last=True) == "cl"
    # [128][400] fp32 tile > 150 KB
    assert ops._pick_layout(shapes, 10, (20, 20), rotated=True, backward=False, channels_last=True) == "nchw"
    assert ops._pick_layout(shapes, 10, (20, 20), rotated=True, backward=True, channels_last=False) == "nchw"


def test_assign_boxes_to_levels_rotated_area_is_w_times_h():
    from detectron2_b200.poolers import assign_boxes_to_levels

    # (cx, cy, w, h, angle): sqrt(w*h) = 112, 224, 448, 56 and 4000 -> levels 3, 4, 5, 2 (clamped) and 5 (clamped); the
    # centre coordinates must not enter the area (the 4-column formula would give (w - cx) * (h - cy))
    rb = torch.tensor([[500.0, 400, 112, 112, 30], [10, 20, 224, 224, -90], [0, 0, 448, 448, 180], [300, 300, 28, 112, 45],
                       [1, 1, 4000, 4000, 0]])
    assert assign_boxes_to_levels([rb[:2], rb[2:]], 2, 5, 224, 4).tolist() == [1, 2, 3, 0, 3]
    ab = torch.tensor([[100.0, 100, 212, 212], [100, 100, 324, 324]])  # the axis-aligned rule is unchanged
    assert assign_boxes_to_levels([ab], 2, 5, 224, 4).tolist() == [1, 2]


def test_rotated_pooler_fake_kernels_trace_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    from detectron2_b200 import ops

    with FakeTensorMode():
        feats = [torch.empty(2, 16, 40 // 2 ** i, 60 // 2 ** i, device="cuda") for i in range(4)]
        rois = torch.empty(7, 6, device="cuda")
        y = ops.roi_pooler_rotated_op(feats, rois, [1 / 4, 1 / 8, 1 / 16, 1 / 32], 14, 14, 0, 2, 5, 4, 224.0)
        assert y.shape == (7, 16, 14, 14)
        shapes = [2, 16] + [s for t in feats for s in t.shape[2:]]
        g = ops.roi_pooler_rotated_backward_op(y, rois, shapes, [1 / 4, 1 / 8, 1 / 16, 1 / 32], 14, 14, 0, 2, 5, 4, 224.0)
        assert [tuple(t.shape) for t in g] == [tuple(t.shape) for t in feats]
