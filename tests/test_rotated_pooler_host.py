"""CPU-side checks of the multi-level rotated pooler: argument validation of its C entry points (every check runs before
anything is launched, so no GPU is needed), the rotated level rule of assign_boxes_to_levels, and the fake kernels."""
import ctypes as C

import torch

EINVAL = -1


def _pyr(num_levels=4, min_level=2):
    from detectron2_b200 import _C

    P = _C.Pyramid()
    P.num_levels = num_levels
    for l in range(num_levels):
        P.H[l], P.W[l] = 64 >> l, 96 >> l
        P.scale[l] = 1.0 / 2 ** (min_level + l)
        P.feat[l] = P.grad[l] = 0x1000 * (l + 1)  # never dereferenced: every call below fails or returns before a launch
    P.min_level, P.max_level, P.canonical_level, P.canonical_box_size = min_level, min_level + num_levels - 1, 4, 224.0
    return P


def test_rotated_pooler_entry_points_validate_arguments_without_a_gpu():
    from detectron2_b200 import _C

    lib = _C.lib()
    fwd = lambda P, n=2, k=3, rois=0x10, out=0x20, dt=None: (  # noqa: E731
        lib.d2b_roi_pooler_rotated_forward(C.byref(P), n, 8, rois, k, 7, 7, 0, out, None) if dt is None else
        lib.d2b_roi_pooler_rotated_forward_nhwc_t(C.byref(P), n, 8, rois, k, 7, 7, 0, out, dt, None))
    bwd = lambda P, n=2, k=3, go=0x10, rois=0x20, dt=None: (  # noqa: E731
        lib.d2b_roi_pooler_rotated_backward(C.byref(P), n, 8, go, rois, k, 7, 7, 0, None) if dt is None else
        lib.d2b_roi_pooler_rotated_backward_nhwc_t(C.byref(P), n, 8, go, dt, rois, k, 7, 7, 0, None))
    calls = [lambda P, **a: fwd(P, **a), lambda P, **a: fwd(P, dt=0, **a), lambda P, **a: bwd(P, **a),
             lambda P, **a: bwd(P, dt=0, **a)]
    for call in calls:
        # level boxes are an axis-aligned notion: rotated RoIs are never rounded to the feature dtype
        P = _pyr()
        P.level_rois = 0x30
        assert call(P) == EINVAL
        # num_levels does not match max_level - min_level + 1
        P = _pyr()
        P.max_level = 6
        assert call(P) == EINVAL
        P = _pyr()
        P.num_levels = 0
        assert call(P) == EINVAL
        P.num_levels = _C.MAX_LEVELS + 1
        assert call(P) == EINVAL
        # negative sizes
        assert call(_pyr(), n=-1) == EINVAL
        assert call(_pyr(), k=-1) == EINVAL
        # no images, no RoIs: nothing to do
        assert call(_pyr(), n=0, k=0) == 0
    # bad dtype codes of the half-precision variants
    assert fwd(_pyr(), dt=3) == EINVAL and fwd(_pyr(), dt=-1) == EINVAL
    assert bwd(_pyr(), dt=7) == EINVAL
    # missing pointers
    assert fwd(_pyr(), rois=None) == EINVAL and fwd(_pyr(), out=None) == EINVAL
    assert fwd(_pyr(), dt=1, rois=None) == EINVAL and fwd(_pyr(), dt=2, out=None) == EINVAL
    assert bwd(_pyr(), go=None) == EINVAL and bwd(_pyr(), rois=None) == EINVAL
    assert bwd(_pyr(), dt=1, go=None) == EINVAL and bwd(_pyr(), dt=2, rois=None) == EINVAL
    for call in calls:
        P = _pyr()
        P.feat[2] = P.grad[2] = None
        assert call(P) == EINVAL
    # the channels-last forms need 16-byte aligned maps
    P = _pyr()
    P.feat[1] = P.grad[1] = 0x1004
    assert fwd(P, dt=0) == EINVAL and bwd(P, dt=0) == EINVAL
    # no images but RoIs: the RoIs point at images that do not exist (both directions)
    for call in calls:
        assert call(_pyr(), n=0, k=3) == EINVAL
    # pooled sizes beyond the channels-last kernel's shared-memory tile: refused before the backward's zero-fill launch
    assert lib.d2b_roi_pooler_rotated_backward_nhwc_t(C.byref(_pyr()), 2, 8, 0x10, 0, 0x20, 3, 20, 20, 0, None) == -3
    assert lib.d2b_roi_pooler_rotated_backward_nhwc_t(C.byref(_pyr()), 2, 6, 0x10, 0, 0x20, 3, 7, 7, 0, None) == -3


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
