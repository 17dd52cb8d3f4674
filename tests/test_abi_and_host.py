"""CPU-side tests: the C-ABI library loads and exports every symbol include/d2b200.h declares, and the host
wrappers keep the reference's surface (names, repr strings, exception types).  No compute calls: there is no GPU."""
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_header_symbols_and_abi_version():
    from detectron2_b200 import _C

    lib = _C.lib()
    header = open(os.path.join(ROOT, "include", "d2b200.h")).read()
    declared = set(re.findall(r"\b(d2b_[a-z0-9_]+)\s*\(", header)) - {"d2b_dcn_params"}
    assert len(declared) >= 14
    for name in declared:
        assert hasattr(lib, name), name
    assert set(_C.EXPORTED) == declared
    assert {n for n in declared if n.startswith(("d2b_roi_", "d2b_pyramid_"))} == {
        "d2b_roi_pooler_forward", "d2b_roi_pooler_backward", "d2b_roi_pooler_nhwc_supported", "d2b_pyramid_nchw_to_nhwc",
        "d2b_pyramid_nhwc_to_nchw"}
    # one entry point per selection stage, the box type and the decode as D2B_SELECT_* flags
    assert {n for n in declared if re.search(r"_(prepare|select)", n)} == {
        "d2b_rpn_prepare", "d2b_frcnn_prepare", "d2b_dense_prepare", "d2b_rpn_select"}
    # the FCOS loss is the dense loss with D2B_LOSS_LINEAR_GIOU
    assert {n for n in declared if n.startswith("d2b_fcos_")} == {"d2b_fcos_assign"}
    assert {n for n in declared if re.match(r"d2b_(dense|frcnn)_loss_", n)} == {
        "d2b_dense_loss_workspace_bytes", "d2b_dense_loss_forward", "d2b_dense_loss_backward",
        "d2b_frcnn_loss_workspace_bytes", "d2b_frcnn_loss_forward", "d2b_frcnn_loss_backward"}
    assert lib.d2b_abi_version() == _C.ABI_VERSION == 7
    assert lib.d2b_arch() == b"sm_90a"
    assert _C.get_cuda_version().startswith("CUDA 12")


def test_workspace_queries_run_on_host():
    from detectron2_b200 import _C

    small, big = _C.lib().d2b_nms_workspace_bytes(1000, 0, 0), _C.lib().d2b_nms_workspace_bytes(10000, 0, 0)
    assert 0 < small < big
    assert _C.lib().d2b_nms_workspace_bytes(10000, 1, 0) > big  # 5 floats per rotated box
    assert _C.lib().d2b_nms_workspace_bytes(10000, 0, 1000) < big / 4  # bounded categories: bitmask linear in M


def test_surface_matches_reference_names():
    import detectron2_b200.layers as L

    for name in ["ROIAlign", "roi_align", "ROIAlignRotated", "roi_align_rotated", "DeformConv", "ModulatedDeformConv",
                 "batched_nms", "nms", "batched_nms_rotated", "nms_rotated", "paste_masks_in_image",
                 "pairwise_iou_rotated"]:
        assert hasattr(L, name), name
    for op in ["nms_rotated", "box_iou_rotated", "roi_align_rotated_forward", "roi_align_rotated_backward"]:
        assert hasattr(torch.ops.detectron2, op)


def test_repr_strings():  # /root/reference/tests/layers/test_deformable.py:157-171
    import detectron2_b200.layers as L

    assert repr(L.DeformConv(3, 10, kernel_size=3, padding=1, deformable_groups=2)) == (
        "DeformConv(in_channels=3, out_channels=10, kernel_size=(3, 3), stride=(1, 1), padding=(1, 1), "
        "dilation=(1, 1), groups=1, deformable_groups=2, bias=False)")
    assert repr(L.ModulatedDeformConv(3, 10, kernel_size=3, padding=1, deformable_groups=2)) == (
        "ModulatedDeformConv(in_channels=3, out_channels=10, kernel_size=(3, 3), stride=1, padding=1, dilation=1, "
        "groups=1, deformable_groups=2, bias=True)")
    assert "aligned=True" in repr(L.ROIAlign((7, 7), 0.25, 0))
    m = L.ModulatedDeformConv(4, 8, 3)
    assert m.weight.shape == (8, 4, 3, 3) and m.bias.shape == (8,) and (m.bias == 0).all()


def test_no_cpu_fallback():
    import detectron2_b200.layers as L

    with pytest.raises(NotImplementedError):
        L.nms(torch.rand(4, 4), torch.rand(4), 0.5)
    with pytest.raises(NotImplementedError):
        L.ROIAlign((7, 7), 1.0, 0)(torch.rand(1, 1, 8, 8), torch.tensor([[0.0, 1, 1, 4, 4]]))
    with pytest.raises(NotImplementedError):
        L.DeformConv(1, 1, 3, padding=1)(torch.rand(1, 1, 5, 5), torch.zeros(1, 18, 5, 5))
    with pytest.raises(ValueError):
        L.deform_conv(torch.rand(1, 5, 5), torch.zeros(1, 18, 5, 5), torch.rand(1, 1, 3, 3))
    with pytest.raises(AssertionError):
        L.ROIAlign((7, 7), 1.0, 0)(torch.rand(1, 1, 8, 8), torch.rand(3, 4))


def test_empty_inputs_host_side():
    import detectron2_b200.layers as L

    assert L.batched_nms_rotated(torch.zeros(0, 5), torch.zeros(0), torch.zeros(0, dtype=torch.int64), 0.5).shape == (0,)
    assert L.batched_nms(torch.zeros(0, 4), torch.zeros(0), torch.zeros(0, dtype=torch.int64), 0.5).shape == (0,)
    out = L.paste_masks_in_image(torch.zeros(0, 28, 28), torch.zeros(0, 4), (10, 12))
    assert out.shape == (0, 10, 12) and out.dtype == torch.uint8
    y = L.DeformConv(2, 4, 3, padding=1)(torch.zeros(0, 2, 8, 8), torch.zeros(0, 18, 8, 8))
    assert y.shape == (0, 4, 8, 8)


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "detectron2_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f
                assert "import torchvision" not in src and "from torchvision" not in src, f


def test_fake_kernels_trace_shapes():
    """Every custom op has a fake (meta) kernel, so the ops trace / compile without touching the GPU library."""
    from torch._subclasses.fake_tensor import FakeTensorMode

    from detectron2_b200 import ops

    with FakeTensorMode():
        x = torch.empty(2, 16, 20, 30, device="cuda")
        rois = torch.empty(7, 5, device="cuda")
        assert ops.roi_align_op(x, rois, 0.25, 7, 7, 0, True).shape == (7, 16, 7, 7)
        assert ops.roi_align_rotated_op(x, torch.empty(7, 6, device="cuda"), 0.25, 5, 4, 2).shape == (7, 16, 5, 4)
        feats = [torch.empty(2, 16, 40 // 2 ** i, 60 // 2 ** i, device="cuda") for i in range(4)]
        y = ops.roi_pooler_op(feats, rois, [1 / 4, 1 / 8, 1 / 16, 1 / 32], 14, 14, 0, True, 2, 5, 4, 224.0)
        assert y.shape == (7, 16, 14, 14)
        w = torch.empty(24, 8, 3, 3, device="cuda")
        off = torch.empty(2, 18, 10, 15, device="cuda")
        out = ops.deform_conv_op(x, off, None, w, None, [2, 2], [1, 1], [1, 1], 2, 1, -1)
        assert out.shape == (2, 24, 10, 15)
        _check_dcn_fakes(ops, x, w, off)
        assert ops.box_iou_rotated_op(torch.empty(5, 5, device="cuda"), torch.empty(9, 5, device="cuda")).shape == (5, 9)
        pm = ops.paste_masks_op(torch.empty(3, 28, 28, device="cuda"), torch.empty(3, 4, device="cuda"), 40, 50, 0.5)
        assert pm.shape == (3, 40, 50) and pm.dtype == torch.bool  # threshold >= 0: bool output like the reference


_DCN_SCHEMAS = {
    "deform_conv": "d2b200::deform_conv(Tensor x, Tensor offset, Tensor? mask, Tensor weight, Tensor? bias, SymInt[] stride, "
                   "SymInt[] padding, SymInt[] dilation, SymInt groups, SymInt deformable_groups, SymInt precision) -> Tensor",
    "deform_conv_train": "d2b200::deform_conv_train(Tensor x, Tensor offset, Tensor? mask, Tensor weight, Tensor? bias, "
                         "SymInt[] stride, SymInt[] padding, SymInt[] dilation, SymInt groups, SymInt deformable_groups, "
                         "SymInt precision) -> (Tensor, Tensor, Tensor)",
    "deform_conv_backward": "d2b200::deform_conv_backward(Tensor x, Tensor offset, Tensor? mask, Tensor weight, "
                            "Tensor grad_out, SymInt[] stride, SymInt[] padding, SymInt[] dilation, SymInt groups, "
                            "SymInt deformable_groups, bool with_bias, bool need_data, bool need_weight, SymInt precision, "
                            "Tensor? cols=None) -> (Tensor, Tensor, Tensor, Tensor, Tensor)",
    "deform_conv_fused": "d2b200::deform_conv_fused(Tensor x, Tensor offset_mask, Tensor weight, Tensor? scale, "
                         "Tensor? shift, bool relu, SymInt[] stride, SymInt[] padding, SymInt[] dilation, SymInt groups, "
                         "SymInt deformable_groups, SymInt precision) -> Tensor",
    "deform_conv_fused_train": "d2b200::deform_conv_fused_train(Tensor x, Tensor offset_mask, Tensor weight, Tensor? scale, "
                               "Tensor? shift, bool relu, SymInt[] stride, SymInt[] padding, SymInt[] dilation, "
                               "SymInt groups, SymInt deformable_groups, SymInt precision) -> (Tensor, Tensor, Tensor)",
    "deform_conv_fused_backward": "d2b200::deform_conv_fused_backward(Tensor x, Tensor offset_mask, Tensor weight, "
                                  "Tensor? scale, bool relu, Tensor y, Tensor grad_out, SymInt[] stride, SymInt[] padding, "
                                  "SymInt[] dilation, SymInt groups, SymInt deformable_groups, SymInt precision, "
                                  "Tensor? cols=None) -> (Tensor, Tensor, Tensor)",
}


def _check_dcn_fakes(ops, x, w, off):
    """The six deformable-conv ops: schemas as released, and the shapes / dtypes of their fake outputs."""
    for name, schema in _DCN_SCHEMAS.items():
        assert str(getattr(torch.ops.d2b200, name).default._schema) == schema, name
    geo = ([2, 2], [1, 1], [1, 1], 2, 1)
    f32, u8, bf16 = torch.float32, torch.uint8, torch.bfloat16
    mask = torch.empty(2, 9, 10, 15, device="cuda")
    om = torch.empty(2, 27, 10, 15, device="cuda")
    sc, sh = torch.empty(24, device="cuda"), torch.empty(24, device="cuda")
    xb = x.to(bf16)

    def meta(ts):
        return [(tuple(t.shape), t.dtype) for t in ts]

    y = ops.deform_conv_op(xb, off, mask, w, sh, *geo, 1)
    assert meta([y]) == [((2, 24, 10, 15), bf16)]
    assert meta(ops.deform_conv_train_op(xb, off, mask, w, sh, *geo, -1)) == [((2, 24, 10, 15), bf16), ((0,), f32),
                                                                               ((0,), u8)]
    go = torch.empty(2, 24, 10, 15, device="cuda")
    assert meta(ops.deform_conv_backward_op(x, off, mask, w, go, *geo, True, True, True, 1)) == [
        ((2, 16, 20, 30), f32), ((2, 18, 10, 15), f32), ((2, 9, 10, 15), f32), ((24, 8, 3, 3), f32), ((24,), f32)]
    assert meta(ops.deform_conv_backward_op(x, off, None, w, go, *geo, False, False, True, 0)) == [
        ((0,), f32), ((0,), f32), ((0,), f32), ((24, 8, 3, 3), f32), ((0,), f32)]
    assert meta(ops.deform_conv_backward_op(x, off, mask, w, go, *geo, True, True, False, -1)) == [
        ((2, 16, 20, 30), f32), ((2, 18, 10, 15), f32), ((2, 9, 10, 15), f32), ((0,), f32), ((0,), f32)]
    y = ops.deform_conv_fused_op(xb, om, w, sc, sh, True, *geo, -1)
    assert meta([y]) == [((2, 24, 10, 15), bf16)]
    assert meta(ops.deform_conv_fused_train_op(xb, om, w, None, sh, False, *geo, 2)) == [((2, 24, 10, 15), bf16),
                                                                                        ((0,), f32), ((0,), u8)]
    assert meta(ops.deform_conv_fused_backward_op(x, om, w, sc, True, go, go, *geo, 1)) == [
        ((2, 16, 20, 30), f32), ((2, 27, 10, 15), f32), ((24, 8, 3, 3), f32)]


def test_pooler_layout_policy_host_logic(monkeypatch):
    """Which RoIAlign kernel a call gets (detectron2_b200/ops.py): pure host logic, checked on CPU tensors."""
    from detectron2_b200 import ops

    nchw = [torch.zeros(1, 256, 200 // 2 ** i, 336 // 2 ** i) for i in range(4)]
    cl = [t.contiguous(memory_format=torch.channels_last) for t in nchw]
    assert all(ops._is_channels_last(t) for t in cl) and not any(ops._is_channels_last(t) for t in nchw)
    # C == 1 or H*W == 1: both layouts coincide, treated as plain NCHW
    assert not ops._is_channels_last(torch.zeros(2, 1, 5, 5).contiguous(memory_format=torch.channels_last))
    monkeypatch.setattr(ops, "POOLER_LAYOUT", "auto")
    assert ops._pick_layout(cl, 1) == "cl"                        # channels_last is consumed in place
    assert ops._pick_layout(nchw, 1000 * 256 * 49) == "xpose"     # box head: layout change + NHWC kernel pays
    assert ops._pick_layout(nchw, 100 * 256 * 196) == "nchw"      # mask head alone: NCHW kernel
    assert ops._pick_layout(nchw, 10 * 256 * 49) == "nchw"
    assert ops._pick_layout([nchw[0], cl[1]], 10) == "nchw"        # mixed pyramid: falls back to the NCHW kernel
    odd = [torch.zeros(1, 6, 8, 8).contiguous(memory_format=torch.channels_last)]
    assert ops._pick_layout(odd, 10 ** 9) == "nchw"                # C % 4 != 0: NHWC kernel not applicable
    monkeypatch.setattr(ops, "POOLER_LAYOUT", "nchw")
    assert ops._pick_layout(cl, 1) == "nchw"
    monkeypatch.setattr(ops, "POOLER_LAYOUT", "nhwc")
    assert ops._pick_layout(nchw, 1) == "xpose"
    with pytest.raises(NotImplementedError):                       # no CPU fallback for the layout change either
        ops.pyramid_to_channels_last(nchw)


def test_channels_last_limits_without_a_gpu(monkeypatch):
    """d2b_roi_pooler_nhwc_supported is the one statement of the channels-last kernels' shape limits; the layout chooser
    sends every shape it refuses to the NCHW kernels.  Every call here is host-only."""
    import ctypes as C

    from detectron2_b200 import _C, ops

    lib = _C.lib()
    EINVAL, UNSUPPORTED = -1, -3
    ROT, BWD = _C.ROI_ROTATED, _C.ROI_BACKWARD

    def pyr(hw):
        P = _C.Pyramid()
        P.num_levels = len(hw)
        for l, (h, w) in enumerate(hw):
            P.H[l], P.W[l] = h, w
        return P

    bench = pyr([(200 // 2 ** l, 336 // 2 ** l) for l in range(4)])  # bench.py's 800x1333 pyramid
    q = lambda P, c, ph, pw, flags: lib.d2b_roi_pooler_nhwc_supported(C.byref(P), c, ph, pw, flags)  # noqa: E731
    for flags in (0, BWD, ROT, ROT | BWD):
        assert q(bench, 256, 7, 7, flags) == 0 and q(bench, 256, 14, 14, flags) == 0, flags
        assert q(bench, 6, 7, 7, flags) == UNSUPPORTED, flags                         # C % 4 != 0
        assert q(pyr([(16384, 16384)]), 4, 7, 7, flags) == UNSUPPORTED, flags        # H*W*C/4 >= 2^28
    assert q(bench, 256, 32, 32, BWD) == UNSUPPORTED and q(bench, 256, 7, 40, BWD) == UNSUPPORTED  # backward tile > 180 KB
    assert q(bench, 256, 32, 32, 0) == 0                                           # ... the forward takes them
    assert q(bench, 256, 20, 20, ROT) == UNSUPPORTED and q(bench, 256, 20, 20, ROT | BWD) == UNSUPPORTED  # tile > 150 KB
    assert lib.d2b_roi_pooler_nhwc_supported(None, 256, 7, 7, 0) == EINVAL

    # the two calls the channels-last kernels refuse go to the NCHW kernels: ROIAlign((32, 32)) backward, single-level
    # ROIAlignRotated((20, 20)) forward and backward -- channels-last inputs, and NCHW inputs under D2B_POOLER_LAYOUT=nhwc
    x = torch.zeros(2, 256, 50, 84)
    xcl = x.contiguous(memory_format=torch.channels_last)
    monkeypatch.setattr(ops, "POOLER_LAYOUT", "auto")
    assert ops._pick_layout([xcl], 10 ** 6, (32, 32)) == "cl"
    assert ops._pick_layout([tuple(x.shape)], 10 ** 6, (32, 32), backward=True, channels_last=True) == "nchw"
    assert ops._pick_layout([xcl], 10 ** 6, (20, 20), rotated=True) == "nchw"
    assert ops._pick_layout([tuple(x.shape)], 10 ** 6, (20, 20), rotated=True, backward=True, channels_last=True) == "nchw"
    monkeypatch.setattr(ops, "POOLER_LAYOUT", "nhwc")
    assert ops._pick_layout([x], 1, (32, 32)) == "xpose"
    assert ops._pick_layout([tuple(x.shape)], 1, (32, 32), backward=True, channels_last=False) == "nchw"
    assert ops._pick_layout([x], 1, (20, 20), rotated=True) == "nchw"
    assert ops._pick_layout([tuple(x.shape)], 1, (20, 20), rotated=True, backward=True, channels_last=False) == "nchw"


# The argument rule of d2b_roi_pooler_forward / _backward (include/d2b200.h), one row per fault: (what, arguments changed
# from a valid call, expected status).  The expected status is a number, or a function of the call's kind that returns None
# where the call is valid (it would launch, so it is not made).  `flag` is a bit added to the call's flags; pyramid keys:
# `h` / `w` / `map` set H, W and feat = grad of the last level, `num_levels`, `max_level` and `level_rois` the fields of the
# same name.
EINVAL, UNSUPPORTED = -1, -3
_ROI_FAULTS = [
    ("no RoIs", dict(k=0), lambda t: None if t.bwd else 0),  # the backward zero-fills its gradient maps
    ("no RoIs, nothing else valid", dict(k=0, n=-1, map=None), lambda t: EINVAL if t.bwd else 0),
    ("no RoIs, no images", dict(k=0, n=0), 0),
    ("no channels", dict(c=0), 0),
    ("no channels, no data", dict(c=0, data=None), 0),
    ("no images", dict(n=0), EINVAL),  # RoIs of images that do not exist
    ("n < 0", dict(n=-1), EINVAL),
    ("c < 0", dict(c=-4), EINVAL),
    ("k < 0", dict(k=-1), EINVAL),
    ("k < 0, no images", dict(k=-2, n=0), EINVAL),
    ("pooled_h < 1", dict(ph=0), EINVAL),
    ("pooled_w < 1", dict(pw=-1), EINVAL),
    ("no rois", dict(rois=None), EINVAL),
    ("no out / grad_out", dict(data=None), EINVAL),
    ("no feature / gradient map", dict(map=None), EINVAL),
    ("empty level", dict(h=0), EINVAL),
    ("negative level height", dict(h=-1), EINVAL),
    ("negative level width", dict(w=-3), EINVAL),
    ("no levels", dict(num_levels=0), EINVAL),
    ("too many levels", dict(num_levels=9), EINVAL),
    ("levels do not match min_level..max_level", dict(max_level=6), lambda t: EINVAL if t.levels > 1 else None),
    ("level boxes of rotated RoIs", dict(level_rois=0x30), lambda t: EINVAL if t.rot else None),
    ("flag D2B_ROI_BACKWARD", dict(flag=2), EINVAL),
    ("unknown flag", dict(flag=8), EINVAL),
    ("dtype code 3", dict(dt=3), EINVAL),
    ("dtype code -1", dict(dt=-1), EINVAL),
    ("dtype code 9", dict(dt=9), EINVAL),
    ("fp16 data", dict(dt=1), lambda t: None if t.nhwc else EINVAL),  # the NCHW kernels read and write fp32 only
    ("bf16 data", dict(dt=2), lambda t: None if t.nhwc else EINVAL),
    ("fp16 data, no rois", dict(dt=1, rois=None), EINVAL),
    ("bf16 data, no out / grad_out", dict(dt=2, data=None), EINVAL),
    ("misaligned map", dict(map=0x1004), lambda t: EINVAL if t.nhwc else None),
    ("misaligned empty map", dict(map=0x1004, h=0), EINVAL),
    ("misaligned map, c % 4 != 0", dict(map=0x1004, c=6), lambda t: EINVAL if t.nhwc else None),  # EINVAL first
    ("c % 4 != 0", dict(c=6), lambda t: UNSUPPORTED if t.nhwc else None),
    ("rotated tile > 150 KB", dict(ph=20, pw=20), lambda t: UNSUPPORTED if t.nhwc and t.rot else None),
    ("tile of the backward > 180 KB", dict(ph=32, pw=32), lambda t: UNSUPPORTED if t.nhwc and (t.rot or t.bwd) else None),
]


def _roi_pooler_call(lib, bwd, flags, levels, n=2, c=8, k=3, ph=7, pw=7, rois=0x10, data=0x20, dt=0, **pyr):
    """One call on a one-level (a single-level op: 16x16 at scale 1/4) or four-level (64x96 .. 8x12) pyramid whose maps are
    16-byte aligned pointers that are never dereferenced."""
    import ctypes as C

    from detectron2_b200 import _C

    P = _C.Pyramid()
    P.num_levels = levels
    for l in range(levels):
        P.H[l], P.W[l] = (16, 16) if levels == 1 else (64 >> l, 96 >> l)
        P.scale[l] = 0.25 / 2 ** l
        P.feat[l] = P.grad[l] = 0x1000 * (l + 1)
    P.min_level, P.max_level, P.canonical_level, P.canonical_box_size = 2, 1 + levels, 4, 224.0
    last = levels - 1
    P.H[last], P.W[last] = pyr.get("h", P.H[last]), pyr.get("w", P.W[last])
    P.feat[last] = P.grad[last] = pyr.get("map", P.feat[last])
    P.num_levels, P.max_level = pyr.get("num_levels", levels), pyr.get("max_level", P.max_level)
    P.level_rois = pyr.get("level_rois")
    if bwd:
        return lib.d2b_roi_pooler_backward(C.byref(P), n, c, data, dt, rois, k, ph, pw, 0, 1, flags, None)
    return lib.d2b_roi_pooler_forward(C.byref(P), n, c, rois, k, ph, pw, 0, 1, flags, data, dt, None)


def test_roi_pooler_entry_points_validate_arguments_without_a_gpu():
    """Every fault gets its status before anything is launched, in each of the eight forward / backward x axis-aligned /
    rotated x NCHW / channels-last kinds of call.  Without a GPU a launch attempt returns a positive CUDA error, so a negative
    status here also shows that no launch came first (the gradient maps were not written)."""
    import itertools
    import types

    from detectron2_b200 import _C

    lib = _C.lib()
    for bwd, rot, nhwc, levels in itertools.product((False, True), (False, True), (False, True), (1, 4)):
        flags = (_C.ROI_ROTATED if rot else 0) | (_C.ROI_NHWC if nhwc else 0)
        kind = types.SimpleNamespace(bwd=bwd, rot=rot, nhwc=nhwc, levels=levels)
        for what, args, want in _ROI_FAULTS:
            want = want(kind) if callable(want) else want
            if want is not None:
                a = dict(args)
                got = _roi_pooler_call(lib, bwd, flags | a.pop("flag", 0), levels, **a)
                assert got == want, (what, "bwd" if bwd else "fwd", flags, levels, got)


# The inference selection entry points.  Each row is one fault in an otherwise valid call whose pointers are dummy addresses,
# never dereferenced: (entry point, fault, arguments that differ, expected status or a function of the call's flags giving
# it, None where the row does not apply).  A flag set with ROT runs the rotated box type, one without it xyxy.
ROT, SEG, NOOFF, LIN = 1, 2, 4, 8  # D2B_SELECT_ROTATED / _SEG_PER_IMAGE / _NO_OFFSETS / _LINEAR
_SELECT_KINDS = {  # every flag set each entry point takes
    "d2b_rpn_prepare": (0, NOOFF, ROT, ROT | SEG),
    "d2b_frcnn_prepare": (0, ROT, ROT | SEG),
    "d2b_dense_prepare": (0, LIN),
    "d2b_rpn_select": (0, ROT),
}
_P = 0x1000  # a 16-byte aligned dummy address
_SELECT_PARAMS = {  # every parameter in order, with its value in a valid call (lv: the levels built by _select_call)
    "d2b_rpn_prepare": dict(lv=None, N=2, image_hw=_P, min_box_size=0.0, flags=0, flat_boxes=_P, nms_boxes=_P, nms_scores=_P,
                            raw_scores=_P, cat_ids=_P, nonfinite=_P),
    "d2b_frcnn_prepare": dict(boxes=_P, scores=_P, row_start=(0, 4, 9), N=2, num_classes=3, kreg=3, image_hw=_P,
                              score_thresh=0.05, cap=16, flags=0, cand_boxes=_P, nms_boxes=_P, nms_scores=_P, raw_scores=_P,
                              cand_flat=_P, cat_ids=_P, n_cand=_P, row_map=_P),
    "d2b_dense_prepare": dict(lv=None, N=2, num_classes=80, weights=(1.0, 1.0, 1.0, 1.0), scale_clamp=4.135, flags=0,
                              flat_boxes=_P, nms_boxes=_P, nms_scores=_P, raw_scores=_P, classes=_P, cat_ids=_P),
    "d2b_rpn_select": dict(keep=_P, num_keep=_P, N=2, T=10, post_nms_topk=5, flags=0, flat_boxes=_P, raw_scores=_P,
                           cat_ids=_P, out_boxes=_P, out_scores=_P, out_index=_P, counts=_P),
}
_MISALIGNED = 0x1004
_XYXY_ONLY = lambda f: EINVAL if not f & ROT else None  # noqa: E731  (rotated boxes have no alignment requirement)
_SELECT_FAULTS = [
    ("d2b_rpn_prepare", "no level struct", dict(lv=None), EINVAL),
    ("d2b_rpn_prepare", "nonfinite NULL", dict(nonfinite=None), EINVAL),
    ("d2b_rpn_prepare", "N < 0", dict(N=-1), EINVAL),
    ("d2b_rpn_prepare", "no level", dict(num_levels=0), EINVAL),
    ("d2b_rpn_prepare", "9 levels", dict(num_levels=9), EINVAL),
    ("d2b_rpn_prepare", "k > A", dict(k=[11]), EINVAL),
    ("d2b_rpn_prepare", "top-k indices NULL", dict(topk_idx=[None]), EINVAL),
    ("d2b_rpn_prepare", "T > INT_MAX", dict(num_levels=2, A=[2 ** 30] * 2, k=[2 ** 30] * 2), EINVAL),
    ("d2b_rpn_prepare", "image_hw NULL", dict(image_hw=None), EINVAL),
    ("d2b_rpn_prepare", "nms_boxes NULL", dict(nms_boxes=None), EINVAL),
    ("d2b_rpn_prepare", "proposals misaligned", dict(proposals=[_MISALIGNED]), _XYXY_ONLY),
    ("d2b_rpn_prepare", "flat_boxes misaligned", dict(flat_boxes=_MISALIGNED), _XYXY_ONLY),
    ("d2b_frcnn_prepare", "more images than D2B_MAX_IMAGES", dict(N=65), EINVAL),
    ("d2b_frcnn_prepare", "N < 0", dict(N=-1), EINVAL),
    ("d2b_frcnn_prepare", "no class", dict(num_classes=0), EINVAL),
    ("d2b_frcnn_prepare", "kreg neither 1 nor K", dict(kreg=2), EINVAL),
    ("d2b_frcnn_prepare", "cap < 0", dict(cap=-1), EINVAL),
    ("d2b_frcnn_prepare", "row_start NULL", dict(row_start=None), EINVAL),
    ("d2b_frcnn_prepare", "row_start decreasing", dict(row_start=(0, 4, 3)), EINVAL),
    ("d2b_frcnn_prepare", "row_start[0] < 0: rows before boxes[0]", dict(row_start=(-1, 4, 9)), EINVAL),
    ("d2b_frcnn_prepare", "image_hw NULL", dict(image_hw=None), EINVAL),
    ("d2b_frcnn_prepare", "n_cand NULL", dict(n_cand=None), EINVAL),
    ("d2b_frcnn_prepare", "boxes NULL", dict(boxes=None), EINVAL),
    ("d2b_frcnn_prepare", "row_map NULL", dict(row_map=None), EINVAL),
    ("d2b_frcnn_prepare", "cand_boxes NULL", dict(cand_boxes=None), EINVAL),
    ("d2b_frcnn_prepare", "cat_ids NULL", dict(cat_ids=None), EINVAL),
    ("d2b_frcnn_prepare", "cand_boxes misaligned", dict(cand_boxes=_MISALIGNED), _XYXY_ONLY),
    ("d2b_frcnn_prepare", "nms_boxes misaligned", dict(nms_boxes=_MISALIGNED), _XYXY_ONLY),
    ("d2b_frcnn_prepare", "no images: nothing to do", dict(N=0, image_hw=None, n_cand=None), 0),
    ("d2b_dense_prepare", "no level struct", dict(lv=None), EINVAL),
    ("d2b_dense_prepare", "no level", dict(num_levels=0), EINVAL),
    ("d2b_dense_prepare", "9 levels", dict(num_levels=9), EINVAL),
    ("d2b_dense_prepare", "N < 0", dict(N=-1), EINVAL),
    ("d2b_dense_prepare", "no class", dict(num_classes=0), EINVAL),
    ("d2b_dense_prepare", "weights NULL", dict(weights=None), lambda f: None if f & LIN else EINVAL),
    ("d2b_dense_prepare", "weights NULL, no images", dict(weights=None, N=0), lambda f: 0 if f & LIN else EINVAL),
    ("d2b_dense_prepare", "no images: nothing to do", dict(N=0, flat_boxes=None), 0),
    ("d2b_dense_prepare", "R < 0", dict(R=[-1]), EINVAL),
    ("d2b_dense_prepare", "k < 0", dict(k=[-1]), EINVAL),
    ("d2b_dense_prepare", "anchors NULL", dict(anchors=[None]), EINVAL),
    ("d2b_dense_prepare", "deltas misaligned", dict(deltas=[_MISALIGNED]), EINVAL),
    ("d2b_dense_prepare", "T > INT_MAX", dict(num_levels=2, k=[2 ** 30] * 2), EINVAL),
    ("d2b_dense_prepare", "no candidate: nothing to do", dict(k=[0], flat_boxes=None), 0),
    ("d2b_dense_prepare", "classes NULL", dict(classes=None), EINVAL),
    ("d2b_dense_prepare", "flat_boxes misaligned", dict(flat_boxes=_MISALIGNED), EINVAL),
    ("d2b_dense_prepare", "nms_boxes misaligned", dict(nms_boxes=_MISALIGNED), EINVAL),
    ("d2b_rpn_select", "N < 0", dict(N=-1), EINVAL),
    ("d2b_rpn_select", "T < 0", dict(T=-1), EINVAL),
    ("d2b_rpn_select", "post_nms_topk < 0", dict(post_nms_topk=-1), EINVAL),
    ("d2b_rpn_select", "no images: nothing to do", dict(N=0, counts=None), 0),
    ("d2b_rpn_select", "counts NULL", dict(counts=None), EINVAL),
] + [("d2b_rpn_select", name + " NULL", {name: None}, EINVAL)
     for name in ("keep", "num_keep", "flat_boxes", "raw_scores", "cat_ids", "out_boxes", "out_scores", "out_index")] + [
    ("d2b_rpn_select", "flat_boxes misaligned", dict(flat_boxes=_MISALIGNED), _XYXY_ONLY),
    ("d2b_rpn_select", "out_boxes misaligned", dict(out_boxes=_MISALIGNED), _XYXY_ONLY),
]


def _select_call(lib, entry, flags, **over):
    import ctypes as C

    from detectron2_b200 import _C

    args = dict(_SELECT_PARAMS[entry], flags=flags)
    if "lv" in args:  # levels of 10 boxes with a top-k of 5 each
        lv = _C.RpnLevels() if entry == "d2b_rpn_prepare" else _C.DenseLevels()
        lv.num_levels = over.pop("num_levels", 1)
        for name, _ in lv._fields_[1:]:
            default = 10 if name in ("A", "R") else 5 if name == "k" else _P
            for l, v in enumerate(over.pop(name, [default] * _C.MAX_LEVELS)):
                getattr(lv, name)[l] = v
        args["lv"] = C.byref(lv)
    args.update(over)
    if args.get("row_start") is not None:
        args["row_start"] = (C.c_int * 3)(*args["row_start"])
    if args.get("weights") is not None:
        args["weights"] = (C.c_float * 4)(*args["weights"])
    return getattr(lib, entry)(*args.values(), None)


def test_selection_entry_points_validate_arguments_without_a_gpu():
    """Every fault of the four selection entry points gets its status before anything is launched, for each flag set the
    entry point takes; every other flag value is D2B_EINVAL.  Without a GPU a launch attempt returns a positive CUDA error,
    so a status <= 0 here also shows that nothing was launched or written (not even rpn_prepare's zeroing of nonfinite)."""
    from detectron2_b200 import _C

    lib = _C.lib()
    assert (_C.SELECT_ROTATED, _C.SELECT_SEG_PER_IMAGE, _C.SELECT_NO_OFFSETS, _C.SELECT_LINEAR) == (ROT, SEG, NOOFF, LIN)
    for entry, kinds in _SELECT_KINDS.items():
        for flags in [f for f in range(32) if f not in kinds] + [-1, 1 << 30]:
            assert _select_call(lib, entry, flags) == EINVAL, (entry, flags)
    for entry, what, args, want in _SELECT_FAULTS:
        for flags in _SELECT_KINDS[entry]:
            w = want(flags) if callable(want) else want
            if w is not None:
                got = _select_call(lib, entry, flags, **args)
                assert got == w, (entry, what, flags, got)


def test_roi_pooler_no_images():  # /root/reference/tests/modeling/test_roi_pooler.py:107-115
    from detectron2_b200.poolers import ROIPooler

    feature = torch.rand(0, 32, 32, 32) - 0.5
    pooler = ROIPooler(output_size=14, scales=(1.0,), sampling_ratio=0.0, pooler_type="ROIAlignV2")
    assert pooler.forward([feature], []).shape == (0, 32, 14, 14)
    with pytest.raises(ValueError):
        ROIPooler(output_size=7, scales=(0.25,), sampling_ratio=0, pooler_type="ROIPool")
    with pytest.raises(AssertionError):  # scales that do not form a pyramid (poolers.py:186-190)
        ROIPooler(output_size=7, scales=(0.25, 0.0625), sampling_ratio=0, pooler_type="ROIAlignV2")


class _RotNms(torch.nn.Module):  # /root/reference/tests/layers/test_nms_rotated.py:153-168
    def forward(self, boxes, scores, threshold: float):
        import detectron2_b200.layers as L

        return L.nms_rotated(boxes, scores, threshold)


def test_wrappers_are_scriptable():
    """The wrappers the reference scripts in its own tests (tests/layers/test_nms.py:16-29, test_nms_rotated.py:153-168,
    test_mask_ops.py:156-165) compile with torch.jit.script: their bodies are dispatcher ops only.  (Scripted == eager
    is checked on the GPU in tests/test_gpu_parity.py.)"""
    import detectron2_b200.layers as L

    for fn in (L.batched_nms, L.nms, L.batched_nms_rotated, L.paste_masks_in_image):
        f = fn.__original_fn if hasattr(fn, "__original_fn") else fn  # script_if_tracing wrapper
        assert torch.jit.script(f) is not None
    assert "detectron2::nms_rotated" in str(torch.jit.script(_nms_rotated_fn).graph)


def _nms_rotated_fn(boxes: torch.Tensor, scores: torch.Tensor, threshold: float) -> torch.Tensor:
    return torch.ops.detectron2.nms_rotated(boxes, scores, threshold)


def test_layout_change_and_packed_paste_validate_arguments_without_a_gpu():
    """Status codes of the pyramid layout changes and the bit-packed paste on invalid arguments (checked before anything is
    launched): negative = d2b error (include/d2b200.h), what the Python host turns into RuntimeError."""
    import ctypes as C

    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL = -1
    # dtype codes of the half-precision variants
    P = _C.Pyramid()
    P.num_levels = 1
    P.H[0], P.W[0] = 8, 8
    dst = (C.c_void_p * 1)(None)
    assert lib.d2b_pyramid_nchw_to_nhwc(C.byref(P), 1, 4, dst, 7, None) == EINVAL
    assert lib.d2b_pyramid_nhwc_to_nchw(C.byref(P), 1, 4, dst, -1, None) == EINVAL
    assert _C.DTYPE_CODE == {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}
    # bit-packed paste: boolean output only
    assert lib.d2b_paste_masks_packed(None, None, 3, 28, 10, 10, -1.0, None, None) == EINVAL
    assert lib.d2b_paste_masks_packed(None, None, 0, 28, 10, 10, 0.5, None, None) == 0


def test_post_processing_dispatch_and_pyramid_struct():
    """CPU tensors take the torch-op restatements (pinned to the real reference functions in test_host_logic_cpu.py); the ABI
    struct carries the level_rois field of ABI v4."""
    from detectron2_b200 import _C, dense_inference, fast_rcnn_inference

    assert [n for n, _ in _C.Pyramid._fields_][-1] == "level_rois"
    assert callable(fast_rcnn_inference.fast_rcnn_inference_fixed) and callable(dense_inference.dense_detector_inference_fixed)
    with pytest.raises(NotImplementedError):  # the fixed-capacity forms are CUDA only
        fast_rcnn_inference.fast_rcnn_inference_fixed([torch.zeros(2, 4)], [torch.zeros(2, 3)], [(10, 10)], 0.05, 0.5, 10)
    with pytest.raises(NotImplementedError):
        dense_inference.dense_detector_inference_fixed([torch.zeros(4, 4)], [torch.zeros(1, 4, 2)], [torch.zeros(1, 4, 4)], 1,
                                                       0.05, 10, 0.5, 10)


def test_unpack_mask_bits_host_side():
    """The receiving side of the bit-packed paste: plain torch ops, CPU tensors (bit b of word w = pixel 32 w + b)."""
    import detectron2_b200.layers as L

    g = torch.Generator().manual_seed(0)
    ref = torch.rand(3, 5, 70, generator=g) > 0.5
    words = torch.zeros(3, 5, 3, dtype=torch.int64)
    for x in range(70):
        words[..., x // 32] |= ref[..., x].to(torch.int64) << (x % 32)
    packed = torch.where(words >= 2 ** 31, words - 2 ** 32, words).to(torch.int32)  # two's-complement int32 words
    assert torch.equal(L.unpack_mask_bits(packed, 70), ref)
    assert L.paste_masks_in_image_packed(torch.zeros(0, 28, 28), torch.zeros(0, 4), (10, 40)).shape == (0, 10, 2)


def test_ctypes_signatures_match_the_header_arity():
    """Every prototype of include/d2b200.h against the ctypes binding: same number of parameters (a missing / extra argument in
    the binding would shift every following pointer)."""
    from detectron2_b200 import _C

    _C.lib()
    header = open(os.path.join(ROOT, "include", "d2b200.h")).read()
    header = re.sub(r"/\*.*?\*/", "", header, flags=re.S)
    protos = re.findall(r"\b(d2b_[a-z0-9_]+)\s*\(([^;{]*?)\)\s*;", header, flags=re.S)
    assert len(protos) >= 30
    for name, params in protos:
        params = params.strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert len(_C.EXPORTED[name][1]) == n, (name, n, len(_C.EXPORTED[name][1]))
