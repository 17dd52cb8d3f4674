"""torch custom-op registration over the C ABI (libd2b200.so).

Two op namespaces are served:
  * ``d2b200::*``      -- our own ops (autograd + fake/meta kernels, so they trace and compile);
  * ``detectron2::*``  -- the four dispatcher ops the reference registers in csrc/vision.cpp:115-120
    (nms_rotated, box_iou_rotated, roi_align_rotated_forward, roi_align_rotated_backward) with the same
    schemas, so reference call sites ``torch.ops.detectron2.*`` (layers/roi_align_rotated.py:20,33,89,
    layers/nms.py:89, layers/rotated_boxes.py:21) run unchanged on CUDA tensors.  If the reference's own
    library already defined them (e.g. the CPU oracle build is loaded) only a CUDA kernel is added.

PyTorch is plumbing here: allocation, streams, autograd graph.  All arithmetic happens in the hand-written kernels.
"""
import ctypes as C
import os
from typing import List, Optional, Tuple

import torch

from . import _C
from ._C import check, ptr, stream_ptr

Tensor = torch.Tensor


def _f32c(t: Optional[Tensor]) -> Optional[Tensor]:
    if t is None:
        return None
    return t.to(dtype=torch.float32).contiguous()


# =================================================================================== RoIAlign
# Feature-map layout policy of the axis-aligned forward (D2B_POOLER_LAYOUT = auto | nchw | nhwc):
#   * channels_last inputs are consumed in place by the NHWC kernel (torchvision would .contiguous() them first);
#   * NCHW inputs go to the NCHW kernel, unless the call is large enough that "one layout-change launch + NHWC
#     pooling" is cheaper.  Cost model fitted to tools/bench_pooler_layouts.py on an H100 80GB HBM3 SXM at 700 W
#     (bench.py's 800x1333 pyramid, 256 channels; 1 000 / 512 / 2 000 RoIs at 7x7 and 100 at 14x14); it picks the faster
#     path on all four.
POOLER_LAYOUT = os.environ.get("D2B_POOLER_LAYOUT", "auto")
_NCHW_PS_PER_OUT = 21.0      # NCHW kernel: picoseconds per output element (13.9 mask head .. 27.5 box head, 512 RoIs)
_NHWC_PS_PER_OUT = 9.0       # NHWC kernel (7.8 .. 16.8)
_XPOSE_PS_PER_BYTE = 0.72    # layout change: 91.4 MB of fp32 features in 65-68 us (reads + writes each byte once)


def _is_channels_last(t: Tensor) -> bool:
    return t.dim() == 4 and not t.is_contiguous() and t.is_contiguous(memory_format=torch.channels_last)


def _nhwc_ok(feats, c: int) -> bool:
    return c % 4 == 0 and all(t.shape[2] * t.shape[3] * (c // 4) < 2 ** 28 for t in feats)


def _pick_layout(feats, n_out: int) -> str:
    """'cl' = channels_last inputs used in place, 'xpose' = layout change + NHWC kernel, 'nchw' = NCHW kernel."""
    c = feats[0].shape[1]
    if POOLER_LAYOUT == "nchw" or not _nhwc_ok(feats, c):
        return "nchw"
    if all(_is_channels_last(t) and t.data_ptr() % 16 == 0 for t in feats):
        return "cl"
    if POOLER_LAYOUT == "nhwc":
        return "xpose"
    feat_bytes = 4 * sum(t.numel() for t in feats)
    return "xpose" if (n_out * _NHWC_PS_PER_OUT + feat_bytes * _XPOSE_PS_PER_BYTE < n_out * _NCHW_PS_PER_OUT) else "nchw"


def _to_nhwc(fs, P, n: int, c: int, device):
    """One launch: every level of the NCHW pyramid `P` (fp32, fp16 or bf16 elements, all levels alike) -> freshly allocated
    fp32 NHWC buffers; returns them.  For half-precision levels the layout change is also the up-cast."""
    bufs = [torch.empty((t.shape[0], t.shape[2], t.shape[3], t.shape[1]), dtype=torch.float32, device=device) for t in fs]
    dst = (C.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])
    check(_C.lib().d2b_pyramid_nchw_to_nhwc_t(C.byref(P), n, c, dst, _C.DTYPE_CODE[fs[0].dtype], stream_ptr(device)),
          "pyramid_nchw_to_nhwc")
    return bufs


def _same_half_dtype(ts) -> bool:
    return ts[0].dtype in _HALF and all(t.dtype == ts[0].dtype for t in ts)


def pyramid_to_channels_last(feats: List[Tensor]) -> List[Tensor]:
    """All levels of an NCHW fp32 feature pyramid -> channels_last tensors (same logical [N,C,H,W] shape, NHWC storage)
    with ONE kernel launch.  A caller that pools the same features more than once per image (box head + mask head,
    roi_heads.py:798,843 in the reference) converts once and hands the result to every ROIPooler / ROIAlign call, which
    then run the channels-last kernel in place.  Inputs that are already channels_last, need autograd, are not fp32 or
    do not fit the NHWC kernel's limits are returned through torch's own (autograd-aware) conversion / unchanged."""
    _C.require_cuda(*feats)
    if len(feats) == 0 or len(feats) > _C.MAX_LEVELS:
        raise RuntimeError("pyramid_to_channels_last: need 1..%d levels" % _C.MAX_LEVELS)
    c = feats[0].shape[1]
    if not _nhwc_ok(feats, c) or any(t.shape[:2] != feats[0].shape[:2] for t in feats):
        return list(feats)
    if any(t.dtype != torch.float32 for t in feats) or (torch.is_grad_enabled() and any(t.requires_grad for t in feats)):
        return [t.contiguous(memory_format=torch.channels_last) for t in feats]
    if all(_is_channels_last(t) for t in feats):
        return list(feats)
    fs = [t.contiguous() for t in feats]
    n = fs[0].shape[0]
    if n == 0 or c == 0:
        return list(feats)
    with torch.cuda.device(fs[0].device):
        P = _pyramid(fs, None, [1.0] * len(fs), 0, len(fs) - 1, 0, 1.0)
        bufs = _to_nhwc(fs, P, n, c, fs[0].device)
    return [b.permute(0, 3, 1, 2) for b in bufs]


def _roi_common(input: Tensor, rois: Tensor, cols: int):
    _C.require_cuda(input, rois)
    if input.dim() != 4:
        raise RuntimeError("roi_align: input must be NCHW")
    if rois.dim() != 2 or rois.size(1) != cols:
        raise RuntimeError("roi_align: rois must be K x %d" % cols)


@torch.library.custom_op("d2b200::roi_align", mutates_args=(), device_types="cuda")
def roi_align_op(input: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int,
                 sampling_ratio: int, aligned: bool) -> Tensor:
    _roi_common(input, rois, 5)
    r = _f32c(rois)
    n, c, h, w = input.shape
    k = r.shape[0]
    out = torch.empty((k, c, pooled_h, pooled_w), dtype=torch.float32, device=input.device)
    if out.numel():
        x = input.to(dtype=torch.float32)
        layout = _pick_layout([x], out.numel())
        with torch.cuda.device(x.device):
            if layout == "nchw":
                x = x.contiguous()
                check(_C.lib().d2b_roi_align_forward(ptr(x), n, c, h, w, ptr(r), k, spatial_scale, pooled_h, pooled_w,
                                                     sampling_ratio, int(aligned), ptr(out), stream_ptr(x.device)),
                      "roi_align_forward")
            else:
                if layout == "xpose":
                    x = x.contiguous()
                    x = _to_nhwc([x], _pyramid([x], None, [spatial_scale], 0, 0, 0, 1.0), n, c, x.device)[0]
                check(_C.lib().d2b_roi_align_forward_nhwc(ptr(x), n, c, h, w, ptr(r), k, spatial_scale, pooled_h,
                                                          pooled_w, sampling_ratio, int(aligned), ptr(out),
                                                          stream_ptr(x.device)), "roi_align_forward_nhwc")
    return out.to(input.dtype)


@roi_align_op.register_fake
def _(input, rois, spatial_scale, pooled_h, pooled_w, sampling_ratio, aligned):
    return input.new_empty((rois.shape[0], input.shape[1], pooled_h, pooled_w))


# Backward and rotated per-element costs are carried over from the kernels' first tuning and have not been re-measured on an
# H100 (the layout-change cost per byte above has); the choice only changes speed, every path computes the same result.
_NCHW_BWD_PS_PER_OUT = 40.0  # NCHW backward kernel: picoseconds per grad_out element
_NHWC_BWD_PS_PER_OUT = 8.0   # channels-last backward (one red.v4 per footprint pixel)


def _bwd_layout(shapes_nchw, n_out: int, channels_last: bool) -> str:
    """'cl': gradients produced channels-last in place; 'xpose': channels-last kernel into scratch + one layout-change
    launch back to NCHW; 'nchw': the NCHW kernel.  shapes_nchw: [(n, c, h, w)] per level."""
    c = shapes_nchw[0][1]
    ok = c % 4 == 0 and POOLER_LAYOUT != "nchw" and all(h * w * (c // 4) < 2 ** 28 for (_, _, h, w) in shapes_nchw)
    if not ok:
        return "nchw"
    if channels_last:
        return "cl"
    if POOLER_LAYOUT == "nhwc":
        return "xpose"
    feat_bytes = 4 * sum(n * c * h * w for (n, c, h, w) in shapes_nchw)
    return "xpose" if n_out * _NHWC_BWD_PS_PER_OUT + feat_bytes * _XPOSE_PS_PER_BYTE < n_out * _NCHW_BWD_PS_PER_OUT else "nchw"


def _from_nhwc(bufs, n: int, c: int, device, dtype=torch.float32):
    """One launch: fp32 NHWC buffers -> freshly allocated NCHW tensors of `dtype` (fp32, or fp16 / bf16: the layout change
    is also the down-cast of the gradients of half-precision features)."""
    outs = [torch.empty((b.shape[0], b.shape[3], b.shape[1], b.shape[2]), dtype=dtype, device=device) for b in bufs]
    P = _C.Pyramid()
    P.num_levels = len(bufs)
    for l, b in enumerate(bufs):
        P.feat[l] = b.data_ptr()
        P.H[l], P.W[l] = b.shape[1], b.shape[2]
    dst = (C.c_void_p * len(outs))(*[o.data_ptr() for o in outs])
    check(_C.lib().d2b_pyramid_nhwc_to_nchw_t(C.byref(P), n, c, dst, _C.DTYPE_CODE[dtype], stream_ptr(device)),
          "pyramid_nhwc_to_nchw")
    return outs


@torch.library.custom_op("d2b200::roi_align_backward", mutates_args=(), device_types="cuda")
def roi_align_backward_op(grad: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int, n: int,
                          c: int, h: int, w: int, sampling_ratio: int, aligned: bool,
                          channels_last: bool = False) -> Tensor:
    _C.require_cuda(grad, rois)
    g, r = _f32c(grad), _f32c(rois)
    layout = _bwd_layout([(n, c, h, w)], g.numel(), channels_last) if n * c * h * w else "nchw"
    with torch.cuda.device(g.device):
        if layout == "nchw":
            gin = torch.empty((n, c, h, w), dtype=torch.float32, device=g.device)
            check(_C.lib().d2b_roi_align_backward(ptr(g), ptr(r), r.shape[0], spatial_scale, pooled_h, pooled_w, n, c, h,
                                                  w, sampling_ratio, int(aligned), ptr(gin), stream_ptr(g.device)),
                  "roi_align_backward")
        else:
            buf = torch.empty((n, h, w, c), dtype=torch.float32, device=g.device)
            check(_C.lib().d2b_roi_align_backward_nhwc(ptr(g), ptr(r), r.shape[0], spatial_scale, pooled_h, pooled_w, n, c,
                                                       h, w, sampling_ratio, int(aligned), ptr(buf),
                                                       stream_ptr(g.device)), "roi_align_backward_nhwc")
            gin = buf.permute(0, 3, 1, 2) if layout == "cl" else _from_nhwc([buf], n, c, g.device)[0]
    return gin.to(grad.dtype)


@roi_align_backward_op.register_fake
def _(grad, rois, spatial_scale, pooled_h, pooled_w, n, c, h, w, sampling_ratio, aligned, channels_last=False):
    out = grad.new_empty((n, c, h, w))
    return out.contiguous(memory_format=torch.channels_last) if channels_last else out


def _roi_align_setup(ctx, inputs, output):
    input, rois, spatial_scale, ph, pw, sr, aligned = inputs
    ctx.save_for_backward(rois)
    ctx.args = (spatial_scale, ph, pw, tuple(input.shape), sr, aligned, _is_channels_last(input))


def _roi_align_bwd(ctx, grad):
    (rois,) = ctx.saved_tensors
    scale, ph, pw, (n, c, h, w), sr, aligned, cl = ctx.args
    gin = roi_align_backward_op(grad, rois, scale, ph, pw, n, c, h, w, sr, aligned, cl)
    return gin, None, None, None, None, None, None


roi_align_op.register_autograd(_roi_align_bwd, setup_context=_roi_align_setup)


# ----------------------------------------------------------------------------------- fused multi-level pooler
_HALF = (torch.float16, torch.bfloat16)


def _pyramid(feats, grads, scales, min_level, max_level, canonical_level, canonical_box_size, level_rois=None):
    P = _C.Pyramid()
    P.level_rois = level_rois.data_ptr() if level_rois is not None else None
    P.num_levels = len(feats)
    for l, t in enumerate(feats):
        P.feat[l] = t.data_ptr()
        P.grad[l] = grads[l].data_ptr() if grads is not None else None
        P.H[l], P.W[l] = t.shape[2], t.shape[3]
        P.scale[l] = scales[l]
    P.min_level, P.max_level, P.canonical_level = min_level, max_level, canonical_level
    P.canonical_box_size = canonical_box_size
    return P


@torch.library.custom_op("d2b200::roi_pooler", mutates_args=(), device_types="cuda")
def roi_pooler_op(feats: List[Tensor], rois: Tensor, scales: List[float], pooled_h: int, pooled_w: int,
                  sampling_ratio: int, aligned: bool, min_level: int, max_level: int, canonical_level: int,
                  canonical_box_size: float) -> Tensor:
    _C.require_cuda(rois, *feats)
    if len(feats) < 1 or len(feats) > _C.MAX_LEVELS or len(feats) != len(scales):
        raise RuntimeError("roi_pooler: need 1..%d feature levels with one scale each" % _C.MAX_LEVELS)
    r_lvl = _f32c(rois)
    # half-precision feature maps: the reference samples with the rois cast to the feature dtype (layers/roi_align.py:60,
    # then torchvision's autocast wrapper upcasts both) while the FPN level comes from the fp32 boxes (poolers.py:245)
    half = feats[0].dtype in _HALF
    r = r_lvl.to(feats[0].dtype).to(torch.float32) if half else r_lvl
    n, c = feats[0].shape[:2]
    k = r.shape[0]
    numel = k * c * pooled_h * pooled_w
    layout = _pick_layout(feats, numel) if numel else "nchw"
    # half-precision NCHW levels: the layout-change launch reads them as they are (it is also the up-cast) and the pooling
    # kernel writes the result in their dtype -- no cast passes; every other combination computes on fp32 copies
    fused_half = layout == "xpose" and _same_half_dtype(feats)
    fs = list(feats) if fused_half else [t.to(dtype=torch.float32) for t in feats]
    out_dt = feats[0].dtype if (layout != "nchw" and feats[0].dtype in _C.DTYPE_CODE) else torch.float32
    out = torch.empty((k, c, pooled_h, pooled_w), dtype=out_dt, device=r.device)
    if numel:
        with torch.cuda.device(r.device):
            if layout != "cl":
                fs = [t.contiguous() for t in fs]
            # channels_last tensors: same logical shape, NHWC storage -- _pyramid only takes pointers and H, W
            P = _pyramid(fs, None, scales, min_level, max_level, canonical_level, canonical_box_size, r_lvl if half else None)
            if layout == "nchw":
                check(_C.lib().d2b_roi_pooler_forward(C.byref(P), n, c, ptr(r), k, pooled_h, pooled_w, sampling_ratio,
                                                      int(aligned), ptr(out), stream_ptr(r.device)), "roi_pooler_forward")
            else:
                if layout == "xpose":
                    bufs = _to_nhwc(fs, P, n, c, r.device)
                    for l, b in enumerate(bufs):
                        P.feat[l] = b.data_ptr()
                check(_C.lib().d2b_roi_pooler_forward_nhwc_t(C.byref(P), n, c, ptr(r), k, pooled_h, pooled_w, sampling_ratio,
                                                             int(aligned), ptr(out), _C.DTYPE_CODE[out_dt],
                                                             stream_ptr(r.device)), "roi_pooler_forward_nhwc")
    return out if out.dtype == feats[0].dtype else out.to(feats[0].dtype)


@roi_pooler_op.register_fake
def _(feats, rois, scales, pooled_h, pooled_w, sampling_ratio, aligned, min_level, max_level, canonical_level,
      canonical_box_size):
    return feats[0].new_empty((rois.shape[0], feats[0].shape[1], pooled_h, pooled_w))


@torch.library.custom_op("d2b200::roi_pooler_backward", mutates_args=(), device_types="cuda")
def roi_pooler_backward_op(grad: Tensor, rois: Tensor, shapes: List[int], scales: List[float], pooled_h: int,
                           pooled_w: int, sampling_ratio: int, aligned: bool, min_level: int, max_level: int,
                           canonical_level: int, canonical_box_size: float,
                           channels_last: bool = False, level_rois: Optional[Tensor] = None,
                           half_grads: bool = False) -> List[Tensor]:
    """`level_rois`: the fp32 boxes the FPN level was assigned from when `rois` are the feature-dtype-rounded ones the forward
    sampled with (half-precision features, see roi_pooler_op).  `half_grads`: return NCHW gradients in `grad`'s fp16 / bf16
    dtype (written by the layout-change launch) instead of fp32."""
    _C.require_cuda(grad, rois, level_rois)
    r = _f32c(rois)
    lr = _f32c(level_rois)
    nl = len(scales)
    n, c = shapes[0], shapes[1]
    hw = [(shapes[2 + 2 * l], shapes[3 + 2 * l]) for l in range(nl)]
    layout = _bwd_layout([(n, c, h, w) for (h, w) in hw], grad.numel(), channels_last) if n * c else "nchw"
    # the channels-last kernel reads fp16 / bf16 gradients in place; the NCHW kernel takes fp32
    g = grad.contiguous() if (layout != "nchw" and grad.dtype in _C.DTYPE_CODE) else _f32c(grad)
    with torch.cuda.device(g.device):
        if layout == "nchw":
            grads = [torch.empty((n, c, h, w), dtype=torch.float32, device=g.device) for (h, w) in hw]
            P = _pyramid(grads, grads, scales, min_level, max_level, canonical_level, canonical_box_size, lr)
            check(_C.lib().d2b_roi_pooler_backward(C.byref(P), n, c, ptr(g), ptr(r), r.shape[0], pooled_h, pooled_w,
                                                   sampling_ratio, int(aligned), stream_ptr(g.device)), "roi_pooler_backward")
        else:
            bufs = [torch.empty((n, h, w, c), dtype=torch.float32, device=g.device) for (h, w) in hw]
            views = [b.permute(0, 3, 1, 2) for b in bufs]  # logical NCHW shape: _pyramid reads H, W from dims 2, 3
            P = _pyramid(views, views, scales, min_level, max_level, canonical_level, canonical_box_size, lr)
            check(_C.lib().d2b_roi_pooler_backward_nhwc_t(C.byref(P), n, c, ptr(g), _C.DTYPE_CODE[g.dtype], ptr(r), r.shape[0],
                                                          pooled_h, pooled_w, sampling_ratio, int(aligned),
                                                          stream_ptr(g.device)), "roi_pooler_backward_nhwc")
            if layout == "cl":
                grads = views
            else:
                grads = _from_nhwc(bufs, n, c, g.device, grad.dtype if (half_grads and grad.dtype in _HALF) else torch.float32)
    if half_grads and grad.dtype in _HALF:
        grads = [t if t.dtype == grad.dtype else t.to(grad.dtype) for t in grads]
    return grads


@roi_pooler_backward_op.register_fake
def _(grad, rois, shapes, scales, pooled_h, pooled_w, sampling_ratio, aligned, min_level, max_level, canonical_level,
      canonical_box_size, channels_last=False, level_rois=None, half_grads=False):
    n, c = shapes[0], shapes[1]
    dt = grad.dtype if half_grads else torch.float32
    outs = [grad.new_empty((n, c, shapes[2 + 2 * l], shapes[3 + 2 * l]), dtype=dt) for l in range(len(scales))]
    return [o.contiguous(memory_format=torch.channels_last) for o in outs] if channels_last else outs


def _pooler_setup(ctx, inputs, output):
    feats, rois, scales, ph, pw, sr, aligned, lo, hi, cl, cs = inputs
    ctx.save_for_backward(rois)
    shapes = [feats[0].shape[0], feats[0].shape[1]]
    for t in feats:
        shapes += [t.shape[2], t.shape[3]]
    ctx.args = (shapes, scales, ph, pw, sr, aligned, lo, hi, cl, cs, [t.dtype for t in feats],
                all(_is_channels_last(t) for t in feats))


def _pooler_bwd(ctx, grad):
    (rois,) = ctx.saved_tensors
    shapes, scales, ph, pw, sr, aligned, lo, hi, cl, cs, dts, chl = ctx.args
    half = dts[0] in _HALF  # same rois as the forward: rounded to the feature dtype for sampling, fp32 for the level
    grads = roi_pooler_backward_op(grad, rois.to(dts[0]).to(torch.float32) if half else rois, shapes, scales, ph, pw, sr,
                                   aligned, lo, hi, cl, cs, chl, rois if half else None,
                                   half and grad.dtype == dts[0] and all(d == dts[0] for d in dts))
    return [g.to(dt) for g, dt in zip(grads, dts)], None, None, None, None, None, None, None, None, None, None


roi_pooler_op.register_autograd(_pooler_bwd, setup_context=_pooler_setup)


_ROT_NCHW_PS = (30.0, 64.0)  # rotated NCHW kernels: picoseconds per output element (forward, backward); not re-measured, above
_ROT_NHWC_PS = (10.0, 16.0)  # rotated channels-last kernels


def _rot_layout(n: int, c: int, h: int, w: int, n_out: int, channels_last: bool, bwd: bool) -> str:
    return _rot_pyramid_layout([(n, c, h, w)], n_out, channels_last, bwd)


def _rot_pyramid_layout(shapes_nchw, n_out: int, channels_last: bool, bwd: bool, bins: int = 0) -> str:
    """Rotated kernels: 'cl', 'xpose' or 'nchw' as in _bwd_layout, for a pyramid of (n, c, h, w) levels.  bins: pooled
    h * w when known; the channels-last kernel keeps a [128 channels][bins] fp32 tile in shared memory (<= 150 KB)."""
    c = shapes_nchw[0][1]
    if c % 4 != 0 or POOLER_LAYOUT == "nchw" or any(h * w * (c // 4) >= 2 ** 28 for (_, _, h, w) in shapes_nchw):
        return "nchw"
    if 4 * 128 * (bins | 1) > 150 * 1024:
        return "nchw"
    if channels_last:
        return "cl"
    if POOLER_LAYOUT == "nhwc":
        return "xpose"
    i = 1 if bwd else 0
    feat_bytes = 4 * sum(n * c * h * w for (n, c, h, w) in shapes_nchw)
    return "xpose" if n_out * _ROT_NHWC_PS[i] + feat_bytes * _XPOSE_PS_PER_BYTE < n_out * _ROT_NCHW_PS[i] else "nchw"


@torch.library.custom_op("d2b200::roi_align_rotated", mutates_args=(), device_types="cuda")
def roi_align_rotated_op(input: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int,
                         sampling_ratio: int) -> Tensor:
    _roi_common(input, rois, 6)
    x, r = input.to(dtype=torch.float32), _f32c(rois)
    n, c, h, w = x.shape
    k = r.shape[0]
    out = torch.empty((k, c, pooled_h, pooled_w), dtype=torch.float32, device=x.device)
    if out.numel():
        layout = _rot_layout(n, c, h, w, out.numel(), _is_channels_last(x) and x.data_ptr() % 16 == 0, False)
        with torch.cuda.device(x.device):
            if layout == "nchw":
                x = x.contiguous()
                check(_C.lib().d2b_roi_align_rotated_forward(ptr(x), n, c, h, w, ptr(r), k, spatial_scale, pooled_h,
                                                             pooled_w, sampling_ratio, ptr(out), stream_ptr(x.device)),
                      "roi_align_rotated_forward")
            else:
                if layout == "xpose":
                    x = x.contiguous()
                    x = _to_nhwc([x], _pyramid([x], None, [spatial_scale], 0, 0, 0, 1.0), n, c, x.device)[0]
                check(_C.lib().d2b_roi_align_rotated_forward_nhwc(ptr(x), n, c, h, w, ptr(r), k, spatial_scale, pooled_h,
                                                                  pooled_w, sampling_ratio, ptr(out),
                                                                  stream_ptr(x.device)), "roi_align_rotated_forward_nhwc")
    return out.to(input.dtype)


@roi_align_rotated_op.register_fake
def _(input, rois, spatial_scale, pooled_h, pooled_w, sampling_ratio):
    return input.new_empty((rois.shape[0], input.shape[1], pooled_h, pooled_w))


@torch.library.custom_op("d2b200::roi_align_rotated_backward", mutates_args=(), device_types="cuda")
def roi_align_rotated_backward_op(grad: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int,
                                  n: int, c: int, h: int, w: int, sampling_ratio: int,
                                  channels_last: bool = False) -> Tensor:
    _C.require_cuda(grad, rois)
    g, r = _f32c(grad), _f32c(rois)
    layout = _rot_layout(n, c, h, w, g.numel(), channels_last, True) if n * c * h * w else "nchw"
    with torch.cuda.device(g.device):
        if layout == "nchw":
            gin = torch.empty((n, c, h, w), dtype=torch.float32, device=g.device)
            check(_C.lib().d2b_roi_align_rotated_backward(ptr(g), ptr(r), r.shape[0], spatial_scale, pooled_h, pooled_w,
                                                          n, c, h, w, sampling_ratio, ptr(gin), stream_ptr(g.device)),
                  "roi_align_rotated_backward")
        else:
            buf = torch.empty((n, h, w, c), dtype=torch.float32, device=g.device)
            check(_C.lib().d2b_roi_align_rotated_backward_nhwc(ptr(g), ptr(r), r.shape[0], spatial_scale, pooled_h,
                                                               pooled_w, n, c, h, w, sampling_ratio, ptr(buf),
                                                               stream_ptr(g.device)), "roi_align_rotated_backward_nhwc")
            gin = buf.permute(0, 3, 1, 2) if layout == "cl" else _from_nhwc([buf], n, c, g.device)[0]
    return gin.to(grad.dtype)


@roi_align_rotated_backward_op.register_fake
def _(grad, rois, spatial_scale, pooled_h, pooled_w, n, c, h, w, sampling_ratio, channels_last=False):
    out = grad.new_empty((n, c, h, w))
    return out.contiguous(memory_format=torch.channels_last) if channels_last else out


def _roi_rot_setup(ctx, inputs, output):
    input, rois, spatial_scale, ph, pw, sr = inputs
    ctx.save_for_backward(rois)
    ctx.args = (spatial_scale, ph, pw, tuple(input.shape), sr, _is_channels_last(input))


def _roi_rot_bwd(ctx, grad):
    (rois,) = ctx.saved_tensors
    scale, ph, pw, (n, c, h, w), sr, cl = ctx.args
    return roi_align_rotated_backward_op(grad, rois, scale, ph, pw, n, c, h, w, sr, cl), None, None, None, None, None


roi_align_rotated_op.register_autograd(_roi_rot_bwd, setup_context=_roi_rot_setup)


# ----------------------------------------------------------------------------------- fused multi-level rotated pooler
@torch.library.custom_op("d2b200::roi_pooler_rotated", mutates_args=(), device_types="cuda")
def roi_pooler_rotated_op(feats: List[Tensor], rois: Tensor, scales: List[float], pooled_h: int, pooled_w: int,
                          sampling_ratio: int, min_level: int, max_level: int, canonical_level: int,
                          canonical_box_size: float) -> Tensor:
    """ROIPooler(pooler_type="ROIAlignRotated") over several levels in one launch: rois [K,6] = (batch, cx, cy, w, h, angle),
    the level of each from w*h.  The rois are used in fp32 whatever the feature dtype (layers/roi_align_rotated.py:81-83)."""
    _C.require_cuda(rois, *feats)
    if len(feats) < 1 or len(feats) > _C.MAX_LEVELS or len(feats) != len(scales):
        raise RuntimeError("roi_pooler_rotated: need 1..%d feature levels with one scale each" % _C.MAX_LEVELS)
    _roi_common(feats[0], rois, 6)
    r = _f32c(rois)
    n, c = feats[0].shape[:2]
    k = r.shape[0]
    numel = k * c * pooled_h * pooled_w
    cl = all(_is_channels_last(t) and t.data_ptr() % 16 == 0 for t in feats)
    layout = (_rot_pyramid_layout([(n, c, t.shape[2], t.shape[3]) for t in feats], numel, cl, False, pooled_h * pooled_w)
              if numel else "nchw")
    # half-precision NCHW levels: the layout-change launch reads them as they are (it is also the up-cast) and the pooling
    # kernel writes the result in their dtype; every other combination computes on fp32 copies
    fused_half = layout == "xpose" and _same_half_dtype(feats)
    fs = list(feats) if fused_half else [t.to(dtype=torch.float32) for t in feats]
    out_dt = feats[0].dtype if (layout != "nchw" and feats[0].dtype in _C.DTYPE_CODE) else torch.float32
    out = torch.empty((k, c, pooled_h, pooled_w), dtype=out_dt, device=r.device)
    if numel:
        with torch.cuda.device(r.device):
            if layout != "cl":
                fs = [t.contiguous() for t in fs]
            P = _pyramid(fs, None, scales, min_level, max_level, canonical_level, canonical_box_size)
            if layout == "nchw":
                check(_C.lib().d2b_roi_pooler_rotated_forward(C.byref(P), n, c, ptr(r), k, pooled_h, pooled_w, sampling_ratio,
                                                              ptr(out), stream_ptr(r.device)), "roi_pooler_rotated_forward")
            else:
                if layout == "xpose":
                    bufs = _to_nhwc(fs, P, n, c, r.device)
                    for l, b in enumerate(bufs):
                        P.feat[l] = b.data_ptr()
                check(_C.lib().d2b_roi_pooler_rotated_forward_nhwc_t(C.byref(P), n, c, ptr(r), k, pooled_h, pooled_w,
                                                                     sampling_ratio, ptr(out), _C.DTYPE_CODE[out_dt],
                                                                     stream_ptr(r.device)), "roi_pooler_rotated_forward_nhwc")
    return out if out.dtype == feats[0].dtype else out.to(feats[0].dtype)


@roi_pooler_rotated_op.register_fake
def _(feats, rois, scales, pooled_h, pooled_w, sampling_ratio, min_level, max_level, canonical_level, canonical_box_size):
    return feats[0].new_empty((rois.shape[0], feats[0].shape[1], pooled_h, pooled_w))


@torch.library.custom_op("d2b200::roi_pooler_rotated_backward", mutates_args=(), device_types="cuda")
def roi_pooler_rotated_backward_op(grad: Tensor, rois: Tensor, shapes: List[int], scales: List[float], pooled_h: int,
                                   pooled_w: int, sampling_ratio: int, min_level: int, max_level: int, canonical_level: int,
                                   canonical_box_size: float, channels_last: bool = False,
                                   half_grads: bool = False) -> List[Tensor]:
    """Gradients of roi_pooler_rotated for every level; shapes = [n, c, h0, w0, h1, w1, ...].  `half_grads`: return NCHW
    gradients in `grad`'s fp16 / bf16 dtype (written by the layout-change launch) instead of fp32."""
    _C.require_cuda(grad, rois)
    r = _f32c(rois)
    nl = len(scales)
    n, c = shapes[0], shapes[1]
    hw = [(shapes[2 + 2 * l], shapes[3 + 2 * l]) for l in range(nl)]
    layout = (_rot_pyramid_layout([(n, c, h, w) for (h, w) in hw], grad.numel(), channels_last, True, pooled_h * pooled_w)
              if n * c else "nchw")
    # the channels-last kernel reads fp16 / bf16 gradients in place; the NCHW kernel takes fp32
    g = grad.contiguous() if (layout != "nchw" and grad.dtype in _C.DTYPE_CODE) else _f32c(grad)
    with torch.cuda.device(g.device):
        if layout == "nchw":
            grads = [torch.empty((n, c, h, w), dtype=torch.float32, device=g.device) for (h, w) in hw]
            P = _pyramid(grads, grads, scales, min_level, max_level, canonical_level, canonical_box_size)
            check(_C.lib().d2b_roi_pooler_rotated_backward(C.byref(P), n, c, ptr(g), ptr(r), r.shape[0], pooled_h, pooled_w,
                                                           sampling_ratio, stream_ptr(g.device)), "roi_pooler_rotated_backward")
        else:
            bufs = [torch.empty((n, h, w, c), dtype=torch.float32, device=g.device) for (h, w) in hw]
            views = [b.permute(0, 3, 1, 2) for b in bufs]  # logical NCHW shape: _pyramid reads H, W from dims 2, 3
            P = _pyramid(views, views, scales, min_level, max_level, canonical_level, canonical_box_size)
            check(_C.lib().d2b_roi_pooler_rotated_backward_nhwc_t(C.byref(P), n, c, ptr(g), _C.DTYPE_CODE[g.dtype], ptr(r),
                                                                  r.shape[0], pooled_h, pooled_w, sampling_ratio,
                                                                  stream_ptr(g.device)), "roi_pooler_rotated_backward_nhwc")
            if layout == "cl":
                grads = views
            else:
                grads = _from_nhwc(bufs, n, c, g.device, grad.dtype if (half_grads and grad.dtype in _HALF) else torch.float32)
    if half_grads and grad.dtype in _HALF:
        grads = [t if t.dtype == grad.dtype else t.to(grad.dtype) for t in grads]
    return grads


@roi_pooler_rotated_backward_op.register_fake
def _(grad, rois, shapes, scales, pooled_h, pooled_w, sampling_ratio, min_level, max_level, canonical_level,
      canonical_box_size, channels_last=False, half_grads=False):
    n, c = shapes[0], shapes[1]
    dt = grad.dtype if half_grads else torch.float32
    outs = [grad.new_empty((n, c, shapes[2 + 2 * l], shapes[3 + 2 * l]), dtype=dt) for l in range(len(scales))]
    return [o.contiguous(memory_format=torch.channels_last) for o in outs] if channels_last else outs


def _pooler_rot_setup(ctx, inputs, output):
    feats, rois, scales, ph, pw, sr, lo, hi, cl, cs = inputs
    ctx.save_for_backward(rois)
    shapes = [feats[0].shape[0], feats[0].shape[1]]
    for t in feats:
        shapes += [t.shape[2], t.shape[3]]
    ctx.args = (shapes, scales, ph, pw, sr, lo, hi, cl, cs, [t.dtype for t in feats],
                all(_is_channels_last(t) for t in feats))


def _pooler_rot_bwd(ctx, grad):
    (rois,) = ctx.saved_tensors
    shapes, scales, ph, pw, sr, lo, hi, cl, cs, dts, chl = ctx.args
    half = dts[0] in _HALF and grad.dtype == dts[0] and all(d == dts[0] for d in dts)
    grads = roi_pooler_rotated_backward_op(grad, rois, shapes, scales, ph, pw, sr, lo, hi, cl, cs, chl, half)
    return [g.to(dt) for g, dt in zip(grads, dts)], None, None, None, None, None, None, None, None, None


roi_pooler_rotated_op.register_autograd(_pooler_rot_bwd, setup_context=_pooler_rot_setup)


# =================================================================================== NMS / rotated IoU
def nms_fixed(boxes: Tensor, scores: Tensor, idxs: Optional[Tensor], iou_threshold: float,
              rotated: bool, apply_offsets: bool = True, max_segment: int = 0) -> Tuple[Tensor, Tensor]:
    """Sync-free NMS: returns (keep[M] int64, 0-padded, num_keep[1] int64 device tensor).
    keep[:num_keep] are the kept original indices in descending-score order.  CUDA-graph friendly.
    max_segment: upper bound on the boxes per category when the caller knows one (sizes the IoU bitmask; 0 = M).  If a
    category exceeds it num_keep comes back as -1 (the eager op below raises)."""
    _C.require_cuda(boxes, scores, idxs)
    b, s = _f32c(boxes), _f32c(scores)
    ix = None if idxs is None else idxs.to(dtype=torch.int64).contiguous()
    m = b.shape[0]
    keep = torch.empty((m,), dtype=torch.int64, device=b.device)
    num = torch.zeros((1,), dtype=torch.int64, device=b.device) if m == 0 else torch.empty((1,), dtype=torch.int64, device=b.device)
    if m:
        flags = (1 if rotated else 0) | (0 if apply_offsets else 2)  # D2B_NMS_ROTATED | D2B_NMS_NO_OFFSET
        ws_bytes = _C.lib().d2b_nms_workspace_bytes(m, flags, int(max_segment))
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=b.device)
        with torch.cuda.device(b.device):
            check(_C.lib().d2b_nms(ptr(b), ptr(s), ptr(ix), m, float(iou_threshold), flags, int(max_segment), ptr(keep),
                                   ptr(num), ptr(ws), ws_bytes, stream_ptr(b.device)), "nms")
    return keep, num


@torch.library.custom_op("d2b200::nms", mutates_args=(), device_types="cuda")
def nms_op(boxes: Tensor, scores: Tensor, idxs: Optional[Tensor], iou_threshold: float, rotated: bool,
           apply_offsets: bool = True) -> Tensor:
    keep, num = nms_fixed(boxes, scores, idxs, iou_threshold, rotated, apply_offsets)
    n = int(num.item())  # the one host sync: the reference contract returns an exactly-sized tensor
    if n < 0:
        raise RuntimeError("nms: a category exceeded the max_segment bound")
    return keep[:n].clone()


@nms_op.register_fake
def _(boxes, scores, idxs, iou_threshold, rotated, apply_offsets=True):
    ctx = torch.library.get_ctx()
    n = ctx.new_dynamic_size()
    return boxes.new_empty((n,), dtype=torch.int64)


@torch.library.custom_op("d2b200::box_iou_rotated", mutates_args=(), device_types="cuda")
def box_iou_rotated_op(boxes1: Tensor, boxes2: Tensor) -> Tensor:
    _C.require_cuda(boxes1, boxes2)
    b1, b2 = _f32c(boxes1), _f32c(boxes2)
    n, m = b1.shape[0], b2.shape[0]
    out = torch.empty((n, m), dtype=torch.float32, device=b1.device)
    if n and m:
        with torch.cuda.device(b1.device):
            check(_C.lib().d2b_box_iou_rotated(ptr(b1), n, ptr(b2), m, ptr(out), stream_ptr(b1.device)),
                  "box_iou_rotated")
    return out


@box_iou_rotated_op.register_fake
def _(boxes1, boxes2):
    return boxes1.new_empty((boxes1.shape[0], boxes2.shape[0]), dtype=torch.float32)


# =================================================================================== deformable conv
def _dcn_params(x, weight, stride, padding, dilation, groups, deformable_groups):
    n, cin, h, w = x.shape
    cout, _, kh, kw = weight.shape
    return _C.DcnParams(n, cin, h, w, cout, kh, kw, stride[0], stride[1], padding[0], padding[1], dilation[0],
                        dilation[1], groups, deformable_groups)


def dcn_output_shape(x, weight, stride, padding, dilation):
    n, _, h, w = x.shape
    cout, _, kh, kw = weight.shape
    ho = (h + 2 * padding[0] - (dilation[0] * (kh - 1) + 1)) // stride[0] + 1
    wo = (w + 2 * padding[1] - (dilation[1] * (kw - 1) + 1)) // stride[1] + 1
    return n, cout, ho, wo


def _dcn_check(x, offset, mask, weight, stride, padding, dilation, groups, dg):
    """Shape checks of deform_conv_cuda.cu:140-270 / :894-905 -> RuntimeError like TORCH_CHECK."""
    if x.dim() != 4:
        raise ValueError("Expected 4D tensor as input, got {}D tensor instead.".format(x.dim()))
    if weight.dim() != 4:
        raise RuntimeError("deform_conv: weight must be 4D")
    n, cout, ho, wo = dcn_output_shape(x, weight, stride, padding, dilation)
    kh, kw = weight.shape[2:]
    if ho < 1 or wo < 1:
        raise RuntimeError("deform_conv: output size is too small")
    if x.shape[1] != weight.shape[1] * groups:
        raise RuntimeError("deform_conv: input channels and weight/groups do not match")
    if tuple(offset.shape) != (n, 2 * dg * kh * kw, ho, wo):
        raise RuntimeError("invalid spatial size or number of channels of offset: got %s, expected %s" %
                           (tuple(offset.shape), (n, 2 * dg * kh * kw, ho, wo)))
    if mask is not None and tuple(mask.shape) != (n, dg * kh * kw, ho, wo):
        raise RuntimeError("invalid spatial size or number of channels of mask: got %s, expected %s" %
                           (tuple(mask.shape), (n, dg * kh * kw, ho, wo)))


def _dcn_x(x: Tensor, p, precision: int, backward: bool):
    """(fp32 tensor to hand to the kernel, flags).  channels_last inputs are consumed in place by the tensor-core
    kernels (D2B_DCN_X_NHWC); everything else is made NCHW-contiguous."""
    xf = x.to(dtype=torch.float32)
    if (precision != 0 and _is_channels_last(xf) and xf.data_ptr() % 16 == 0
            and _C.lib().d2b_deform_conv_tc_shape_supported(C.byref(p), int(backward))):
        return xf, _C.DCN_X_NHWC
    return xf.contiguous(), 0


def _ws(nbytes: int, device):
    # torch's caching allocator hands out 512-byte aligned blocks: satisfies the ABI's 256-byte requirement
    return torch.empty((nbytes,), dtype=torch.uint8, device=device) if nbytes else None


@torch.library.custom_op("d2b200::deform_conv", mutates_args=(), device_types="cuda")
def deform_conv_op(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, bias: Optional[Tensor],
                   stride: List[int], padding: List[int], dilation: List[int], groups: int, deformable_groups: int,
                   precision: int) -> Tensor:
    _C.require_cuda(x, offset, mask, weight, bias)
    _dcn_check(x, offset, mask, weight, stride, padding, dilation, groups, deformable_groups)
    of, mf, wf, bf = _f32c(offset), _f32c(mask), _f32c(weight), _f32c(bias)
    p = _dcn_params(x, wf, stride, padding, dilation, groups, deformable_groups)
    xf, flags = _dcn_x(x, p, precision, False)
    out = torch.empty(dcn_output_shape(xf, wf, stride, padding, dilation), dtype=torch.float32, device=x.device)
    ws_bytes = _C.lib().d2b_deform_conv_forward_workspace_bytes(C.byref(p), precision, flags)
    ws = _ws(ws_bytes, x.device)
    with torch.cuda.device(x.device):
        check(_C.lib().d2b_deform_conv_forward(ptr(xf), ptr(of), ptr(mf), ptr(wf), ptr(bf), C.byref(p), precision, flags,
                                               ptr(out), None, ptr(ws), ws_bytes, stream_ptr(x.device)),
              "deform_conv_forward")
    return out.to(x.dtype)


@deform_conv_op.register_fake
def _(x, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups, precision):
    return x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation))


@torch.library.custom_op("d2b200::deform_conv_backward", mutates_args=(), device_types="cuda")
def deform_conv_backward_op(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, grad_out: Tensor,
                            stride: List[int], padding: List[int], dilation: List[int], groups: int,
                            deformable_groups: int, with_bias: bool, need_data: bool,
                            need_weight: bool, precision: int,
                            cols: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """All gradients of deform_conv.  `cols`: the column tiles saved by deform_conv_train (same shapes / precision); the
    weight gradient then streams them back instead of sampling x again.  grad_x has x's memory format."""
    _C.require_cuda(x, offset, mask, weight, grad_out, cols)
    of, mf, wf, gf = _f32c(offset), _f32c(mask), _f32c(weight), _f32c(grad_out)
    p = _dcn_params(x, wf, stride, padding, dilation, groups, deformable_groups)
    xf, flags = _dcn_x(x, p, precision, True)
    dev = x.device
    e = lambda: torch.empty((0,), dtype=torch.float32, device=dev)  # noqa: E731
    gx = torch.empty_like(xf) if need_data else e()  # preserves channels_last strides when flags say NHWC
    go = torch.empty_like(of) if need_data else e()
    gm = torch.empty_like(mf) if (need_data and mf is not None) else e()
    gw = torch.empty_like(wf) if need_weight else e()
    gb = torch.empty((wf.shape[0],), dtype=torch.float32, device=dev) if (with_bias and need_weight) else e()
    P = lambda t: ptr(t) if t.numel() else None  # noqa: E731
    ws_bytes = _C.lib().d2b_deform_conv_backward_workspace_bytes(C.byref(p), precision, flags, int(need_data),
                                                                 int(need_weight))
    ws = _ws(ws_bytes, dev)
    if cols is not None and cols.numel() != _C.lib().d2b_deform_conv_cols_bytes(C.byref(p), precision):
        raise RuntimeError("deform_conv_backward: `cols` does not belong to this shape / precision")
    with torch.cuda.device(dev):
        check(_C.lib().d2b_deform_conv_backward(ptr(xf), ptr(of), ptr(mf), ptr(wf), ptr(gf), C.byref(p), precision, flags,
                                                ptr(cols), P(gx), P(go), P(gm), P(gw), P(gb), ptr(ws), ws_bytes,
                                                stream_ptr(dev)),
              "deform_conv_backward")
    return gx, go, gm, gw, gb


@deform_conv_backward_op.register_fake
def _(x, offset, mask, weight, grad_out, stride, padding, dilation, groups, deformable_groups, with_bias, need_data,
      need_weight, precision, cols=None):
    e = lambda: x.new_empty((0,))  # noqa: E731
    return (torch.empty_like(x) if need_data else e(), torch.empty_like(offset) if need_data else e(),
            torch.empty_like(mask) if (need_data and mask is not None) else e(),
            torch.empty_like(weight) if need_weight else e(),
            x.new_empty((weight.shape[0],)) if (with_bias and need_weight) else e())


def _dcn_setup(ctx, inputs, output):
    x, offset, mask, weight, bias, stride, padding, dilation, groups, dg, precision = inputs
    ctx.save_for_backward(x, offset, mask, weight)
    ctx.args = (stride, padding, dilation, groups, dg, bias is not None, precision)
    ctx.has_mask = mask is not None


def _dcn_bwd(ctx, grad):
    x, offset, mask, weight = ctx.saved_tensors
    stride, padding, dilation, groups, dg, with_bias, precision = ctx.args
    need_data = ctx.needs_input_grad[0] or ctx.needs_input_grad[1] or (ctx.has_mask and ctx.needs_input_grad[2])
    need_weight = ctx.needs_input_grad[3] or (with_bias and ctx.needs_input_grad[4])
    gx, go, gm, gw, gb = deform_conv_backward_op(x, offset, mask, weight, grad, stride, padding, dilation, groups, dg,
                                                 with_bias, need_data, need_weight, precision)
    return (gx.to(x.dtype) if need_data else None, go.to(offset.dtype) if need_data else None,
            gm.to(mask.dtype) if (need_data and ctx.has_mask) else None,
            gw.to(weight.dtype) if need_weight else None, gb if (with_bias and need_weight) else None,
            None, None, None, None, None, None)


deform_conv_op.register_autograd(_dcn_bwd, setup_context=_dcn_setup)


# ----------------------------------------------------------------------------------- training forward: keeps what the backward needs
def _dcn_train_layout(x: Tensor, p, precision: int):
    """(x for the kernel, flags, saved channels-last copy or None, cols or None).  When the tensor-core kernels take the
    shape in both directions, x is laid out channels-last ONCE (our layout kernel) and that copy serves the forward and both
    gradient kernels; the forward also keeps its sampled columns for the weight gradient."""
    lib = _C.lib()
    if precision != 0 and lib.d2b_deform_conv_tc_shape_supported(C.byref(p), 0) and \
            lib.d2b_deform_conv_tc_shape_supported(C.byref(p), 1) and x.numel():
        xf = x.to(dtype=torch.float32) if (_is_channels_last(x) or x.dtype not in _C.DTYPE_CODE) else None
        if xf is not None and _is_channels_last(xf) and xf.data_ptr() % 16 == 0:
            xs = None
            xk = xf
        else:
            # NCHW fp32 / fp16 / bf16 -> fp32 channels-last in ONE launch (for half inputs it is also the up-cast)
            src = (xf if xf is not None else x).detach().contiguous()
            with torch.cuda.device(x.device):
                buf = _to_nhwc([src], _pyramid([src], None, [1.0], 0, 0, 0, 1.0), src.shape[0], src.shape[1], x.device)[0]
            xs = buf.permute(0, 3, 1, 2)
            xk = xs
        if _is_channels_last(xk) and xk.data_ptr() % 16 == 0:
            nb = lib.d2b_deform_conv_cols_bytes(C.byref(p), precision)
            cols = torch.empty((nb,), dtype=torch.uint8, device=x.device) if nb else None
            return xk, _C.DCN_X_NHWC, xs, cols
    xk, flags = _dcn_x(x, p, precision, False)
    return xk, flags, None, None


@torch.library.custom_op("d2b200::deform_conv_train", mutates_args=(), device_types="cuda")
def deform_conv_train_op(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, bias: Optional[Tensor],
                         stride: List[int], padding: List[int], dilation: List[int], groups: int, deformable_groups: int,
                         precision: int) -> Tuple[Tensor, Tensor, Tensor]:
    """deform_conv for a step that will be differentiated: (out, x_saved, cols).  x_saved is the channels-last fp32 copy of x
    the kernels ran on (empty when x itself was usable), cols the saved column tiles (empty when the shape has no
    tensor-core path); both go to deform_conv_backward."""
    _C.require_cuda(x, offset, mask, weight, bias)
    _dcn_check(x, offset, mask, weight, stride, padding, dilation, groups, deformable_groups)
    of, mf, wf, bf = _f32c(offset), _f32c(mask), _f32c(weight), _f32c(bias)
    p = _dcn_params(x, wf, stride, padding, dilation, groups, deformable_groups)
    xk, flags, xs, cols = _dcn_train_layout(x, p, precision)
    out = torch.empty(dcn_output_shape(xk, wf, stride, padding, dilation), dtype=torch.float32, device=x.device)
    ws_bytes = _C.lib().d2b_deform_conv_forward_workspace_bytes(C.byref(p), precision, flags)
    ws = _ws(ws_bytes, x.device)
    with torch.cuda.device(x.device):
        check(_C.lib().d2b_deform_conv_forward(ptr(xk), ptr(of), ptr(mf), ptr(wf), ptr(bf), C.byref(p), precision, flags,
                                               ptr(out), ptr(cols), ptr(ws), ws_bytes, stream_ptr(x.device)),
              "deform_conv_forward")
    e = lambda dt: torch.empty((0,), dtype=dt, device=x.device)  # noqa: E731
    return out.to(x.dtype), xs if xs is not None else e(torch.float32), cols if cols is not None else e(torch.uint8)


@deform_conv_train_op.register_fake
def _(x, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups, precision):
    return (x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation)), x.new_empty((0,), dtype=torch.float32),
            x.new_empty((0,), dtype=torch.uint8))


def _dcnt_setup(ctx, inputs, output):
    x, offset, mask, weight, bias, stride, padding, dilation, groups, dg, precision = inputs
    _, xs, cols = output
    ctx.save_for_backward(x if xs.numel() == 0 else xs, offset, mask, weight, cols)
    ctx.args = (stride, padding, dilation, groups, dg, bias is not None, precision, x.dtype)
    ctx.has_mask = mask is not None
    # the saved copy of x and the column tiles are outputs only so that autograd can keep them: nobody differentiates through
    # them, and materialising their (zero) gradients would fill 155 MB per res3 layer in every backward
    ctx.set_materialize_grads(False)


def _dcnt_bwd(ctx, grad, _gxs, _gcols):
    if grad is None:
        return (None,) * 11
    x, offset, mask, weight, cols = ctx.saved_tensors
    stride, padding, dilation, groups, dg, with_bias, precision, xdtype = ctx.args
    need_data = ctx.needs_input_grad[0] or ctx.needs_input_grad[1] or (ctx.has_mask and ctx.needs_input_grad[2])
    need_weight = ctx.needs_input_grad[3] or (with_bias and ctx.needs_input_grad[4])
    gx, go, gm, gw, gb = deform_conv_backward_op(x, offset, mask, weight, grad, stride, padding, dilation, groups, dg,
                                                 with_bias, need_data, need_weight, precision,
                                                 cols if cols.numel() else None)
    return (gx.to(xdtype) if need_data else None, go.to(offset.dtype) if need_data else None,
            gm.to(mask.dtype) if (need_data and ctx.has_mask) else None,
            gw.to(weight.dtype) if need_weight else None, gb if (with_bias and need_weight) else None,
            None, None, None, None, None, None)


deform_conv_train_op.register_autograd(_dcnt_bwd, setup_context=_dcnt_setup)


def deform_conv(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, bias: Optional[Tensor],
                stride: List[int], padding: List[int], dilation: List[int], groups: int, deformable_groups: int,
                precision: int) -> Tensor:
    """The entry the layers call: the training op (which keeps the channels-last copy of x and the sampled columns for the
    backward) when a gradient can flow, the plain forward otherwise."""
    if torch.is_grad_enabled() and (x.requires_grad or offset.requires_grad or weight.requires_grad
                                    or (mask is not None and mask.requires_grad)
                                    or (bias is not None and bias.requires_grad)):
        return deform_conv_train_op(x, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups,
                                    precision)[0]
    return deform_conv_op(x, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups, precision)


# ----------------------------------------------------------------------------------- DeformBottleneckBlock conv2, fused
@torch.library.custom_op("d2b200::deform_conv_fused", mutates_args=(), device_types="cuda")
def deform_conv_fused_op(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor], shift: Optional[Tensor],
                         relu: bool, stride: List[int], padding: List[int], dilation: List[int], groups: int,
                         deformable_groups: int, precision: int) -> Tensor:
    """y = relu(modulated_deform_conv(x, offset, sigmoid(mask), weight) * scale + shift) with offset / mask taken straight
    from the raw conv2_offset output `offset_mask` [N, 3*dg*kh*kw, Ho, Wo] (detectron2/modeling/backbone/resnet.py:305-318):
    the chunk / cat / sigmoid happen while the sampling taps are built, scale / shift / relu in the accumulator epilogue."""
    _C.require_cuda(x, offset_mask, weight, scale, shift)
    kh, kw = weight.shape[2:]
    n, cout, ho, wo = dcn_output_shape(x, weight, stride, padding, dilation)
    if x.dim() != 4:
        raise ValueError("Expected 4D tensor as input, got {}D tensor instead.".format(x.dim()))
    if tuple(offset_mask.shape) != (n, 3 * deformable_groups * kh * kw, ho, wo):
        raise RuntimeError("invalid shape of offset_mask: got %s, expected %s" %
                           (tuple(offset_mask.shape), (n, 3 * deformable_groups * kh * kw, ho, wo)))
    om, wf, sc, sh = _f32c(offset_mask), _f32c(weight), _f32c(scale), _f32c(shift)
    p = _dcn_params(x, wf, stride, padding, dilation, groups, deformable_groups)
    if precision == 0 or not _C.lib().d2b_deform_conv_tc_shape_supported(C.byref(p), 0):
        raise RuntimeError("deform_conv_fused: the tensor-core kernels do not take this shape / precision "
                           "(use layers.modulated_deform_conv and apply the epilogue separately)")
    xf, flags = _dcn_x(x, p, precision, False)
    out = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=x.device)
    ws_bytes = _C.lib().d2b_deform_conv_forward_workspace_bytes(C.byref(p), 1, flags)
    ws = _ws(ws_bytes, x.device)
    with torch.cuda.device(x.device):
        check(_C.lib().d2b_deform_conv_fused_forward(ptr(xf), ptr(om), ptr(wf), ptr(sc), ptr(sh), int(relu), C.byref(p),
                                                     precision, flags, ptr(out), None, ptr(ws), ws_bytes,
                                                     stream_ptr(x.device)),
              "deform_conv_fused_forward")
    return out.to(x.dtype)


@deform_conv_fused_op.register_fake
def _(x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups, deformable_groups, precision):
    return x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation))


@torch.library.custom_op("d2b200::deform_conv_fused_backward", mutates_args=(), device_types="cuda")
def deform_conv_fused_backward_op(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor], relu: bool,
                                  y: Tensor, grad_out: Tensor, stride: List[int], padding: List[int],
                                  dilation: List[int], groups: int, deformable_groups: int,
                                  precision: int, cols: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor]:
    _C.require_cuda(x, offset_mask, weight, scale, y, grad_out, cols)
    om, wf, sc, yf, gf = _f32c(offset_mask), _f32c(weight), _f32c(scale), _f32c(y), _f32c(grad_out)
    p = _dcn_params(x, wf, stride, padding, dilation, groups, deformable_groups)
    if not _C.lib().d2b_deform_conv_tc_shape_supported(C.byref(p), 1):
        raise RuntimeError("deform_conv_fused_backward: the tensor-core backward does not take this shape")
    xf, flags = _dcn_x(x, p, precision, True)
    gx, gom, gw = torch.empty_like(xf), torch.empty_like(om), torch.empty_like(wf)
    ws_bytes = _C.lib().d2b_deform_conv_backward_workspace_bytes(C.byref(p), 1, flags, 1, 1)
    ws = _ws(ws_bytes, x.device)
    if cols is not None and cols.numel() != _C.lib().d2b_deform_conv_cols_bytes(C.byref(p), precision):
        raise RuntimeError("deform_conv_fused_backward: `cols` does not belong to this shape / precision")
    with torch.cuda.device(x.device):
        check(_C.lib().d2b_deform_conv_fused_backward(ptr(xf), ptr(om), ptr(wf), ptr(sc), int(relu), ptr(yf), ptr(gf),
                                                      C.byref(p), precision, flags, ptr(cols), ptr(gx), ptr(gom), ptr(gw),
                                                      ptr(ws), ws_bytes, stream_ptr(x.device)), "deform_conv_fused_backward")
    return gx, gom, gw


@deform_conv_fused_backward_op.register_fake
def _(x, offset_mask, weight, scale, relu, y, grad_out, stride, padding, dilation, groups, deformable_groups, precision,
      cols=None):
    return torch.empty_like(x), torch.empty_like(offset_mask), torch.empty_like(weight)


def _dcnf_setup(ctx, inputs, output):
    x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups, dg, precision = inputs
    ctx.save_for_backward(x, offset_mask, weight, scale, output)
    ctx.args = (relu, stride, padding, dilation, groups, dg, precision)


def _dcnf_bwd(ctx, grad):
    x, offset_mask, weight, scale, y = ctx.saved_tensors
    relu, stride, padding, dilation, groups, dg, precision = ctx.args
    gx, gom, gw = deform_conv_fused_backward_op(x, offset_mask, weight, scale, relu, y, grad, stride, padding, dilation,
                                                groups, dg, precision)
    # scale / shift are FrozenBatchNorm buffers (or a folded bias): no gradient is produced for them
    return (gx.to(x.dtype), gom.to(offset_mask.dtype), gw.to(weight.dtype), None, None, None, None, None, None, None, None,
            None)


deform_conv_fused_op.register_autograd(_dcnf_bwd, setup_context=_dcnf_setup)


@torch.library.custom_op("d2b200::deform_conv_fused_train", mutates_args=(), device_types="cuda")
def deform_conv_fused_train_op(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor],
                               shift: Optional[Tensor], relu: bool, stride: List[int], padding: List[int],
                               dilation: List[int], groups: int, deformable_groups: int,
                               precision: int) -> Tuple[Tensor, Tensor, Tensor]:
    """deform_conv_fused for a step that will be differentiated: (y, x_saved, cols) like deform_conv_train."""
    _C.require_cuda(x, offset_mask, weight, scale, shift)
    kh, kw = weight.shape[2:]
    n, cout, ho, wo = dcn_output_shape(x, weight, stride, padding, dilation)
    if tuple(offset_mask.shape) != (n, 3 * deformable_groups * kh * kw, ho, wo):
        raise RuntimeError("invalid shape of offset_mask: got %s, expected %s" %
                           (tuple(offset_mask.shape), (n, 3 * deformable_groups * kh * kw, ho, wo)))
    om, wf, sc, sh = _f32c(offset_mask), _f32c(weight), _f32c(scale), _f32c(shift)
    p = _dcn_params(x, wf, stride, padding, dilation, groups, deformable_groups)
    if precision == 0 or not _C.lib().d2b_deform_conv_tc_shape_supported(C.byref(p), 0):
        raise RuntimeError("deform_conv_fused: the tensor-core kernels do not take this shape / precision")
    prec = 1 if precision == -1 else precision
    xk, flags, xs, cols = _dcn_train_layout(x, p, prec)
    out = torch.empty((n, cout, ho, wo), dtype=torch.float32, device=x.device)
    ws_bytes = _C.lib().d2b_deform_conv_forward_workspace_bytes(C.byref(p), 1, flags)
    ws = _ws(ws_bytes, x.device)
    with torch.cuda.device(x.device):
        check(_C.lib().d2b_deform_conv_fused_forward(ptr(xk), ptr(om), ptr(wf), ptr(sc), ptr(sh), int(relu), C.byref(p),
                                                     prec, flags, ptr(out), ptr(cols), ptr(ws), ws_bytes,
                                                     stream_ptr(x.device)),
              "deform_conv_fused_forward")
    e = lambda dt: torch.empty((0,), dtype=dt, device=x.device)  # noqa: E731
    return out.to(x.dtype), xs if xs is not None else e(torch.float32), cols if cols is not None else e(torch.uint8)


@deform_conv_fused_train_op.register_fake
def _(x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups, deformable_groups, precision):
    return (x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation)), x.new_empty((0,), dtype=torch.float32),
            x.new_empty((0,), dtype=torch.uint8))


def _dcnft_setup(ctx, inputs, output):
    x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups, dg, precision = inputs
    y, xs, cols = output
    ctx.save_for_backward(x if xs.numel() == 0 else xs, offset_mask, weight, scale, y, cols)
    ctx.args = (relu, stride, padding, dilation, groups, dg, 1 if precision == -1 else precision, x.dtype)
    ctx.set_materialize_grads(False)  # see _dcnt_setup


def _dcnft_bwd(ctx, grad, _gxs, _gcols):
    if grad is None:
        return (None,) * 12
    x, offset_mask, weight, scale, y, cols = ctx.saved_tensors
    relu, stride, padding, dilation, groups, dg, precision, xdtype = ctx.args
    gx, gom, gw = deform_conv_fused_backward_op(x, offset_mask, weight, scale, relu, y, grad, stride, padding, dilation,
                                                groups, dg, precision, cols if cols.numel() else None)
    return (gx.to(xdtype), gom.to(offset_mask.dtype), gw.to(weight.dtype), None, None, None, None, None, None, None, None,
            None)


deform_conv_fused_train_op.register_autograd(_dcnft_bwd, setup_context=_dcnft_setup)


def deform_conv_fused(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor], shift: Optional[Tensor],
                      relu: bool, stride: List[int], padding: List[int], dilation: List[int], groups: int,
                      deformable_groups: int, precision: int) -> Tensor:
    """The entry DeformBottleneckConv2 calls: the training op when a gradient can flow, the plain forward otherwise."""
    if torch.is_grad_enabled() and (x.requires_grad or offset_mask.requires_grad or weight.requires_grad):
        return deform_conv_fused_train_op(x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups,
                                          deformable_groups, precision)[0]
    return deform_conv_fused_op(x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups,
                                deformable_groups, precision)


# =================================================================================== paste masks
@torch.library.custom_op("d2b200::paste_masks", mutates_args=(), device_types="cuda")
def paste_masks_op(masks: Tensor, boxes: Tensor, img_h: int, img_w: int, threshold: float) -> Tensor:
    _C.require_cuda(masks, boxes)
    mk, bx = _f32c(masks), _f32c(boxes)
    n, m = mk.shape[0], mk.shape[-1]
    # bool output (1 byte per pixel, 0/1) for threshold >= 0, uint8 (value * 255) otherwise: mask_ops.py:137-141
    out = torch.empty((n, img_h, img_w), dtype=torch.bool if threshold >= 0 else torch.uint8, device=mk.device)
    if out.numel():
        with torch.cuda.device(mk.device):
            check(_C.lib().d2b_paste_masks(ptr(mk), ptr(bx), n, m, img_h, img_w, threshold, ptr(out),
                                           stream_ptr(mk.device)), "paste_masks")
    return out


@paste_masks_op.register_fake
def _(masks, boxes, img_h, img_w, threshold):
    return masks.new_empty((masks.shape[0], img_h, img_w), dtype=torch.bool if threshold >= 0 else torch.uint8)


@torch.library.custom_op("d2b200::paste_masks_packed", mutates_args=(), device_types="cuda")
def paste_masks_packed_op(masks: Tensor, boxes: Tensor, img_h: int, img_w: int, threshold: float) -> Tensor:
    """Bit-packed boolean paste: int32 [N, H, ceil(W / 32)], bit b of word w of row y = pixel (y, 32 w + b)."""
    _C.require_cuda(masks, boxes)
    if not threshold >= 0:
        raise RuntimeError("paste_masks_packed: boolean output only (threshold >= 0)")
    mk, bx = _f32c(masks), _f32c(boxes)
    n, m = mk.shape[0], mk.shape[-1]
    out = torch.empty((n, img_h, (img_w + 31) // 32), dtype=torch.int32, device=mk.device)
    if out.numel():
        with torch.cuda.device(mk.device):
            check(_C.lib().d2b_paste_masks_packed(ptr(mk), ptr(bx), n, m, img_h, img_w, threshold, ptr(out),
                                                  stream_ptr(mk.device)), "paste_masks_packed")
    return out


@paste_masks_packed_op.register_fake
def _(masks, boxes, img_h, img_w, threshold):
    return masks.new_empty((masks.shape[0], img_h, (img_w + 31) // 32), dtype=torch.int32)


# =================================================================================== detectron2::* dispatcher ops
def _d2_nms_rotated(dets: Tensor, scores: Tensor, iou_threshold: float) -> Tensor:
    return nms_op(dets, scores, None, iou_threshold, True)


def _d2_box_iou_rotated(boxes1: Tensor, boxes2: Tensor) -> Tensor:
    return box_iou_rotated_op(boxes1, boxes2)


def _d2_roi_align_rotated_forward(input: Tensor, rois: Tensor, spatial_scale: float, pooled_height: int,
                                  pooled_width: int, sampling_ratio: int) -> Tensor:
    return roi_align_rotated_op(input, rois, spatial_scale, pooled_height, pooled_width, sampling_ratio)


def _d2_roi_align_rotated_backward(grad: Tensor, rois: Tensor, spatial_scale: float, pooled_height: int,
                                   pooled_width: int, batch_size: int, channels: int, height: int, width: int,
                                   sampling_ratio: int) -> Tensor:
    return roi_align_rotated_backward_op(grad, rois, spatial_scale, pooled_height, pooled_width, batch_size, channels,
                                         height, width, sampling_ratio)


_D2_SCHEMAS = {  # schemas as registered by the reference (dumped from the compiled csrc, SURVEY.md 8b)
    "nms_rotated": ("(Tensor dets, Tensor scores, float iou_threshold) -> Tensor", _d2_nms_rotated),
    "box_iou_rotated": ("(Tensor boxes1, Tensor boxes2) -> Tensor", _d2_box_iou_rotated),
    "roi_align_rotated_forward": ("(Tensor input, Tensor rois, float spatial_scale, int pooled_height, "
                                  "int pooled_width, int sampling_ratio) -> Tensor", _d2_roi_align_rotated_forward),
    "roi_align_rotated_backward": ("(Tensor grad, Tensor rois, float spatial_scale, int pooled_height, "
                                   "int pooled_width, int batch_size, int channels, int height, int width, "
                                   "int sampling_ratio) -> Tensor", _d2_roi_align_rotated_backward),
}

_d2_lib = None


def register_detectron2_namespace():
    """Expose our CUDA kernels under torch.ops.detectron2.* (idempotent).

    Coexistence with the reference's own extension: if `detectron2._C` (or the oracle's build of its csrc) was loaded
    first, its TORCH_LIBRARY(detectron2) block already defined the schemas -- we then only add a CUDA kernel, and only where
    none is registered (a CUDA build of the reference keeps its own kernels: registering a second one would raise).
    Loading the reference extension AFTER this module is not supported by the dispatcher (its `def` would collide with
    the schemas defined here): import detectron2 first, or set D2B_NO_D2_NAMESPACE=1 and call the d2b200::* ops."""
    global _d2_lib
    if _d2_lib is not None or os.environ.get("D2B_NO_D2_NAMESPACE", "0") == "1":
        return
    _d2_lib = torch.library.Library("detectron2", "FRAGMENT")
    for name, (schema, fn) in _D2_SCHEMAS.items():
        qual = "detectron2::" + name
        exists = True
        try:
            torch._C._dispatch_find_schema_or_throw(qual, "")
        except RuntimeError:
            exists = False
        if not exists:
            _d2_lib.define(name + schema)
        elif torch._C._dispatch_has_kernel_for_dispatch_key(qual, "CUDA"):
            continue  # the reference's own CUDA kernel is present: leave it
        _d2_lib.impl(name, fn, "CUDA")


register_detectron2_namespace()
