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
import functools
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
# One host path serves the eight RoIAlign ops: axis-aligned or rotated, each as a single-level op (a one-level pyramid) or
# a multi-level pooler op, forward and backward.  Feature-map layout policy (D2B_POOLER_LAYOUT = auto | nchw | nhwc):
#   * shapes the channels-last kernels do not take (d2b_roi_pooler_nhwc_supported) go to the NCHW kernels;
#   * channels_last inputs are consumed in place by the channels-last kernels (torchvision would .contiguous() them first);
#   * NCHW inputs go to the NCHW kernels, unless the call is large enough that "one layout-change launch + channels-last
#     kernel" is cheaper.  Cost model of the axis-aligned forward fitted to tools/bench_pooler_layouts.py on an H100 80GB
#     HBM3 SXM at 700 W (bench.py's 800x1333 pyramid, 256 channels; 1 000 / 512 / 2 000 RoIs at 7x7 and 100 at 14x14); it
#     picks the faster path on all four.  The backward and rotated per-element costs are carried over from the kernels'
#     first tuning and have not been re-measured on an H100 (the layout-change cost per byte has); the choice only changes
#     speed, every path computes the same result.
POOLER_LAYOUT = os.environ.get("D2B_POOLER_LAYOUT", "auto")
# picoseconds per output element (forward) / grad_out element (backward): (NCHW kernel, channels-last kernel)
_PS_PER_OUT = {  # (rotated, backward)
    (False, False): (21.0, 9.0),  # NCHW 13.9 mask head .. 27.5 box head (512 RoIs); channels-last 7.8 .. 16.8
    (False, True): (40.0, 8.0),   # channels-last: one red.v4 per footprint pixel
    (True, False): (30.0, 10.0),
    (True, True): (64.0, 16.0),
}
_XPOSE_PS_PER_BYTE = 0.72    # layout change: 91.4 MB of fp32 features in 65-68 us (reads + writes each byte once)
_HALF = (torch.float16, torch.bfloat16)
_ONE_LEVEL = (0, 0, 0, 1.0)  # min_level, max_level, canonical_level, canonical_box_size of a single-level call


def _is_channels_last(t: Tensor) -> bool:
    return t.dim() == 4 and not t.is_contiguous() and t.is_contiguous(memory_format=torch.channels_last)


@functools.lru_cache(maxsize=256)
def _nhwc_supported(c: int, hw: Tuple[Tuple[int, int], ...], pooled_h: int, pooled_w: int, flags: int) -> bool:
    """d2b_roi_pooler_nhwc_supported: the channels-last kernels take `c` channels over levels of (h, w) sizes `hw`."""
    P = _C.Pyramid()
    P.num_levels = len(hw)
    for l, (h, w) in enumerate(hw):
        P.H[l], P.W[l] = h, w
    return _C.lib().d2b_roi_pooler_nhwc_supported(C.byref(P), c, pooled_h, pooled_w, flags) == 0


def _pick_layout(feats, n_out: int, pooled: Tuple[int, int] = (1, 1), rotated: bool = False, backward: bool = False,
                 channels_last: Optional[bool] = None) -> str:
    """'cl' = channels-last levels used in place (forward) / gradients produced channels-last (backward), 'xpose' = layout
    change + channels-last kernel, 'nchw' = NCHW kernel.  feats: the levels as tensors or as (n, c, h, w) sizes;
    channels_last defaults to "every level is a 16-byte aligned channels_last tensor"."""
    shapes = [tuple(t.shape) if isinstance(t, Tensor) else tuple(t) for t in feats]
    flags = (_C.ROI_ROTATED if rotated else 0) | (_C.ROI_BACKWARD if backward else 0)
    if POOLER_LAYOUT == "nchw" or not _nhwc_supported(shapes[0][1], tuple(s[2:] for s in shapes), *pooled, flags):
        return "nchw"
    if channels_last is None:
        channels_last = all(_is_channels_last(t) and t.data_ptr() % 16 == 0 for t in feats)
    if channels_last:
        return "cl"
    if POOLER_LAYOUT == "nhwc":
        return "xpose"
    nchw_ps, nhwc_ps = _PS_PER_OUT[(rotated, backward)]
    feat_bytes = 4 * sum(n * c * h * w for (n, c, h, w) in shapes)
    return "xpose" if n_out * nhwc_ps + feat_bytes * _XPOSE_PS_PER_BYTE < n_out * nchw_ps else "nchw"


def _to_nhwc(fs, P, n: int, c: int, device):
    """One launch: every level of the NCHW pyramid `P` (fp32, fp16 or bf16 elements, all levels alike) -> freshly allocated
    fp32 NHWC buffers; returns them.  For half-precision levels the layout change is also the up-cast."""
    bufs = [torch.empty((t.shape[0], t.shape[2], t.shape[3], t.shape[1]), dtype=torch.float32, device=device) for t in fs]
    dst = (C.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])
    check(_C.lib().d2b_pyramid_nchw_to_nhwc(C.byref(P), n, c, dst, _C.DTYPE_CODE[fs[0].dtype], stream_ptr(device)),
          "pyramid_nchw_to_nhwc")
    return bufs


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
    check(_C.lib().d2b_pyramid_nhwc_to_nchw(C.byref(P), n, c, dst, _C.DTYPE_CODE[dtype], stream_ptr(device)),
          "pyramid_nhwc_to_nchw")
    return outs


def _same_half_dtype(ts) -> bool:
    return ts[0].dtype in _HALF and all(t.dtype == ts[0].dtype for t in ts)


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


def pyramid_to_channels_last(feats: List[Tensor]) -> List[Tensor]:
    """All levels of an NCHW fp32 feature pyramid -> channels_last tensors (same logical [N,C,H,W] shape, NHWC storage)
    with ONE kernel launch.  A caller that pools the same features more than once per image (box head + mask head,
    roi_heads.py:798,843 in the reference) converts once and hands the result to every ROIPooler / ROIAlign call, which
    then run the channels-last kernel in place.  Inputs that are already channels_last, need autograd, are not fp32 or
    do not fit the channels-last kernels' limits are returned through torch's own (autograd-aware) conversion / unchanged."""
    _C.require_cuda(*feats)
    if len(feats) == 0 or len(feats) > _C.MAX_LEVELS:
        raise RuntimeError("pyramid_to_channels_last: need 1..%d levels" % _C.MAX_LEVELS)
    c = feats[0].shape[1]
    if (not _nhwc_supported(c, tuple((t.shape[2], t.shape[3]) for t in feats), 1, 1, 0)
            or any(t.shape[:2] != feats[0].shape[:2] for t in feats)):
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


def _check_levels(what: str, feats, scales):
    if len(feats) < 1 or len(feats) > _C.MAX_LEVELS or len(feats) != len(scales):
        raise RuntimeError("%s: need 1..%d feature levels with one scale each" % (what, _C.MAX_LEVELS))


def _roi_forward(feats, rois, scales, pooled_h: int, pooled_w: int, sampling_ratio: int, levels, rotated: bool,
                 aligned: bool = True, level_rois: Optional[Tensor] = None) -> Tensor:
    """The forward of every RoIAlign op.  feats: the levels (one for a single-level op); levels: (min_level, max_level,
    canonical_level, canonical_box_size); rois: the boxes sampled with, level_rois: the ones the FPN level is assigned
    from when they differ.  The output has the dtype of the features."""
    r, lr = _f32c(rois), _f32c(level_rois)
    n, c = feats[0].shape[:2]
    k = r.shape[0]
    numel = k * c * pooled_h * pooled_w
    layout = _pick_layout(feats, numel, (pooled_h, pooled_w), rotated) if numel else "nchw"
    # half-precision NCHW levels: the layout-change launch reads them as they are (it is also the up-cast) and the pooling
    # kernel writes the result in their dtype -- no cast passes; every other combination computes on fp32 copies
    fused_half = layout == "xpose" and _same_half_dtype(feats)
    fs = list(feats) if fused_half else [t.to(dtype=torch.float32) for t in feats]
    out_dt = feats[0].dtype if (layout != "nchw" and feats[0].dtype in _C.DTYPE_CODE) else torch.float32
    out = torch.empty((k, c, pooled_h, pooled_w), dtype=out_dt, device=r.device)
    if numel:
        flags = (_C.ROI_ROTATED if rotated else 0) | (_C.ROI_NHWC if layout != "nchw" else 0)
        with torch.cuda.device(r.device):
            if layout != "cl":
                fs = [t.contiguous() for t in fs]
            # channels_last tensors: same logical shape, NHWC storage -- _pyramid only takes pointers and H, W
            P = _pyramid(fs, None, scales, *levels, lr)
            if layout == "xpose":
                bufs = _to_nhwc(fs, P, n, c, r.device)
                for l, b in enumerate(bufs):
                    P.feat[l] = b.data_ptr()
            check(_C.lib().d2b_roi_pooler_forward(C.byref(P), n, c, ptr(r), k, pooled_h, pooled_w, sampling_ratio,
                                                  int(aligned), flags, ptr(out), _C.DTYPE_CODE[out_dt],
                                                  stream_ptr(r.device)),
                  "roi_pooler_forward")
    return out if out.dtype == feats[0].dtype else out.to(feats[0].dtype)


def _roi_backward(grad, rois, shapes, scales, pooled_h: int, pooled_w: int, sampling_ratio: int, levels, rotated: bool,
                  channels_last: bool, aligned: bool = True, level_rois: Optional[Tensor] = None,
                  half_grads: bool = False) -> List[Tensor]:
    """The backward of every RoIAlign op: the gradient of each level, shapes = [n, c, h0, w0, h1, w1, ...].  fp32 NCHW
    tensors, or channels-last ones when `channels_last` and the channels-last kernel ran; `half_grads`: NCHW gradients in
    `grad`'s fp16 / bf16 dtype (written by the layout-change launch) instead of fp32."""
    r, lr = _f32c(rois), _f32c(level_rois)
    n, c = shapes[0], shapes[1]
    hw = [(shapes[2 + 2 * l], shapes[3 + 2 * l]) for l in range(len(scales))]
    layout = (_pick_layout([(n, c, h, w) for (h, w) in hw], grad.numel(), (pooled_h, pooled_w), rotated, True,
                           channels_last) if n * c else "nchw")
    # the channels-last kernels read fp16 / bf16 gradients in place; the NCHW kernels take fp32
    g = grad.contiguous() if (layout != "nchw" and grad.dtype in _C.DTYPE_CODE) else _f32c(grad)
    flags = (_C.ROI_ROTATED if rotated else 0) | (_C.ROI_NHWC if layout != "nchw" else 0)
    with torch.cuda.device(g.device):
        if layout == "nchw":
            grads = [torch.empty((n, c, h, w), dtype=torch.float32, device=g.device) for (h, w) in hw]
        else:
            bufs = [torch.empty((n, h, w, c), dtype=torch.float32, device=g.device) for (h, w) in hw]
            grads = [b.permute(0, 3, 1, 2) for b in bufs]  # logical NCHW shape: _pyramid reads H, W from dims 2, 3
        P = _pyramid(grads, grads, scales, *levels, lr)
        check(_C.lib().d2b_roi_pooler_backward(C.byref(P), n, c, ptr(g), _C.DTYPE_CODE[g.dtype], ptr(r), r.shape[0], pooled_h,
                                               pooled_w, sampling_ratio, int(aligned), flags, stream_ptr(g.device)),
              "roi_pooler_backward")
        if layout == "xpose":
            grads = _from_nhwc(bufs, n, c, g.device, grad.dtype if (half_grads and grad.dtype in _HALF) else torch.float32)
    if half_grads and grad.dtype in _HALF:
        grads = [t if t.dtype == grad.dtype else t.to(grad.dtype) for t in grads]
    return grads


def _one_level_backward(grad, rois, spatial_scale, pooled_h, pooled_w, n, c, h, w, sampling_ratio, rotated, channels_last,
                        aligned=True) -> Tensor:
    _C.require_cuda(grad, rois)
    if n * c * h * w == 0:  # nothing to write (and a pyramid level needs h, w > 0)
        return torch.empty((n, c, h, w), dtype=grad.dtype, device=grad.device)
    return _roi_backward(grad, rois, [n, c, h, w], [spatial_scale], pooled_h, pooled_w, sampling_ratio, _ONE_LEVEL, rotated,
                         channels_last, aligned)[0].to(grad.dtype)


def _register_roi_autograd(op, backward_op, rotated: bool):
    """The autograd pair of the four RoIAlign ops.  Their inputs are (input or feats, rois, *args); the backward op takes
    args with the feature shapes and the channels-last flag added, and for the axis-aligned pooler the level boxes."""

    def setup_context(ctx, inputs, output):
        feats, rois, *args = inputs
        ctx.pyramid = isinstance(feats, (list, tuple))
        fs = list(feats) if ctx.pyramid else [feats]
        ctx.save_for_backward(rois)
        ctx.args = args
        ctx.shapes = [fs[0].shape[0], fs[0].shape[1]] + [s for t in fs for s in t.shape[2:]]
        ctx.dtypes = [t.dtype for t in fs]
        ctx.channels_last = all(_is_channels_last(t) for t in fs)

    def backward(ctx, grad):
        (rois,) = ctx.saved_tensors
        a, dts, cl = ctx.args, ctx.dtypes, ctx.channels_last
        nones = (None,) * (len(a) + 1)
        if not ctx.pyramid:  # args (scale, ph, pw, sr[, aligned]) -> (scale, ph, pw, n, c, h, w, sr[, aligned], channels_last)
            return (backward_op(grad, rois, *a[:3], *ctx.shapes, *a[3:], cl).to(dts[0]),) + nones
        half = dts[0] in _HALF
        half_grads = half and grad.dtype == dts[0] and all(d == dts[0] for d in dts)
        if rotated:
            grads = backward_op(grad, rois, ctx.shapes, *a, cl, half_grads)
        else:  # same rois as the forward: rounded to the feature dtype for sampling, fp32 for the level
            grads = backward_op(grad, rois.to(dts[0]).to(torch.float32) if half else rois, ctx.shapes, *a, cl,
                                rois if half else None, half_grads)
        return ([g.to(dt) for g, dt in zip(grads, dts)],) + nones

    op.register_autograd(backward, setup_context=setup_context)


@torch.library.custom_op("d2b200::roi_align", mutates_args=(), device_types="cuda")
def roi_align_op(input: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int,
                 sampling_ratio: int, aligned: bool) -> Tensor:
    _roi_common(input, rois, 5)
    return _roi_forward([input], rois, [spatial_scale], pooled_h, pooled_w, sampling_ratio, _ONE_LEVEL, False, aligned)


@roi_align_op.register_fake
def _(input, rois, spatial_scale, pooled_h, pooled_w, sampling_ratio, aligned):
    return input.new_empty((rois.shape[0], input.shape[1], pooled_h, pooled_w))


@torch.library.custom_op("d2b200::roi_align_backward", mutates_args=(), device_types="cuda")
def roi_align_backward_op(grad: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int, n: int,
                          c: int, h: int, w: int, sampling_ratio: int, aligned: bool,
                          channels_last: bool = False) -> Tensor:
    return _one_level_backward(grad, rois, spatial_scale, pooled_h, pooled_w, n, c, h, w, sampling_ratio, False,
                               channels_last, aligned)


@roi_align_backward_op.register_fake
def _(grad, rois, spatial_scale, pooled_h, pooled_w, n, c, h, w, sampling_ratio, aligned, channels_last=False):
    out = grad.new_empty((n, c, h, w))
    return out.contiguous(memory_format=torch.channels_last) if channels_last else out


# ----------------------------------------------------------------------------------- fused multi-level pooler
@torch.library.custom_op("d2b200::roi_pooler", mutates_args=(), device_types="cuda")
def roi_pooler_op(feats: List[Tensor], rois: Tensor, scales: List[float], pooled_h: int, pooled_w: int,
                  sampling_ratio: int, aligned: bool, min_level: int, max_level: int, canonical_level: int,
                  canonical_box_size: float) -> Tensor:
    _C.require_cuda(rois, *feats)
    _check_levels("roi_pooler", feats, scales)
    r = _f32c(rois)
    # half-precision feature maps: the reference samples with the rois cast to the feature dtype (layers/roi_align.py:60,
    # then torchvision's autocast wrapper upcasts both) while the FPN level comes from the fp32 boxes (poolers.py:245)
    half = feats[0].dtype in _HALF
    return _roi_forward(feats, r.to(feats[0].dtype).to(torch.float32) if half else r, scales, pooled_h, pooled_w,
                        sampling_ratio, (min_level, max_level, canonical_level, canonical_box_size), False, aligned,
                        r if half else None)


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
    return _roi_backward(grad, rois, shapes, scales, pooled_h, pooled_w, sampling_ratio,
                         (min_level, max_level, canonical_level, canonical_box_size), False, channels_last, aligned,
                         level_rois, half_grads)


@roi_pooler_backward_op.register_fake
def _(grad, rois, shapes, scales, pooled_h, pooled_w, sampling_ratio, aligned, min_level, max_level, canonical_level,
      canonical_box_size, channels_last=False, level_rois=None, half_grads=False):
    n, c = shapes[0], shapes[1]
    dt = grad.dtype if half_grads else torch.float32
    outs = [grad.new_empty((n, c, shapes[2 + 2 * l], shapes[3 + 2 * l]), dtype=dt) for l in range(len(scales))]
    return [o.contiguous(memory_format=torch.channels_last) for o in outs] if channels_last else outs


# ----------------------------------------------------------------------------------- rotated
@torch.library.custom_op("d2b200::roi_align_rotated", mutates_args=(), device_types="cuda")
def roi_align_rotated_op(input: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int,
                         sampling_ratio: int) -> Tensor:
    _roi_common(input, rois, 6)
    return _roi_forward([input], rois, [spatial_scale], pooled_h, pooled_w, sampling_ratio, _ONE_LEVEL, True)


@roi_align_rotated_op.register_fake
def _(input, rois, spatial_scale, pooled_h, pooled_w, sampling_ratio):
    return input.new_empty((rois.shape[0], input.shape[1], pooled_h, pooled_w))


@torch.library.custom_op("d2b200::roi_align_rotated_backward", mutates_args=(), device_types="cuda")
def roi_align_rotated_backward_op(grad: Tensor, rois: Tensor, spatial_scale: float, pooled_h: int, pooled_w: int,
                                  n: int, c: int, h: int, w: int, sampling_ratio: int,
                                  channels_last: bool = False) -> Tensor:
    return _one_level_backward(grad, rois, spatial_scale, pooled_h, pooled_w, n, c, h, w, sampling_ratio, True,
                               channels_last)


@roi_align_rotated_backward_op.register_fake
def _(grad, rois, spatial_scale, pooled_h, pooled_w, n, c, h, w, sampling_ratio, channels_last=False):
    out = grad.new_empty((n, c, h, w))
    return out.contiguous(memory_format=torch.channels_last) if channels_last else out


@torch.library.custom_op("d2b200::roi_pooler_rotated", mutates_args=(), device_types="cuda")
def roi_pooler_rotated_op(feats: List[Tensor], rois: Tensor, scales: List[float], pooled_h: int, pooled_w: int,
                          sampling_ratio: int, min_level: int, max_level: int, canonical_level: int,
                          canonical_box_size: float) -> Tensor:
    """ROIPooler(pooler_type="ROIAlignRotated") over several levels in one launch: rois [K,6] = (batch, cx, cy, w, h, angle),
    the level of each from w*h.  The rois are used in fp32 whatever the feature dtype (layers/roi_align_rotated.py:81-83)."""
    _C.require_cuda(rois, *feats)
    _check_levels("roi_pooler_rotated", feats, scales)
    _roi_common(feats[0], rois, 6)
    return _roi_forward(feats, rois, scales, pooled_h, pooled_w, sampling_ratio,
                        (min_level, max_level, canonical_level, canonical_box_size), True)


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
    return _roi_backward(grad, rois, shapes, scales, pooled_h, pooled_w, sampling_ratio,
                         (min_level, max_level, canonical_level, canonical_box_size), True, channels_last,
                         half_grads=half_grads)


@roi_pooler_rotated_backward_op.register_fake
def _(grad, rois, shapes, scales, pooled_h, pooled_w, sampling_ratio, min_level, max_level, canonical_level,
      canonical_box_size, channels_last=False, half_grads=False):
    n, c = shapes[0], shapes[1]
    dt = grad.dtype if half_grads else torch.float32
    outs = [grad.new_empty((n, c, shapes[2 + 2 * l], shapes[3 + 2 * l]), dtype=dt) for l in range(len(scales))]
    return [o.contiguous(memory_format=torch.channels_last) for o in outs] if channels_last else outs


_register_roi_autograd(roi_align_op, roi_align_backward_op, False)
_register_roi_autograd(roi_pooler_op, roi_pooler_backward_op, False)
_register_roi_autograd(roi_align_rotated_op, roi_align_rotated_backward_op, True)
_register_roi_autograd(roi_pooler_rotated_op, roi_pooler_rotated_backward_op, True)


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


# =================================================================================== label sampling
@torch.library.custom_op("d2b200::sample_labels", mutates_args=(), device_types="cuda")
def sample_labels_op(labels: Tensor, num_samples: int, max_pos: int, bg_label: int, seed: Tensor, want_labels: bool,
                     want_sampled: bool) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """d2b_sample_labels on labels [N, P] (int8 read as int8, any other integer type as int64) with seed [1] int64 (its
    64 bits are the SplitMix64 seed).  Returns (out_labels [N, P] int8 in the RPN form, sampled [N, num_samples] int64,
    num_pos [N] int64, num_neg [N] int64); an output not asked for is an empty tensor."""
    _C.require_cuda(labels, seed)
    if labels.dim() != 2 or seed.dtype != torch.int64 or seed.numel() != 1:
        raise ValueError("sample_labels: labels [N, P] and seed [1] int64")
    dev = labels.device
    kind = _C.LABELS_I8 if labels.dtype == torch.int8 else _C.LABELS_I64
    lab = labels.contiguous() if kind == _C.LABELS_I8 else labels.to(torch.int64).contiguous()
    n, p = lab.shape
    sd = seed.to(dev).contiguous()
    out_labels = torch.empty((n, p) if want_labels else (0,), dtype=torch.int8, device=dev)
    sampled = torch.empty((n, num_samples) if want_sampled else (0,), dtype=torch.int64, device=dev)
    num_pos = torch.zeros((n,), dtype=torch.int64, device=dev)
    num_neg = torch.zeros((n,), dtype=torch.int64, device=dev)
    if out_labels.numel() or sampled.numel():  # else num_samples or P is 0: nothing is sampled, the counts are 0
        lib = _C.lib()
        ws_bytes = int(lib.d2b_sample_labels_workspace_bytes(n, p, num_samples))
        ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=dev)
        with torch.cuda.device(dev):
            check(lib.d2b_sample_labels(ptr(lab), kind, n, p, int(bg_label), int(num_samples), int(max_pos), ptr(sd),
                                        ptr(out_labels) if want_labels else None, ptr(sampled) if want_sampled else None,
                                        ptr(num_pos), ptr(num_neg), ptr(ws), ws_bytes, stream_ptr(dev)), "sample_labels")
    return out_labels, sampled, num_pos, num_neg


@sample_labels_op.register_fake
def _(labels, num_samples, max_pos, bg_label, seed, want_labels, want_sampled):
    n, p = labels.shape
    e = labels.new_empty
    return (e((n, p) if want_labels else (0,), dtype=torch.int8),
            e((n, num_samples) if want_sampled else (0,), dtype=torch.int64), e((n,), dtype=torch.int64),
            e((n,), dtype=torch.int64))


# =================================================================================== deformable conv
# One host path serves the six DCN ops: plain (DeformConv / ModulatedDeformConv) or fused (conv2 of a DeformBottleneckBlock:
# the raw offset + mask-logit tensor in, relu(conv * scale + shift) out), each as an inference op, a training op that keeps
# what the backward needs, and a backward op.  `conv` = (stride, padding, dilation, groups, deformable_groups).
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


def _dcn_check(x, offset, mask, weight, stride, padding, dilation, groups, dg, fused: bool):
    """Shape checks of deform_conv_cuda.cu:140-270 / :894-905 -> RuntimeError like TORCH_CHECK.  fused: `offset` is the
    offset + mask-logit tensor.  The kernels read the weight with the strides of Cin / groups input channels, so a weight
    that does not match is refused here."""
    if x.dim() != 4:
        raise ValueError("Expected 4D tensor as input, got {}D tensor instead.".format(x.dim()))
    if weight.dim() != 4:
        raise RuntimeError("deform_conv: weight must be 4D")
    n, cout, ho, wo = dcn_output_shape(x, weight, stride, padding, dilation)
    kk = dg * weight.shape[2] * weight.shape[3]
    if ho < 1 or wo < 1:
        raise RuntimeError("deform_conv: output size is too small")
    if x.shape[1] != weight.shape[1] * groups:
        raise RuntimeError("deform_conv: input channels and weight/groups do not match")
    if fused:
        if tuple(offset.shape) != (n, 3 * kk, ho, wo):
            raise RuntimeError("invalid shape of offset_mask: got %s, expected %s" %
                               (tuple(offset.shape), (n, 3 * kk, ho, wo)))
        return
    if tuple(offset.shape) != (n, 2 * kk, ho, wo):
        raise RuntimeError("invalid spatial size or number of channels of offset: got %s, expected %s" %
                           (tuple(offset.shape), (n, 2 * kk, ho, wo)))
    if mask is not None and tuple(mask.shape) != (n, kk, ho, wo):
        raise RuntimeError("invalid spatial size or number of channels of mask: got %s, expected %s" %
                           (tuple(mask.shape), (n, kk, ho, wo)))


def _dcn_precision(precision: int, fused: bool) -> int:
    """The fused ops run on the tensor-core kernels only, so their "auto" (-1) is bf16x3 (1)."""
    return 1 if fused and precision == -1 else precision


def _dcn_layout(x: Tensor, p, precision: int, backward: bool = False, train: bool = False):
    """(x to hand to the kernel, flags, channels-last copy of x made here or None, cols or None).  channels_last fp32 x
    that is 16-byte aligned is used in place by the tensor-core kernels (D2B_DCN_X_NHWC).  A training forward whose shape
    the tensor-core kernels take in both directions lays any other x out channels-last ONCE (our layout kernel; for half
    inputs it is also the up-cast): that copy serves the forward and both gradient kernels, and the forward keeps its
    sampled columns in `cols` for the weight gradient.  Any other x is made fp32 NCHW-contiguous and the kernels change
    its layout themselves."""
    lib, q = _C.lib(), C.byref(p)
    tc = precision != 0 and lib.d2b_deform_conv_tc_shape_supported(q, int(backward))
    if train and tc and x.numel() and lib.d2b_deform_conv_tc_shape_supported(q, 1):
        xk, xs = (x.to(dtype=torch.float32) if (_is_channels_last(x) or x.dtype not in _C.DTYPE_CODE) else x), None
        if not (_is_channels_last(xk) and xk.data_ptr() % 16 == 0):
            src = xk.detach().contiguous()
            with torch.cuda.device(x.device):
                buf = _to_nhwc([src], _pyramid([src], None, [1.0], 0, 0, 0, 1.0), src.shape[0], src.shape[1], x.device)[0]
            xk = xs = buf.permute(0, 3, 1, 2)
        if _is_channels_last(xk):  # else a 1x1 map, whose copy is NCHW-contiguous as well: it runs as an inference call
            nb = lib.d2b_deform_conv_cols_bytes(q, precision)
            return xk, _C.DCN_X_NHWC, xs, (torch.empty((nb,), dtype=torch.uint8, device=x.device) if nb else None)
    xf = x.to(dtype=torch.float32)
    if tc and _is_channels_last(xf) and xf.data_ptr() % 16 == 0:
        return xf, _C.DCN_X_NHWC, None, None
    return xf.contiguous(), 0, None, None


def _ws(nbytes: int, device):
    # torch's caching allocator hands out 512-byte aligned blocks: satisfies the ABI's 256-byte requirement
    return torch.empty((nbytes,), dtype=torch.uint8, device=device) if nbytes else None


def _dcn_forward(x, offset, mask, weight, bias, conv, precision: int, train: bool, fused=None):
    """The forward of the four DCN forward ops: the output in x's dtype; for `train` also the channels-last fp32 copy of x
    the kernels ran on (empty when x itself was usable) and the saved column tiles (empty when the shape has no tensor-core
    path), both for the backward.  fused = (scale, relu) of a fused op: `offset` is the offset + mask-logit tensor, `mask`
    is None and `bias` is the shift of the epilogue."""
    scale, relu = fused or (None, False)
    _C.require_cuda(x, offset, mask, weight, bias, scale)
    _dcn_check(x, offset, mask, weight, *conv, fused is not None)
    of, mf, wf, bf, sc = _f32c(offset), _f32c(mask), _f32c(weight), _f32c(bias), _f32c(scale)
    p = _dcn_params(x, wf, *conv)
    lib = _C.lib()
    if fused is not None and (precision == 0 or not lib.d2b_deform_conv_tc_shape_supported(C.byref(p), 0)):
        raise RuntimeError("deform_conv_fused: the tensor-core kernels do not take this shape / precision "
                           "(use layers.modulated_deform_conv and apply the epilogue separately)")
    precision = _dcn_precision(precision, fused is not None)
    xk, flags, xs, cols = _dcn_layout(x, p, precision, train=train)
    out = torch.empty(dcn_output_shape(x, wf, *conv[:3]), dtype=torch.float32, device=x.device)
    ws_bytes = lib.d2b_deform_conv_forward_workspace_bytes(C.byref(p), precision, flags)
    ws = _ws(ws_bytes, x.device)
    with torch.cuda.device(x.device):
        if fused is None:
            check(lib.d2b_deform_conv_forward(ptr(xk), ptr(of), ptr(mf), ptr(wf), ptr(bf), C.byref(p), precision, flags,
                                              ptr(out), ptr(cols), ptr(ws), ws_bytes, stream_ptr(x.device)),
                  "deform_conv_forward")
        else:
            check(lib.d2b_deform_conv_fused_forward(ptr(xk), ptr(of), ptr(wf), ptr(sc), ptr(bf), int(relu), C.byref(p),
                                                    precision, flags, ptr(out), ptr(cols), ptr(ws), ws_bytes,
                                                    stream_ptr(x.device)),
                  "deform_conv_fused_forward")
    if not train:
        return out.to(x.dtype)
    e = lambda dt: torch.empty((0,), dtype=dt, device=x.device)  # noqa: E731
    return out.to(x.dtype), xs if xs is not None else e(torch.float32), cols if cols is not None else e(torch.uint8)


def _dcn_backward(x, offset, mask, weight, grad_out, conv, precision: int, cols, need_data: bool = True,
                  need_weight: bool = True, with_bias: bool = False, fused=None):
    """The gradients of every DCN op: (grad_x, grad_offset, grad_mask, grad_weight, grad_bias), one not asked for being
    empty; fused = (scale, relu, y) of a fused op: (grad_x, grad_offset_mask, grad_weight), all three computed.  `cols`: the
    column tiles saved by a training forward of the same shape / precision.  grad_x has x's memory format."""
    scale, relu, y = fused or (None, False, None)
    _C.require_cuda(x, offset, mask, weight, grad_out, cols, scale, y)
    of, mf, wf, gf, sc, yf = _f32c(offset), _f32c(mask), _f32c(weight), _f32c(grad_out), _f32c(scale), _f32c(y)
    p = _dcn_params(x, wf, *conv)
    lib = _C.lib()
    what = "deform_conv_backward" if fused is None else "deform_conv_fused_backward"
    if fused is not None and not lib.d2b_deform_conv_tc_shape_supported(C.byref(p), 1):
        raise RuntimeError(what + ": the tensor-core backward does not take this shape")
    if cols is not None and cols.numel() != lib.d2b_deform_conv_cols_bytes(C.byref(p), precision):
        raise RuntimeError(what + ": `cols` does not belong to this shape / precision")
    xk, flags, _, _ = _dcn_layout(x, p, precision, backward=True)
    dev = x.device
    gx = torch.empty_like(xk) if need_data else None  # preserves channels_last strides when flags say NHWC
    go = torch.empty_like(of) if need_data else None
    gm = torch.empty_like(mf) if (need_data and mf is not None) else None
    gw = torch.empty_like(wf) if need_weight else None
    gb = torch.empty((wf.shape[0],), dtype=torch.float32, device=dev) if (with_bias and need_weight) else None
    ws_bytes = lib.d2b_deform_conv_backward_workspace_bytes(C.byref(p), precision, flags, int(need_data),
                                                            int(need_weight))
    ws = _ws(ws_bytes, dev)
    P = lambda t: ptr(t) if t is not None and t.numel() else None  # noqa: E731
    with torch.cuda.device(dev):
        if fused is None:
            check(lib.d2b_deform_conv_backward(ptr(xk), ptr(of), ptr(mf), ptr(wf), ptr(gf), C.byref(p), precision, flags,
                                               ptr(cols), P(gx), P(go), P(gm), P(gw), P(gb), ptr(ws), ws_bytes,
                                               stream_ptr(dev)), what)
        else:
            check(lib.d2b_deform_conv_fused_backward(ptr(xk), ptr(of), ptr(wf), ptr(sc), int(relu), ptr(yf), ptr(gf),
                                                     C.byref(p), precision, flags, ptr(cols), P(gx), P(go), P(gw), ptr(ws),
                                                     ws_bytes, stream_ptr(dev)), what)
    if fused is not None:
        return gx, go, gw
    e = lambda t: t if t is not None else torch.empty((0,), dtype=torch.float32, device=dev)  # noqa: E731
    return e(gx), e(go), e(gm), e(gw), e(gb)


def _register_dcn_autograd(op, backward_op, fused: bool, train: bool):
    """The autograd pair of the four DCN forward ops.  Their inputs are (x, offset, mask, weight, bias, *conv, precision)
    or, fused, (x, offset_mask, weight, scale, shift, relu, *conv, precision); a training op's outputs are (y, x_saved,
    cols) and its backward runs on the saved channels-last copy of x and streams the saved columns back."""

    def setup_context(ctx, inputs, output):
        if fused:
            x, offset, weight, scale, _, ctx.relu, *conv, precision = inputs
            mask, ctx.with_bias = None, False
        else:
            x, offset, mask, weight, bias, *conv, precision = inputs
            scale, ctx.with_bias = None, bias is not None
        y, xs, cols = output if train else (output, None, None)
        ctx.save_for_backward(xs if xs is not None and xs.numel() else x, offset, mask, weight, scale,
                              y if fused else None, cols if cols is not None and cols.numel() else None)
        ctx.conv, ctx.precision, ctx.x_dtype = conv, _dcn_precision(precision, fused), x.dtype
        if train:
            # the saved copy of x and the column tiles are outputs only so that autograd can keep them: nobody
            # differentiates through them, and materialising their (zero) gradients would fill 155 MB per res3 layer in
            # every backward
            ctx.set_materialize_grads(False)

    def backward(ctx, grad, *_):
        n_in = len(ctx.needs_input_grad)
        if grad is None:  # a training op of which only x_saved / cols were used
            return (None,) * n_in
        x, offset, mask, weight, scale, y, cols = ctx.saved_tensors
        if fused:  # scale / shift are FrozenBatchNorm buffers (or a folded bias): no gradient is produced for them
            gx, go, gw = backward_op(x, offset, weight, scale, ctx.relu, y, grad, *ctx.conv, ctx.precision, cols)
            return (gx.to(ctx.x_dtype), go.to(offset.dtype), gw.to(weight.dtype)) + (None,) * (n_in - 3)
        need = ctx.needs_input_grad
        need_data = need[0] or need[1] or (mask is not None and need[2])
        need_weight = need[3] or (ctx.with_bias and need[4])
        gx, go, gm, gw, gb = backward_op(x, offset, mask, weight, grad, *ctx.conv, ctx.with_bias, need_data, need_weight,
                                         ctx.precision, cols)
        return (gx.to(ctx.x_dtype) if need_data else None, go.to(offset.dtype) if need_data else None,
                gm.to(mask.dtype) if (need_data and mask is not None) else None,
                gw.to(weight.dtype) if need_weight else None, gb if (ctx.with_bias and need_weight) else None,
                ) + (None,) * (n_in - 5)

    op.register_autograd(backward, setup_context=setup_context)


@torch.library.custom_op("d2b200::deform_conv", mutates_args=(), device_types="cuda")
def deform_conv_op(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, bias: Optional[Tensor],
                   stride: List[int], padding: List[int], dilation: List[int], groups: int, deformable_groups: int,
                   precision: int) -> Tensor:
    return _dcn_forward(x, offset, mask, weight, bias, (stride, padding, dilation, groups, deformable_groups), precision,
                        False)


@deform_conv_op.register_fake
def _(x, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups, precision):
    return x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation))


@torch.library.custom_op("d2b200::deform_conv_train", mutates_args=(), device_types="cuda")
def deform_conv_train_op(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, bias: Optional[Tensor],
                         stride: List[int], padding: List[int], dilation: List[int], groups: int, deformable_groups: int,
                         precision: int) -> Tuple[Tensor, Tensor, Tensor]:
    """deform_conv for a step that will be differentiated: (out, x_saved, cols).  x_saved is the channels-last fp32 copy of x
    the kernels ran on (empty when x itself was usable), cols the saved column tiles (empty when the shape has no
    tensor-core path); both go to deform_conv_backward."""
    return _dcn_forward(x, offset, mask, weight, bias, (stride, padding, dilation, groups, deformable_groups), precision,
                        True)


@deform_conv_train_op.register_fake
def _(x, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups, precision):
    return (x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation)), x.new_empty((0,), dtype=torch.float32),
            x.new_empty((0,), dtype=torch.uint8))


@torch.library.custom_op("d2b200::deform_conv_backward", mutates_args=(), device_types="cuda")
def deform_conv_backward_op(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, grad_out: Tensor,
                            stride: List[int], padding: List[int], dilation: List[int], groups: int,
                            deformable_groups: int, with_bias: bool, need_data: bool,
                            need_weight: bool, precision: int,
                            cols: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """All gradients of deform_conv.  `cols`: the column tiles saved by deform_conv_train (same shapes / precision); the
    weight gradient then streams them back instead of sampling x again.  grad_x has x's memory format."""
    return _dcn_backward(x, offset, mask, weight, grad_out, (stride, padding, dilation, groups, deformable_groups),
                         precision, cols, need_data, need_weight, with_bias)


@deform_conv_backward_op.register_fake
def _(x, offset, mask, weight, grad_out, stride, padding, dilation, groups, deformable_groups, with_bias, need_data,
      need_weight, precision, cols=None):
    e = lambda: x.new_empty((0,))  # noqa: E731
    return (torch.empty_like(x) if need_data else e(), torch.empty_like(offset) if need_data else e(),
            torch.empty_like(mask) if (need_data and mask is not None) else e(),
            torch.empty_like(weight) if need_weight else e(),
            x.new_empty((weight.shape[0],)) if (with_bias and need_weight) else e())


# ----------------------------------------------------------------------------------- DeformBottleneckBlock conv2, fused
@torch.library.custom_op("d2b200::deform_conv_fused", mutates_args=(), device_types="cuda")
def deform_conv_fused_op(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor], shift: Optional[Tensor],
                         relu: bool, stride: List[int], padding: List[int], dilation: List[int], groups: int,
                         deformable_groups: int, precision: int) -> Tensor:
    """y = relu(modulated_deform_conv(x, offset, sigmoid(mask), weight) * scale + shift) with offset / mask taken straight
    from the raw conv2_offset output `offset_mask` [N, 3*dg*kh*kw, Ho, Wo] (detectron2/modeling/backbone/resnet.py:305-318):
    the chunk / cat / sigmoid happen while the sampling taps are built, scale / shift / relu in the accumulator epilogue."""
    return _dcn_forward(x, offset_mask, None, weight, shift, (stride, padding, dilation, groups, deformable_groups),
                        precision, False, (scale, relu))


@deform_conv_fused_op.register_fake
def _(x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups, deformable_groups, precision):
    return x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation))


@torch.library.custom_op("d2b200::deform_conv_fused_train", mutates_args=(), device_types="cuda")
def deform_conv_fused_train_op(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor],
                               shift: Optional[Tensor], relu: bool, stride: List[int], padding: List[int],
                               dilation: List[int], groups: int, deformable_groups: int,
                               precision: int) -> Tuple[Tensor, Tensor, Tensor]:
    """deform_conv_fused for a step that will be differentiated: (y, x_saved, cols) like deform_conv_train."""
    return _dcn_forward(x, offset_mask, None, weight, shift, (stride, padding, dilation, groups, deformable_groups),
                        precision, True, (scale, relu))


@deform_conv_fused_train_op.register_fake
def _(x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups, deformable_groups, precision):
    return (x.new_empty(dcn_output_shape(x, weight, stride, padding, dilation)), x.new_empty((0,), dtype=torch.float32),
            x.new_empty((0,), dtype=torch.uint8))


@torch.library.custom_op("d2b200::deform_conv_fused_backward", mutates_args=(), device_types="cuda")
def deform_conv_fused_backward_op(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor], relu: bool,
                                  y: Tensor, grad_out: Tensor, stride: List[int], padding: List[int],
                                  dilation: List[int], groups: int, deformable_groups: int,
                                  precision: int, cols: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor]:
    return _dcn_backward(x, offset_mask, None, weight, grad_out, (stride, padding, dilation, groups, deformable_groups),
                         precision, cols, fused=(scale, relu, y))


@deform_conv_fused_backward_op.register_fake
def _(x, offset_mask, weight, scale, relu, y, grad_out, stride, padding, dilation, groups, deformable_groups, precision,
      cols=None):
    return torch.empty_like(x), torch.empty_like(offset_mask), torch.empty_like(weight)


_register_dcn_autograd(deform_conv_op, deform_conv_backward_op, fused=False, train=False)
_register_dcn_autograd(deform_conv_train_op, deform_conv_backward_op, fused=False, train=True)
_register_dcn_autograd(deform_conv_fused_op, deform_conv_fused_backward_op, fused=True, train=False)
_register_dcn_autograd(deform_conv_fused_train_op, deform_conv_fused_backward_op, fused=True, train=True)


def _grad_can_flow(*tensors) -> bool:
    return torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in tensors)


def deform_conv(x: Tensor, offset: Tensor, mask: Optional[Tensor], weight: Tensor, bias: Optional[Tensor],
                stride: List[int], padding: List[int], dilation: List[int], groups: int, deformable_groups: int,
                precision: int) -> Tensor:
    """The entry the layers call: the training op (which keeps the channels-last copy of x and the sampled columns for the
    backward) when a gradient can flow, the plain forward otherwise."""
    args = (x, offset, mask, weight, bias, stride, padding, dilation, groups, deformable_groups, precision)
    return deform_conv_train_op(*args)[0] if _grad_can_flow(x, offset, mask, weight, bias) else deform_conv_op(*args)


def deform_conv_fused(x: Tensor, offset_mask: Tensor, weight: Tensor, scale: Optional[Tensor], shift: Optional[Tensor],
                      relu: bool, stride: List[int], padding: List[int], dilation: List[int], groups: int,
                      deformable_groups: int, precision: int) -> Tensor:
    """The entry DeformBottleneckConv2 calls: the training op when a gradient can flow, the plain forward otherwise."""
    args = (x, offset_mask, weight, scale, shift, relu, stride, padding, dilation, groups, deformable_groups, precision)
    return deform_conv_fused_train_op(*args)[0] if _grad_can_flow(x, offset_mask, weight) else deform_conv_fused_op(*args)


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
