"""Semantic segmentation training loss: bilinear upsampling fused into the pixel cross-entropy, on two native entry points.

  * `sem_seg_fpn_losses` -- SemSegFPNHead.losses (modeling/meta_arch/semantic_seg.py:255-267): predictions.float(),
    F.interpolate(scale_factor=common_stride, bilinear, align_corners=False), F.cross_entropy(mean, ignore_index).
  * `deeplab_losses` -- DeepLabV3PlusHead.losses / DeepLabV3Head.losses (projects/DeepLab/deeplab/semantic_seg.py) and
    PanopticDeepLabSemSegHead.losses (projects/Panoptic-DeepLab/panoptic_deeplab/panoptic_seg.py), with loss_type
    "cross_entropy" or "hard_pixel_mining" (DeepLabCE, projects/DeepLab/deeplab/loss.py, per-pixel `weights` optional).
  * `sem_seg_loss_fixed` -- the sync-free form behind both: (loss, valid count, status) as device tensors.

The reference materialises the upsampled [N, C, H, W] fp32 map and its log_softmax (464 MB each at 2 x 54 x 800 x 1344)
and its backward goes through upsample_bilinear2d_backward's float atomics.  `d2b_sem_seg_loss_forward` evaluates the
upsampled values from the low-res logits inside the logsumexp and keeps one fp32 per pixel (lse); the backward recomputes
them and writes every logit gradient once, in a fixed order.  Logits of any dtype are upsampled in fp32 (the reference's
`predictions.float()`; the DeepLab heads interpolate half-precision logits in half precision).

Top-k ties: pixels tied at the k-th largest value are taken in ascending flat index; the reference's torch.topk choice
among ties is unspecified and changes only the gradient of the tied pixels.  A NaN per-pixel loss ranks above +inf.
CPU tensors take `_sem_seg_loss_host`, the reference's torch composition with that tie rule; run on CUDA tensors it is what
the GPU tests compare the kernels against.
"""
import ctypes as C
from typing import Dict, Optional, Tuple

import torch
from torch.nn import functional as F

from . import _C
from ._C import check, ptr, stream_ptr

Tensor = torch.Tensor

__all__ = ["sem_seg_fpn_losses", "deeplab_losses", "sem_seg_loss_fixed", "sem_seg_loss_op", "sem_seg_loss_backward_op",
           "SEMSEG_MAX_STRIDE"]

SEMSEG_MEAN, SEMSEG_TOP_K = 0, 1  # D2B_SEMSEG_MEAN / D2B_SEMSEG_TOP_K
SEMSEG_MAX_STRIDE = 32            # D2B_SEMSEG_MAX_STRIDE
STATUS_BAD_LABEL = 1              # D2B_SEMSEG_STATUS_BAD_LABEL


def _selects(top_k_percent_pixels: Optional[float]) -> bool:
    """True when the top-k reduction runs a selection (every value but 1.0)."""
    return top_k_percent_pixels is not None and top_k_percent_pixels != 1.0


def _as_logits(logits: Tensor) -> Tensor:
    if logits.dim() != 4:
        raise RuntimeError("sem_seg_loss: predictions must be N x C x Hp x Wp")
    return (logits if logits.dtype in _C.DTYPE_CODE else logits.to(torch.float32)).contiguous()


def _out_shape(logits: Tensor, stride: int) -> Tuple[int, int, int]:
    return logits.shape[0], logits.shape[2] * stride, logits.shape[3] * stride


def _check_inputs(logits: Tensor, targets: Tensor, stride: int, weights: Optional[Tensor]):
    if not 1 <= stride <= SEMSEG_MAX_STRIDE:
        raise RuntimeError("sem_seg_loss: the stride must be in 1..%d" % SEMSEG_MAX_STRIDE)
    shape = _out_shape(logits, stride)
    if tuple(targets.shape) != shape:
        raise RuntimeError("sem_seg_loss: targets must be N x (Hp * stride) x (Wp * stride) = %s, got %s"
                           % (shape, tuple(targets.shape)))
    if weights is not None and tuple(weights.shape) != shape:
        raise RuntimeError("sem_seg_loss: weights must have the targets' shape")


@torch.library.custom_op("d2b200::sem_seg_loss", mutates_args=(), device_types="cuda")
def sem_seg_loss_op(logits: Tensor, targets: Tensor, stride: int, ignore_value: int,
                    top_k_percent_pixels: Optional[float], weights: Optional[Tensor]
                    ) -> Tuple[Tensor, Tensor, Tensor, Tensor, Tensor]:
    """logits [N, C, Hp, Wp] (fp32 / fp16 / bf16), targets [N, Hp * stride, Wp * stride] int64.  top_k_percent_pixels
    None: the mean over the valid pixels (loss_sum / count); otherwise DeepLabCE's top-k (loss_sum / k, weights allowed).
    Returns (loss_sum [] fp32, count [] int64, status [] int32, lse [N, H, W] fp32, selected [N, H, W] uint8 -- empty unless
    a selection runs)."""
    _C.require_cuda(logits, targets, weights)
    lg = _as_logits(logits)
    _check_inputs(lg, targets, stride, weights)
    n, h, w = _out_shape(lg, stride)
    _, c, hp, wp = lg.shape
    device = lg.device
    tg = targets.to(torch.int64).contiguous()
    wt = None if weights is None else weights.to(torch.float32).contiguous()
    reduction = SEMSEG_MEAN if top_k_percent_pixels is None else SEMSEG_TOP_K
    top_k = -1.0 if top_k_percent_pixels is None else float(top_k_percent_pixels)
    loss_sum = torch.empty((), dtype=torch.float32, device=device)
    count = torch.empty((), dtype=torch.int64, device=device)
    status = torch.empty((), dtype=torch.int32, device=device)
    lse = torch.empty((n, h, w), dtype=torch.float32, device=device)
    selected = torch.empty((n, h, w) if _selects(top_k_percent_pixels) else (0,), dtype=torch.uint8, device=device)
    lib = _C.lib()
    dt = _C.DTYPE_CODE[lg.dtype]
    ws_bytes = lib.d2b_sem_seg_loss_workspace_bytes(n, c, hp, wp, stride, dt, reduction, top_k)
    if ws_bytes == 0:
        raise RuntimeError("sem_seg_loss: unsupported arguments (N %d, C %d, %d x %d, stride %d, top_k %r)"
                           % (n, c, hp, wp, stride, top_k_percent_pixels))
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        check(lib.d2b_sem_seg_loss_forward(ptr(lg), dt, n, c, hp, wp, stride, ptr(tg), int(ignore_value), reduction, top_k,
                                           ptr(wt), ptr(lse), ptr(selected) if selected.numel() else None, ptr(loss_sum),
                                           ptr(count), ptr(status), ptr(ws), ws_bytes, stream_ptr(device)),
              "sem_seg_loss_forward")
    return loss_sum, count, status, lse, selected


@sem_seg_loss_op.register_fake
def _(logits, targets, stride, ignore_value, top_k_percent_pixels, weights):
    n, h, w = _out_shape(logits, stride)
    return (logits.new_empty((), dtype=torch.float32), logits.new_empty((), dtype=torch.int64),
            logits.new_empty((), dtype=torch.int32), logits.new_empty((n, h, w), dtype=torch.float32),
            logits.new_empty((n, h, w) if _selects(top_k_percent_pixels) else (0,), dtype=torch.uint8))


@torch.library.custom_op("d2b200::sem_seg_loss_backward", mutates_args=(), device_types="cuda")
def sem_seg_loss_backward_op(logits: Tensor, targets: Tensor, stride: int, ignore_value: int, weights: Optional[Tensor],
                             selected: Tensor, lse: Tensor, grad_sum: Tensor) -> Tensor:
    """d loss / d logits from grad_sum = d loss / d loss_sum (a device scalar); selected empty = every valid pixel.
    Returns the gradient in the dtype of `_as_logits(logits)`."""
    _C.require_cuda(logits, targets, weights, selected, lse, grad_sum)
    lg = _as_logits(logits)
    n, _, hp, wp = lg.shape
    out = torch.empty_like(lg)
    if n:
        gs = grad_sum.to(torch.float32).reshape(1).contiguous()
        tg = targets.to(torch.int64).contiguous()
        wt = None if weights is None else weights.to(torch.float32).contiguous()
        with torch.cuda.device(lg.device):
            check(_C.lib().d2b_sem_seg_loss_backward(ptr(lg), _C.DTYPE_CODE[lg.dtype], n, lg.shape[1], hp, wp, stride,
                                                     ptr(tg), int(ignore_value), ptr(wt),
                                                     ptr(selected) if selected.numel() else None, ptr(lse.contiguous()),
                                                     ptr(gs), ptr(out), stream_ptr(lg.device)), "sem_seg_loss_backward")
    return out


@sem_seg_loss_backward_op.register_fake
def _(logits, targets, stride, ignore_value, weights, selected, lse, grad_sum):
    return torch.empty_like(_as_logits(logits))


def _ssl_setup(ctx, inputs, output):
    logits, targets, stride, ignore_value, _, weights = inputs
    ctx.stride, ctx.ignore_value = stride, ignore_value
    ctx.save_for_backward(logits, targets, weights, output[4], output[3])


def _ssl_bwd(ctx, grad_sum, grad_count, grad_status, grad_lse, grad_selected):
    logits, targets, weights, selected, lse = ctx.saved_tensors
    if grad_sum is None:
        grad_sum = lse.new_zeros(())
    grad = sem_seg_loss_backward_op(logits, targets, ctx.stride, ctx.ignore_value, weights, selected, lse, grad_sum)
    return grad.to(logits.dtype), None, None, None, None, None


sem_seg_loss_op.register_autograd(_ssl_bwd, setup_context=_ssl_setup)


def sem_seg_loss_fixed(predictions: Tensor, targets: Tensor, common_stride: int, ignore_value: int,
                       top_k_percent_pixels: Optional[float] = None,
                       weights: Optional[Tensor] = None) -> Tuple[Tensor, Tensor, Tensor]:
    """Sync-free loss of CUDA tensors: returns (loss, count, status) as device tensors -- loss the mean cross-entropy over
    the valid pixels (top_k_percent_pixels None) or DeepLabCE's top-k mean, count the valid pixels, status nonzero when a
    target is outside [0, C) and not ignore_value.  Static shapes: capturable in a CUDA graph."""
    if top_k_percent_pixels is None and weights is not None:
        raise ValueError("sem_seg_loss: per-pixel weights need the top-k (DeepLabCE) reduction")
    loss_sum, count, status, _, _ = sem_seg_loss_op(predictions, targets, int(common_stride), int(ignore_value),
                                                    None if top_k_percent_pixels is None else float(top_k_percent_pixels),
                                                    weights)
    if top_k_percent_pixels is None:
        loss = loss_sum / count.to(torch.float32)  # 0 / 0 = NaN without a valid pixel, as F.cross_entropy
    else:
        numel = targets.numel()
        k = numel if top_k_percent_pixels == 1.0 else int(top_k_percent_pixels * numel)
        loss = loss_sum / k if k else loss_sum * float("nan")
    return loss, count, status


def _raise_on_bad_label(status: Tensor):
    if int(status.item()) & STATUS_BAD_LABEL:  # the one host read
        raise RuntimeError("sem_seg_loss: a target is outside [0, num_classes) and not the ignore value")


def _sem_seg_loss_host(predictions: Tensor, targets: Tensor, common_stride: int, ignore_value: int,
                       top_k_percent_pixels: Optional[float] = None, weights: Optional[Tensor] = None) -> Tensor:
    """The reference composition: predictions.float(), F.interpolate, F.cross_entropy; for top-k DeepLabCE with the
    documented tie rule (a stable descending sort: ties in ascending flat index, NaN first)."""
    up = F.interpolate(predictions.float(), scale_factor=common_stride, mode="bilinear", align_corners=False)
    if top_k_percent_pixels is None:
        return F.cross_entropy(up, targets, reduction="mean", ignore_index=ignore_value)
    pixel = F.cross_entropy(up, targets, reduction="none", ignore_index=ignore_value)
    if weights is not None:
        pixel = pixel * weights
    pixel = pixel.contiguous().view(-1)
    if top_k_percent_pixels == 1.0:
        return pixel.mean()
    k = int(top_k_percent_pixels * pixel.numel())
    order = torch.sort(pixel.detach(), descending=True, stable=True).indices[:k]
    return pixel[order].mean()


def _loss(predictions, targets, common_stride, ignore_value, top_k_percent_pixels, weights) -> Tensor:
    if not predictions.is_cuda:
        return _sem_seg_loss_host(predictions, targets, common_stride, ignore_value, top_k_percent_pixels, weights)
    loss, _, status = sem_seg_loss_fixed(predictions, targets, common_stride, ignore_value, top_k_percent_pixels, weights)
    _raise_on_bad_label(status)
    return loss


def sem_seg_fpn_losses(predictions: Tensor, targets: Tensor, common_stride: int, ignore_value: int,
                       loss_weight: float) -> Dict[str, Tensor]:
    """SemSegFPNHead.losses: predictions [N, C, Hp, Wp] at 1 / common_stride, targets [N, H, W] int64.  Returns
    {"loss_sem_seg": mean cross-entropy * loss_weight}.  On CUDA one forward and one backward launch sequence, and one host
    read of the status (a target outside [0, C) raises, as the reference does)."""
    return {"loss_sem_seg": _loss(predictions, targets, common_stride, ignore_value, None, None) * loss_weight}


def deeplab_losses(predictions: Tensor, targets: Tensor, common_stride: int, ignore_value: int, loss_weight: float,
                   loss_type: str, top_k_percent_pixels: float = 0.2,
                   weights: Optional[Tensor] = None) -> Dict[str, Tensor]:
    """DeepLabV3PlusHead.losses / DeepLabV3Head.losses (loss_type "cross_entropy" or "hard_pixel_mining" with
    top_k_percent_pixels 0.2) and PanopticDeepLabSemSegHead.losses (its loss_top_k and per-pixel `weights` [N, H, W]).
    Returns {"loss_sem_seg": loss * loss_weight}."""
    if loss_type == "cross_entropy":
        if weights is not None:
            raise ValueError("deeplab_losses: nn.CrossEntropyLoss takes no per-pixel weights")
        top_k = None
    elif loss_type == "hard_pixel_mining":
        top_k = float(top_k_percent_pixels)
    else:
        raise ValueError("Unexpected loss type: %s" % loss_type)
    return {"loss_sem_seg": _loss(predictions, targets, common_stride, ignore_value, top_k, weights) * loss_weight}
