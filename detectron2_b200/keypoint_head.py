"""Keypoint R-CNN head: heatmap decoding for inference and the keypoint loss for training, on two native entry points.

  * `heatmaps_to_keypoints` / `keypoint_rcnn_inference` -- detectron2/structures/keypoints.py:164-235 and
    modeling/roi_heads/keypoint_head.py:99-132.  The reference loops over the detections: one host sync
    (int(heights_ceil[i])), a materialised K x ceil(h) x ceil(w) bicubic map and about ten small launches per detection.
    Here `d2b_keypoints_from_heatmaps` evaluates the bicubic maps on the fly in pixel tiles spread over the whole GPU, with
    no host sync (three launches, capturable in a CUDA graph).
  * `keypoint_rcnn_loss` / `keypoint_rcnn_loss_fixed` -- modeling/roi_heads/keypoint_head.py:40-96 (the per-image
    Keypoints.to_heatmap loop, `nonzero()` host sync, gather of the valid rows, cross_entropy).  Here one launch computes the
    heatmap targets of every proposal of the batch and the per-keypoint cross-entropy; the backward writes the full logits
    gradient.  The normalizer "number of valid keypoints" stays on the device.
  * `keypoints_to_heatmap` -- the training targets alone (structures/keypoints.py:105-161).

CPU tensors take `_heatmaps_to_keypoints_host` / `_keypoint_rcnn_loss_host`, the same computation written with torch ops
(as fast_rcnn_inference does); run on CUDA tensors they are the reference the GPU tests compare the kernels against.
The containers (`Instances`, `Keypoints`, `Boxes`) are out of scope: tensors and per-image lists are used.
"""
from typing import List, Optional, Tuple

import torch
from torch.nn import functional as F

from . import _C
from ._C import check, ptr, stream_ptr

Tensor = torch.Tensor

__all__ = ["heatmaps_to_keypoints", "keypoint_rcnn_inference", "keypoint_rcnn_loss", "keypoint_rcnn_loss_fixed",
           "keypoints_to_heatmap", "keypoints_from_heatmaps_op", "keypoint_loss_op"]


# ---- inference ------------------------------------------------------------------------------------------------------
@torch.library.custom_op("d2b200::keypoints_from_heatmaps", mutates_args=(), device_types="cuda")
def keypoints_from_heatmaps_op(maps: Tensor, rois: Tensor) -> Tensor:
    """maps [R, K, S, S] logits, rois [R, 4] xyxy -> [R, K, 4] fp32 (x, y, logit, score)."""
    _C.require_cuda(maps, rois)
    if maps.dim() != 4 or maps.shape[2] != maps.shape[3] or rois.shape != (maps.shape[0], 4):
        raise RuntimeError("keypoints_from_heatmaps: maps must be R x K x S x S and rois R x 4")
    m = maps.to(dtype=torch.float32).contiguous()
    r, k, s, _ = m.shape
    bx = rois.to(dtype=torch.float32).contiguous()
    out = torch.empty((r, k, 4), dtype=torch.float32, device=m.device)
    if r:
        lib = _C.lib()
        ws_bytes = lib.d2b_keypoints_workspace_bytes(r, k)
        ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=m.device)
        with torch.cuda.device(m.device):
            check(lib.d2b_keypoints_from_heatmaps(ptr(m), r, k, s, ptr(bx), ptr(out), ptr(ws), ws_bytes,
                                                  stream_ptr(m.device)), "keypoints_from_heatmaps")
    return out


@keypoints_from_heatmaps_op.register_fake
def _(maps, rois):
    return maps.new_empty((maps.shape[0], maps.shape[1], 4), dtype=torch.float32)


def _heatmaps_to_keypoints_host(maps: Tensor, rois: Tensor) -> Tensor:
    """Per ROI: bicubic resize of the K maps to (ceil(h), ceil(w)), spatial argmax, score of the argmax normalised over the
    S x S map -- the reference's operations in the reference's order (one host read of all output sizes up front)."""
    x0, y0 = rois[:, 0], rois[:, 1]
    w = (rois[:, 2] - rois[:, 0]).clamp(min=1)
    h = (rois[:, 3] - rois[:, 1]).clamp(min=1)
    w_ceil, h_ceil = w.ceil(), h.ceil()
    corr_w, corr_h = w / w_ceil, h / h_ceil
    r, k = maps.shape[:2]
    out = maps.new_zeros(r, k, 4)
    sizes = torch.stack([h_ceil, w_ceil], dim=1).tolist() if r else []
    kidx = torch.arange(k, device=maps.device)
    for i, (hi, wi) in enumerate(sizes):
        hi, wi = int(hi), int(wi)
        resized = F.interpolate(maps[[i]], size=(hi, wi), mode="bicubic", align_corners=False).reshape(k, hi * wi)
        top = resized.max(1).values
        pos = resized.argmax(1)
        norm = (maps[i] - top.view(k, 1, 1)).exp().sum((1, 2))
        val = resized[kidx, pos]
        xi = pos % wi
        yi = (pos - xi) // wi
        out[i, :, 0] = (xi.float() + 0.5) * corr_w[i] + x0[i]
        out[i, :, 1] = (yi.float() + 0.5) * corr_h[i] + y0[i]
        out[i, :, 2] = val
        out[i, :, 3] = (val - top).exp() / norm
    return out


def heatmaps_to_keypoints(maps: Tensor, rois: Tensor) -> Tensor:
    """Reference signature (structures/keypoints.py:164-235): maps [R, K, S, S] logits, rois [R, 4] xyxy -> [R, K, 4] with
    (x, y, logit, score).  On CUDA one native call without host synchronisation; S <= 241.

    Ties of the spatial argmax go to the first pixel in row-major order; a NaN in a resized map wins (first NaN, logit
    NaN), as torch.argmax / max on CUDA.  Half-precision maps are cast to fp32 first (the reference interpolates them in
    half precision), so parity with the reference holds for fp32 maps.  A box with a non-finite coordinate, or with more than
    2^32 pixels, gives a NaN row on CUDA (the reference raises in int()); CPU tensors follow the reference."""
    if not maps.is_cuda:
        return _heatmaps_to_keypoints_host(maps, rois)
    return keypoints_from_heatmaps_op(maps, rois)


def keypoint_rcnn_inference(pred_keypoint_logits: Tensor, pred_boxes: List[Tensor]) -> List[Tuple[Tensor, Tensor]]:
    """keypoint_head.py:99-132 without Instances: pred_keypoint_logits [R, K, S, S] of all images, pred_boxes[i] [n_i, 4].
    Returns per image (pred_keypoints [n_i, K, 3] with (x, y, score), pred_keypoint_heatmaps [n_i, K, S, S])."""
    logits = pred_keypoint_logits.detach()
    boxes = torch.cat([b.detach() for b in pred_boxes], dim=0) if len(pred_boxes) else logits.new_zeros((0, 4))
    results = heatmaps_to_keypoints(logits, boxes)[:, :, [0, 1, 3]]
    counts = [int(b.shape[0]) for b in pred_boxes]
    return list(zip(results.split(counts, dim=0), logits.split(counts, dim=0)))


# ---- training -------------------------------------------------------------------------------------------------------
def _loss_forward(logits: Optional[Tensor], keypoints: Tensor, boxes: Tensor, n: int, k: int, s: int):
    device = keypoints.device
    kp = keypoints.to(dtype=torch.float32).contiguous()
    bx = boxes.to(dtype=torch.float32).contiguous()
    if kp.shape != (n, k, 3) or bx.shape != (n, 4):
        raise RuntimeError("keypoint_loss: keypoints must be N x K x 3 and boxes N x 4")
    target = torch.empty((n, k), dtype=torch.int64, device=device)
    valid = torch.empty((n, k), dtype=torch.uint8, device=device)
    num_valid = torch.empty((), dtype=torch.int64, device=device)
    loss = None if logits is None else torch.empty((n, k), dtype=torch.float32, device=device)
    dt = 0 if logits is None else _C.DTYPE_CODE[logits.dtype]
    with torch.cuda.device(device):
        check(_C.lib().d2b_keypoint_loss_forward(ptr(logits), dt, n, k, s, ptr(kp), ptr(bx), ptr(target), ptr(valid),
                                                 ptr(loss), ptr(num_valid), stream_ptr(device)), "keypoint_loss_forward")
    return loss, target, valid, num_valid


def _loss_logits(logits: Tensor) -> Tensor:
    if logits.dim() != 4 or logits.shape[2] != logits.shape[3]:
        raise RuntimeError("keypoint_loss: logits must be N x K x S x S")
    return logits if logits.dtype in _C.DTYPE_CODE else logits.to(torch.float32)


@torch.library.custom_op("d2b200::keypoint_loss", mutates_args=(), device_types="cuda")
def keypoint_loss_op(logits: Tensor, keypoints: Tensor, boxes: Tensor) -> Tuple[Tensor, Tensor, Tensor, Tensor]:
    """logits [N, K, S, S] (fp32 / fp16 / bf16), keypoints [N, K, 3] matched ground truth (x, y, v), boxes [N, 4] proposals.
    Returns (loss_per_kp [N, K] fp32, target [N, K] int64, valid [N, K] uint8, num_valid [] int64)."""
    _C.require_cuda(logits, keypoints, boxes)
    lg = _loss_logits(logits).contiguous()
    n, k, s, _ = lg.shape
    return _loss_forward(lg, keypoints, boxes, n, k, s)


@keypoint_loss_op.register_fake
def _(logits, keypoints, boxes):
    n, k = logits.shape[:2]
    return (logits.new_empty((n, k), dtype=torch.float32), logits.new_empty((n, k), dtype=torch.int64),
            logits.new_empty((n, k), dtype=torch.uint8), logits.new_empty((), dtype=torch.int64))


@torch.library.custom_op("d2b200::keypoint_loss_backward", mutates_args=(), device_types="cuda")
def keypoint_loss_backward_op(logits: Tensor, target: Tensor, valid: Tensor, grad_loss: Tensor) -> Tensor:
    lg = _loss_logits(logits).contiguous()
    n, k, s, _ = lg.shape
    gs = grad_loss.to(dtype=torch.float32).contiguous()
    out = torch.empty_like(lg)
    if n:
        with torch.cuda.device(lg.device):
            check(_C.lib().d2b_keypoint_loss_backward(ptr(lg), _C.DTYPE_CODE[lg.dtype], n, k, s, ptr(target.contiguous()),
                                                      ptr(valid.contiguous()), ptr(gs), ptr(out), stream_ptr(lg.device)),
                  "keypoint_loss_backward")
    return out


@keypoint_loss_backward_op.register_fake
def _(logits, target, valid, grad_loss):
    return torch.empty_like(_loss_logits(logits))


def _kl_setup(ctx, inputs, output):
    ctx.save_for_backward(inputs[0], output[1], output[2])


def _kl_bwd(ctx, grad_loss, grad_target, grad_valid, grad_num_valid):
    logits, target, valid = ctx.saved_tensors
    return keypoint_loss_backward_op(logits, target, valid, grad_loss).to(logits.dtype), None, None


keypoint_loss_op.register_autograd(_kl_bwd, setup_context=_kl_setup)


def _cat(ts: List[Tensor], width: Tuple[int, ...], like: Tensor) -> Tensor:
    return torch.cat(ts, dim=0) if len(ts) else like.new_zeros((0,) + width, dtype=torch.float32)


def keypoint_rcnn_loss_fixed(pred_keypoint_logits: Tensor, gt_keypoints: List[Tensor], proposal_boxes: List[Tensor],
                             normalizer: Optional[float] = None) -> Tuple[Tensor, Tensor]:
    """Sync-free form of `keypoint_rcnn_loss` (CUDA tensors): returns (loss, num_valid) as device tensors.  Static shapes:
    capturable in a CUDA graph.  Without a valid keypoint the loss and the gradient are 0, also when a logit is NaN or
    infinite (the reference's pred.sum() * 0 is NaN then)."""
    k = pred_keypoint_logits.shape[1]
    kps = _cat(gt_keypoints, (k, 3), pred_keypoint_logits)
    boxes = _cat(proposal_boxes, (4,), pred_keypoint_logits)
    loss_per_kp, _, _, num_valid = keypoint_loss_op(pred_keypoint_logits, kps, boxes)
    total = loss_per_kp.sum()
    # without valid keypoints every row's loss and gradient is 0.  The reference's pred.sum() * 0 is also 0 then, except
    # when a logit is NaN or infinite, where it is NaN: here the loss stays 0 (no reduction over the logits only to carry it)
    if normalizer is None:
        return total / num_valid.clamp(min=1).to(total.dtype), num_valid
    return total / normalizer, num_valid


def keypoint_rcnn_loss(pred_keypoint_logits: Tensor, gt_keypoints: List[Tensor], proposal_boxes: List[Tensor],
                       normalizer: Optional[float] = None) -> Tensor:
    """keypoint_head.py:40-96 without Instances: pred_keypoint_logits [N, K, S, S] of all images (image order),
    gt_keypoints[i] [n_i, K, 3] the matched ground-truth keypoints of image i's proposals (Instances.gt_keypoints.tensor),
    proposal_boxes[i] [n_i, 4].  normalizer None: divide by the number of valid keypoints (read on the device).
    The reference's "kpts_num_skipped_batches" event-storage counter of a batch without valid keypoints is not kept.
    fp16 / bf16 logits are read in place with fp32 arithmetic (the reference's cross_entropy runs in fp32 under autocast);
    the gradient comes back in the logits' dtype."""
    if not pred_keypoint_logits.is_cuda:
        return _keypoint_rcnn_loss_host(pred_keypoint_logits, gt_keypoints, proposal_boxes, normalizer)
    return keypoint_rcnn_loss_fixed(pred_keypoint_logits, gt_keypoints, proposal_boxes, normalizer)[0]


def keypoints_to_heatmap(keypoints: Tensor, rois: Tensor, heatmap_size: int) -> Tuple[Tensor, Tensor]:
    """Keypoints.to_heatmap (structures/keypoints.py:105-161): keypoints [N, K, 3], rois [N, 4] -> (target [N, K] int64 =
    y * S + x of the keypoint's cell, 0 where not valid; valid [N, K] int64).  A NaN cell (a NaN coordinate, or 0 * inf
    at x1 of a subnormal-width box) is not valid: the reference's floor().long() gives INT64_MIN for NaN on CUDA (and on
    x86 CPUs)."""
    if not keypoints.is_cuda:
        return _keypoints_to_heatmap_host(keypoints, rois, heatmap_size)
    _C.require_cuda(rois)
    n, k = keypoints.shape[:2]
    if rois.numel() == 0:
        return rois.new_zeros((0,), dtype=torch.int64), rois.new_zeros((0,), dtype=torch.int64)
    _, target, valid, _ = _loss_forward(None, keypoints, rois, n, k, int(heatmap_size))
    return target, valid.to(torch.int64)


def _keypoints_to_heatmap_host(keypoints: Tensor, rois: Tensor, heatmap_size: int) -> Tuple[Tensor, Tensor]:
    """The cell of every keypoint in its ROI's heatmap: floor((c - x1) * (S / (x2 - x1))), c == x2 -> S - 1."""
    if rois.numel() == 0:
        return rois.new().long(), rois.new().long()
    x, y = keypoints[..., 0], keypoints[..., 1]
    on_x2 = x == rois[:, 2][:, None]
    on_y2 = y == rois[:, 3][:, None]
    cx = ((x - rois[:, 0][:, None]) * (heatmap_size / (rois[:, 2] - rois[:, 0]))[:, None]).floor().long()
    cy = ((y - rois[:, 1][:, None]) * (heatmap_size / (rois[:, 3] - rois[:, 1]))[:, None]).floor().long()
    cx[on_x2] = heatmap_size - 1
    cy[on_y2] = heatmap_size - 1
    inside = (cx >= 0) & (cy >= 0) & (cx < heatmap_size) & (cy < heatmap_size)
    valid = (inside & (keypoints[..., 2] > 0)).long()
    return (cy * heatmap_size + cx) * valid, valid


def _keypoint_rcnn_loss_host(pred_keypoint_logits: Tensor, gt_keypoints: List[Tensor], proposal_boxes: List[Tensor],
                             normalizer: Optional[float] = None) -> Tensor:
    """Targets of every image, the valid rows gathered (host sync), cross-entropy summed and normalised."""
    s = pred_keypoint_logits.shape[2]
    targets, valids = [], []
    for kp, boxes in zip(gt_keypoints, proposal_boxes):
        if len(boxes) == 0:
            continue
        t, v = _keypoints_to_heatmap_host(kp, boxes, s)
        targets.append(t.view(-1))
        valids.append(v.view(-1))
    rows = torch.nonzero(torch.cat(valids).to(torch.uint8)).squeeze(1) if valids else None
    if rows is None or rows.numel() == 0:
        return pred_keypoint_logits.sum() * 0
    n, k, h, w = pred_keypoint_logits.shape
    flat = pred_keypoint_logits.view(n * k, h * w)
    loss = F.cross_entropy(flat[rows], torch.cat(targets)[rows], reduction="sum")
    return loss / (rows.numel() if normalizer is None else normalizer)
