"""mask_rcnn_loss -- mask-head training targets + loss in one kernel per image (SURVEY 8f-4).

Same value as detectron2/modeling/roi_heads/mask_head.py:33-112 (`mask_rcnn_loss`): for every sampled foreground proposal the
ground-truth bitmask is cropped to the proposal box and resized to the mask-head resolution (BitMasks.crop_and_resize,
structures/masks.py:193-224: RoIAlign, sampling_ratio 0, aligned, >= 0.5), the logits of the proposal's class are gathered
and `binary_cross_entropy_with_logits(..., reduction="mean")` is taken over all proposals of the batch.

Mechanism: the reference indexes the image's BitMasks by the matched ground-truth index (K x H x W bytes per image, e.g.
136 MB for 128 proposals of an 800 x 1333 image), converts them to fp32, pools, thresholds, gathers, reduces.  Here one CTA
per proposal samples the matched ground-truth mask straight from the [G, H, W] byte tensor (`mask_index`), and writes the
0/1 target and the proposal's loss sum; the backward writes the full logits gradient (zero off the class channel).
"""
import ctypes as C
from typing import List, Optional, Tuple, Union

import torch

from . import _C
from ._C import check, ptr, stream_ptr
from .polygon_masks import PackedPolygons, batch_mask_index

Tensor = torch.Tensor

__all__ = ["mask_rcnn_loss", "mask_loss_per_roi", "mask_loss_polygons"]


@torch.library.custom_op("d2b200::mask_loss", mutates_args=(), device_types="cuda")
def mask_loss_per_roi(logits: Tensor, gt_masks: Tensor, boxes: Tensor, mask_index: Optional[Tensor],
                      classes: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """One image.  logits [K,C,S,S]; gt_masks [G,H,W] bool / uint8 / float (nonzero = 1); boxes [K,4]; mask_index [K]
    (None: proposal k <-> mask k); classes [K] (None: class-agnostic).  Returns (loss sum per proposal [K] fp32, targets
    [K,S,S] bool)."""
    _C.require_cuda(logits, gt_masks, boxes, mask_index, classes)
    if logits.dim() != 4 or logits.shape[2] != logits.shape[3]:
        raise RuntimeError("mask_loss: logits must be K x C x S x S")
    lg = logits.to(dtype=torch.float32).contiguous()
    k, c, s, _ = lg.shape
    gm = gt_masks.contiguous()
    gm = (gm if gm.dtype == torch.bool else gm != 0).view(torch.uint8)  # any nonzero value is 1, as BitMasks reads it
    if gm.dim() != 3 or boxes.shape != (k, 4):
        raise RuntimeError("mask_loss: gt_masks must be G x H x W and boxes K x 4")
    bx = boxes.to(dtype=torch.float32).contiguous()
    mi = None if mask_index is None else mask_index.to(dtype=torch.int64).contiguous()
    cl = None if classes is None else classes.to(dtype=torch.int64).contiguous()
    loss = torch.zeros((k,), dtype=torch.float32, device=lg.device)
    targets = torch.zeros((k, s, s), dtype=torch.bool, device=lg.device)
    if k:
        with torch.cuda.device(lg.device):
            check(_C.lib().d2b_mask_loss_forward(ptr(lg), k, c, s, ptr(gm), gm.shape[0], gm.shape[1], gm.shape[2], ptr(bx),
                                                 ptr(mi), ptr(cl), ptr(loss), ptr(targets), stream_ptr(lg.device)),
                  "mask_loss_forward")
    return loss, targets


@mask_loss_per_roi.register_fake
def _(logits, gt_masks, boxes, mask_index, classes):
    k, s = logits.shape[0], logits.shape[2]
    return logits.new_empty((k,), dtype=torch.float32), logits.new_empty((k, s, s), dtype=torch.bool)


@torch.library.custom_op("d2b200::mask_loss_backward", mutates_args=(), device_types="cuda")
def mask_loss_backward(logits: Tensor, targets: Tensor, classes: Optional[Tensor], grad_loss: Tensor) -> Tensor:
    lg = logits.to(dtype=torch.float32).contiguous()
    k, c, s, _ = lg.shape
    cl = None if classes is None else classes.to(dtype=torch.int64).contiguous()
    gs = grad_loss.to(dtype=torch.float32).contiguous()
    out = torch.empty_like(lg)
    if k:
        with torch.cuda.device(lg.device):
            check(_C.lib().d2b_mask_loss_backward(ptr(lg), k, c, s, ptr(targets.contiguous()), ptr(cl), ptr(gs), ptr(out),
                                                  stream_ptr(lg.device)), "mask_loss_backward")
    return out


@mask_loss_backward.register_fake
def _(logits, targets, classes, grad_loss):
    return torch.empty_like(logits, dtype=torch.float32)


def _ml_setup(ctx, inputs, output):
    logits, gt_masks, boxes, mask_index, classes = inputs
    ctx.save_for_backward(logits, output[1], classes)


def _ml_bwd(ctx, grad_loss, grad_targets):
    logits, targets, classes = ctx.saved_tensors
    return mask_loss_backward(logits, targets, classes, grad_loss).to(logits.dtype), None, None, None, None


mask_loss_per_roi.register_autograd(_ml_bwd, setup_context=_ml_setup)


@torch.library.custom_op("d2b200::mask_loss_polygons", mutates_args=(), device_types="cuda")
def mask_loss_polygons(logits: Tensor, coords: Tensor, poly_start: Tensor, inst_start: Tensor, boxes: Tensor,
                       mask_index: Optional[Tensor], classes: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
    """All images at once.  logits [K,C,S,S]; the packed polygons (polygon_masks.PackedPolygons); boxes [K,4]; mask_index
    [K] batch-wide instance index (None: proposal k <-> instance k; outside [0, G): all-zero target); classes [K] (None:
    class-agnostic).  Returns (loss sum per proposal [K] fp32, targets [K,S,S] bool), as mask_loss_per_roi with the
    targets of PolygonMasks.crop_and_resize."""
    _C.require_cuda(logits, coords, poly_start, inst_start, boxes, mask_index, classes)
    if logits.dim() != 4 or logits.shape[2] != logits.shape[3] or boxes.shape != (logits.shape[0], 4):
        raise RuntimeError("mask_loss_polygons: logits must be K x C x S x S and boxes K x 4")
    if not logits.shape[2] <= _C.POLYGON_MAX_S:
        raise RuntimeError("mask_loss_polygons: S must be at most %d" % _C.POLYGON_MAX_S)
    if (coords.dtype != torch.float64 or poly_start.dtype != torch.int32 or inst_start.dtype != torch.int32
            or coords.dim() != 2 or coords.shape[1] != 2):
        raise RuntimeError("mask_loss_polygons: expected coords [V, 2] float64, poly_start and inst_start int32")
    lg = logits.to(dtype=torch.float32).contiguous()
    k, c, s, _ = lg.shape
    bx = boxes.to(dtype=torch.float32).contiguous()
    mi = None if mask_index is None else mask_index.to(dtype=torch.int64).contiguous()
    cl = None if classes is None else classes.to(dtype=torch.int64).contiguous()
    cd, ps, ist = coords.contiguous(), poly_start.contiguous(), inst_start.contiguous()
    loss = torch.zeros((k,), dtype=torch.float32, device=lg.device)
    targets = torch.zeros((k, s, s), dtype=torch.bool, device=lg.device)
    if k:
        with torch.cuda.device(lg.device):
            check(_C.lib().d2b_mask_loss_polygons_forward(ptr(lg), k, c, s, ptr(cd), cd.shape[0], ptr(ps), ps.shape[0] - 1,
                                                          ptr(ist), ist.shape[0] - 1, ptr(bx), ptr(mi), ptr(cl), ptr(loss),
                                                          ptr(targets), stream_ptr(lg.device)),
                  "mask_loss_polygons_forward")
    return loss, targets


@mask_loss_polygons.register_fake
def _(logits, coords, poly_start, inst_start, boxes, mask_index, classes):
    k, s = logits.shape[0], logits.shape[2]
    return logits.new_empty((k,), dtype=torch.float32), logits.new_empty((k, s, s), dtype=torch.bool)


def _mlp_setup(ctx, inputs, output):
    logits, coords, poly_start, inst_start, boxes, mask_index, classes = inputs
    ctx.save_for_backward(logits, output[1], classes)


def _mlp_bwd(ctx, grad_loss, grad_targets):
    logits, targets, classes = ctx.saved_tensors
    return (mask_loss_backward(logits, targets, classes, grad_loss).to(logits.dtype),) + (None,) * 6


mask_loss_polygons.register_autograd(_mlp_bwd, setup_context=_mlp_setup)


def mask_rcnn_loss(pred_mask_logits: Tensor, gt_masks: Union[List[Tensor], PackedPolygons], proposal_boxes: List[Tensor],
                   gt_classes: Optional[List[Tensor]] = None, mask_index: Optional[List[Tensor]] = None):
    """pred_mask_logits [sum K_i, C, S, S] in image order; per image i: gt_masks[i] [G_i,H_i,W_i] bitmasks, proposal_boxes[i]
    [K_i,4], gt_classes[i] [K_i] (omit for a class-agnostic head, C == 1), mask_index[i] [K_i] matched ground-truth index
    (omit when gt_masks[i] already holds one mask per proposal, as the reference's Instances do).
    gt_masks may instead be the batch's polygons, packed by polygon_masks.pack_polygons (the reference's PolygonMasks):
    then every image's targets and losses come from one forward launch and one backward launch, without a host sync.
    Returns (loss, targets [sum K_i, S, S] bool) -- loss == mask_rcnn_loss of the reference (mask_head.py:112)."""
    total = pred_mask_logits.shape[0]
    if total == 0:
        return pred_mask_logits.sum() * 0, pred_mask_logits.new_zeros((0,) + tuple(pred_mask_logits.shape[2:]), dtype=torch.bool)
    s = pred_mask_logits.shape[2]
    if isinstance(gt_masks, PackedPolygons):
        dev = pred_mask_logits.device
        ks = [b.shape[0] for b in proposal_boxes]
        assert sum(ks) == total, "proposal counts do not match the logits"
        lo, tg = mask_loss_polygons(pred_mask_logits, gt_masks.coords, gt_masks.poly_start, gt_masks.inst_start,
                                    torch.cat(list(proposal_boxes)), batch_mask_index(gt_masks, ks, mask_index, dev),
                                    None if gt_classes is None else torch.cat(list(gt_classes)))
        return lo.sum() / float(total * s * s), tg
    k0, losses, targets = 0, [], []
    for i, boxes in enumerate(proposal_boxes):
        k = boxes.shape[0]
        lo, tg = mask_loss_per_roi(pred_mask_logits[k0:k0 + k], gt_masks[i], boxes,
                                   None if mask_index is None else mask_index[i],
                                   None if gt_classes is None else gt_classes[i])
        losses.append(lo)
        targets.append(tg)
        k0 += k
    assert k0 == total, "proposal counts do not match the logits"
    return torch.cat(losses).sum() / float(total * s * s), torch.cat(targets)
