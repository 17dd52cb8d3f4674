"""FCOS training targets, losses and inference (detectron2/modeling/meta_arch/fcos.py) on the library's kernels.

  * `fcos_label_anchors_fixed` / `fcos_label_anchors` -- FCOS._match_anchors + label_anchors (fcos.py:97-191): centre
    sampling, the inside test and the per-level scale range, the smallest-area GT per point.  `d2b_fcos_assign` does all
    images in one launch (one thread per point, the GT boxes staged in shared memory); the reference builds several
    [G, R, 4] tensors per image.
  * `fcos_losses_fixed` / `fcos_losses` -- FCOS.losses + compute_ctrness_targets (fcos.py:193-251): the focal loss, the
    GIoU of Box2BoxTransformLinear's decode and the centerness BCE, on the dense loss kernel (`d2b200::dense_loss`), read in
    place from the per-level predictions, normalised by the EMA of the positive count (initial value 300).
  * `fcos_inference_fixed` / `fcos_inference` -- FCOS.forward_inference (fcos.py:253-301): scores
    sqrt(sigmoid(logits) * sigmoid(centerness)) by torch's elementwise ops, then RetinaNet's batched selection
    (dense_inference.py) with the linear decode.

The `_fixed` forms take padded GT tensors, return device tensors only, make no host read and can be captured in a CUDA graph.
The reference-shaped wrappers take per-image lists, make one host read and raise where the reference asserts.  CPU tensors
take the torch restatements (`_*_host`), which the tests pin to the fixture taken from the reference and run on CUDA tensors
as the reference the kernels are compared against.
"""
import ctypes as C
from typing import List, Optional, Sequence, Tuple, Union

import torch
from torch.nn import functional as F

from . import _C
from ._C import check, ptr, stream_ptr
from .dense_inference import apply_deltas_linear, dense_detector_inference, dense_detector_inference_fixed
from .losses import _ema_update, _giou_loss, _raise_status, _sigmoid_focal_loss, _stack, dense_loss_op
from .matching import _pad

Tensor = torch.Tensor

__all__ = ["fcos_label_anchors", "fcos_label_anchors_fixed", "fcos_losses", "fcos_losses_fixed", "fcos_inference",
           "fcos_inference_fixed", "fcos_assign_op"]

_EMA_INIT = 300.0  # FCOS.losses: self._ema_update("loss_normalizer", ..., 300)


def _levels(anchors: Union[Tensor, Sequence[Tensor]], level_counts: Optional[Sequence[int]]):
    if isinstance(anchors, Tensor):
        if level_counts is None:
            raise ValueError("fcos: pass level_counts with concatenated anchors (or the per-level list)")
        return anchors, [int(c) for c in level_counts]
    return torch.cat(list(anchors), dim=0), [int(a.shape[0]) for a in anchors]


# ---- assignment ------------------------------------------------------------------------------------------------------
@torch.library.custom_op("d2b200::fcos_assign", mutates_args=(), device_types="cuda")
def fcos_assign_op(anchors: Tensor, level_counts: List[int], gt_boxes: Tensor, gt_count: Tensor, gt_classes: Tensor,
                   num_classes: int, center_sampling_radius: float) -> Tuple[Tensor, Tensor, Tensor]:
    """anchors [R, 4] (levels concatenated, R = sum level_counts), gt_boxes [N, Gmax, 4], gt_count [N] int64, gt_classes
    [N, Gmax] int64.  Returns (labels [N, R] int64, matched_gt_boxes [N, R, 4] fp32, matches [N, R] int64, -1 unmatched)."""
    _C.require_cuda(anchors, gt_boxes, gt_count, gt_classes)
    n, gmax = gt_boxes.shape[0], gt_boxes.shape[1]
    r = sum(level_counts)
    if anchors.shape != (r, 4) or gt_boxes.shape != (n, gmax, 4) or gt_count.shape != (n,) or \
            gt_classes.shape != (n, gmax):
        raise ValueError("fcos_assign: anchors [R, 4], gt_boxes [N, Gmax, 4], gt_count [N], gt_classes [N, Gmax]")
    dev = anchors.device
    an = anchors.float().contiguous()
    gt = gt_boxes.float().contiguous()
    cnt = gt_count.to(torch.int64).contiguous()
    cls = gt_classes.to(torch.int64).contiguous()
    matches = torch.empty((n, r), dtype=torch.int64, device=dev)
    labels = torch.empty((n, r), dtype=torch.int64, device=dev)
    boxes = torch.empty((n, r, 4), dtype=torch.float32, device=dev)
    lc = (C.c_int * max(len(level_counts), 1))(*level_counts)
    with torch.cuda.device(dev):
        check(_C.lib().d2b_fcos_assign(ptr(an), lc, len(level_counts), ptr(gt), ptr(cnt), n, gmax, ptr(cls),
                                       int(num_classes), float(center_sampling_radius), ptr(matches), ptr(labels),
                                       ptr(boxes), stream_ptr(dev)), "fcos_assign")
    return labels, boxes, matches


@fcos_assign_op.register_fake
def _(anchors, level_counts, gt_boxes, gt_count, gt_classes, num_classes, center_sampling_radius):
    n, r = gt_boxes.shape[0], anchors.shape[0]
    return (anchors.new_empty((n, r), dtype=torch.int64), anchors.new_empty((n, r, 4), dtype=torch.float32),
            anchors.new_empty((n, r), dtype=torch.int64))


def fcos_label_anchors_fixed(anchors, gt_boxes: Tensor, gt_count: Tensor, gt_classes: Tensor, *, num_classes: int,
                             center_sampling_radius: float = 1.5, level_counts: Optional[Sequence[int]] = None):
    """FCOS.label_anchors on padded device tensors (CUDA only, no host read, capturable in a CUDA graph).
    anchors: per-level list of [R_l, 4] point boxes (or [R, 4] with level_counts); gt_boxes [N, Gmax, 4] with gt_count [N]
    (rows past the count are never read), gt_classes [N, Gmax].  Returns (gt_labels [N, R] int64, matched_gt_boxes
    [N, R, 4], matches [N, R] int64, -1 unmatched)."""
    an, counts = _levels(anchors, level_counts)
    return fcos_assign_op(an, counts, gt_boxes, gt_count, gt_classes, int(num_classes), float(center_sampling_radius))


def fcos_label_anchors(anchors, gt_boxes: List[Tensor], gt_classes: List[Tensor], *, num_classes: int,
                       center_sampling_radius: float = 1.5, level_counts: Optional[Sequence[int]] = None):
    """FCOS.label_anchors (fcos.py:153-191) with per-image lists of GT boxes [G_i, 4] and classes [G_i].  Returns
    (gt_labels, matched_gt_boxes) as per-image lists, as the reference."""
    an, counts = _levels(anchors, level_counts)
    if not an.is_cuda:
        return _fcos_label_anchors_host(an, counts, gt_boxes, gt_classes, num_classes, center_sampling_radius)[:2]
    gt, cnt = _pad(list(gt_boxes), 4, an.device)
    cls = torch.zeros(gt.shape[:2], dtype=torch.int64, device=an.device)
    for i, c in enumerate(gt_classes):
        cls[i, :len(c)] = c.to(an.device)
    labels, boxes, _ = fcos_assign_op(an, counts, gt, cnt, cls, int(num_classes), float(center_sampling_radius))
    return list(labels.unbind(0)), list(boxes.unbind(0))


# ---- losses ----------------------------------------------------------------------------------------------------------
def fcos_losses_fixed(anchors, pred_logits: List[Tensor], gt_labels, pred_anchor_deltas: List[Tensor], gt_boxes,
                      pred_centerness: List[Tensor], loss_normalizer: Tensor, *, num_classes: int,
                      focal_loss_alpha: float = 0.25, focal_loss_gamma: float = 2.0):
    """FCOS.losses on device tensors (CUDA only, no host read, capturable in a CUDA graph).
    pred_logits[l] [N, R_l, K], pred_anchor_deltas[l] [N, R_l, 4], pred_centerness[l] [N, R_l] or [N, R_l, 1];
    gt_labels [N, R] int64 and gt_boxes [N, R, 4] (fcos_label_anchors_fixed's).  loss_normalizer: caller-held fp64 [1]
    tensor holding the EMA of DenseDetector._ema_update (set it to 300 before the first call); it is updated in place as
    retinanet_losses_fixed's.  Returns (losses {"loss_fcos_cls", "loss_fcos_loc", "loss_fcos_ctr"}, num_pos, status)."""
    an = anchors if isinstance(anchors, Tensor) else torch.cat(list(anchors), dim=0)
    sums, counts, status = dense_loss_op(list(pred_logits), list(pred_anchor_deltas), list(pred_centerness), an,
                                         _stack(gt_boxes), _stack(gt_labels), int(num_classes), False,
                                         float(focal_loss_gamma), float(focal_loss_alpha), 0.0, _C.LOSS_LINEAR_GIOU,
                                         0.0, None)
    num_pos, _ = counts.unbind(0)
    cls, reg, ctr = (sums * _ema_update(loss_normalizer, num_pos, "fcos_losses_fixed")).unbind(0)
    return {"loss_fcos_cls": cls, "loss_fcos_loc": reg, "loss_fcos_ctr": ctr}, num_pos, status


def fcos_losses(anchors, pred_logits: List[Tensor], gt_labels: List[Tensor], pred_anchor_deltas: List[Tensor],
                gt_boxes: List[Tensor], pred_centerness: List[Tensor], *, num_classes: int,
                loss_normalizer: Optional[float] = None, focal_loss_alpha: float = 0.25, focal_loss_gamma: float = 2.0):
    """FCOS.losses (fcos.py:193-238) with the `self` attributes as arguments; loss_normalizer is the previous EMA value
    (None: the first call, 300).  Returns (losses, num_pos_anchors, the new normaliser as a Python float).  One host read."""
    an = anchors if isinstance(anchors, Tensor) else torch.cat(list(anchors), dim=0)
    old = _EMA_INIT if loss_normalizer is None else float(loss_normalizer)
    if not an.is_cuda:
        return _fcos_losses_host(an, pred_logits, gt_labels, pred_anchor_deltas, gt_boxes, pred_centerness, num_classes,
                                 old, focal_loss_alpha, focal_loss_gamma)
    ema = torch.tensor([old], dtype=torch.float64).to(an.device)
    losses, num_pos, status = fcos_losses_fixed(an, pred_logits, gt_labels, pred_anchor_deltas, gt_boxes, pred_centerness,
                                                ema, num_classes=num_classes, focal_loss_alpha=focal_loss_alpha,
                                                focal_loss_gamma=focal_loss_gamma)
    st, p = torch.stack([status.to(torch.int64), num_pos]).tolist()
    _raise_status(st, "Box2BoxTransformLinear")
    return losses, p, old * 0.9 + max(p, 1) * (1 - 0.9)


# ---- inference -------------------------------------------------------------------------------------------------------
def _scores(pred_logits: List[Tensor], pred_centerness: List[Tensor]) -> List[Tensor]:
    """torch.sqrt(x.sigmoid_() * y.sigmoid_()) of fcos.py:269, all images at once (elementwise: the same bits)."""
    out = []
    for x, y in zip(pred_logits, pred_centerness):
        y = y.reshape(x.shape[0], x.shape[1], 1)
        out.append(torch.sqrt(x.sigmoid() * y.sigmoid()))
    return out


def fcos_inference_fixed(anchors: List[Tensor], pred_logits: List[Tensor], pred_anchor_deltas: List[Tensor],
                         pred_centerness: List[Tensor], num_images: int, test_score_thresh: float = 0.2,
                         test_topk_candidates: int = 1000, test_nms_thresh: float = 0.6,
                         max_detections_per_image: int = 100):
    """FCOS.forward_inference after _transpose_dense_predictions, sync-free (CUDA only): (boxes [N, D, 4], scores [N, D],
    classes [N, D], counts [N]) with D = max_detections_per_image, as dense_detector_inference_fixed."""
    return dense_detector_inference_fixed(list(anchors), _scores(pred_logits, pred_centerness), list(pred_anchor_deltas),
                                          num_images, test_score_thresh, test_topk_candidates, test_nms_thresh,
                                          max_detections_per_image, transform="linear")


def fcos_inference(anchors: List[Tensor], pred_logits: List[Tensor], pred_anchor_deltas: List[Tensor],
                   pred_centerness: List[Tensor], image_sizes: List[Tuple[int, int]], test_score_thresh: float = 0.2,
                   test_topk_candidates: int = 1000, test_nms_thresh: float = 0.6, max_detections_per_image: int = 100):
    """FCOS.forward_inference (fcos.py:253-301): pred_logits[l] (N, R_l, K) raw logits, pred_anchor_deltas[l] (N, R_l, 4),
    pred_centerness[l] (N, R_l, 1) raw logits.  Returns one `Detections` per image; the defaults are FCOS's."""
    return dense_detector_inference(list(anchors), _scores(pred_logits, pred_centerness), list(pred_anchor_deltas),
                                    image_sizes, test_score_thresh, test_topk_candidates, test_nms_thresh,
                                    max_detections_per_image, transform="linear")


# ---- torch restatement (CPU tensors; the reference of the GPU tests) --------------------------------------------------
def _match_quality_host(anchors: Tensor, level_counts: Sequence[int], gt: Tensor, radius: float) -> Tensor:
    """FCOS._match_anchors (fcos.py:97-151): the [G, R] quality matrix."""
    centers = (anchors[:, :2] + anchors[:, 2:]) / 2
    sizes = anchors[:, 2] - anchors[:, 0]
    lower = sizes * 4
    lower[: level_counts[0]] = 0
    upper = sizes * 8
    upper[-level_counts[-1]:] = float("inf")
    gt_centers = (gt[:, :2] + gt[:, 2:]) / 2
    dists = (centers[None, :, :] - gt_centers[:, None, :]).abs_()
    q = dists.max(dim=2).values < float(radius) * sizes[None, :]
    x, y = centers.unsqueeze(dim=2).unbind(dim=1)
    x0, y0, x1, y1 = gt.unsqueeze(dim=0).unbind(dim=2)
    pd = torch.stack([x - x0, y - y0, x1 - x, y1 - y], dim=2).permute(1, 0, 2)
    q &= pd.min(dim=2).values > 0
    pd = pd.max(dim=2).values
    q &= (pd > lower[None, :]) & (pd < upper[None, :])
    areas = (gt[:, 2] - gt[:, 0]) * (gt[:, 3] - gt[:, 1])
    q = q.to(torch.float32)
    q *= 1e8 - areas[:, None]
    return q


def _fcos_label_anchors_host(anchors: Tensor, level_counts: Sequence[int], gt_boxes: List[Tensor],
                             gt_classes: List[Tensor], num_classes: int, radius: float = 1.5):
    """FCOS.label_anchors (fcos.py:153-191).  Returns (gt_labels, matched_gt_boxes, matches) per-image lists."""
    labels, boxes, matches = [], [], []
    for gt, cls in zip(gt_boxes, gt_classes):
        if len(gt) > 0:
            quality, idx = _match_quality_host(anchors, level_counts, gt, radius).max(dim=0)
            idx[quality < 1e-5] = -1
            boxes.append(gt[idx.clip(min=0)])
            lab = cls[idx.clip(min=0)]
            lab[idx < 0] = num_classes
            labels.append(lab)
            matches.append(idx)
        else:
            boxes.append(torch.zeros_like(anchors))
            labels.append(torch.full((len(anchors),), num_classes, dtype=torch.long, device=anchors.device))
            matches.append(torch.full((len(anchors),), -1, dtype=torch.long, device=anchors.device))
    return labels, boxes, matches


def _get_deltas_linear(src: Tensor, tgt: Tensor) -> Tensor:
    """Box2BoxTransformLinear(normalize_by_size=True).get_deltas (box_regression.py:243-273)."""
    cx = 0.5 * (src[:, 0] + src[:, 2])
    cy = 0.5 * (src[:, 1] + src[:, 3])
    d = torch.stack((cx - tgt[:, 0], cy - tgt[:, 1], tgt[:, 2] - cx, tgt[:, 3] - cy), dim=1)
    sw = src[:, 2] - src[:, 0]
    sh = src[:, 3] - src[:, 1]
    return d / torch.stack([sw, sh, sw, sh], dim=1)


def _ctrness_targets_host(anchors: Tensor, gt_boxes: List[Tensor]) -> Tensor:
    """FCOS.compute_ctrness_targets (fcos.py:240-251)."""
    reg = torch.stack([_get_deltas_linear(anchors, m) for m in gt_boxes], dim=0)
    if len(reg) == 0:
        return reg.new_zeros(len(reg))
    lr = reg[:, :, [0, 2]]
    tb = reg[:, :, [1, 3]]
    return torch.sqrt((lr.min(dim=-1)[0] / lr.max(dim=-1)[0]) * (tb.min(dim=-1)[0] / tb.max(dim=-1)[0]))


def _fcos_losses_host(anchors: Tensor, pred_logits, gt_labels, pred_anchor_deltas, gt_boxes, pred_centerness, num_classes,
                      old, alpha, gamma):
    """FCOS.losses (fcos.py:193-238) with the previous EMA value `old`; rows labelled -1 are left out of the
    classification sum (the reference's one_hot rejects them).  Returns (losses, num_pos, normalizer)."""
    gt_labels = _stack(gt_labels)
    valid = gt_labels >= 0
    pos_mask = valid & (gt_labels != num_classes)
    num_pos = int(pos_mask.sum().item())
    normalizer = old * 0.9 + max(num_pos, 1) * (1 - 0.9)
    target = F.one_hot(gt_labels[valid], num_classes=num_classes + 1)[:, :-1]
    loss_cls = _sigmoid_focal_loss(torch.cat(list(pred_logits), dim=1)[valid], target.to(pred_logits[0].dtype), alpha,
                                   gamma)
    boxes = torch.stack([apply_deltas_linear(k, anchors) for k in torch.cat(list(pred_anchor_deltas), dim=1)])
    loss_loc = _giou_loss(boxes[pos_mask], _stack(gt_boxes)[pos_mask])
    ctr_t = _ctrness_targets_host(anchors, list(gt_boxes))
    n, r = gt_labels.shape
    pred_ctr = torch.cat([c.reshape(n, -1) for c in pred_centerness], dim=1)
    loss_ctr = F.binary_cross_entropy_with_logits(pred_ctr[pos_mask], ctr_t[pos_mask], reduction="sum")
    return ({"loss_fcos_cls": loss_cls / normalizer, "loss_fcos_loc": loss_loc / normalizer,
             "loss_fcos_ctr": loss_ctr / normalizer}, num_pos, normalizer)
