"""Box-branch training losses of the RPN / RRPN, RetinaNet and Fast R-CNN heads on two native entry points.

  * `rpn_losses` / `rpn_losses_fixed` -- RPN.losses (proposal_generator/rpn.py:366-429), RRPN's with [R, 5] anchors:
    binary_cross_entropy_with_logits over the sampled anchors plus smooth-L1 box regression over the positive ones.
  * `retinanet_losses` / `retinanet_losses_fixed` -- RetinaNet.losses (meta_arch/retinanet.py:160-210): sigmoid focal loss
    over the valid anchors plus box regression, normalised by the EMA of the positive count (DenseDetector._ema_update).
  * `fast_rcnn_losses` / `fast_rcnn_losses_fixed` -- FastRCNNOutputLayers.losses / box_reg_loss and
    _log_classification_stats (roi_heads/fast_rcnn.py:88-115, 307-352, 424-463), for the standard, cascade and rotated heads.
  * FCOS.losses (meta_arch/fcos.py:193-251) is `dense_loss_op` with `LOSS_LINEAR_GIOU` and the centerness logits: the
    GIoU of the linear decode plus the centerness term; its Python surface is detectron2_b200/fcos.py.

The reference concatenates the levels, gathers the valid rows behind a boolean mask, builds an int64 one-hot target and
reads the host about ten times per step (.item() counts, get_deltas' assertion, nonzero).  Here `d2b_dense_loss_*` reads the
per-level logits in place (one read forward, one read and one write backward) and computes the box targets on the fly;
`d2b_frcnn_loss_*` runs one warp per proposal.  The `_fixed` forms return device tensors only (losses, counts, status),
have static shapes and can be captured in a CUDA graph; the reference-shaped wrappers make one host read per call, of the
status and the counts, and raise AssertionError where the reference asserts.

Regression loss types: "smooth_l1" and "giou" (axis-aligned boxes, as in the reference) run on the kernels.  "diou" and
"ciou" are not fused: the wrappers run the torch restatement below (`_*_host`) for them, on any device.  CPU tensors always
take the restatement, which the tests also run on CUDA tensors as the reference the kernels are compared against, and which
reproduces the fixture taken from the real reference functions.  Sigmoid-CE and the federated loss of FastRCNNOutputLayers
are not provided.
"""
import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
from torch.nn import functional as F

from . import _C
from ._C import check, ptr, stream_ptr
from .dense_inference import apply_deltas as _apply_deltas

Tensor = torch.Tensor

__all__ = ["rpn_losses", "rpn_losses_fixed", "retinanet_losses", "retinanet_losses_fixed", "fast_rcnn_losses",
           "fast_rcnn_losses_fixed", "dense_loss_op", "frcnn_loss_op"]

_SCALE_CLAMP = 4.135166556742356  # math.log(1000.0 / 16), box_regression.py:14


# ---- custom ops -----------------------------------------------------------------------------------------------------
def _pred(t: Tensor, dtype: torch.dtype) -> Tensor:
    """Contiguous, of the kernel's element type, 16-byte aligned (vector loads)."""
    t = t.to(dtype).contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _pred_dtype(t: Tensor) -> torch.dtype:
    return t.dtype if t.dtype in _C.DTYPE_CODE else torch.float32


def _c_weights(weights: Optional[Sequence[float]]):
    """The HOST weights array, or NULL for None (D2B_LOSS_LINEAR_GIOU reads no weights)."""
    return None if weights is None else (C.c_float * len(weights))(*[float(w) for w in weights])


def _dense_prepare(logits, deltas, ctr, anchors, gt_boxes, labels, num_classes, rpn):
    if len(logits) == 0 or len(logits) != len(deltas) or len(logits) > _C.MAX_LEVELS:
        raise ValueError("dense_loss: 1 to %d levels of logits and deltas" % _C.MAX_LEVELS)
    if len(ctr) not in (0, len(logits)):
        raise ValueError("dense_loss: no centerness, or one centerness tensor per level")
    dt = _pred_dtype(logits[0])
    xs = [_pred(x, dt) for x in logits]
    ds = [_pred(d, dt) for d in deltas]
    n, d = gt_boxes.shape[0], anchors.shape[-1]
    for x, dl in zip(xs, ds):
        if x.dim() != 3 or x.shape[0] != n or x.shape[2] != num_classes or dl.shape != (n, x.shape[1], d):
            raise ValueError("dense_loss: logits must be [N, R_l, K] and deltas [N, R_l, %d]" % d)
    cs = []
    for c, x in zip(ctr, xs):
        if c.shape not in ((n, x.shape[1]), (n, x.shape[1], 1)):
            raise ValueError("dense_loss: centerness must be [N, R_l] or [N, R_l, 1]")
        cs.append(c.reshape(n, x.shape[1]).to(dt).contiguous())
    r = sum(int(x.shape[1]) for x in xs)
    if anchors.shape != (r, d) or gt_boxes.shape != (n, r, d) or labels.shape != (n, r):
        raise ValueError("dense_loss: anchors [R, D], gt_boxes [N, R, D] and labels [N, R] with R = sum of R_l")
    lab = labels.to(torch.int8 if rpn else torch.int64).contiguous()
    return dt, xs, ds, cs, anchors.float().contiguous(), gt_boxes.float().contiguous(), lab


def _dense_levels(xs, ds, cs, gxs=None, gds=None, gcs=None):
    lv = _C.DenseLossLevels()
    lv.num_levels = len(xs)
    for l, (x, d) in enumerate(zip(xs, ds)):
        lv.logits[l], lv.deltas[l], lv.R[l] = x.data_ptr(), d.data_ptr(), int(x.shape[1])
        if gxs is not None:
            lv.grad_logits[l], lv.grad_deltas[l] = gxs[l].data_ptr(), gds[l].data_ptr()
    for l, c in enumerate(cs):
        lv.ctr[l] = c.data_ptr()
        if gcs is not None:
            lv.grad_ctr[l] = gcs[l].data_ptr()
    return lv


@torch.library.custom_op("d2b200::dense_loss", mutates_args=(), device_types="cuda")
def dense_loss_op(logits: List[Tensor], deltas: List[Tensor], ctr: List[Tensor], anchors: Tensor, gt_boxes: Tensor,
                  labels: Tensor, num_classes: int, rpn: bool, gamma: float, alpha: float, beta: float, loss_type: int,
                  scale_clamp: float, weights: Optional[List[float]]) -> Tuple[Tensor, Tensor, Tensor]:
    """Per level logits [N, R_l, K] and deltas [N, R_l, D] (fp32 / fp16 / bf16), anchors [R, D], matched gt_boxes
    [N, R, D], labels [N, R] (rpn: int8 {-1, 0, 1} and K = 1; else int64 classes with K = background).  ctr: empty, or
    with loss_type LOSS_LINEAR_GIOU (FCOS; weights None) the centerness logits [N, R_l] or [N, R_l, 1] of every level.
    Returns (sums [3] fp32: classification, regression, centerness; counts [2] int64: num_pos, num_neg; status [] int32)."""
    _C.require_cuda(anchors, gt_boxes, labels, *logits, *deltas, *ctr)
    dt, xs, ds, cs, an, gt, lab = _dense_prepare(logits, deltas, ctr, anchors, gt_boxes, labels, num_classes, rpn)
    dev = an.device
    n, d = gt.shape[0], an.shape[-1]
    lv = _dense_levels(xs, ds, cs)
    sums = torch.empty((3,), dtype=torch.float32, device=dev)
    counts = torch.empty((2,), dtype=torch.int64, device=dev)
    status = torch.empty((), dtype=torch.int32, device=dev)
    lib = _C.lib()
    code = _C.DTYPE_CODE[dt]
    ws_bytes = int(lib.d2b_dense_loss_workspace_bytes(C.byref(lv), n, num_classes, code))
    ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        check(lib.d2b_dense_loss_forward(C.byref(lv), n, num_classes, d, code, ptr(an), ptr(gt), ptr(lab),
                                         _C.LABELS_I8 if rpn else _C.LABELS_I64, float(gamma), float(alpha), float(beta),
                                         int(loss_type), float(scale_clamp), _c_weights(weights), ptr(sums), ptr(counts),
                                         ptr(status), ptr(ws), ws_bytes, stream_ptr(dev)), "dense_loss_forward")
    return sums, counts, status


@dense_loss_op.register_fake
def _(logits, deltas, ctr, anchors, gt_boxes, labels, num_classes, rpn, gamma, alpha, beta, loss_type, scale_clamp,
      weights):
    e = anchors.new_empty
    return e((3,), dtype=torch.float32), e((2,), dtype=torch.int64), e((), dtype=torch.int32)


@torch.library.custom_op("d2b200::dense_loss_backward", mutates_args=(), device_types="cuda")
def dense_loss_backward_op(logits: List[Tensor], deltas: List[Tensor], ctr: List[Tensor], anchors: Tensor,
                           gt_boxes: Tensor, labels: Tensor, num_classes: int, rpn: bool, gamma: float, alpha: float,
                           beta: float, loss_type: int, scale_clamp: float, weights: Optional[List[float]],
                           grad_sums: Tensor) -> List[Tensor]:
    """Gradients of every level's logits, then deltas, then centerness logits, in the inputs' dtypes and shapes."""
    dt, xs, ds, cs, an, gt, lab = _dense_prepare(logits, deltas, ctr, anchors, gt_boxes, labels, num_classes, rpn)
    dev = an.device
    gxs, gds, gcs = ([torch.empty_like(t) for t in ts] for ts in (xs, ds, cs))
    lv = _dense_levels(xs, ds, cs, gxs, gds, gcs)
    g = grad_sums.to(torch.float32).contiguous()
    with torch.cuda.device(dev):
        check(_C.lib().d2b_dense_loss_backward(C.byref(lv), gt.shape[0], num_classes, an.shape[-1], _C.DTYPE_CODE[dt],
                                               ptr(an), ptr(gt), ptr(lab), _C.LABELS_I8 if rpn else _C.LABELS_I64,
                                               float(gamma), float(alpha), float(beta), int(loss_type),
                                               float(scale_clamp), _c_weights(weights), ptr(g), stream_ptr(dev)),
              "dense_loss_backward")
    ins = list(logits) + list(deltas) + list(ctr)
    return [gr.to(x.dtype).reshape(x.shape) for gr, x in zip(gxs + gds + gcs, ins)]


@dense_loss_backward_op.register_fake
def _(logits, deltas, ctr, anchors, gt_boxes, labels, num_classes, rpn, gamma, alpha, beta, loss_type, scale_clamp,
      weights, grad_sums):
    return [torch.empty_like(t) for t in list(logits) + list(deltas) + list(ctr)]


def _dense_setup(ctx, inputs, output):
    logits, deltas, ctr, anchors, gt_boxes, labels = inputs[:6]
    ctx.save_for_backward(*logits, *deltas, *ctr, anchors, gt_boxes, labels)
    ctx.num_levels, ctx.num_ctr = len(logits), len(ctr)
    ctx.params = inputs[6:]


def _dense_bwd(ctx, g_sums, *_):
    saved = ctx.saved_tensors
    nl, nc = ctx.num_levels, ctx.num_ctr
    logits, deltas, ctr = list(saved[:nl]), list(saved[nl:2 * nl]), list(saved[2 * nl:2 * nl + nc])
    anchors, gt_boxes, labels = saved[2 * nl + nc:]
    grads = dense_loss_backward_op(logits, deltas, ctr, anchors, gt_boxes, labels, *ctx.params, g_sums)
    return (grads[:nl], grads[nl:2 * nl], grads[2 * nl:]) + (None,) * 11


dense_loss_op.register_autograd(_dense_bwd, setup_context=_dense_setup)


def _frcnn_prepare(scores, deltas, proposals, gt_boxes, gt_classes):
    r, k1 = scores.shape
    d = proposals.shape[-1]
    if scores.dim() != 2 or deltas.shape[0] != r or deltas.shape[1] not in (d, (k1 - 1) * d) or k1 < 2:
        raise ValueError("frcnn_loss: scores [R, K+1] and deltas [R, K*D] or [R, D]")
    if proposals.shape != (r, d) or gt_boxes.shape != (r, d) or gt_classes.shape != (r,):
        raise ValueError("frcnn_loss: proposal_boxes and gt_boxes [R, D], gt_classes [R]")
    dt = _pred_dtype(scores)
    return (dt, scores.to(dt).contiguous(), deltas.to(dt).contiguous(), proposals.float().contiguous(),
            gt_boxes.float().contiguous(), gt_classes.to(torch.int64).contiguous(), k1 - 1, deltas.shape[1] // d)


@torch.library.custom_op("d2b200::frcnn_loss", mutates_args=(), device_types="cuda")
def frcnn_loss_op(scores: Tensor, deltas: Tensor, proposals: Tensor, gt_boxes: Tensor, gt_classes: Tensor, beta: float,
                  loss_type: int, scale_clamp: float, weights: List[float]) -> Tuple[Tensor, Tensor, Tensor]:
    """scores [R, K+1], deltas [R, K*D] or [R, D] (fp32 / fp16 / bf16), proposals / gt_boxes [R, D], gt_classes [R].
    Returns (sums [2] fp32: cross-entropy sum, smooth-L1 sum; counts [4] int64: num_fg, num_accurate, fg_num_accurate,
    num_false_negative; status [] int32)."""
    _C.require_cuda(scores, deltas, proposals, gt_boxes, gt_classes)
    dt, sc, dl, pr, gt, cls, k, kreg = _frcnn_prepare(scores, deltas, proposals, gt_boxes, gt_classes)
    dev = sc.device
    r, d = sc.shape[0], pr.shape[-1]
    sums = torch.empty((2,), dtype=torch.float32, device=dev)
    counts = torch.empty((4,), dtype=torch.int64, device=dev)
    status = torch.empty((), dtype=torch.int32, device=dev)
    lib = _C.lib()
    ws_bytes = int(lib.d2b_frcnn_loss_workspace_bytes(r))
    ws = torch.empty((max(ws_bytes, 16),), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        check(lib.d2b_frcnn_loss_forward(ptr(sc), ptr(dl), r, k, kreg, d, _C.DTYPE_CODE[dt], ptr(pr), ptr(gt), ptr(cls),
                                         float(beta), int(loss_type), float(scale_clamp), _c_weights(weights), ptr(sums),
                                         ptr(counts), ptr(status), ptr(ws), ws_bytes, stream_ptr(dev)), "frcnn_loss_forward")
    return sums, counts, status


@frcnn_loss_op.register_fake
def _(scores, deltas, proposals, gt_boxes, gt_classes, beta, loss_type, scale_clamp, weights):
    e = scores.new_empty
    return e((2,), dtype=torch.float32), e((4,), dtype=torch.int64), e((), dtype=torch.int32)


@torch.library.custom_op("d2b200::frcnn_loss_backward", mutates_args=(), device_types="cuda")
def frcnn_loss_backward_op(scores: Tensor, deltas: Tensor, proposals: Tensor, gt_boxes: Tensor, gt_classes: Tensor,
                           beta: float, loss_type: int, scale_clamp: float, weights: List[float],
                           grad_sums: Tensor) -> Tuple[Tensor, Tensor]:
    dt, sc, dl, pr, gt, cls, k, kreg = _frcnn_prepare(scores, deltas, proposals, gt_boxes, gt_classes)
    dev = sc.device
    g = grad_sums.to(torch.float32).contiguous()
    gs, gd = torch.empty_like(sc), torch.empty_like(dl)
    if sc.shape[0]:
        with torch.cuda.device(dev):
            check(_C.lib().d2b_frcnn_loss_backward(ptr(sc), ptr(dl), sc.shape[0], k, kreg, pr.shape[-1], _C.DTYPE_CODE[dt],
                                                   ptr(pr), ptr(gt), ptr(cls), float(beta), int(loss_type),
                                                   float(scale_clamp), _c_weights(weights), ptr(g), ptr(gs), ptr(gd),
                                                   stream_ptr(dev)),
                  "frcnn_loss_backward")
    return gs.to(scores.dtype), gd.to(deltas.dtype)


@frcnn_loss_backward_op.register_fake
def _(scores, deltas, proposals, gt_boxes, gt_classes, beta, loss_type, scale_clamp, weights, grad_sums):
    return torch.empty_like(scores), torch.empty_like(deltas)


def _frcnn_setup(ctx, inputs, output):
    ctx.save_for_backward(*inputs[:5])
    ctx.params = inputs[5:]


def _frcnn_bwd(ctx, g_sums, *_):
    gs, gd = frcnn_loss_backward_op(*ctx.saved_tensors, *ctx.params, g_sums)
    return gs, gd, None, None, None, None, None, None, None


frcnn_loss_op.register_autograd(_frcnn_bwd, setup_context=_frcnn_setup)


# ---- sync-free forms ------------------------------------------------------------------------------------------------
def _stack(t: Union[Tensor, Sequence[Tensor]]) -> Tensor:
    return t if isinstance(t, Tensor) else torch.stack(list(t))


def _cat_anchors(anchors: Union[Tensor, Sequence[Tensor]]) -> Tensor:
    return anchors if isinstance(anchors, Tensor) else torch.cat(list(anchors), dim=0)


def _ema_update(loss_normalizer: Tensor, num_pos: Tensor, what: str) -> Tensor:
    """DenseDetector._ema_update on the caller-held fp64 [1] `loss_normalizer`, in place: old * 0.9 + max(num_pos, 1) *
    (1 - 0.9), in fp64 with separately rounded operations, as the Python float recurrence.  Returns the fp32 reciprocal of
    the new value: the reference divides by the normaliser as a Python float, and torch's CUDA kernel then multiplies by
    the fp32 reciprocal."""
    if loss_normalizer.dtype != torch.float64 or loss_normalizer.numel() != 1:
        raise ValueError("%s: loss_normalizer must be a float64 tensor with one element" % what)
    momentum = 0.9
    loss_normalizer.copy_(loss_normalizer * momentum + num_pos.clamp(min=1).to(torch.float64) * (1 - momentum))
    return torch.reciprocal(loss_normalizer.reshape(()).to(torch.float32))


def rpn_losses_fixed(anchors, pred_objectness_logits: List[Tensor], gt_labels, pred_anchor_deltas: List[Tensor],
                     gt_boxes, *, batch_size_per_image: int, smooth_l1_beta: float = 0.0,
                     box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0), box_reg_loss_type: str = "smooth_l1",
                     scale_clamp: float = _SCALE_CLAMP, loss_weight: Optional[Dict[str, float]] = None):
    """RPN.losses on device tensors (CUDA only, no host read, capturable in a CUDA graph).
    anchors [R, D] (or per-level list), pred_objectness_logits[l] [N, R_l], gt_labels [N, R] int8 (or a list of [R]),
    pred_anchor_deltas[l] [N, R_l, D], gt_boxes [N, R, D] (or a list).  D = 5 with five weights: RRPN.
    Returns (losses {"loss_rpn_cls", "loss_rpn_loc"}, num_pos_anchors, num_neg_anchors, status), all device tensors."""
    labels = _stack(gt_labels)
    n = labels.shape[0]
    sums, counts, status = dense_loss_op([x.unsqueeze(-1) for x in pred_objectness_logits], list(pred_anchor_deltas), [],
                                         _cat_anchors(anchors), _stack(gt_boxes), labels, 1, True, 0.0, -1.0,
                                         float(smooth_l1_beta), _fused_type(box_reg_loss_type), float(scale_clamp),
                                         [float(w) for w in box2box_weights])
    cls, reg, _ = (sums / (batch_size_per_image * n)).unbind(0)
    num_pos, num_neg = counts.unbind(0)
    lw = loss_weight or {}
    losses = {"loss_rpn_cls": cls, "loss_rpn_loc": reg}
    return {k: v * lw.get(k, 1.0) for k, v in losses.items()}, num_pos, num_neg, status


def retinanet_losses_fixed(anchors, pred_logits: List[Tensor], gt_labels, pred_anchor_deltas: List[Tensor], gt_boxes,
                           loss_normalizer: Tensor, *, num_classes: int, focal_loss_alpha: float = 0.25,
                           focal_loss_gamma: float = 2.0, smooth_l1_beta: float = 0.1,
                           box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0), box_reg_loss_type: str = "smooth_l1",
                           scale_clamp: float = _SCALE_CLAMP):
    """RetinaNet.losses on device tensors (CUDA only, no host read, capturable in a CUDA graph).
    pred_logits[l] [N, R_l, K], gt_labels [N, R] int64 (the `classes` of match_boxes_fixed), gt_boxes [N, R, 4].
    loss_normalizer: caller-held fp64 [1] tensor holding the EMA of DenseDetector._ema_update (set it to 100 before the
    first call); it is updated in place, old * 0.9 + max(num_pos, 1) * (1 - 0.9), in fp64 with separately rounded
    operations, as the Python float recurrence.  Returns (losses {"loss_cls", "loss_box_reg"}, num_pos_anchors, status)."""
    sums, counts, status = dense_loss_op(list(pred_logits), list(pred_anchor_deltas), [], _cat_anchors(anchors),
                                         _stack(gt_boxes), _stack(gt_labels), int(num_classes), False,
                                         float(focal_loss_gamma), float(focal_loss_alpha), float(smooth_l1_beta),
                                         _fused_type(box_reg_loss_type), float(scale_clamp),
                                         [float(w) for w in box2box_weights])
    num_pos, _ = counts.unbind(0)
    cls, reg, _ = (sums * _ema_update(loss_normalizer, num_pos, "retinanet_losses_fixed")).unbind(0)
    return {"loss_cls": cls, "loss_box_reg": reg}, num_pos, status


def fast_rcnn_losses_fixed(scores: Tensor, proposal_deltas: Tensor, proposal_boxes: Tensor, gt_boxes: Tensor,
                           gt_classes: Tensor, *, smooth_l1_beta: float = 0.0,
                           box2box_weights: Sequence[float] = (10.0, 10.0, 5.0, 5.0), box_reg_loss_type: str = "smooth_l1",
                           scale_clamp: float = _SCALE_CLAMP, loss_weight: Optional[Dict[str, float]] = None):
    """FastRCNNOutputLayers.losses on device tensors (CUDA only, no host read, capturable in a CUDA graph).
    scores [R, K+1], proposal_deltas [R, K*D] or [R, D], proposal_boxes / gt_boxes [R, D] (the proposals of all images
    concatenated), gt_classes [R] int64.  Cascade stages pass their stage's weights; D = 5 with five weights: rotated heads.
    Returns (losses {"loss_cls", "loss_box_reg"}, counts [4] int64 = (num_fg, num_accurate, fg_num_accurate,
    num_false_negative) of _log_classification_stats, status)."""
    sums, counts, status = frcnn_loss_op(scores, proposal_deltas, proposal_boxes, gt_boxes, gt_classes,
                                            float(smooth_l1_beta), _fused_type(box_reg_loss_type), float(scale_clamp),
                                            [float(w) for w in box2box_weights])
    # cross_entropy(mean) of no rows is the reference's scores.sum() * 0: a zero loss (the sum is 0 here)
    cls, reg = (sums / max(scores.shape[0], 1)).unbind(0)
    losses = {"loss_cls": cls, "loss_box_reg": reg}
    lw = loss_weight or {}
    return {k: v * lw.get(k, 1.0) for k, v in losses.items()}, counts, status


# ---- reference-shaped wrappers --------------------------------------------------------------------------------------
def _fused_type(loss_type: str) -> int:
    if loss_type not in _C.LOSS_TYPES:
        raise ValueError("box regression loss %r has no kernel (smooth_l1, giou); the reference-shaped wrappers run diou and "
                         "ciou through the torch restatement" % (loss_type,))
    return _C.LOSS_TYPES[loss_type]


def _use_kernels(loss_type: str, on_cuda: bool) -> bool:
    if loss_type not in ("smooth_l1", "giou", "diou", "ciou"):
        raise ValueError(f"Invalid dense box regression loss type '{loss_type}'")
    return on_cuda and loss_type in _C.LOSS_TYPES


def _raise_status(status: int, what: str):
    if status & _C.LOSS_STATUS_INVALID_CLASS:  # F.one_hot / cross_entropy reject such labels
        raise RuntimeError("class labels out of range [-1, num_classes]")
    if status & _C.LOSS_STATUS_INVALID_BOX:
        raise AssertionError("Input boxes to %s are not valid!" % what)
    if status & _C.LOSS_STATUS_INVALID_BOX_ORDER:
        raise AssertionError("bad box: x1 larger than x2 or y1 larger than y2")


def _transform_name(d: int) -> str:
    return "Box2BoxTransformRotated" if d == 5 else "Box2BoxTransform"


def rpn_losses(anchors, pred_objectness_logits: List[Tensor], gt_labels: List[Tensor], pred_anchor_deltas: List[Tensor],
               gt_boxes: List[Tensor], *, batch_size_per_image: int, box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0),
               scale_clamp: float = _SCALE_CLAMP, box_reg_loss_type: str = "smooth_l1", smooth_l1_beta: float = 0.0,
               loss_weight: Optional[Dict[str, float]] = None):
    """RPN.losses (rpn.py:366-429) with the `self` attributes as arguments.  Returns (losses, {"num_pos_anchors",
    "num_neg_anchors"} as Python ints, the batch totals the reference logs divided by the image count).  One host read."""
    anchors = _cat_anchors(anchors)
    if not _use_kernels(box_reg_loss_type, anchors.is_cuda):
        return _rpn_losses_host(anchors, pred_objectness_logits, gt_labels, pred_anchor_deltas, gt_boxes,
                                batch_size_per_image, box2box_weights, scale_clamp, box_reg_loss_type, smooth_l1_beta,
                                loss_weight)
    losses, num_pos, num_neg, status = rpn_losses_fixed(anchors, pred_objectness_logits, gt_labels, pred_anchor_deltas,
                                                        gt_boxes, batch_size_per_image=batch_size_per_image,
                                                        smooth_l1_beta=smooth_l1_beta, box2box_weights=box2box_weights,
                                                        box_reg_loss_type=box_reg_loss_type, scale_clamp=scale_clamp,
                                                        loss_weight=loss_weight)
    st, p, q = torch.stack([status.to(torch.int64), num_pos, num_neg]).tolist()
    _raise_status(st, _transform_name(anchors.shape[-1]))
    return losses, {"num_pos_anchors": p, "num_neg_anchors": q}


def retinanet_losses(anchors, pred_logits: List[Tensor], gt_labels: List[Tensor], pred_anchor_deltas: List[Tensor],
                     gt_boxes: List[Tensor], *, num_classes: int, loss_normalizer: Optional[float] = None,
                     focal_loss_alpha: float = 0.25, focal_loss_gamma: float = 2.0,
                     box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0), scale_clamp: float = _SCALE_CLAMP,
                     box_reg_loss_type: str = "smooth_l1", smooth_l1_beta: float = 0.1):
    """RetinaNet.losses (retinanet.py:160-210) with the `self` attributes as arguments; loss_normalizer is the previous EMA
    value (None: the first call, 100).  Returns (losses, num_pos_anchors, the new normaliser as a Python float).
    One host read."""
    anchors = _cat_anchors(anchors)
    old = 100.0 if loss_normalizer is None else float(loss_normalizer)
    if not _use_kernels(box_reg_loss_type, anchors.is_cuda):
        return _retinanet_losses_host(anchors, pred_logits, gt_labels, pred_anchor_deltas, gt_boxes, num_classes, old,
                                      focal_loss_alpha, focal_loss_gamma, box2box_weights, scale_clamp,
                                      box_reg_loss_type, smooth_l1_beta)
    ema = torch.tensor([old], dtype=torch.float64).to(anchors.device)
    losses, num_pos, status = retinanet_losses_fixed(anchors, pred_logits, gt_labels, pred_anchor_deltas, gt_boxes, ema,
                                                     num_classes=num_classes, focal_loss_alpha=focal_loss_alpha,
                                                     focal_loss_gamma=focal_loss_gamma, smooth_l1_beta=smooth_l1_beta,
                                                     box2box_weights=box2box_weights, box_reg_loss_type=box_reg_loss_type,
                                                     scale_clamp=scale_clamp)
    st, p = torch.stack([status.to(torch.int64), num_pos]).tolist()
    _raise_status(st, _transform_name(anchors.shape[-1]))
    return losses, p, old * 0.9 + max(p, 1) * (1 - 0.9)


def fast_rcnn_losses(scores: Tensor, proposal_deltas: Tensor, proposal_boxes: Tensor, gt_boxes: Tensor,
                     gt_classes: Tensor, *, box2box_weights: Sequence[float] = (10.0, 10.0, 5.0, 5.0),
                     scale_clamp: float = _SCALE_CLAMP, box_reg_loss_type: str = "smooth_l1", smooth_l1_beta: float = 0.0,
                     loss_weight: Optional[Dict[str, float]] = None):
    """FastRCNNOutputLayers.losses (fast_rcnn.py:307-352) with (scores, proposal_deltas) = predictions and the proposals'
    fields concatenated over the images (gt_boxes: the proposal boxes for images without GT, as the reference).
    Returns (losses, stats) with stats the counts of _log_classification_stats as Python ints.  One host read."""
    if not _use_kernels(box_reg_loss_type, scores.is_cuda):
        return _fast_rcnn_losses_host(scores, proposal_deltas, proposal_boxes, gt_boxes, gt_classes, box2box_weights,
                                      scale_clamp, box_reg_loss_type, smooth_l1_beta, loss_weight)
    losses, counts, status = fast_rcnn_losses_fixed(scores, proposal_deltas, proposal_boxes, gt_boxes, gt_classes,
                                                    smooth_l1_beta=smooth_l1_beta, box2box_weights=box2box_weights,
                                                    box_reg_loss_type=box_reg_loss_type, scale_clamp=scale_clamp,
                                                    loss_weight=loss_weight)
    vals = torch.cat([status.to(torch.int64).reshape(1), counts]).tolist()
    _raise_status(vals[0], _transform_name(proposal_boxes.shape[-1]))
    return losses, dict(zip(("num_fg", "num_accurate", "fg_num_accurate", "num_false_negative"), vals[1:]))


# ---- torch restatement (CPU tensors; the reference of the GPU tests) ------------------------------------------------
def _get_deltas(src: Tensor, tgt: Tensor, weights: Sequence[float]) -> Tensor:
    """Box2BoxTransform.get_deltas / Box2BoxTransformRotated.get_deltas (box_regression.py:43-76, 145-180)."""
    import math

    if src.shape[-1] == 5:
        sx, sy, sw, sh, sa = src.unbind(1)
        tx, ty, tw, th, ta = tgt.unbind(1)
        wx, wy, ww, wh, wa = weights
        da = ta - sa
        da = (da + 180.0) % 360.0 - 180.0
        da *= wa * math.pi / 180.0
        out = [wx * (tx - sx) / sw, wy * (ty - sy) / sh, ww * torch.log(tw / sw), wh * torch.log(th / sh), da]
    else:
        sw = src[:, 2] - src[:, 0]
        sh = src[:, 3] - src[:, 1]
        sx, sy = src[:, 0] + 0.5 * sw, src[:, 1] + 0.5 * sh
        tw = tgt[:, 2] - tgt[:, 0]
        th = tgt[:, 3] - tgt[:, 1]
        tx, ty = tgt[:, 0] + 0.5 * tw, tgt[:, 1] + 0.5 * th
        wx, wy, ww, wh = weights
        out = [wx * (tx - sx) / sw, wy * (ty - sy) / sh, ww * torch.log(tw / sw), wh * torch.log(th / sh)]
    assert bool((sw > 0).all()), "Input boxes to %s are not valid!" % _transform_name(src.shape[-1])
    return torch.stack(out, dim=1)


def _smooth_l1_loss(input: Tensor, target: Tensor, beta: float) -> Tensor:
    """fvcore smooth_l1_loss, reduction "sum"."""
    if beta < 1e-5:
        return torch.abs(input - target).sum()
    n = torch.abs(input - target)
    return torch.where(n < beta, 0.5 * n ** 2 / beta, n - 0.5 * beta).sum()


def _giou_loss(boxes1: Tensor, boxes2: Tensor, eps: float = 1e-7) -> Tensor:
    """fvcore giou_loss, reduction "sum"."""
    x1, y1, x2, y2 = boxes1.unbind(dim=-1)
    x1g, y1g, x2g, y2g = boxes2.unbind(dim=-1)
    assert bool((x2 >= x1).all()), "bad box: x1 larger than x2"
    assert bool((y2 >= y1).all()), "bad box: y1 larger than y2"
    xk1, yk1 = torch.max(x1, x1g), torch.max(y1, y1g)
    xk2, yk2 = torch.min(x2, x2g), torch.min(y2, y2g)
    inter = torch.zeros_like(x1)
    mask = (yk2 > yk1) & (xk2 > xk1)
    inter[mask] = (xk2[mask] - xk1[mask]) * (yk2[mask] - yk1[mask])
    union = (x2 - x1) * (y2 - y1) + (x2g - x1g) * (y2g - y1g) - inter
    iou = inter / (union + eps)
    xc1, yc1 = torch.min(x1, x1g), torch.min(y1, y1g)
    xc2, yc2 = torch.max(x2, x2g), torch.max(y2, y2g)
    area_c = (xc2 - xc1) * (yc2 - yc1)
    return (1 - (iou - (area_c - union) / (area_c + eps))).sum()


def _iou_terms(boxes1: Tensor, boxes2: Tensor, eps: float):
    """The shared part of diou_loss / ciou_loss (layers/losses.py): IoU with eps in the union, the squared diagonal of the
    enclosing box plus eps, and the squared distance of the centres."""
    x1, y1, x2, y2 = boxes1.unbind(dim=-1)
    x1g, y1g, x2g, y2g = boxes2.unbind(dim=-1)
    assert bool((x2 >= x1).all()), "bad box: x1 larger than x2"
    assert bool((y2 >= y1).all()), "bad box: y1 larger than y2"
    xk1, yk1 = torch.max(x1, x1g), torch.max(y1, y1g)
    xk2, yk2 = torch.min(x2, x2g), torch.min(y2, y2g)
    inter = torch.zeros_like(x1)
    mask = (yk2 > yk1) & (xk2 > xk1)
    inter[mask] = (xk2[mask] - xk1[mask]) * (yk2[mask] - yk1[mask])
    iou = inter / ((x2 - x1) * (y2 - y1) + (x2g - x1g) * (y2g - y1g) - inter + eps)
    diag = ((torch.max(x2, x2g) - torch.min(x1, x1g)) ** 2) + ((torch.max(y2, y2g) - torch.min(y1, y1g)) ** 2) + eps
    dist = (((x2 + x1) / 2 - (x1g + x2g) / 2) ** 2) + (((y2 + y1) / 2 - (y1g + y2g) / 2) ** 2)
    return iou, diag, dist


def _diou_loss(boxes1: Tensor, boxes2: Tensor, eps: float = 1e-7) -> Tensor:
    """diou_loss (layers/losses.py:5-63), reduction "sum"."""
    iou, diag, dist = _iou_terms(boxes1, boxes2, eps)
    return (1 - iou + (dist / diag)).sum()


def _ciou_loss(boxes1: Tensor, boxes2: Tensor, eps: float = 1e-7) -> Tensor:
    """ciou_loss (layers/losses.py:66-133), reduction "sum": diou plus the aspect-ratio term, its weight without gradient."""
    import math

    iou, diag, dist = _iou_terms(boxes1, boxes2, eps)
    x1, y1, x2, y2 = boxes1.unbind(dim=-1)
    x1g, y1g, x2g, y2g = boxes2.unbind(dim=-1)
    v = (4 / (math.pi ** 2)) * torch.pow(torch.atan((x2g - x1g) / (y2g - y1g)) - torch.atan((x2 - x1) / (y2 - y1)), 2)
    with torch.no_grad():
        alpha = v / (1 - iou + v + eps)
    return (1 - iou + (dist / diag) + alpha * v).sum()


def _sigmoid_focal_loss(inputs: Tensor, targets: Tensor, alpha: float, gamma: float) -> Tensor:
    """fvcore sigmoid_focal_loss, reduction "sum" (fp32)."""
    inputs, targets = inputs.float(), targets.float()
    p = torch.sigmoid(inputs)
    ce = F.binary_cross_entropy_with_logits(inputs, targets, reduction="none")
    p_t = p * targets + (1 - p) * (1 - targets)
    loss = ce * ((1 - p_t) ** gamma)
    if alpha >= 0:
        loss = (alpha * targets + (1 - alpha) * (1 - targets)) * loss
    return loss.sum()


def _dense_box_regression_loss(anchors: Tensor, weights, scale_clamp, pred_anchor_deltas: List[Tensor],
                               gt_boxes: List[Tensor], fg_mask, loss_type: str, beta: float) -> Tensor:
    """_dense_box_regression_loss (box_regression.py:310-369): smooth_l1, giou, diou and ciou."""
    pred = torch.cat(list(pred_anchor_deltas), dim=1)
    if loss_type == "smooth_l1":
        gt_deltas = torch.stack([_get_deltas(anchors, k, weights) for k in gt_boxes])
        return _smooth_l1_loss(pred[fg_mask], gt_deltas[fg_mask], beta)
    boxes = torch.stack([_apply_deltas(k, anchors, weights, scale_clamp) for k in pred])
    loss = {"giou": _giou_loss, "diou": _diou_loss, "ciou": _ciou_loss}[loss_type]
    return loss(boxes[fg_mask], torch.stack(list(gt_boxes))[fg_mask])


def _rpn_losses_host(anchors, pred_objectness_logits, gt_labels, pred_anchor_deltas, gt_boxes, batch_size_per_image,
                     weights, scale_clamp, loss_type, beta, loss_weight):
    num_images = len(gt_labels)
    gt_labels = _stack(gt_labels)
    pos_mask = gt_labels == 1
    num_pos, num_neg = int(pos_mask.sum().item()), int((gt_labels == 0).sum().item())
    loc = _dense_box_regression_loss(anchors, weights, scale_clamp, pred_anchor_deltas, list(gt_boxes), pos_mask,
                                     loss_type, beta)
    valid = gt_labels >= 0
    obj = F.binary_cross_entropy_with_logits(torch.cat(list(pred_objectness_logits), dim=1)[valid],
                                             gt_labels[valid].to(torch.float32), reduction="sum")
    normalizer = batch_size_per_image * num_images
    lw = loss_weight or {}
    losses = {"loss_rpn_cls": obj / normalizer, "loss_rpn_loc": loc / normalizer}
    return {k: v * lw.get(k, 1.0) for k, v in losses.items()}, {"num_pos_anchors": num_pos, "num_neg_anchors": num_neg}


def _retinanet_losses_host(anchors, pred_logits, gt_labels, pred_anchor_deltas, gt_boxes, num_classes, old, alpha, gamma,
                           weights, scale_clamp, loss_type, beta):
    gt_labels = _stack(gt_labels)
    valid = gt_labels >= 0
    pos_mask = valid & (gt_labels != num_classes)
    num_pos = int(pos_mask.sum().item())
    normalizer = old * 0.9 + max(num_pos, 1) * (1 - 0.9)
    target = F.one_hot(gt_labels[valid], num_classes=num_classes + 1)[:, :-1]
    loss_cls = _sigmoid_focal_loss(torch.cat(list(pred_logits), dim=1)[valid], target.to(pred_logits[0].dtype), alpha,
                                   gamma)
    loss_box = _dense_box_regression_loss(anchors, weights, scale_clamp, pred_anchor_deltas, list(gt_boxes), pos_mask,
                                          loss_type, beta)
    return {"loss_cls": loss_cls / normalizer, "loss_box_reg": loss_box / normalizer}, num_pos, normalizer


def _fast_rcnn_losses_host(scores, proposal_deltas, proposal_boxes, gt_boxes, gt_classes, weights, scale_clamp,
                           loss_type, beta, loss_weight):
    k = scores.shape[1] - 1
    stats = {"num_fg": 0, "num_accurate": 0, "fg_num_accurate": 0, "num_false_negative": 0}
    if gt_classes.numel():
        pred = scores.argmax(dim=1)
        fg = (gt_classes >= 0) & (gt_classes < k)
        stats = {"num_fg": int(fg.sum()), "num_accurate": int((pred == gt_classes).sum()),
                 "fg_num_accurate": int((pred[fg] == gt_classes[fg]).sum()),
                 "num_false_negative": int((pred[fg] == k).sum())}
    loss_cls = F.cross_entropy(scores, gt_classes, reduction="mean") if gt_classes.numel() else scores.sum() * 0.0
    d = proposal_boxes.shape[1]
    fg_inds = torch.nonzero((gt_classes >= 0) & (gt_classes < k), as_tuple=True)[0]
    if proposal_deltas.shape[1] == d:
        fg_deltas = proposal_deltas[fg_inds]
    else:
        fg_deltas = proposal_deltas.view(-1, k, d)[fg_inds, gt_classes[fg_inds]]
    loss_box = _dense_box_regression_loss(proposal_boxes[fg_inds], weights, scale_clamp, [fg_deltas.unsqueeze(0)],
                                          [gt_boxes[fg_inds]], ..., loss_type, beta)
    lw = loss_weight or {}
    losses = {"loss_cls": loss_cls, "loss_box_reg": loss_box / max(gt_classes.numel(), 1.0)}
    return {n: v * lw.get(n, 1.0) for n, v in losses.items()}, stats
