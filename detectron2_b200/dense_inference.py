"""Batched dense-detector (RetinaNet / FCOS-style) inference post-processing (SURVEY 8f-2), same results as the reference's
per-image path: `RetinaNet.forward_inference` / `inference_single_image` (detectron2/modeling/meta_arch/retinanet.py:
256-308) on top of `DenseDetector._decode_per_level_predictions` / `_decode_multi_level_predictions`
(meta_arch/dense_detector.py:186-258) and `Box2BoxTransform.apply_deltas` (modeling/box_regression.py:78-116).

The reference loops over images and, inside, over feature levels: boolean filtering, `nonzero()` (host sync), `topk`,
box decoding, then one `batched_nms` per image and a slice.  Here every image and every level goes through ONE NMS
pipeline and there is a single host synchronisation (the read of the per-image output lengths):

  * per level, the candidates of all images are taken with one batched `topk` over the (anchor, class) scores with the
    entries that fail `score > score_thresh` set to -inf -- the same set, in the same (descending-score) order, as the
    reference's filter + `topk(min(count, topk_candidates))`; slots beyond an image's real candidate count stay dead;
  * boxes are decoded for the candidates only, with the reference's fp32 expression order;
  * NMS category = image * (K + 1) + class with torchvision's `batched_nms` coordinate offsets reproduced per image
    (`class * (max coordinate of that image's candidates + 1)` in fp32, applied while the image has at most 25 000
    candidates, as `torchvision.ops.boxes.batched_nms` does on CUDA), dead slots parked in a dummy category;
  * the first `max_detections_per_image` survivors of every image are extracted from the score-ordered keep list on the
    device.
On CUDA the decode, class ids, offsets (`d2b_dense_prepare`) and the final selection (`d2b_rpn_select`) are one kernel each
for all levels and images; the torch-op form below is the host-logic restatement used for CPU tensors.
"""
import math
from typing import List, Sequence, Tuple

import torch

from . import ops
from ._batched_select import first_k_per_image, nms_select
from .fast_rcnn_inference import Detections

__all__ = ["apply_deltas", "apply_deltas_linear", "dense_detector_inference", "retinanet_inference"]

_DEFAULT_SCALE_CLAMP = math.log(1000.0 / 16)  # box_regression.py:17


def apply_deltas(deltas: torch.Tensor, boxes: torch.Tensor, weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0),
                 scale_clamp: float = _DEFAULT_SCALE_CLAMP) -> torch.Tensor:
    """Box2BoxTransform.apply_deltas (box_regression.py:78-116), op for op: deltas (R, k*4), boxes (R, 4) -> (R, k*4)."""
    deltas = deltas.float()
    boxes = boxes.to(deltas.dtype)
    widths = boxes[:, 2] - boxes[:, 0]
    heights = boxes[:, 3] - boxes[:, 1]
    ctr_x = boxes[:, 0] + 0.5 * widths
    ctr_y = boxes[:, 1] + 0.5 * heights
    wx, wy, ww, wh = weights
    dx = deltas[:, 0::4] / wx
    dy = deltas[:, 1::4] / wy
    dw = deltas[:, 2::4] / ww
    dh = deltas[:, 3::4] / wh
    dw = torch.clamp(dw, max=scale_clamp)
    dh = torch.clamp(dh, max=scale_clamp)
    pred_ctr_x = dx * widths[:, None] + ctr_x[:, None]
    pred_ctr_y = dy * heights[:, None] + ctr_y[:, None]
    pred_w = torch.exp(dw) * widths[:, None]
    pred_h = torch.exp(dh) * heights[:, None]
    x1 = pred_ctr_x - 0.5 * pred_w
    y1 = pred_ctr_y - 0.5 * pred_h
    x2 = pred_ctr_x + 0.5 * pred_w
    y2 = pred_ctr_y + 0.5 * pred_h
    return torch.stack((x1, y1, x2, y2), dim=-1).reshape(deltas.shape)


def apply_deltas_linear(deltas: torch.Tensor, boxes: torch.Tensor) -> torch.Tensor:
    """Box2BoxTransformLinear(normalize_by_size=True).apply_deltas (box_regression.py:275-307), op for op: deltas (R, k*4),
    boxes (R, 4) -> (R, k*4)."""
    deltas = torch.nn.functional.relu(deltas)
    boxes = boxes.to(deltas.dtype)
    ctr_x = 0.5 * (boxes[:, 0] + boxes[:, 2])
    ctr_y = 0.5 * (boxes[:, 1] + boxes[:, 3])
    stride_w = boxes[:, 2] - boxes[:, 0]
    stride_h = boxes[:, 3] - boxes[:, 1]
    deltas = deltas * torch.stack([stride_w, stride_h, stride_w, stride_h], dim=1).repeat(1, deltas.shape[1] // 4)
    pred = torch.zeros_like(deltas)
    pred[:, 0::4] = ctr_x[:, None] - deltas[:, 0::4]
    pred[:, 1::4] = ctr_y[:, None] - deltas[:, 1::4]
    pred[:, 2::4] = ctr_x[:, None] + deltas[:, 2::4]
    pred[:, 3::4] = ctr_y[:, None] + deltas[:, 3::4]
    return pred


_TRANSFORMS = ("delta", "linear")  # Box2BoxTransform (RetinaNet), Box2BoxTransformLinear (FCOS)


def _check_transform(transform: str):
    if transform not in _TRANSFORMS:
        raise ValueError("box transform must be one of %s, got %r" % (_TRANSFORMS, transform))


def dense_detector_inference_fixed(anchors: List[torch.Tensor], pred_scores: List[torch.Tensor],
                                   pred_deltas: List[torch.Tensor], num_images: int, score_thresh: float,
                                   topk_candidates: int, nms_thresh: float, max_detections_per_image: int,
                                   box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0),
                                   scale_clamp: float = _DEFAULT_SCALE_CLAMP, transform: str = "delta"):
    """Sync-free, fixed-capacity form (CUDA tensors only): (boxes [N, D, 4], scores [N, D], classes [N, D], counts [N]) with
    D = max_detections_per_image, rows beyond counts[i] zero.  Launch sequence: per level one `where` + batched `topk`
    (library), then d2b_dense_prepare (decode + class ids + NMS offsets of ALL levels and images), memset + 3 NMS kernels,
    d2b_rpn_select, one gather.  Static shapes: capturable in a CUDA graph.
    transform: "delta" decodes with Box2BoxTransform(box2box_weights, scale_clamp) (RetinaNet), "linear" with
    Box2BoxTransformLinear(normalize_by_size=True) (FCOS, D2B_SELECT_LINEAR; weights and scale_clamp unused)."""
    import ctypes as C

    from . import _C
    from ._C import check, ptr, stream_ptr

    n = int(num_images)
    device = pred_scores[0].device
    _C.require_cuda(*anchors, *pred_scores, *pred_deltas)
    L = len(anchors)
    if L > _C.MAX_LEVELS:
        raise RuntimeError("dense_detector_inference: at most %d feature levels" % _C.MAX_LEVELS)
    ncls = pred_scores[0].shape[2]
    lv = _C.DenseLevels()
    lv.num_levels = L
    keepalive = []
    t = 0
    for l, (a_l, s_l, d_l) in enumerate(zip(anchors, pred_scores, pred_deltas)):
        _, r, k_cls = s_l.shape
        flat = s_l.reshape(n, r * k_cls)
        k = min(int(topk_candidates), r * k_cls)
        # score threshold + top-k (dense_detector.py:211-224): failing entries can never be selected ahead of passing ones
        masked = torch.where(flat > score_thresh, flat.float(), torch.full_like(flat, float("-inf"), dtype=torch.float32))
        top_s, top_i = masked.topk(k, dim=1)
        a_c, d_c = a_l.float().contiguous(), d_l.float().contiguous()
        keepalive += [top_s, top_i, a_c, d_c]
        lv.anchors[l], lv.deltas[l], lv.topk_idx[l], lv.topk_scores[l] = a_c.data_ptr(), d_c.data_ptr(), top_i.data_ptr(), top_s.data_ptr()
        lv.R[l], lv.k[l] = r, k
        t += k
    m = n * t
    topk = int(max_detections_per_image) if max_detections_per_image >= 0 else t
    f32 = dict(dtype=torch.float32, device=device)
    i64 = dict(dtype=torch.int64, device=device)
    flat_boxes, nms_boxes = torch.empty((m, 4), **f32), torch.empty((m, 4), **f32)
    nms_scores, raw_scores = torch.empty((m,), **f32), torch.empty((m,), **f32)
    classes, cat_ids = torch.empty((m,), **i64), torch.empty((m,), **i64)
    _check_transform(transform)
    w = (C.c_float * 4)(*[float(x) for x in box2box_weights])
    flags = _C.SELECT_LINEAR if transform == "linear" else 0
    with torch.cuda.device(device):
        check(_C.lib().d2b_dense_prepare(C.byref(lv), n, ncls, w, float(scale_clamp), flags, ptr(flat_boxes), ptr(nms_boxes),
                                         ptr(nms_scores), ptr(raw_scores), ptr(classes), ptr(cat_ids), stream_ptr(device)),
              "dense_prepare")
    out_boxes, out_scores, out_index, counts = nms_select(nms_boxes, nms_scores, cat_ids, flat_boxes, raw_scores, n, t, topk,
                                                          nms_thresh, False, max(t, 1))
    out_classes = classes[out_index.reshape(-1)].reshape(n, topk) if m else out_index
    del keepalive
    return out_boxes, out_scores, out_classes, counts


def dense_detector_inference(anchors: List[torch.Tensor], pred_scores: List[torch.Tensor],
                             pred_deltas: List[torch.Tensor], image_sizes: List[Tuple[int, int]], score_thresh: float,
                             topk_candidates: int, nms_thresh: float, max_detections_per_image: int,
                             box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0),
                             scale_clamp: float = _DEFAULT_SCALE_CLAMP, transform: str = "delta") -> List[Detections]:
    """anchors[l]: (R_l, 4) anchors of level l; pred_scores[l]: (N, R_l, K) class scores (already sigmoid-ed);
    pred_deltas[l]: (N, R_l, 4) box regression outputs.  Returns one `Detections` per image with the fields of the
    reference's `Instances` (pred_boxes, scores, pred_classes), in the reference's order (descending score).
    transform: "delta" (Box2BoxTransform, RetinaNet) or "linear" (Box2BoxTransformLinear, FCOS)."""
    if not pred_scores[0].is_cuda:
        return _dense_detector_inference_host(anchors, pred_scores, pred_deltas, image_sizes, score_thresh, topk_candidates,
                                              nms_thresh, max_detections_per_image, box2box_weights, scale_clamp,
                                              transform)
    ob, osc, ocl, counts = dense_detector_inference_fixed(anchors, pred_scores, pred_deltas, len(image_sizes), score_thresh,
                                                          topk_candidates, nms_thresh, max_detections_per_image,
                                                          box2box_weights, scale_clamp, transform)
    counts_host = counts.tolist()  # the one host sync: the reference contract returns exactly-sized results
    return [Detections(sz, ob[i, :counts_host[i]], osc[i, :counts_host[i]], ocl[i, :counts_host[i]])
            for i, sz in enumerate(image_sizes)]


def _dense_detector_inference_host(anchors: List[torch.Tensor], pred_scores: List[torch.Tensor],
                                   pred_deltas: List[torch.Tensor], image_sizes: List[Tuple[int, int]], score_thresh: float,
                                   topk_candidates: int, nms_thresh: float, max_detections_per_image: int,
                                   box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0),
                                   scale_clamp: float = _DEFAULT_SCALE_CLAMP, transform: str = "delta") -> List[Detections]:
    """The same selection written with torch ops (host-logic restatement pinned to the real reference functions by
    tests/test_host_logic_cpu.py with the NMS replaced by the oracle; the CUDA path above is the product)."""
    _check_transform(transform)
    num_images = len(image_sizes)
    device = pred_scores[0].device
    ncls = pred_scores[0].shape[2]
    batch_idx = torch.arange(num_images, device=device)
    boxes_l, scores_l, cls_l, live_l = [], [], [], []
    for anchors_i, scores_i, deltas_i in zip(anchors, pred_scores, pred_deltas):
        n, r, k_cls = scores_i.shape
        flat = scores_i.reshape(n, r * k_cls)
        k = min(int(topk_candidates), r * k_cls)
        # 1. score threshold + top-k (dense_detector.py:211-224): failing entries can never be selected ahead of passing ones
        masked = torch.where(flat > score_thresh, flat.float(), torch.full_like(flat, float("-inf"), dtype=torch.float32))
        top_s, top_i = masked.topk(k, dim=1)
        live = top_s > float("-inf")
        anchor_idxs = torch.div(top_i, k_cls, rounding_mode="floor")
        classes = top_i - anchor_idxs * k_cls
        # 2. decode the selected boxes only (:226-230)
        sel_deltas = deltas_i[batch_idx[:, None], anchor_idxs]                       # N x k x 4
        sel_anchors = anchors_i[anchor_idxs]                                         # N x k x 4
        if transform == "linear":
            decoded = apply_deltas_linear(sel_deltas.reshape(-1, 4), sel_anchors.reshape(-1, 4))
        else:
            decoded = apply_deltas(sel_deltas.reshape(-1, 4), sel_anchors.reshape(-1, 4), box2box_weights, scale_clamp)
        boxes_l.append(decoded.reshape(n, k, 4))
        scores_l.append(top_s)
        cls_l.append(classes)
        live_l.append(live)
    # 3. concatenate the levels (`Instances.cat`, :258): candidate order = level-major, descending score inside a level
    boxes = torch.cat(boxes_l, dim=1)      # N x T x 4
    scores = torch.cat(scores_l, dim=1)    # N x T
    classes = torch.cat(cls_l, dim=1)      # N x T
    live = torch.cat(live_l, dim=1)        # N x T
    n, t = scores.shape

    # 4. one NMS for all images (retinanet.py:305-307 per image): torchvision's coordinate trick reproduced per image
    zeros = torch.zeros_like(boxes)
    neg = torch.full_like(boxes, float("-inf"))
    n_live = live.sum(dim=1)
    mx = torch.where(live[..., None], boxes, neg).reshape(n, -1).max(dim=1).values if t > 0 else boxes.new_zeros((n,))
    mx = torch.where(n_live > 0, mx, torch.zeros_like(mx))  # image without candidates (torchvision returns early)
    use_trick = (n_live * 4 <= 100_000)    # torchvision/ops/boxes.py batched_nms: coordinate trick up to 100k elements on CUDA
    offs = classes.to(torch.float32) * (mx[:, None] + 1.0)
    offs = torch.where(use_trick[:, None] & live, offs, torch.zeros_like(offs))
    nms_boxes = torch.where(live[..., None], boxes + offs[..., None], zeros).reshape(-1, 4)
    nms_scores = torch.where(live, scores, torch.full_like(scores, float("-inf"))).reshape(-1)
    cat_ids = torch.where(live, classes + batch_idx[:, None] * (ncls + 1), torch.full_like(classes, -1)).reshape(-1)  # -1: ignored
    keep, num_keep = ops.nms_fixed(nms_boxes, nms_scores, cat_ids, float(nms_thresh), False, apply_offsets=False,
                                   max_segment=max(t, 1))

    # 5. per-image first max_detections_per_image of the score-ordered keep list (:308), on the device
    topk = int(max_detections_per_image) if max_detections_per_image >= 0 else keep.shape[0]
    img_of = batch_idx[:, None].expand(n, t).reshape(-1)
    out_idx, counts = first_k_per_image(keep, num_keep, img_of, live.reshape(-1), num_images, topk)
    flat_boxes, flat_scores, flat_cls = boxes.reshape(-1, 4), scores.reshape(-1), classes.reshape(-1)

    counts_host = counts.tolist()  # the one host sync: the reference contract returns exactly-sized results
    results = []
    for i, image_size in enumerate(image_sizes):
        sel_i = out_idx[i, : counts_host[i]]
        results.append(Detections(image_size, flat_boxes[sel_i], flat_scores[sel_i], flat_cls[sel_i]))
    return results


def retinanet_inference(anchors: List[torch.Tensor], pred_logits: List[torch.Tensor],
                        pred_anchor_deltas: List[torch.Tensor], image_sizes: List[Tuple[int, int]],
                        test_score_thresh: float = 0.05, test_topk_candidates: int = 1000, test_nms_thresh: float = 0.5,
                        max_detections_per_image: int = 100,
                        box2box_weights: Sequence[float] = (1.0, 1.0, 1.0, 1.0)) -> List[Detections]:
    """`RetinaNet.forward_inference` after `_transpose_dense_predictions` (retinanet.py:256-273): pred_logits[l] is
    (N, H_l*W_l*A, K) raw logits (the reference applies `sigmoid_()` per image at :267), pred_anchor_deltas[l] is
    (N, H_l*W_l*A, 4).  Defaults are the reference config defaults (config/defaults.py MODEL.RETINANET.*)."""
    scores = [x.sigmoid() for x in pred_logits]
    return dense_detector_inference(anchors, scores, pred_anchor_deltas, image_sizes, test_score_thresh,
                                    test_topk_candidates, test_nms_thresh, max_detections_per_image, box2box_weights)
