"""fast_rcnn_inference_rotated -- batched rotated Fast R-CNN inference post-processing, same results as
detectron2/modeling/roi_heads/rotated_fast_rcnn.py:46-132 (`fast_rcnn_inference_rotated`,
`fast_rcnn_inference_single_image_rotated`).

The reference processes one image at a time: boolean row filtering, `RotatedBoxes.clip` (a `torch.where(...)[0]` host
sync), `nonzero()` on the R x K score matrix (another sync), one `batched_nms_rotated`, slicing.  Here every image of the
batch goes through ONE rotated NMS: the functions below are `fast_rcnn_inference.fast_rcnn_inference[_fixed]` with
`rotated=True`:

  * `d2b_frcnn_prepare` with `D2B_SELECT_ROTATED` (one CTA per image) drops the non-finite rows, compacts the (row, class)
    pairs with score > score_thresh IN ROW-MAJOR ORDER into `CAP` slots per image, normalises the angles and clips the boxes,
    and adds batched_nms_rotated's offsets class * (max - min + 1) over the image's candidates to the centres;
  * one `d2b_nms(D2B_NMS_ROTATED | D2B_NMS_NO_OFFSET)` with category image * (K + 1) + class, empty slots -1 (ignored);
  * `d2b_rpn_select` with `D2B_SELECT_ROTATED` hands every image the first `topk_per_image` entries of the score-ordered
    keep list.
An image whose candidates overflow `fast_rcnn_inference.CANDIDATE_CAP` is recomputed with the exact (synchronising)
candidate list.  CPU tensors take the same selection written with torch ops.
"""
from typing import List, Tuple

import torch

from .fast_rcnn_inference import _fast_rcnn_inference_host, fast_rcnn_inference, fast_rcnn_inference_fixed

__all__ = ["fast_rcnn_inference_rotated", "fast_rcnn_inference_single_image_rotated", "fast_rcnn_inference_rotated_fixed"]


def fast_rcnn_inference_rotated_fixed(boxes: List[torch.Tensor], scores: List[torch.Tensor], image_shapes,
                                      score_thresh: float, nms_thresh: float, topk_per_image: int, cap: int = 0):
    """Sync-free, fixed-capacity form (CUDA tensors only, at most D2B_MAX_IMAGES images).  Returns a dict of device
    tensors: `boxes` [N, topk, 5], `scores` / `classes` / `rows` [N, topk] (rows = index among the image's valid rows),
    `counts` [N] and `n_cand` [N] (an image with n_cand > cap overflowed its candidate slots and must be redone exactly).
    `image_shapes` is a list of (h, w) or an [N, 2] CUDA tensor.  Static shapes: capturable in a CUDA graph."""
    return fast_rcnn_inference_fixed(boxes, scores, image_shapes, score_thresh, nms_thresh, topk_per_image, cap,
                                     rotated=True)


def fast_rcnn_inference_rotated(boxes: List[torch.Tensor], scores: List[torch.Tensor], image_shapes: List[Tuple[int, int]],
                                score_thresh: float, nms_thresh: float, topk_per_image: int):
    """boxes[i]: R_i x (K*5) or R_i x 5 predicted rotated boxes, scores[i]: R_i x (K+1) class scores (last = background).
    Returns (list[Detections], list[Tensor of kept row indices]) exactly like the reference."""
    return fast_rcnn_inference(boxes, scores, image_shapes, score_thresh, nms_thresh, topk_per_image, rotated=True)


def fast_rcnn_inference_single_image_rotated(boxes, scores, image_shape, score_thresh: float, nms_thresh: float,
                                             topk_per_image: int):
    """Single-image form with the reference's signature (rotated_fast_rcnn.py:84-86)."""
    res, rows = fast_rcnn_inference_rotated([boxes], [scores], [image_shape], score_thresh, nms_thresh, topk_per_image)
    return res[0], rows[0]


def _fast_rcnn_inference_rotated_host(boxes: List[torch.Tensor], scores: List[torch.Tensor],
                                      image_shapes: List[Tuple[int, int]], score_thresh: float, nms_thresh: float,
                                      topk_per_image: int):
    """The torch-op restatement of the same selection (also for CUDA tensors, with the GPU NMS): the kernels are tested
    against it."""
    return _fast_rcnn_inference_host(boxes, scores, image_shapes, score_thresh, nms_thresh, topk_per_image, rotated=True)
