"""find_top_rrpn_proposals -- batched rotated RPN proposal selection, same signature and results as
detectron2/modeling/proposal_generator/rrpn.py:20-127.

The reference loops over images in Python: per image it filters non-finite boxes with boolean indexing, clips the rotated
boxes (`RotatedBoxes.clip`, whose `torch.where(...)[0]` is a host sync), drops empty boxes after a `.item()` (:110) and runs
one `batched_nms_rotated`.  Here all images go through ONE rotated NMS: the functions below are
`proposal_utils.find_top_rpn_proposals[_fixed]` with `rotated=True`:

  * `d2b_rpn_prepare` with `D2B_SELECT_ROTATED` (one CTA per image) gathers the per-level top-k, normalises the angles and
    clips, and moves removed boxes (non-finite, or not larger than `min_box_size` after clipping) to the ignored category -1
    instead of removing them; it adds batched_nms_rotated's offsets -- level * (max - min + 1) over THAT image's surviving
    boxes, fp32 -- to the centres;
  * one `d2b_nms(D2B_NMS_ROTATED | D2B_NMS_NO_OFFSET)` with category image * L + level (image alone for a threshold <= 0,
    which IoU 0 passes: the reference's one NMS per image then suppresses across levels too; `D2B_SELECT_SEG_PER_IMAGE`);
  * `d2b_rpn_select` with `D2B_SELECT_ROTATED` hands every image the first `post_nms_topk` survivors of the score-ordered
    keep list.
The only host synchronisation is the final read of the N output lengths.  `clip_rotated` and `rotated_offset_scale` are
the torch-op forms of the clip and the offsets that the host restatements use.
"""
from typing import List, Tuple

import torch

from .proposal_utils import _find_top_rpn_proposals_host, find_top_rpn_proposals, find_top_rpn_proposals_fixed

__all__ = ["find_top_rrpn_proposals", "find_top_rrpn_proposals_fixed", "clip_rotated"]


def clip_rotated(boxes: torch.Tensor, h, w) -> torch.Tensor:
    """RotatedBoxes.clip(box_size=(h, w), clip_angle_threshold=1.0) (structures/rotated_boxes.py:248-303) of [..., 5] boxes,
    out of place.  `h` / `w` are numbers or tensors that broadcast against boxes[..., 0]."""
    a = (boxes[..., 4] + 180.0) % 360.0 - 180.0  # normalize_angles
    near = a.abs() <= 1.0
    cx, cy, bw, bh = boxes[..., 0], boxes[..., 1], boxes[..., 2], boxes[..., 3]
    x1 = torch.minimum((cx - bw / 2.0).clamp(min=0), torch.as_tensor(w, dtype=boxes.dtype, device=boxes.device))
    y1 = torch.minimum((cy - bh / 2.0).clamp(min=0), torch.as_tensor(h, dtype=boxes.dtype, device=boxes.device))
    x2 = torch.minimum((cx + bw / 2.0).clamp(min=0), torch.as_tensor(w, dtype=boxes.dtype, device=boxes.device))
    y2 = torch.minimum((cy + bh / 2.0).clamp(min=0), torch.as_tensor(h, dtype=boxes.dtype, device=boxes.device))
    return torch.stack([torch.where(near, (x1 + x2) / 2.0, cx), torch.where(near, (y1 + y2) / 2.0, cy),
                        torch.where(near, torch.min(bw, x2 - x1), bw), torch.where(near, torch.min(bh, y2 - y1), bh), a], -1)


def rotated_offset_scale(boxes: torch.Tensor, valid: torch.Tensor) -> torch.Tensor:
    """batched_nms_rotated's offset unit (layers/nms.py:137-143) per image: max - min + 1 over the valid boxes of
    boxes [N, M, 5] (1 for an image without valid boxes).  Returns [N]."""
    hi = torch.max(boxes[..., 0], boxes[..., 1]) + torch.max(boxes[..., 2], boxes[..., 3]) / 2
    lo = torch.min(boxes[..., 0], boxes[..., 1]) - torch.max(boxes[..., 2], boxes[..., 3]) / 2
    mx = torch.where(valid, hi, torch.full_like(hi, float("-inf"))).max(dim=1).values
    mn = torch.where(valid, lo, torch.full_like(lo, float("inf"))).min(dim=1).values
    any_valid = valid.any(dim=1)
    return torch.where(any_valid, mx - mn, torch.zeros_like(mx)) + 1


def find_top_rrpn_proposals_fixed(proposals: List[torch.Tensor], pred_objectness_logits: List[torch.Tensor],
                                  image_sizes, nms_thresh: float, pre_nms_topk: int, post_nms_topk: int,
                                  min_box_size: float):
    """Sync-free, fixed-capacity form (CUDA tensors only): returns (boxes [N, post_nms_topk, 5], objectness logits
    [N, post_nms_topk], counts [N] int64, nonfinite [1] int32) -- rows beyond counts[i] are zero.  `image_sizes` is a list
    of (h, w) or an [N, 2] CUDA tensor.  The launch sequence (torch.topk per level, d2b_rpn_prepare, d2b_nms, d2b_rpn_select,
    with D2B_SELECT_ROTATED) has static shapes: it can be captured in a CUDA graph."""
    return find_top_rpn_proposals_fixed(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk,
                                        post_nms_topk, min_box_size, rotated=True)


def find_top_rrpn_proposals(proposals: List[torch.Tensor], pred_objectness_logits: List[torch.Tensor],
                            image_sizes: List[Tuple[int, int]], nms_thresh: float, pre_nms_topk: int, post_nms_topk: int,
                            min_box_size: float, training: bool):
    """proposals[l]: [N, Hi*Wi*A, 5] rotated boxes, pred_objectness_logits[l]: [N, Hi*Wi*A].  Returns N `Proposals` with
    [k, 5] `proposal_boxes.tensor` and [k] `objectness_logits`, exactly like the reference."""
    return find_top_rpn_proposals(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk, post_nms_topk,
                                  min_box_size, training, rotated=True)


def _find_top_rrpn_proposals_host(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk, post_nms_topk,
                                  min_box_size, training):
    """The torch-op restatement of the same selection (also for CUDA tensors, with the GPU NMS): the kernels are tested
    against it."""
    return _find_top_rpn_proposals_host(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk,
                                        post_nms_topk, min_box_size, training, rotated=True)
