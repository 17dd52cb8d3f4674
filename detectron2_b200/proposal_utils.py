"""find_top_rpn_proposals -- batched RPN proposal selection (SURVEY 8f-2), same signature and results as
detectron2/modeling/proposal_generator/proposal_utils.py:22-135; with `rotated=True` the same for rotated boxes
(find_top_rrpn_proposals, rrpn.py:20-127, whose public names live in `rrpn.py`).

The reference loops over images in Python: per image it filters non-finite / small boxes with boolean indexing, calls
`.item()` (host sync, :118), runs one `batched_nms` and slices.  Here all images go through ONE NMS pipeline:

  * the NMS category of a candidate is `image * L + level`, so one `d2b_nms` call (per-class segments scanned by
    parallel CTAs) covers every (image, level) pair;
  * boxes the reference removes before NMS (non-finite, or smaller than `min_box_size` after clipping) are not
    removed -- which would need a data-dependent shape -- but moved to a private dummy category with score -inf:
    they cannot suppress anything and are dropped from the output, which gives the same kept set and order;
  * the per-image top `post_nms_topk` of the score-ordered keep list is extracted on the device; the only host
    synchronisation is the final read of the N output lengths.
The box type changes the clip (`Boxes.clip` / `RotatedBoxes.clip`), the NMS offsets (torchvision's `batched_nms` /
`batched_nms_rotated`, see `rrpn.py`) and, for a rotated threshold <= 0, the NMS segments; the kernels take it as a
template policy (csrc/postproc.cu).
"""
from typing import List, Tuple

import torch

from . import ops
from ._batched_select import first_k_per_image, image_hw, nms_select, topk_levels

__all__ = ["find_top_rpn_proposals", "find_top_rpn_proposals_fixed", "ProposalBoxes", "Proposals"]


class ProposalBoxes:
    """Minimal stand-in for detectron2.structures.Boxes (the containers are out of scope): `.tensor`, `len()`."""

    def __init__(self, tensor: torch.Tensor):
        self.tensor = tensor

    def __len__(self):
        return self.tensor.shape[0]


class Proposals:
    """Minimal stand-in for detectron2.structures.Instances with the two fields RPN produces."""

    def __init__(self, image_size, proposal_boxes: ProposalBoxes, objectness_logits: torch.Tensor):
        self.image_size = image_size
        self.proposal_boxes = proposal_boxes
        self.objectness_logits = objectness_logits

    def __len__(self):
        return len(self.proposal_boxes)


def find_top_rpn_proposals_fixed(proposals: List[torch.Tensor], pred_objectness_logits: List[torch.Tensor],
                                 image_sizes: List[Tuple[int, int]], nms_thresh: float, pre_nms_topk: int,
                                 post_nms_topk: int, min_box_size: float, *, rotated: bool = False):
    """Sync-free, fixed-capacity form (CUDA tensors only): returns (boxes [N, post_nms_topk, 4], or 5 with `rotated`,
    objectness logits [N, post_nms_topk], counts [N] int64, nonfinite [1] int32) -- rows beyond counts[i] are zero.
    `image_sizes` is a list of (h, w) or an [N, 2] CUDA tensor (needed inside a CUDA-graph capture).  The launch sequence
    (torch.topk per level, d2b_rpn_prepare, d2b_nms, d2b_rpn_select; D2B_SELECT_ROTATED with `rotated`) has static shapes:
    it can be captured in a CUDA graph."""
    import ctypes as C

    from . import _C
    from ._C import check, ptr, stream_ptr

    n = len(image_sizes)
    device = proposals[0].device
    _C.require_cuda(*proposals, *pred_objectness_logits)
    lv, t, ks, keepalive = topk_levels(proposals, pred_objectness_logits, pre_nms_topk)
    hw = image_hw(image_sizes, device)
    m, d = n * t, (5 if rotated else 4)
    f32 = dict(dtype=torch.float32, device=device)
    flat_boxes, nms_boxes = torch.empty((m, d), **f32), torch.empty((m, d), **f32)
    nms_scores, raw_scores = torch.empty((m,), **f32), torch.empty((m,), **f32)
    cat_ids = torch.empty((m,), dtype=torch.int64, device=device)
    nonfinite = torch.empty((1,), dtype=torch.int32, device=device)
    # IoU 0 passes a rotated threshold <= 0: the reference's one NMS per image then suppresses across levels as well
    per_image = rotated and float(nms_thresh) <= 0.0
    flags = (_C.SELECT_ROTATED if rotated else 0) | (_C.SELECT_SEG_PER_IMAGE if per_image else 0)
    if not rotated and t * 4 > 100_000:  # torchvision's batched_nms offsets at most 100 000 coordinates (25 000 boxes)
        flags |= _C.SELECT_NO_OFFSETS
    with torch.cuda.device(device):
        check(_C.lib().d2b_rpn_prepare(C.byref(lv), n, ptr(hw), float(min_box_size), flags, ptr(flat_boxes), ptr(nms_boxes),
                                       ptr(nms_scores), ptr(raw_scores), ptr(cat_ids), ptr(nonfinite), stream_ptr(device)),
              "rpn_prepare")
    out_boxes, out_scores, _, counts = nms_select(nms_boxes, nms_scores, cat_ids, flat_boxes, raw_scores, n, t,
                                                  int(post_nms_topk), nms_thresh, rotated, t if per_image else max(ks))
    del keepalive
    return out_boxes, out_scores, counts, nonfinite


def find_top_rpn_proposals(proposals: List[torch.Tensor], pred_objectness_logits: List[torch.Tensor],
                           image_sizes: List[Tuple[int, int]], nms_thresh: float, pre_nms_topk: int,
                           post_nms_topk: int, min_box_size: float, training: bool, *, rotated: bool = False):
    """proposals[l]: [N, Hi*Wi*A, 4] boxes, or [N, Hi*Wi*A, 5] rotated boxes with `rotated` (find_top_rrpn_proposals),
    pred_objectness_logits[l]: [N, Hi*Wi*A].  Returns N `Proposals` exactly like the reference."""
    if proposals[0].is_cuda:  # fused, fixed-capacity kernels + ONE host read of the output lengths
        out_boxes, out_scores, counts, nonfinite = find_top_rpn_proposals_fixed(
            proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk, post_nms_topk, min_box_size,
            rotated=rotated)
        host = torch.cat([counts, nonfinite.to(torch.int64)]).tolist()  # the one host sync: exactly-sized results
        if training and host[-1]:  # same failure mode as the reference (:106-110); training only
            raise FloatingPointError("Predicted boxes or scores contain Inf/NaN. Training has diverged.")
        dt = pred_objectness_logits[0].dtype
        return [Proposals(sz, ProposalBoxes(out_boxes[i, :host[i]]), out_scores[i, :host[i]].to(dt))
                for i, sz in enumerate(image_sizes)]
    return _find_top_rpn_proposals_host(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk,
                                        post_nms_topk, min_box_size, training, rotated=rotated)


def _find_top_rpn_proposals_host(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk, post_nms_topk,
                                 min_box_size, training, *, rotated=False):
    """The same selection written with torch ops (the host-logic restatement that tests/test_host_logic_cpu.py and
    tests/test_rotated_inference_host.py pin to the real reference functions with the NMS call replaced by the oracle; the
    CUDA path above is the product)."""
    num_images = len(image_sizes)
    device = proposals[0].device
    num_levels = len(proposals)
    # 1. top-k per level and image (proposal_utils.py:70-94, rrpn.py:62-88)
    batch_idx = torch.arange(num_images, device=device)
    boxes_l, scores_l, level_l = [], [], []
    for level_id, (proposals_i, logits_i) in enumerate(zip(proposals, pred_objectness_logits)):
        k = min(logits_i.shape[1], pre_nms_topk)
        topk_scores_i, topk_idx = logits_i.topk(k, dim=1)
        boxes_l.append(proposals_i[batch_idx[:, None], topk_idx])
        scores_l.append(topk_scores_i)
        level_l.append(torch.full((k,), level_id, dtype=torch.int64, device=device))
    boxes = torch.cat(boxes_l, dim=1).float()   # N x T x 4 (5)
    scores = torch.cat(scores_l, dim=1)         # N x T
    levels = torch.cat(level_l, dim=0)          # T
    n, t = scores.shape
    d = boxes.shape[2]

    # 2. validity, clip, small-box filter -- as masks, not as shape changes (:104-120, rrpn.py:97-111)
    finite = torch.isfinite(boxes).all(dim=2) & torch.isfinite(scores)
    if training and not bool(finite.all()):  # same failure mode as the reference (:106-110); training only
        raise FloatingPointError("Predicted boxes or scores contain Inf/NaN. Training has diverged.")
    hw = image_hw(image_sizes, device)  # N x 2
    if rotated:
        from .rrpn import clip_rotated, rotated_offset_scale  # (rrpn imports this module)

        clipped = clip_rotated(boxes, hw[:, 0:1], hw[:, 1:2])
        valid = finite & (clipped[..., 2] > min_box_size) & (clipped[..., 3] > min_box_size)
    else:
        x1 = torch.minimum(boxes[..., 0].clamp(min=0), hw[:, 1:2])
        y1 = torch.minimum(boxes[..., 1].clamp(min=0), hw[:, 0:1])
        x2 = torch.minimum(boxes[..., 2].clamp(min=0), hw[:, 1:2])
        y2 = torch.minimum(boxes[..., 3].clamp(min=0), hw[:, 0:1])
        clipped = torch.stack([x1, y1, x2, y2], dim=2)
        valid = finite & ((x2 - x1) > min_box_size) & ((y2 - y1) > min_box_size)

    # 3. one NMS over all images: category = image * L + level (rotated with a threshold IoU 0 passes: the image alone);
    #    removed boxes get category -1 (ignored by the kernels).  Every category holds at most `pre_nms_topk` boxes: the IoU
    #    bitmask and the scans stay linear in the batch size.
    per_image = rotated and float(nms_thresh) <= 0.0
    img_of = batch_idx[:, None].expand(n, t)
    cat_ids = img_of if per_image else img_of * num_levels + levels[None, :]
    cat_ids = torch.where(valid, cat_ids, torch.full_like(cat_ids, -1)).reshape(-1)
    max_segment = t if per_image else max(x.shape[1] for x in scores_l)
    zeros = torch.zeros_like(clipped)
    flat_boxes = torch.where(valid[..., None], clipped, zeros).reshape(-1, d)
    flat_scores = torch.where(valid, scores.float(), torch.full_like(scores, float("-inf"), dtype=torch.float32)).reshape(-1)
    if rotated:  # batched_nms_rotated's offsets: level * (max - min + 1) over THAT image's valid boxes, on the centres
        offs = levels[None, :].to(torch.float32) * rotated_offset_scale(clipped, valid)[:, None]  # N x T
        nms_boxes = torch.cat([clipped[..., :2] + offs[..., None], clipped[..., 2:]], dim=2)
    elif t * 4 <= 100_000:
        # torchvision's batched_nms (reached per image from proposal_utils.py:121) shifts the boxes of level l by
        # l * (max coordinate of THAT image's boxes + 1) in fp32 before computing IoU, as long as the image has at most
        # 25 000 candidates; reproduce exactly those per-image offsets so that every IoU rounds like the reference's.
        neg = torch.full_like(clipped, float("-inf"))
        max_img = torch.where(valid[..., None], clipped, neg).reshape(n, -1).max(dim=1).values  # N
        offs = levels[None, :].to(torch.float32) * (max_img[:, None] + 1.0)                # N x T
        nms_boxes = clipped + offs[..., None]
    else:
        nms_boxes = clipped
    nms_boxes = torch.where(valid[..., None], nms_boxes, zeros).reshape(-1, d)
    keep, num_keep = ops.nms_fixed(nms_boxes, flat_scores, cat_ids, float(nms_thresh), rotated, apply_offsets=False,
                                   max_segment=max_segment)

    # 4. per-image top post_nms_topk of the score-ordered keep list (:129), on the device
    out_idx, counts = first_k_per_image(keep, num_keep, img_of.reshape(-1), valid.reshape(-1), n, post_nms_topk)
    out_boxes = flat_boxes[out_idx.reshape(-1)].reshape(n, post_nms_topk, d)
    out_scores = scores.reshape(-1)[out_idx.reshape(-1)].reshape(n, post_nms_topk)

    counts_host = counts.tolist()  # the one host sync: the reference contract returns exactly-sized results
    return [Proposals(image_size, ProposalBoxes(out_boxes[i, :counts_host[i]]), out_scores[i, :counts_host[i]])
            for i, image_size in enumerate(image_sizes)]
