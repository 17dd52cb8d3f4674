"""find_top_rrpn_proposals -- batched rotated RPN proposal selection, same signature and results as
detectron2/modeling/proposal_generator/rrpn.py:20-127.

The reference loops over images in Python: per image it filters non-finite boxes with boolean indexing, clips the rotated
boxes (`RotatedBoxes.clip`, whose `torch.where(...)[0]` is a host sync), drops empty boxes after a `.item()` (:110) and runs
one `batched_nms_rotated`.  Here all images go through ONE rotated NMS, as in `proposal_utils.find_top_rpn_proposals`:

  * `d2b_rrpn_prepare` (one CTA per image) gathers the per-level top-k, normalises the angles and clips, and moves removed
    boxes (non-finite, or not larger than `min_box_size` after clipping) to the ignored category -1 instead of removing them;
    it adds batched_nms_rotated's offsets -- level * (max - min + 1) over THAT image's surviving boxes, fp32 -- to the centres;
  * one `d2b_nms(D2B_NMS_ROTATED | D2B_NMS_NO_OFFSET)` with category image * L + level;
  * `d2b_rpn_select_rotated` hands every image the first `post_nms_topk` survivors of the score-ordered keep list.
The only host synchronisation is the final read of the N output lengths.
"""
from typing import List, Tuple

import torch

from . import ops
from .proposal_utils import ProposalBoxes, Proposals

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
    of (h, w) or an [N, 2] CUDA tensor.  The launch sequence (torch.topk per level, d2b_rrpn_prepare, d2b_nms,
    d2b_rpn_select_rotated) has static shapes: it can be captured in a CUDA graph."""
    import ctypes as C

    from . import _C
    from ._C import check, ptr, stream_ptr

    n = len(image_sizes)
    device = proposals[0].device
    _C.require_cuda(*proposals, *pred_objectness_logits)
    L = len(proposals)
    if L > _C.MAX_LEVELS:
        raise RuntimeError("find_top_rrpn_proposals: at most %d feature levels" % _C.MAX_LEVELS)
    lv = _C.RpnLevels()
    lv.num_levels = L
    keepalive = []
    t = 0
    for l, (p_l, s_l) in enumerate(zip(proposals, pred_objectness_logits)):
        k = min(s_l.shape[1], pre_nms_topk)
        top_s, top_i = s_l.float().topk(k, dim=1)  # rrpn.py:76 (library top-k, one call per level)
        p_c = p_l.float().contiguous()
        keepalive += [top_s, top_i, p_c]
        lv.proposals[l], lv.topk_idx[l], lv.topk_scores[l] = p_c.data_ptr(), top_i.data_ptr(), top_s.data_ptr()
        lv.A[l], lv.k[l] = p_c.shape[1], k
        t += k
    if isinstance(image_sizes, torch.Tensor):
        hw = image_sizes.to(device=device, dtype=torch.float32).contiguous()
    else:
        hw = torch.tensor([[float(h), float(w)] for (h, w) in image_sizes], dtype=torch.float32).to(device)
    m = n * t
    f32 = dict(dtype=torch.float32, device=device)
    flat_boxes, nms_boxes = torch.empty((m, 5), **f32), torch.empty((m, 5), **f32)
    nms_scores, raw_scores = torch.empty((m,), **f32), torch.empty((m,), **f32)
    cat_ids = torch.empty((m,), dtype=torch.int64, device=device)
    nonfinite = torch.empty((1,), dtype=torch.int32, device=device)
    out_boxes = torch.empty((n, post_nms_topk, 5), **f32)
    out_scores = torch.empty((n, post_nms_topk), **f32)
    out_index = torch.empty((n, post_nms_topk), dtype=torch.int64, device=device)
    counts = torch.zeros((n,), dtype=torch.int64, device=device)
    # IoU 0 passes a threshold <= 0: the reference's one NMS per image then suppresses across levels as well
    per_image = float(nms_thresh) <= 0.0
    with torch.cuda.device(device):
        check(_C.lib().d2b_rrpn_prepare(C.byref(lv), n, ptr(hw), float(min_box_size), int(per_image), ptr(flat_boxes),
                                        ptr(nms_boxes), ptr(nms_scores), ptr(raw_scores), ptr(cat_ids), ptr(nonfinite),
                                        stream_ptr(device)), "rrpn_prepare")
        if m:
            max_segment = t if per_image else max(int(lv.k[l]) for l in range(L))
            keep, num_keep = ops.nms_fixed(nms_boxes, nms_scores, cat_ids, float(nms_thresh), True, apply_offsets=False,
                                           max_segment=max_segment)
            check(_C.lib().d2b_rpn_select_rotated(ptr(keep), ptr(num_keep), n, t, int(post_nms_topk), ptr(flat_boxes),
                                                  ptr(raw_scores), ptr(cat_ids), ptr(out_boxes), ptr(out_scores),
                                                  ptr(out_index), ptr(counts), stream_ptr(device)), "rrpn_select")
    del keepalive
    return out_boxes, out_scores, counts, nonfinite


def find_top_rrpn_proposals(proposals: List[torch.Tensor], pred_objectness_logits: List[torch.Tensor],
                            image_sizes: List[Tuple[int, int]], nms_thresh: float, pre_nms_topk: int, post_nms_topk: int,
                            min_box_size: float, training: bool):
    """proposals[l]: [N, Hi*Wi*A, 5] rotated boxes, pred_objectness_logits[l]: [N, Hi*Wi*A].  Returns N `Proposals` with
    [k, 5] `proposal_boxes.tensor` and [k] `objectness_logits`, exactly like the reference."""
    if proposals[0].is_cuda:  # fused, fixed-capacity kernels + ONE host read of the output lengths
        out_boxes, out_scores, counts, nonfinite = find_top_rrpn_proposals_fixed(
            proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk, post_nms_topk, min_box_size)
        host = torch.cat([counts, nonfinite.to(torch.int64)]).tolist()  # the one host sync: exactly-sized results
        if training and host[-1]:  # same failure mode as the reference (:98-102); training only
            raise FloatingPointError("Predicted boxes or scores contain Inf/NaN. Training has diverged.")
        dt = pred_objectness_logits[0].dtype
        return [Proposals(sz, ProposalBoxes(out_boxes[i, :host[i]]), out_scores[i, :host[i]].to(dt))
                for i, sz in enumerate(image_sizes)]
    return _find_top_rrpn_proposals_host(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk,
                                         post_nms_topk, min_box_size, training)


def _find_top_rrpn_proposals_host(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk, post_nms_topk,
                                  min_box_size, training):
    """The same selection written with torch ops (the host-logic restatement that tests/test_rotated_inference_host.py pins
    to the real reference function with the NMS call replaced by the oracle; the CUDA path above is the product)."""
    num_images = len(image_sizes)
    device = proposals[0].device
    num_levels = len(proposals)
    # 1. top-k per level and image (rrpn.py:62-88)
    batch_idx = torch.arange(num_images, device=device)
    boxes_l, scores_l, level_l = [], [], []
    for level_id, (proposals_i, logits_i) in enumerate(zip(proposals, pred_objectness_logits)):
        k = min(logits_i.shape[1], pre_nms_topk)
        topk_scores_i, topk_idx = logits_i.topk(k, dim=1)
        boxes_l.append(proposals_i[batch_idx[:, None], topk_idx])
        scores_l.append(topk_scores_i)
        level_l.append(torch.full((k,), level_id, dtype=torch.int64, device=device))
    boxes = torch.cat(boxes_l, dim=1).float()   # N x T x 5
    scores = torch.cat(scores_l, dim=1)         # N x T
    levels = torch.cat(level_l, dim=0)          # T
    n, t = scores.shape

    # 2. validity, clip, empty-box filter -- as masks, not as shape changes (:97-111)
    finite = torch.isfinite(boxes).all(dim=2) & torch.isfinite(scores)
    if training and not bool(finite.all()):  # same failure mode as the reference (:98-102); training only
        raise FloatingPointError("Predicted boxes or scores contain Inf/NaN. Training has diverged.")
    hw = torch.tensor([[float(h), float(w)] for (h, w) in image_sizes], device=device)  # N x 2
    clipped = clip_rotated(boxes, hw[:, 0:1], hw[:, 1:2])
    valid = finite & (clipped[..., 2] > min_box_size) & (clipped[..., 3] > min_box_size)

    # 3. one rotated NMS over all images: category = image * L + level (image alone for a threshold IoU 0 passes),
    #    removed boxes get category -1; centres carry batched_nms_rotated's per-image offsets
    per_image = float(nms_thresh) <= 0.0
    img_of = batch_idx[:, None].expand(n, t)
    cat_ids = img_of if per_image else img_of * num_levels + levels[None, :]
    cat_ids = torch.where(valid, cat_ids, torch.full_like(cat_ids, -1)).reshape(-1)
    max_segment = t if per_image else max(x.shape[1] for x in scores_l)
    zeros = torch.zeros_like(clipped)
    flat_boxes = torch.where(valid[..., None], clipped, zeros).reshape(-1, 5)
    flat_scores = torch.where(valid, scores.float(), torch.full_like(scores, float("-inf"), dtype=torch.float32)).reshape(-1)
    offs = levels[None, :].to(torch.float32) * rotated_offset_scale(clipped, valid)[:, None]  # N x T
    nms_boxes = torch.cat([clipped[..., :2] + offs[..., None], clipped[..., 2:]], dim=2)
    nms_boxes = torch.where(valid[..., None], nms_boxes, zeros).reshape(-1, 5)
    keep, num_keep = ops.nms_fixed(nms_boxes, flat_scores, cat_ids, float(nms_thresh), True, apply_offsets=False,
                                   max_segment=max_segment)

    # 4. per-image top post_nms_topk of the score-ordered keep list (:121)
    m = keep.shape[0]
    live = torch.arange(m, device=device) < num_keep          # keep[] beyond num_keep is padding
    kidx = torch.where(live, keep, torch.zeros_like(keep))
    kimg = torch.div(kidx, t, rounding_mode="floor")
    kvalid = live & valid.reshape(-1)[kidx]
    onehot = (kimg[None, :] == batch_idx[:, None]) & kvalid[None, :]          # N x M
    rank = torch.cumsum(onehot.to(torch.int32), dim=1) - 1
    sel = onehot & (rank < post_nms_topk)
    counts = sel.sum(dim=1)
    out_idx = torch.zeros((num_images, post_nms_topk + 1), dtype=torch.int64, device=device)
    col = torch.where(sel, rank.long(), torch.full_like(rank, post_nms_topk, dtype=torch.int64))
    out_idx.scatter_(1, col, kidx[None, :].expand(n, m))
    out_idx = out_idx[:, :post_nms_topk].contiguous()
    out_boxes = flat_boxes[out_idx.reshape(-1)].reshape(num_images, post_nms_topk, 5)
    out_scores = scores.reshape(-1)[out_idx.reshape(-1)].reshape(num_images, post_nms_topk)

    counts_host = counts.tolist()  # the one host sync: the reference contract returns exactly-sized results
    return [Proposals(image_size, ProposalBoxes(out_boxes[i, :counts_host[i]]), out_scores[i, :counts_host[i]])
            for i, image_size in enumerate(image_sizes)]
