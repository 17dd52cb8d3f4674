"""CPU restatements of find_top_rrpn_proposals (detectron2/modeling/proposal_generator/rrpn.py:20-127) and
fast_rcnn_inference_single_image_rotated (modeling/roi_heads/rotated_fast_rcnn.py:83-132), TEST INFRASTRUCTURE.

They follow the reference step by step -- per-image loop, boolean filtering, RotatedBoxes.clip written the reference's way
(in-place on the rows `torch.where` selects), batched_nms_rotated through the CPU oracle (stable score order) -- and are
pinned to fixtures from the real reference functions (tests/golden/make_golden_rotated.py) by
tests/test_rotated_inference_host.py."""
import torch

from oracle import oracle as orc


def clip_(boxes, image_size, clip_angle_threshold=1.0):
    """RotatedBoxes.clip (structures/rotated_boxes.py:255-303), in place on a [R, 5] tensor."""
    h, w = image_size
    boxes[:, 4] = (boxes[:, 4] + 180.0) % 360.0 - 180.0
    idx = torch.where(torch.abs(boxes[:, 4]) <= clip_angle_threshold)[0]
    x1 = boxes[idx, 0] - boxes[idx, 2] / 2.0
    y1 = boxes[idx, 1] - boxes[idx, 3] / 2.0
    x2 = boxes[idx, 0] + boxes[idx, 2] / 2.0
    y2 = boxes[idx, 1] + boxes[idx, 3] / 2.0
    x1.clamp_(min=0, max=w)
    y1.clamp_(min=0, max=h)
    x2.clamp_(min=0, max=w)
    y2.clamp_(min=0, max=h)
    boxes[idx, 0] = (x1 + x2) / 2.0
    boxes[idx, 1] = (y1 + y2) / 2.0
    boxes[idx, 2] = torch.min(boxes[idx, 2], x2 - x1)
    boxes[idx, 3] = torch.min(boxes[idx, 3], y2 - y1)
    return boxes


def find_top_rrpn_proposals(proposals, pred_objectness_logits, image_sizes, nms_thresh, pre_nms_topk, post_nms_topk,
                            min_box_size, training):
    """Returns [(boxes [k, 5], logits [k])] per image."""
    num_images = len(image_sizes)
    batch_idx = torch.arange(num_images)
    topk_scores, topk_proposals, level_ids = [], [], []
    for level_id, (p_i, l_i) in enumerate(zip(proposals, pred_objectness_logits)):  # :67-83
        k = min(l_i.shape[1], pre_nms_topk)
        s_i, idx = l_i.topk(k, dim=1)
        topk_proposals.append(p_i[batch_idx[:, None], idx])
        topk_scores.append(s_i)
        level_ids.append(torch.full((k,), level_id, dtype=torch.int64))
    topk_scores = torch.cat(topk_scores, dim=1)
    topk_proposals = torch.cat(topk_proposals, dim=1)
    level_ids = torch.cat(level_ids, dim=0)
    results = []
    for n, image_size in enumerate(image_sizes):  # :92-126
        boxes, scores, lvl = topk_proposals[n].clone(), topk_scores[n], level_ids
        valid = torch.isfinite(boxes).all(dim=1) & torch.isfinite(scores)
        if not valid.all():
            if training:
                raise FloatingPointError("Predicted boxes or scores contain Inf/NaN. Training has diverged.")
            boxes, scores, lvl = boxes[valid], scores[valid], lvl[valid]
        clip_(boxes, image_size)
        keep = (boxes[:, 2] > min_box_size) & (boxes[:, 3] > min_box_size)  # RotatedBoxes.nonempty
        boxes, scores, lvl = boxes[keep], scores[keep], lvl[keep]
        keep = orc.batched_nms_rotated(boxes, scores, lvl, nms_thresh)[:post_nms_topk]
        results.append((boxes[keep], scores[keep]))
    return results


def fast_rcnn_inference_single_image_rotated(boxes, scores, image_shape, score_thresh, nms_thresh, topk_per_image):
    """Returns (boxes [k, 5], scores [k], classes [k], rows [k])."""
    valid = torch.isfinite(boxes).all(dim=1) & torch.isfinite(scores).all(dim=1)
    if not valid.all():
        boxes, scores = boxes[valid], scores[valid]
    scores = scores[:, :-1]
    k = boxes.shape[1] // 5
    boxes = clip_(boxes.reshape(-1, 5).clone(), image_shape).view(-1, k, 5)
    filter_mask = scores > score_thresh
    filter_inds = filter_mask.nonzero()
    boxes = boxes[filter_inds[:, 0], 0] if k == 1 else boxes[filter_mask]
    scores = scores[filter_mask]
    keep = orc.batched_nms_rotated(boxes, scores, filter_inds[:, 1], nms_thresh)
    if topk_per_image >= 0:
        keep = keep[:topk_per_image]
    return boxes[keep], scores[keep], filter_inds[keep, 1], filter_inds[keep, 0]


def fast_rcnn_inference_rotated(boxes, scores, image_shapes, score_thresh, nms_thresh, topk_per_image):
    return [fast_rcnn_inference_single_image_rotated(b, s, sh, score_thresh, nms_thresh, topk_per_image)
            for b, s, sh in zip(boxes, scores, image_shapes)]
