"""Anchor and proposal matching for the training targets: pairwise IoU + Matcher + the label / box / class gathers of
RPN / RRPN.label_and_sample_anchors, RetinaNet.label_anchors, (R)ROIHeads.label_and_sample_proposals and
CascadeROIHeads._match_and_label_boxes, with the reference's results.

The reference loops over images in Python; per image it builds the dense G x A IoU matrix plus temporaries of the same
size (about 20 launches, two host syncs: the `>= 0` assertion and the `nonzero` of the low-quality matches).  Here all
images go through ONE `d2b_match_boxes` (a zero-fill launch and two kernels, no G x A matrix, no host sync):

  * `match_boxes_fixed` is the static-shape form (CUDA tensors only): GT boxes padded to [N, Gmax, 4|5] with device counts,
    predictions shared ([A, 4|5] anchors) or per image ([N, Pmax, 4|5] with device counts, e.g. the output of
    `find_top_rpn_proposals_fixed`), optionally followed by the image's GT boxes (`proposal_append_gt`).  It can be captured
    in a CUDA graph;
  * the reference-shaped wrappers make one host read (the per-image status: the reference's AssertionError) and then run
    the reference's own `subsample_labels` per image, in the reference's order, so that under the same seed they consume
    the same random numbers and sample the same indices;
  * `rpn_label_and_sample_anchors_fixed` / `label_and_sample_proposals_fixed` follow `match_boxes_fixed` with ONE
    `d2b_sample_labels` for all images (sampling.py): no host read from matching to loss, capturable in a CUDA graph, the
    reference's sampling law but not its random stream.

The box width selects the box type: 4 = (x1, y1, x2, y2), 5 = rotated (cx, cy, w, h, angle_deg).  CPU tensors take the
host restatement below (`Matcher`, `pairwise_iou`; the rotated IoU is `ops.box_iou_rotated_op`).
"""
from typing import List, Optional

import torch

from . import ops

__all__ = ["Matcher", "pairwise_iou", "pairwise_iou_rotated", "subsample_labels", "match_boxes_fixed",
           "rpn_label_and_sample_anchors", "retinanet_label_anchors", "label_and_sample_proposals",
           "cascade_match_and_label_boxes", "rpn_label_and_sample_anchors_fixed", "label_and_sample_proposals_fixed"]


# ----------------------------------------------------------------------------------------------- host restatement
class Matcher:
    """modeling/matcher.py:9-127: the same constructor, assertions and results."""

    def __init__(self, thresholds: List[float], labels: List[int], allow_low_quality_matches: bool = False):
        thresholds = thresholds[:]
        assert thresholds[0] > 0
        thresholds.insert(0, -float("inf"))
        thresholds.append(float("inf"))
        assert all([low <= high for (low, high) in zip(thresholds[:-1], thresholds[1:])])
        assert all([l in [-1, 0, 1] for l in labels])
        assert len(labels) == len(thresholds) - 1
        self.thresholds = thresholds
        self.labels = labels
        self.allow_low_quality_matches = allow_low_quality_matches

    def __call__(self, match_quality_matrix):
        assert match_quality_matrix.dim() == 2
        if match_quality_matrix.numel() == 0:
            default_matches = match_quality_matrix.new_full((match_quality_matrix.size(1),), 0, dtype=torch.int64)
            default_match_labels = match_quality_matrix.new_full((match_quality_matrix.size(1),), self.labels[0],
                                                                 dtype=torch.int8)
            return default_matches, default_match_labels
        assert torch.all(match_quality_matrix >= 0)
        matched_vals, matches = match_quality_matrix.max(dim=0)
        match_labels = matches.new_full(matches.size(), 1, dtype=torch.int8)
        for l, low, high in zip(self.labels, self.thresholds[:-1], self.thresholds[1:]):
            low_high = (matched_vals >= low) & (matched_vals < high)
            match_labels[low_high] = l
        if self.allow_low_quality_matches:
            self.set_low_quality_matches_(match_labels, match_quality_matrix)
        return matches, match_labels

    def set_low_quality_matches_(self, match_labels, match_quality_matrix):
        highest_quality_foreach_gt, _ = match_quality_matrix.max(dim=1)
        _, pred_inds_with_highest_quality = torch.nonzero(
            match_quality_matrix == highest_quality_foreach_gt[:, None], as_tuple=True)
        match_labels[pred_inds_with_highest_quality] = 1


def pairwise_iou(boxes1: torch.Tensor, boxes2: torch.Tensor) -> torch.Tensor:
    """structures/boxes.py:312-358 on [N, 4] / [M, 4] xyxy tensors, op for op."""
    area1 = (boxes1[:, 2] - boxes1[:, 0]) * (boxes1[:, 3] - boxes1[:, 1])
    area2 = (boxes2[:, 2] - boxes2[:, 0]) * (boxes2[:, 3] - boxes2[:, 1])
    width_height = torch.min(boxes1[:, None, 2:], boxes2[:, 2:]) - torch.max(boxes1[:, None, :2], boxes2[:, :2])
    width_height.clamp_(min=0)
    inter = width_height.prod(dim=2)
    return torch.where(inter > 0, inter / (area1[:, None] + area2 - inter),
                       torch.zeros(1, dtype=inter.dtype, device=inter.device))


def pairwise_iou_rotated(boxes1: torch.Tensor, boxes2: torch.Tensor) -> torch.Tensor:
    """structures/rotated_boxes.py:490-505 (box_iou_rotated) on [N, 5] / [M, 5] tensors."""
    return ops.box_iou_rotated_op(boxes1, boxes2)


def _iou(boxes1, boxes2):
    return pairwise_iou_rotated(boxes1, boxes2) if boxes1.shape[-1] == 5 else pairwise_iou(boxes1, boxes2)


def inside_box(boxes: torch.Tensor, box_size, boundary_threshold=0) -> torch.Tensor:
    """Boxes.inside_box (structures/boxes.py:245-262)."""
    height, width = box_size
    return ((boxes[..., 0] >= -boundary_threshold) & (boxes[..., 1] >= -boundary_threshold)
            & (boxes[..., 2] < width + boundary_threshold) & (boxes[..., 3] < height + boundary_threshold))


def subsample_labels(labels: torch.Tensor, num_samples: int, positive_fraction: float, bg_label: int):
    """modeling/sampling.py:9-54, verbatim (two host syncs and two torch.randperm calls on the labels' device)."""
    positive = torch.nonzero((labels != -1) & (labels != bg_label), as_tuple=True)[0]
    negative = torch.nonzero(labels == bg_label, as_tuple=True)[0]
    num_pos = int(num_samples * positive_fraction)
    num_pos = min(positive.numel(), num_pos)
    num_neg = num_samples - num_pos
    num_neg = min(negative.numel(), num_neg)
    perm1 = torch.randperm(positive.numel(), device=positive.device)[:num_pos]
    perm2 = torch.randperm(negative.numel(), device=negative.device)[:num_neg]
    pos_idx = positive[perm1]
    neg_idx = negative[perm2]
    return pos_idx, neg_idx


def _rpn_subsample(label, batch_size_per_image, positive_fraction):
    """RPN._subsample_labels (proposal_generator/rpn.py:286-303)."""
    pos_idx, neg_idx = subsample_labels(label, batch_size_per_image, positive_fraction, 0)
    label.fill_(-1)
    label.scatter_(0, pos_idx, 1)
    label.scatter_(0, neg_idx, 0)
    return label


def _class_targets(matched_idxs, matched_labels, gt_classes, num_classes, ignore=True):
    """The class gather of RetinaNet.label_anchors / ROIHeads._sample_proposals (ignore=True: label -1 -> -1) and of
    CascadeROIHeads._match_and_label_boxes (ignore=False)."""
    if gt_classes.numel() > 0:
        c = gt_classes[matched_idxs]
        c[matched_labels == 0] = num_classes
        if ignore:
            c[matched_labels == -1] = -1
        return c
    return torch.zeros_like(matched_idxs) + num_classes


# ----------------------------------------------------------------------------------------------- fused, fixed form
def _pad(boxes_list: List[torch.Tensor], d: int, device):
    """[N, max(len), d] zero-padded copy of a list of [k_i, d] tensors + the counts (device, int64).  No host sync."""
    n = len(boxes_list)
    kmax = max([int(b.shape[0]) for b in boxes_list] + [0])
    out = torch.zeros((n, kmax, d), dtype=torch.float32, device=device)
    for i, b in enumerate(boxes_list):
        if b.shape[0]:
            out[i, : b.shape[0]] = b.reshape(-1, d)
    counts = torch.tensor([int(b.shape[0]) for b in boxes_list], dtype=torch.int64).to(device, non_blocking=True)
    return out, counts


def match_boxes_fixed(gt_boxes: torch.Tensor, gt_count: torch.Tensor, pred_boxes: torch.Tensor, matcher: Matcher, *,
                      pred_count: Optional[torch.Tensor] = None, append_gt: bool = False, image_hw=None,
                      boundary_thresh: float = -1.0, gt_classes: Optional[torch.Tensor] = None,
                      num_classes: Optional[int] = None, with_boxes: bool = True):
    """Sync-free, static-shape matching of all images (CUDA tensors only).

    gt_boxes [N, Gmax, D] with gt_count [N] (device int64); pred_boxes [A, D] shared by every image, or [N, Pmax, D] with
    pred_count [N] (device int64; None: all Pmax rows).  append_gt: the image's GT boxes follow its predictions.
    image_hw [N, 2] (h, w) and boundary_thresh >= 0: Boxes.inside_box after the matcher (axis-aligned only).
    Returns (matches [N, P] int64, labels [N, P] int8, matched_gt_boxes [N, P, D] or None, classes [N, P] int64 or None,
    status [N] int32), P = Pmax (+ Gmax with append_gt); rows past the image's count are padding (match 0, label -1).
    status != 0: an IoU of that image is negative or NaN (the reference raises AssertionError)."""
    import ctypes as C

    from . import _C
    from ._C import check, ptr, stream_ptr

    _C.require_cuda(gt_boxes, gt_count, pred_boxes, pred_count, gt_classes)
    device = gt_boxes.device
    d = gt_boxes.shape[-1]
    if d not in (4, 5) or pred_boxes.shape[-1] != d or gt_boxes.dim() != 3:
        raise ValueError("match_boxes_fixed: boxes must be [N, G, 4] / [N, G, 5] and predictions of the same width")
    n, gmax = gt_boxes.shape[0], gt_boxes.shape[1]
    gt = gt_boxes.float().contiguous()
    pred = pred_boxes.float().contiguous()
    shared = pred.dim() == 2
    pmax = pred.shape[0] if shared else pred.shape[1]
    if not shared and pred.shape[0] != n:
        raise ValueError("match_boxes_fixed: per-image predictions must be [N, Pmax, D]")
    p = pmax + (gmax if append_gt else 0)
    thr = [float(t) for t in matcher.thresholds[1:-1]]
    lab = [int(l) for l in matcher.labels]
    if len(thr) > _C.MATCH_MAX_THRESHOLDS:
        raise ValueError("match_boxes_fixed: at most %d thresholds" % _C.MATCH_MAX_THRESHOLDS)
    flags = ((_C.MATCH_ROTATED if d == 5 else 0) | (_C.MATCH_LOW_QUALITY if matcher.allow_low_quality_matches else 0)
             | (_C.MATCH_APPEND_GT if append_gt else 0))
    boundary = float(boundary_thresh) >= 0
    hw = None
    if boundary:
        hw = image_hw if isinstance(image_hw, torch.Tensor) else torch.tensor(
            [[float(h), float(w)] for (h, w) in image_hw], dtype=torch.float32).to(device, non_blocking=True)
        hw = hw.to(device=device, dtype=torch.float32).contiguous()
    counts = gt_count.to(torch.int64).contiguous()
    pcounts = None if pred_count is None else pred_count.to(torch.int64).contiguous()
    want_classes = gt_classes is not None
    gcls = gt_classes.to(torch.int64).contiguous() if want_classes else None
    i64 = dict(dtype=torch.int64, device=device)
    matches = torch.empty((n, p), **i64)
    labels = torch.empty((n, p), dtype=torch.int8, device=device)
    out_boxes = torch.empty((n, p, d), dtype=torch.float32, device=device) if with_boxes else None
    classes = torch.empty((n, p), **i64) if want_classes else None
    status = torch.zeros((n,), dtype=torch.int32, device=device)
    ws_bytes = int(_C.lib().d2b_match_workspace_bytes(n, gmax, p))
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=device)
    c_thr = (C.c_double * len(thr))(*thr)
    c_lab = (C.c_int * len(lab))(*lab)
    with torch.cuda.device(device):
        check(_C.lib().d2b_match_boxes(ptr(gt), ptr(counts), n, gmax, ptr(pred), 0 if shared else pmax, ptr(pcounts), pmax,
                                       c_thr, len(thr), c_lab, flags, ptr(hw), float(boundary_thresh) if boundary else -1.0,
                                       ptr(gcls), int(num_classes if num_classes is not None else 0), ptr(matches),
                                       ptr(labels), ptr(out_boxes), ptr(classes), ptr(status), ptr(ws), ws_bytes,
                                       stream_ptr(device)), "match_boxes")
    return matches, labels, out_boxes, classes, status


def rpn_label_and_sample_anchors_fixed(anchors, gt_boxes: torch.Tensor, gt_count: torch.Tensor, matcher: Matcher,
                                       batch_size_per_image: int, positive_fraction: float, *, image_hw=None,
                                       boundary_thresh: float = -1.0, seed: Optional[torch.Tensor] = None):
    """RPN / RRPN.label_and_sample_anchors for all images with no host read (CUDA only, capturable in a CUDA graph):
    match_boxes_fixed, then ONE d2b_sample_labels in the RPN form instead of the per-image _subsample_labels.
    anchors [A, D] (or per-level list), gt_boxes [N, Gmax, D] with gt_count [N]; image_hw [N, 2] and boundary_thresh >= 0:
    the anchor boundary rule (axis-aligned only, as RRPN).  seed: [1] int64 device tensor (None: torch's CUDA generator).
    Returns (gt_labels [N, A] int8: 1 / 0 / -1, matched_gt_boxes [N, A, D], zeros for an image without GT), the inputs of
    losses.rpn_losses_fixed.  The sample follows the reference's law, not its randperm stream (sampling.py)."""
    from .sampling import sample_labels

    if isinstance(anchors, (list, tuple)):
        anchors = torch.cat(list(anchors), dim=0)
    if anchors.shape[-1] == 5 and boundary_thresh >= 0:  # as RRPN.__init__ (proposal_generator/rrpn.py:139-142)
        raise NotImplementedError("anchor_boundary_thresh is a legacy option not implemented for RRPN.")
    _, labels, boxes, _, _ = match_boxes_fixed(gt_boxes, gt_count, anchors, matcher, image_hw=image_hw,
                                               boundary_thresh=boundary_thresh)
    gt_labels, _, _ = sample_labels(labels, batch_size_per_image, positive_fraction, 0, seed=seed, rpn_labels=True)
    return gt_labels, boxes


def label_and_sample_proposals_fixed(proposals: torch.Tensor, proposal_count: Optional[torch.Tensor],
                                     gt_boxes: torch.Tensor, gt_count: torch.Tensor, gt_classes: torch.Tensor,
                                     matcher: Matcher, num_classes: int, batch_size_per_image: int,
                                     positive_fraction: float, *, proposal_append_gt: bool = True,
                                     seed: Optional[torch.Tensor] = None):
    """(R)ROIHeads.label_and_sample_proposals for all images with no host read (CUDA only, capturable in a CUDA graph):
    match_boxes_fixed, then ONE d2b_sample_labels on the classes instead of the per-image _sample_proposals.
    proposals [N, Pmax, D] with proposal_count [N] (device int64; None: all Pmax rows), gt_boxes [N, Gmax, D] with
    gt_count [N], gt_classes [N, Gmax] int64.  Returns (sampled_idx, gt_classes, matched_idx, proposal_boxes, gt_boxes,
    num_fg, num_bg), [N, B] unless noted, B = batch_size_per_image:
      sampled_idx    rows of the image's proposals ++ GT (GT row g at proposal_count[n] + g, match_boxes_fixed's layout);
      gt_classes     their classes (num_classes = background), matched_idx their matched GT (argmax over GT);
      proposal_boxes [N, B, D] the sampled rows' boxes, gt_boxes [N, B, D] their matched GT boxes (zeros without GT);
      num_fg, num_bg [N]: the sampled counts.  Foreground rows are the first num_fg[n] of each image's block.
    Rows past num_fg + num_bg are padding: index, class and match -1, NaN proposal box (ROIPooler pools it to zeros with no
    gradient), zero GT box.  The sample follows the reference's law, not its randperm stream (sampling.py)."""
    from .sampling import sample_labels

    matches, _, boxes, classes, _ = match_boxes_fixed(gt_boxes, gt_count, proposals, matcher, pred_count=proposal_count,
                                                      append_gt=proposal_append_gt, gt_classes=gt_classes,
                                                      num_classes=num_classes)
    sampled, num_fg, num_bg = sample_labels(classes, batch_size_per_image, positive_fraction, num_classes, seed=seed)
    n, pmax, d = proposals.shape
    if classes.shape[1] == 0:  # no rows to sample from: every sample row is padding (keeps the gathers in bounds)
        classes, matches, boxes = classes.new_full((n, 1), -1), matches.new_zeros((n, 1)), boxes.new_zeros((n, 1, d))
    valid = sampled >= 0
    idx = sampled.clamp(min=0)
    # the sampled row's source: proposal p < proposal_count, else GT p - proposal_count (rows of cat([proposals, gt]))
    if proposal_append_gt:
        pc = (proposal_count.to(torch.int64) if proposal_count is not None
              else torch.full((n,), pmax, dtype=torch.int64, device=proposals.device)).clamp(0, pmax)[:, None]
        src = torch.where(idx < pc, idx, pmax + idx - pc)
        rows = torch.cat([proposals.float(), gt_boxes.float()], dim=1)
    else:
        src, rows = idx, proposals.float()
    if rows.shape[1] == 0:  # nothing to sample from: every row is padding
        rows = rows.new_zeros((n, 1, d))
    src = src.clamp(max=rows.shape[1] - 1)
    prop = torch.where(valid[..., None], rows.gather(1, src[..., None].expand(-1, -1, d)), float("nan"))
    gtb = torch.where(valid[..., None], boxes.gather(1, idx[..., None].expand(-1, -1, d)), 0.0)
    return (sampled, torch.where(valid, classes.gather(1, idx), -1), torch.where(valid, matches.gather(1, idx), -1), prop,
            gtb, num_fg, num_bg)


def _fused(gt_boxes_list, preds, matcher, **kw):
    """match_boxes_fixed over lists + the one host read of the status (the reference's assertion)."""
    device = preds.device if isinstance(preds, torch.Tensor) else preds[0].device
    d = gt_boxes_list[0].shape[-1] if len(gt_boxes_list) and gt_boxes_list[0].dim() == 2 else (
        preds.shape[-1] if isinstance(preds, torch.Tensor) else preds[0].shape[-1])
    gt, counts = _pad(gt_boxes_list, d, device)
    if isinstance(preds, torch.Tensor):  # shared anchors
        out = match_boxes_fixed(gt, counts, preds, matcher, **kw)
    else:
        pred, pcounts = _pad(preds, d, device)
        out = match_boxes_fixed(gt, counts, pred, matcher, pred_count=pcounts, **kw)
    if bool(out[4].any()):  # the one host read before the sampling
        raise AssertionError("match_quality_matrix contains a negative or NaN IoU")
    return out


def _pad_classes(gt_classes, device):
    n = len(gt_classes)
    gmax = max([int(c.shape[0]) for c in gt_classes] + [0])
    out = torch.zeros((n, gmax), dtype=torch.int64, device=device)
    for i, c in enumerate(gt_classes):
        if c.shape[0]:
            out[i, : c.shape[0]] = c
    return out


# ----------------------------------------------------------------------------------------------- reference-shaped wrappers
def rpn_label_and_sample_anchors(anchors, gt_boxes: List[torch.Tensor], image_sizes, matcher: Matcher,
                                 anchor_boundary_thresh, batch_size_per_image: int, positive_fraction: float):
    """RPN.label_and_sample_anchors (rpn.py:307-363); RRPN's (rrpn.py:151-195) for [A, 5] anchors, which, like RRPN, refuse
    anchor_boundary_thresh >= 0.
    anchors: [A, D] tensor or a list of per-level tensors; gt_boxes: one [G_i, D] tensor per image.
    Returns (gt_labels, matched_gt_boxes), one [A] int8 and one [A, D] tensor per image."""
    if isinstance(anchors, (list, tuple)):
        anchors = torch.cat(list(anchors), dim=0)
    rotated = anchors.shape[-1] == 5
    if rotated and anchor_boundary_thresh >= 0:  # as RRPN.__init__ (proposal_generator/rrpn.py:139-142)
        raise NotImplementedError("anchor_boundary_thresh is a legacy option not implemented for RRPN.")
    use_boundary = anchor_boundary_thresh >= 0
    if anchors.is_cuda:
        _, labels, boxes, _, _ = _fused(gt_boxes, anchors, matcher, image_hw=image_sizes if use_boundary else None,
                                        boundary_thresh=anchor_boundary_thresh if use_boundary else -1.0)
        gt_labels, matched = [], []
        for i, gt_i in enumerate(gt_boxes):
            gt_labels.append(_rpn_subsample(labels[i].clone(), batch_size_per_image, positive_fraction))
            matched.append(boxes[i] if len(gt_i) else torch.zeros_like(anchors))
        return gt_labels, matched
    gt_labels, matched = [], []
    for image_size_i, gt_i in zip(image_sizes, gt_boxes):
        matched_idxs, gt_labels_i = matcher(_iou(gt_i, anchors))
        if use_boundary:
            gt_labels_i[~inside_box(anchors, image_size_i, anchor_boundary_thresh)] = -1
        gt_labels_i = _rpn_subsample(gt_labels_i, batch_size_per_image, positive_fraction)
        matched.append(torch.zeros_like(anchors) if len(gt_i) == 0 else gt_i[matched_idxs])
        gt_labels.append(gt_labels_i)
    return gt_labels, matched


def retinanet_label_anchors(anchors, gt_boxes: List[torch.Tensor], gt_classes: List[torch.Tensor], matcher: Matcher,
                            num_classes: int):
    """RetinaNet.label_anchors (meta_arch/retinanet.py:213-255).  Returns (gt_labels [A] int64, matched_gt_boxes [A, 4])
    per image."""
    if isinstance(anchors, (list, tuple)):
        anchors = torch.cat(list(anchors), dim=0)
    if anchors.is_cuda:
        _, _, boxes, classes, _ = _fused(gt_boxes, anchors, matcher, gt_classes=_pad_classes(gt_classes, anchors.device),
                                         num_classes=num_classes)
        return ([classes[i] for i in range(len(gt_boxes))],
                [boxes[i] if len(g) else torch.zeros_like(anchors) for i, g in enumerate(gt_boxes)])
    gt_labels, matched = [], []
    for gt_i, cls_i in zip(gt_boxes, gt_classes):
        matched_idxs, anchor_labels = matcher(_iou(gt_i, anchors))
        matched.append(gt_i[matched_idxs] if len(gt_i) else torch.zeros_like(anchors))
        gt_labels.append(_class_targets(matched_idxs, anchor_labels, cls_i, num_classes))
    return gt_labels, matched


def label_and_sample_proposals(proposal_boxes: List[torch.Tensor], gt_boxes: List[torch.Tensor],
                               gt_classes: List[torch.Tensor], matcher: Matcher, num_classes: int,
                               batch_size_per_image: int, positive_fraction: float, proposal_append_gt: bool = True):
    """ROIHeads.label_and_sample_proposals (roi_heads/roi_heads.py:220-302) and its rotated twin
    (rotated_fast_rcnn.py:218-270) up to the Instances indexing.  Returns per image (sampled_idxs into proposals ++ gt
    (proposals alone without proposal_append_gt), their gt_classes, their matched GT indices); a caller indexes its
    Instances with the first and its targets' gt_* fields with the third (meaningful when the image has GT)."""
    out = []
    if len(proposal_boxes) and proposal_boxes[0].is_cuda:
        device = proposal_boxes[0].device
        matches, _, _, classes, _ = _fused(gt_boxes, list(proposal_boxes), matcher, append_gt=proposal_append_gt,
                                           gt_classes=_pad_classes(gt_classes, device), num_classes=num_classes,
                                           with_boxes=False)
        for i, (p_i, g_i) in enumerate(zip(proposal_boxes, gt_boxes)):
            valid = int(p_i.shape[0]) + (int(g_i.shape[0]) if proposal_append_gt else 0)
            cls_i, m_i = classes[i, :valid], matches[i, :valid]
            fg, bg = subsample_labels(cls_i, batch_size_per_image, positive_fraction, num_classes)
            sampled = torch.cat([fg, bg], dim=0)
            out.append((sampled, cls_i[sampled], m_i[sampled]))
        return out
    for p_i, g_i, c_i in zip(proposal_boxes, gt_boxes, gt_classes):
        if proposal_append_gt:
            p_i = torch.cat([p_i, g_i.to(p_i.dtype)], dim=0)
        matched_idxs, matched_labels = matcher(_iou(g_i, p_i))
        cls = _class_targets(matched_idxs, matched_labels, c_i, num_classes)
        fg, bg = subsample_labels(cls, batch_size_per_image, positive_fraction, num_classes)
        sampled = torch.cat([fg, bg], dim=0)
        out.append((sampled, cls[sampled], matched_idxs[sampled]))
    return out


def cascade_match_and_label_boxes(proposal_boxes: List[torch.Tensor], gt_boxes: List[torch.Tensor],
                                  gt_classes: List[torch.Tensor], matcher: Matcher, num_classes: int):
    """CascadeROIHeads._match_and_label_boxes (roi_heads/cascade_rcnn.py:209-256) for one stage.  Returns per image
    (gt_classes [P] int64, gt_boxes [P, 4])."""
    out = []
    if len(proposal_boxes) and proposal_boxes[0].is_cuda:
        device = proposal_boxes[0].device
        matches, labels, boxes, classes, _ = _fused(gt_boxes, list(proposal_boxes), matcher,
                                                    gt_classes=_pad_classes(gt_classes, device), num_classes=num_classes)
        for i, (p_i, g_i) in enumerate(zip(proposal_boxes, gt_boxes)):
            k = int(p_i.shape[0])
            cls = classes[i, :k]
            if len(g_i) and -1 in matcher.labels:  # the cascade keeps gt_classes[match] for ignored proposals
                cls = torch.where(labels[i, :k] == -1, gt_classes[i].to(device)[matches[i, :k]], cls)
            out.append((cls, boxes[i, :k] if len(g_i) else boxes.new_zeros((k, p_i.shape[-1]))))
        return out
    for p_i, g_i, c_i in zip(proposal_boxes, gt_boxes, gt_classes):
        matched_idxs, proposal_labels = matcher(_iou(g_i, p_i))
        if len(g_i) > 0:
            cls = _class_targets(matched_idxs, proposal_labels, c_i, num_classes, ignore=False)
            boxes = g_i[matched_idxs]
        else:
            cls = torch.zeros_like(matched_idxs) + num_classes
            boxes = g_i.new_zeros((len(p_i), p_i.shape[-1]))
        out.append((cls, boxes))
    return out
