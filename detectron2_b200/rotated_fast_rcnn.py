"""fast_rcnn_inference_rotated -- batched rotated Fast R-CNN inference post-processing, same results as
detectron2/modeling/roi_heads/rotated_fast_rcnn.py:46-132 (`fast_rcnn_inference_rotated`,
`fast_rcnn_inference_single_image_rotated`).

The reference processes one image at a time: boolean row filtering, `RotatedBoxes.clip` (a `torch.where(...)[0]` host
sync), `nonzero()` on the R x K score matrix (another sync), one `batched_nms_rotated`, slicing.  Here every image of the
batch goes through ONE rotated NMS, exactly like `fast_rcnn_inference.fast_rcnn_inference`:

  * `d2b_frcnn_rotated_prepare` (one CTA per image) drops the non-finite rows, compacts the (row, class) pairs with
    score > score_thresh IN ROW-MAJOR ORDER into `CAP` slots per image, normalises the angles and clips the boxes, and adds
    batched_nms_rotated's offsets class * (max - min + 1) over the image's candidates to the centres;
  * one `d2b_nms(D2B_NMS_ROTATED | D2B_NMS_NO_OFFSET)` with category image * (K + 1) + class, empty slots -1 (ignored);
  * `d2b_rpn_select_rotated` hands every image the first `topk_per_image` entries of the score-ordered keep list.
An image whose candidates overflow CAP is recomputed with the exact (synchronising) candidate list.  CPU tensors take the
same selection written with torch ops (`_fast_rcnn_inference_rotated_host`).
"""
from typing import List, Tuple

import torch

from . import ops
from .fast_rcnn_inference import CANDIDATE_CAP, Detections
from .rrpn import clip_rotated, rotated_offset_scale

__all__ = ["fast_rcnn_inference_rotated", "fast_rcnn_inference_single_image_rotated", "fast_rcnn_inference_rotated_fixed"]


def _single_image_exact(boxes, scores, image_shape, score_thresh, nms_thresh, topk_per_image):
    """Reference structure (rotated_fast_rcnn.py:98-132) on top of our NMS; data-dependent shapes, hence host syncs.
    Used only for images whose candidate count exceeds the candidate slots."""
    valid = torch.isfinite(boxes).all(dim=1) & torch.isfinite(scores).all(dim=1)
    if not bool(valid.all()):
        boxes, scores = boxes[valid], scores[valid]
    scores = scores[:, :-1]
    k = boxes.shape[1] // 5
    boxes = clip_rotated(boxes.reshape(-1, 5).float(), float(image_shape[0]), float(image_shape[1])).view(-1, k, 5)
    filter_mask = scores > score_thresh
    filter_inds = filter_mask.nonzero()
    boxes = boxes[filter_inds[:, 0], 0] if k == 1 else boxes[filter_mask]
    scores = scores[filter_mask]
    # batched_nms_rotated with the offsets applied here, as the batched path does: one segment per class, or one for the
    # whole image when IoU 0 passes the threshold
    cls = filter_inds[:, 1]
    live = torch.ones_like(scores, dtype=torch.bool)
    off = cls.to(torch.float32) * rotated_offset_scale(boxes[None], live[None])[0]
    nms_boxes = torch.cat([boxes[:, :2] + off[:, None], boxes[:, 2:]], dim=1)
    seg = torch.zeros_like(cls) if float(nms_thresh) <= 0.0 else cls
    keep, num_keep = ops.nms_fixed(nms_boxes, scores, seg, float(nms_thresh), True, apply_offsets=False)
    keep = keep[: int(num_keep.item())]
    if topk_per_image >= 0:
        keep = keep[:topk_per_image]
    return Detections(image_shape, boxes[keep], scores[keep], filter_inds[keep, 1]), filter_inds[keep, 0]


def fast_rcnn_inference_rotated_fixed(boxes: List[torch.Tensor], scores: List[torch.Tensor], image_shapes,
                                      score_thresh: float, nms_thresh: float, topk_per_image: int, cap: int = 0):
    """Sync-free, fixed-capacity form (CUDA tensors only, at most D2B_MAX_IMAGES images).  Returns a dict of device
    tensors: `boxes` [N, topk, 5], `scores` / `classes` / `rows` [N, topk] (rows = index among the image's valid rows),
    `counts` [N] and `n_cand` [N] (an image with n_cand > cap overflowed its candidate slots and must be redone exactly).
    `image_shapes` is a list of (h, w) or an [N, 2] CUDA tensor.  Static shapes: capturable in a CUDA graph."""
    import ctypes as C

    from . import _C
    from ._C import check, ptr, stream_ptr

    n = len(boxes)
    device = boxes[0].device
    _C.require_cuda(*boxes, *scores)
    if n > _C.MAX_IMAGES:
        raise RuntimeError("fast_rcnn_inference_rotated_fixed: at most %d images per call" % _C.MAX_IMAGES)
    ncls = scores[0].shape[1] - 1
    kreg = boxes[0].shape[1] // 5
    rcounts = [int(b.shape[0]) for b in boxes]
    starts = [0]
    for r in rcounts:
        starts.append(starts[-1] + r)
    all_b = (boxes[0] if n == 1 else torch.cat(boxes, dim=0)).float().contiguous()
    all_s = (scores[0] if n == 1 else torch.cat(scores, dim=0)).float().contiguous()
    cap = int(cap) if cap else min(CANDIDATE_CAP, max(rcounts + [0]) * ncls)
    topk = int(topk_per_image) if topk_per_image >= 0 else cap
    if isinstance(image_shapes, torch.Tensor):
        hw = image_shapes.to(device=device, dtype=torch.float32).contiguous()
    else:
        hw = torch.tensor([[float(h), float(w)] for (h, w) in image_shapes], dtype=torch.float32).to(device)
    m = n * cap
    f32 = dict(dtype=torch.float32, device=device)
    i64 = dict(dtype=torch.int64, device=device)
    cand_boxes, nms_boxes = torch.empty((m, 5), **f32), torch.empty((m, 5), **f32)
    nms_scores, raw_scores = torch.empty((m,), **f32), torch.empty((m,), **f32)
    cand_flat, cat_ids = torch.empty((m,), **i64), torch.empty((m,), **i64)
    n_cand = torch.zeros((n,), **i64)
    row_map = torch.empty((starts[-1],), **i64)
    out_boxes = torch.zeros((n, topk, 5), **f32)
    out_scores = torch.zeros((n, topk), **f32)
    out_index = torch.zeros((n, topk), **i64)
    counts = torch.zeros((n,), **i64)
    rs = (C.c_int * (n + 1))(*starts)
    # IoU 0 passes a threshold <= 0: the reference's one NMS per image then suppresses across classes as well
    per_image = float(nms_thresh) <= 0.0
    with torch.cuda.device(device):
        check(_C.lib().d2b_frcnn_rotated_prepare(ptr(all_b), ptr(all_s), rs, n, ncls, kreg, ptr(hw), float(score_thresh), cap,
                                                 int(per_image), ptr(cand_boxes), ptr(nms_boxes), ptr(nms_scores),
                                                 ptr(raw_scores), ptr(cand_flat), ptr(cat_ids), ptr(n_cand), ptr(row_map),
                                                 stream_ptr(device)), "frcnn_rotated_prepare")
        if m and topk:
            # an (image, class) category holds at most one candidate per proposal row; an image segment at most `cap`
            max_segment = cap if per_image else max(min(cap, max(rcounts)), 1)
            keep, num_keep = ops.nms_fixed(nms_boxes, nms_scores, cat_ids, float(nms_thresh), True, apply_offsets=False,
                                           max_segment=max_segment)
            check(_C.lib().d2b_rpn_select_rotated(ptr(keep), ptr(num_keep), n, cap, topk, ptr(cand_boxes), ptr(raw_scores),
                                                  ptr(cat_ids), ptr(out_boxes), ptr(out_scores), ptr(out_index),
                                                  ptr(counts), stream_ptr(device)), "frcnn_rotated_select")
    flat = cand_flat[out_index.reshape(-1)].reshape(n, topk) if m else out_index
    rows_local = torch.div(flat, ncls, rounding_mode="floor")
    classes = flat - rows_local * ncls
    # index of the kept rows among the image's valid rows (padded entries clamped into the image's own rows)
    rows = torch.stack([row_map[starts[j]:starts[j + 1]][rows_local[j].clamp(max=rcounts[j] - 1)] if rcounts[j] else rows_local[j]
                        for j in range(n)]) if n else rows_local
    return {"boxes": out_boxes, "scores": out_scores, "classes": classes, "rows": rows, "counts": counts, "n_cand": n_cand,
            "cap": cap}


def fast_rcnn_inference_rotated(boxes: List[torch.Tensor], scores: List[torch.Tensor], image_shapes: List[Tuple[int, int]],
                                score_thresh: float, nms_thresh: float, topk_per_image: int):
    """boxes[i]: R_i x (K*5) or R_i x 5 predicted rotated boxes, scores[i]: R_i x (K+1) class scores (last = background).
    Returns (list[Detections], list[Tensor of kept row indices]) exactly like the reference."""
    if not boxes[0].is_cuda:
        return _fast_rcnn_inference_rotated_host(boxes, scores, image_shapes, score_thresh, nms_thresh, topk_per_image)
    from . import _C

    results, kept_rows = [], []
    for i0 in range(0, len(boxes), _C.MAX_IMAGES):  # chunks of the ABI's image bound
        sl = slice(i0, i0 + _C.MAX_IMAGES)
        out = fast_rcnn_inference_rotated_fixed(boxes[sl], scores[sl], image_shapes[sl], score_thresh, nms_thresh,
                                                topk_per_image)
        stats = torch.stack([out["counts"], out["n_cand"]], dim=1).tolist()  # the one host sync: exactly-sized results
        dt = scores[i0].dtype
        for j, (c, n_cand) in enumerate(stats):
            i = i0 + j
            if n_cand > out["cap"]:  # candidate list was truncated: redo this image exactly (rare)
                det, rows_i = _single_image_exact(boxes[i], scores[i], image_shapes[i], score_thresh, nms_thresh,
                                                  topk_per_image)
            else:
                det = Detections(image_shapes[i], out["boxes"][j, :c], out["scores"][j, :c].to(dt), out["classes"][j, :c])
                rows_i = out["rows"][j, :c]
            results.append(det)
            kept_rows.append(rows_i)
    return results, kept_rows


def _fast_rcnn_inference_rotated_host(boxes: List[torch.Tensor], scores: List[torch.Tensor],
                                      image_shapes: List[Tuple[int, int]], score_thresh: float, nms_thresh: float,
                                      topk_per_image: int):
    """The same selection written with torch ops: top-`CAP` pairs per image by one `topk` (score -inf for non-candidates)
    re-sorted by flat index = the reference's row-major candidate order.  Host-logic restatement pinned to the real
    reference function by tests/test_rotated_inference_host.py (NMS replaced by the oracle); the CUDA path is the product."""
    num_images = len(boxes)
    device = boxes[0].device
    ncls = scores[0].shape[1] - 1
    kreg = boxes[0].shape[1] // 5
    per_image = float(nms_thresh) <= 0.0
    cand_boxes, nms_boxes_l, cand_scores, cand_cat, cand_flat, cand_live, n_cand_l, row_maps = [], [], [], [], [], [], [], []
    caps = []
    for i in range(num_images):
        b, s = boxes[i].float(), scores[i]
        r = b.shape[0]
        cap = min(CANDIDATE_CAP, r * ncls)  # 0 for an image without proposals
        caps.append(cap)
        row_valid = torch.isfinite(b).all(dim=1) & torch.isfinite(s).all(dim=1)
        # index of a row among the valid rows (what the reference returns after `boxes = boxes[valid_mask]`)
        row_maps.append(torch.cumsum(row_valid.to(torch.int64), dim=0) - 1)
        fg = s[:, :-1]
        cand = (fg > score_thresh) & row_valid[:, None]
        masked = torch.where(cand, fg.float(), torch.full_like(fg, float("-inf"), dtype=torch.float32)).reshape(-1)
        n_cand_l.append(cand.sum())
        top_s, top_f = torch.topk(masked, cap)
        top_f, order = torch.sort(top_f)  # back to row-major candidate order (ties inside NMS follow it)
        top_s = top_s[order]
        live = top_s > float("-inf")
        rows = torch.div(top_f, ncls, rounding_mode="floor")
        cls = top_f - rows * ncls
        clipped = clip_rotated(b.reshape(-1, 5), float(image_shapes[i][0]), float(image_shapes[i][1])).view(r, kreg, 5)
        cb = clipped[rows, 0] if kreg == 1 else clipped[rows, cls]
        cb = torch.where(live[:, None], cb, torch.zeros_like(cb))
        # batched_nms_rotated offsets of this image: class * (max - min + 1) over its candidates, fp32, on the centres
        off = cls.to(torch.float32) * rotated_offset_scale(cb[None], live[None])[0]
        nb = torch.cat([cb[:, :2] + off[:, None], cb[:, 2:]], dim=1)
        nms_boxes_l.append(torch.where(live[:, None], nb, torch.zeros_like(nb)))
        cand_boxes.append(cb)
        cand_scores.append(torch.where(live, top_s, torch.full_like(top_s, float("-inf"))))
        seg = torch.full_like(cls, i) if per_image else cls + i * (ncls + 1)
        cand_cat.append(torch.where(live, seg, torch.full_like(cls, -1)))  # -1: slot ignored by the NMS kernels
        cand_flat.append(top_f)
        cand_live.append(live)
    all_boxes = torch.cat(cand_boxes, dim=0)
    nms_boxes = torch.cat(nms_boxes_l, dim=0)
    all_scores = torch.cat(cand_scores, dim=0)
    all_cat = torch.cat(cand_cat, dim=0)
    all_live = torch.cat(cand_live, dim=0)
    img_of = torch.cat([torch.full((caps[i],), i, dtype=torch.int64, device=device) for i in range(num_images)])
    # an (image, class) category holds at most one candidate per proposal row; an image segment at most its slots
    max_segment = max([caps[i] if per_image else min(caps[i], boxes[i].shape[0]) for i in range(num_images)] + [1])
    keep, num_keep = ops.nms_fixed(nms_boxes, all_scores, all_cat, float(nms_thresh), True, apply_offsets=False,
                                   max_segment=max_segment)

    # per-image first topk of the score-ordered keep list, on the device
    m = keep.shape[0]
    topk = topk_per_image if topk_per_image >= 0 else m
    ar = torch.arange(num_images, device=device)
    kidx = torch.where(torch.arange(m, device=device) < num_keep, keep, torch.zeros_like(keep))
    kok = (torch.arange(m, device=device) < num_keep) & all_live[kidx]
    onehot = (img_of[kidx][None, :] == ar[:, None]) & kok[None, :]
    rank = torch.cumsum(onehot.to(torch.int32), dim=1) - 1
    sel = onehot & (rank < topk)
    counts = sel.sum(dim=1)
    out_idx = torch.zeros((num_images, topk + 1), dtype=torch.int64, device=device)
    col = torch.where(sel, rank.long(), torch.full_like(rank, topk, dtype=torch.int64))
    out_idx.scatter_(1, col, kidx[None, :].expand(num_images, m))
    out_idx = out_idx[:, :topk]

    stats = torch.stack([counts, torch.stack(n_cand_l).to(counts.dtype)], dim=1).tolist()  # the one host sync
    flat_all = torch.cat(cand_flat, dim=0)
    results, kept_rows = [], []
    for i in range(num_images):
        c, n_cand = stats[i]
        if n_cand > caps[i]:  # candidate list was truncated: redo this image exactly (rare)
            det, rows_i = _single_image_exact(boxes[i], scores[i], image_shapes[i], score_thresh, nms_thresh, topk_per_image)
            results.append(det)
            kept_rows.append(rows_i)
            continue
        sel_i = out_idx[i, :c]
        f = flat_all[sel_i]
        rows = torch.div(f, ncls, rounding_mode="floor")
        results.append(Detections(image_shapes[i], all_boxes[sel_i], scores[i][:, :-1].reshape(-1)[f], f - rows * ncls))
        kept_rows.append(row_maps[i][rows])
    return results, kept_rows


def fast_rcnn_inference_single_image_rotated(boxes, scores, image_shape, score_thresh: float, nms_thresh: float,
                                             topk_per_image: int):
    """Single-image form with the reference's signature (rotated_fast_rcnn.py:84-86)."""
    res, rows = fast_rcnn_inference_rotated([boxes], [scores], [image_shape], score_thresh, nms_thresh, topk_per_image)
    return res[0], rows[0]
