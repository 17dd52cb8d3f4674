"""fast_rcnn_inference -- batched Fast R-CNN inference post-processing (SURVEY 8f-2), same results as
detectron2/modeling/roi_heads/fast_rcnn.py:46-173 (`fast_rcnn_inference`, `fast_rcnn_inference_single_image`).

The reference processes one image at a time: boolean row filtering, `nonzero()` on the R x K score matrix (host
sync), one `batched_nms`, slicing.  Here every image of the batch goes through ONE NMS pipeline and there is a single
host synchronisation (the read of the per-image output lengths):

  * candidates are the (row, class) pairs with score > score_thresh; instead of `nonzero()` one kernel
    (`d2b_frcnn_prepare`, one CTA per image) drops the non-finite rows, compacts the pairs IN ROW-MAJOR ORDER (the
    reference's order; it decides ties inside NMS) into `CAP` slots per image, clips the boxes and applies the NMS
    coordinate offsets.  The candidate count is checked on the device and read with the output lengths; an image that
    overflowed CAP is recomputed with the exact (synchronising) candidate list;
  * NMS category = image * (K + 1) + class with the per-image fp32 coordinate offsets of torchvision's
    `batched_nms` reproduced exactly (`D2B_NMS_NO_OFFSET`), empty candidate slots carry category -1 (ignored);
  * `d2b_rpn_select` hands every image the first `topk_per_image` entries of the score-ordered keep list.
Launch sequence for the whole batch: prepare, memset + 3 NMS kernels, select, two small gathers.  CPU tensors take the
same selection written with torch ops (`_fast_rcnn_inference_host`, the host-logic restatement pinned by the CPU tests).

With `rotated=True` the same functions are rotated Fast R-CNN inference (detectron2/modeling/roi_heads/rotated_fast_rcnn.py:
46-132, whose public names live in `rotated_fast_rcnn.py`): 5-wide boxes, `D2B_SELECT_ROTATED` for `d2b_frcnn_prepare`
(RotatedBoxes.clip and batched_nms_rotated's offsets class * (max - min + 1) on the centres) and `d2b_rpn_select`,
`D2B_NMS_ROTATED`, and for a threshold <= 0, which IoU 0 passes, `D2B_SELECT_SEG_PER_IMAGE`: one NMS segment per image (the
reference's one NMS per image then suppresses across classes too).
"""
from typing import List, Tuple

import torch

from . import ops
from ._batched_select import first_k_per_image, image_hw, nms_select
from .rrpn import clip_rotated, rotated_offset_scale

__all__ = ["fast_rcnn_inference", "fast_rcnn_inference_single_image", "Detections"]

CANDIDATE_CAP = 8192  # candidates per image taken without a host sync (the reference's typical count is a few thousand)


class Detections:
    """Minimal stand-in for detectron2.structures.Instances with the three fields this function produces."""

    def __init__(self, image_size, pred_boxes: torch.Tensor, scores: torch.Tensor, pred_classes: torch.Tensor):
        self.image_size = image_size
        self.pred_boxes = pred_boxes
        self.scores = scores
        self.pred_classes = pred_classes

    def __len__(self):
        return self.pred_boxes.shape[0]


def _clip(boxes: torch.Tensor, h: float, w: float) -> torch.Tensor:  # Boxes.clip (structures/boxes.py)
    b = boxes.reshape(-1, 4)
    x1 = b[:, 0].clamp(min=0, max=w)
    y1 = b[:, 1].clamp(min=0, max=h)
    x2 = b[:, 2].clamp(min=0, max=w)
    y2 = b[:, 3].clamp(min=0, max=h)
    return torch.stack([x1, y1, x2, y2], dim=1)


def _single_image_exact(boxes, scores, image_shape, score_thresh, nms_thresh, topk_per_image, rotated=False):
    """Reference structure (fast_rcnn.py:117-173, rotated_fast_rcnn.py:98-132) on top of our NMS; data-dependent shapes,
    hence host syncs.  Used only for images whose candidate count exceeds the candidate slots."""
    valid = torch.isfinite(boxes).all(dim=1) & torch.isfinite(scores).all(dim=1)
    if not bool(valid.all()):
        boxes, scores = boxes[valid], scores[valid]
    scores = scores[:, :-1]
    d = 5 if rotated else 4
    k = boxes.shape[1] // d
    h, w = float(image_shape[0]), float(image_shape[1])
    boxes = (clip_rotated(boxes.reshape(-1, 5).float(), h, w) if rotated else _clip(boxes, h, w)).view(-1, k, d)
    filter_mask = scores > score_thresh
    filter_inds = filter_mask.nonzero()
    boxes = boxes[filter_inds[:, 0], 0] if k == 1 else boxes[filter_mask]
    scores = scores[filter_mask]
    cls = filter_inds[:, 1]
    if rotated:
        # batched_nms_rotated with the offsets applied here, as the batched path does: one segment per class, or one for
        # the whole image when IoU 0 passes the threshold
        live = torch.ones_like(scores, dtype=torch.bool)
        off = cls.to(torch.float32) * rotated_offset_scale(boxes[None], live[None])[0]
        nms_boxes = torch.cat([boxes[:, :2] + off[:, None], boxes[:, 2:]], dim=1)
        seg = torch.zeros_like(cls) if float(nms_thresh) <= 0.0 else cls
        keep, num_keep = ops.nms_fixed(nms_boxes, scores, seg, float(nms_thresh), True, apply_offsets=False)
        keep = keep[: int(num_keep.item())]
    else:
        from .layers import batched_nms

        keep = batched_nms(boxes, scores, cls, nms_thresh)
    if topk_per_image >= 0:
        keep = keep[:topk_per_image]
    return Detections(image_shape, boxes[keep], scores[keep], filter_inds[keep, 1]), filter_inds[keep, 0]


def fast_rcnn_inference_fixed(boxes: List[torch.Tensor], scores: List[torch.Tensor], image_shapes, score_thresh: float,
                              nms_thresh: float, topk_per_image: int, cap: int = 0, *, rotated: bool = False):
    """Sync-free, fixed-capacity form (CUDA tensors only, at most D2B_MAX_IMAGES images).  Returns a dict of device
    tensors: `boxes` [N, topk, 4] (5 with `rotated`), `scores` / `classes` / `rows` [N, topk] (rows = index among the
    image's valid rows), `counts` [N] and `n_cand` [N] (an image with n_cand > cap overflowed its candidate slots and must
    be redone exactly).  `image_shapes` is a list of (h, w) or an [N, 2] CUDA tensor.  Static shapes: capturable."""
    import ctypes as C

    from . import _C
    from ._C import check, ptr, stream_ptr

    n = len(boxes)
    device = boxes[0].device
    _C.require_cuda(*boxes, *scores)
    if n > _C.MAX_IMAGES:
        raise RuntimeError("fast_rcnn_inference_fixed: at most %d images per call" % _C.MAX_IMAGES)
    d = 5 if rotated else 4
    ncls = scores[0].shape[1] - 1
    kreg = boxes[0].shape[1] // d
    rcounts = [int(b.shape[0]) for b in boxes]
    starts = [0]
    for r in rcounts:
        starts.append(starts[-1] + r)
    all_b = (boxes[0] if n == 1 else torch.cat(boxes, dim=0)).float().contiguous()
    all_s = (scores[0] if n == 1 else torch.cat(scores, dim=0)).float().contiguous()
    cap = int(cap) if cap else min(CANDIDATE_CAP, max(rcounts + [0]) * ncls)
    topk = int(topk_per_image) if topk_per_image >= 0 else cap
    hw = image_hw(image_shapes, device)
    m = n * cap
    f32 = dict(dtype=torch.float32, device=device)
    i64 = dict(dtype=torch.int64, device=device)
    cand_boxes, nms_boxes = torch.empty((m, d), **f32), torch.empty((m, d), **f32)
    nms_scores, raw_scores = torch.empty((m,), **f32), torch.empty((m,), **f32)
    cand_flat, cat_ids = torch.empty((m,), **i64), torch.empty((m,), **i64)
    n_cand = torch.zeros((n,), **i64)
    row_map = torch.empty((starts[-1],), **i64)
    rs = (C.c_int * (n + 1))(*starts)
    per_image = rotated and float(nms_thresh) <= 0.0
    flags = (_C.SELECT_ROTATED if rotated else 0) | (_C.SELECT_SEG_PER_IMAGE if per_image else 0)
    with torch.cuda.device(device):
        check(_C.lib().d2b_frcnn_prepare(ptr(all_b), ptr(all_s), rs, n, ncls, kreg, ptr(hw), float(score_thresh), cap, flags,
                                         ptr(cand_boxes), ptr(nms_boxes), ptr(nms_scores), ptr(raw_scores), ptr(cand_flat),
                                         ptr(cat_ids), ptr(n_cand), ptr(row_map), stream_ptr(device)), "frcnn_prepare")
    # an (image, class) category holds at most one candidate per proposal row; an image segment at most `cap`
    max_segment = cap if per_image else max(min(cap, max(rcounts + [0])), 1)
    out_boxes, out_scores, out_index, counts = nms_select(nms_boxes, nms_scores, cat_ids, cand_boxes, raw_scores, n, cap,
                                                          topk, nms_thresh, rotated, max_segment)
    flat = cand_flat[out_index.reshape(-1)].reshape(n, topk) if m else out_index
    rows_local = torch.div(flat, ncls, rounding_mode="floor")
    classes = flat - rows_local * ncls
    # index of the kept rows among the image's valid rows (no host-built offsets: the sequence stays graph-capturable)
    # (padded entries point at candidate 0, possibly another image's: clamp into the image's own rows)
    rows = torch.stack([row_map[starts[j]:starts[j + 1]][rows_local[j].clamp(max=rcounts[j] - 1)] if rcounts[j] else rows_local[j]
                        for j in range(n)]) if n else rows_local
    return {"boxes": out_boxes, "scores": out_scores, "classes": classes, "rows": rows, "counts": counts, "n_cand": n_cand,
            "cap": cap}


def fast_rcnn_inference(boxes: List[torch.Tensor], scores: List[torch.Tensor], image_shapes: List[Tuple[int, int]],
                        score_thresh: float, nms_thresh: float, topk_per_image: int, *, rotated: bool = False):
    """boxes[i]: R_i x (K*4) or R_i x 4 predicted boxes (K*5 or 5 rotated boxes with `rotated`), scores[i]: R_i x (K+1)
    class scores (last = background).  Returns (list[Detections], list[Tensor of kept row indices]) exactly like the
    reference."""
    if not boxes[0].is_cuda:
        return _fast_rcnn_inference_host(boxes, scores, image_shapes, score_thresh, nms_thresh, topk_per_image,
                                         rotated=rotated)
    from . import _C

    results, kept_rows = [], []
    for i0 in range(0, len(boxes), _C.MAX_IMAGES):  # chunks of the ABI's image bound
        sl = slice(i0, i0 + _C.MAX_IMAGES)
        out = fast_rcnn_inference_fixed(boxes[sl], scores[sl], image_shapes[sl], score_thresh, nms_thresh, topk_per_image,
                                        rotated=rotated)
        stats = torch.stack([out["counts"], out["n_cand"]], dim=1).tolist()  # the one host sync: exactly-sized results
        dt = scores[i0].dtype
        for j, (c, n_cand) in enumerate(stats):
            i = i0 + j
            if n_cand > out["cap"]:  # candidate list was truncated: redo this image exactly (rare)
                det, rows_i = _single_image_exact(boxes[i], scores[i], image_shapes[i], score_thresh, nms_thresh,
                                                  topk_per_image, rotated)
            else:
                det = Detections(image_shapes[i], out["boxes"][j, :c], out["scores"][j, :c].to(dt), out["classes"][j, :c])
                rows_i = out["rows"][j, :c]
            results.append(det)
            kept_rows.append(rows_i)
    return results, kept_rows


def _fast_rcnn_inference_host(boxes: List[torch.Tensor], scores: List[torch.Tensor], image_shapes: List[Tuple[int, int]],
                              score_thresh: float, nms_thresh: float, topk_per_image: int, *, rotated: bool = False):
    """The same selection written with torch ops: top-`CAP` pairs per image by one `topk` (score -inf for non-candidates)
    re-sorted by flat index = the reference's row-major candidate order.  Host-logic restatement pinned to the real
    reference functions by tests/test_host_logic_cpu.py and tests/test_rotated_inference_host.py (NMS replaced by the
    oracle); the CUDA path above is the product."""
    num_images = len(boxes)
    device = boxes[0].device
    d = 5 if rotated else 4
    ncls = scores[0].shape[1] - 1
    kreg = boxes[0].shape[1] // d
    per_image = rotated and float(nms_thresh) <= 0.0
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
        h, w = float(image_shapes[i][0]), float(image_shapes[i][1])
        clipped = (clip_rotated(b.reshape(-1, 5), h, w) if rotated else _clip(b, h, w)).view(r, kreg, d)
        cb = clipped[rows, 0] if kreg == 1 else clipped[rows, cls]
        cb = torch.where(live[:, None], cb, torch.zeros_like(cb))
        if rotated:  # batched_nms_rotated offsets of this image: class * (max - min + 1) over its candidates, on the centres
            off = cls.to(torch.float32) * rotated_offset_scale(cb[None], live[None])[0]
            nb = torch.cat([cb[:, :2] + off[:, None], cb[:, 2:]], dim=1)
        else:  # torchvision batched_nms offsets of this image: class * (max coordinate of its candidate boxes + 1), fp32
            if cap > 0:
                mx = torch.where(live[:, None], cb, torch.full_like(cb, float("-inf"))).max()
                mx = torch.where(torch.isfinite(mx), mx, torch.zeros_like(mx))
            else:
                mx = torch.zeros((), dtype=torch.float32, device=device)
            nb = cb + torch.where(live, cls.to(torch.float32) * (mx + 1.0), torch.zeros_like(top_s))[:, None]
        nms_boxes_l.append(torch.where(live[:, None], nb, torch.zeros_like(nb)))
        cand_boxes.append(cb)
        cand_scores.append(torch.where(live, top_s, torch.full_like(top_s, float("-inf"))))
        seg = torch.full_like(cls, i) if per_image else cls + i * (ncls + 1)
        cand_cat.append(torch.where(live, seg, torch.full_like(cls, -1)))  # -1: slot ignored by the NMS kernels
        cand_flat.append(top_f)
        cand_live.append(live)
    all_boxes = torch.cat(cand_boxes, dim=0)
    img_of = torch.cat([torch.full((caps[i],), i, dtype=torch.int64, device=device) for i in range(num_images)])
    # an (image, class) category holds at most one candidate per proposal row; an image segment at most its slots
    max_segment = max([caps[i] if per_image else min(caps[i], boxes[i].shape[0]) for i in range(num_images)] + [1])
    keep, num_keep = ops.nms_fixed(torch.cat(nms_boxes_l, dim=0), torch.cat(cand_scores, dim=0), torch.cat(cand_cat, dim=0),
                                   float(nms_thresh), rotated, apply_offsets=False, max_segment=max_segment)

    # per-image first topk of the score-ordered keep list, on the device
    topk = topk_per_image if topk_per_image >= 0 else keep.shape[0]
    out_idx, counts = first_k_per_image(keep, num_keep, img_of, torch.cat(cand_live, dim=0), num_images, topk)

    stats = torch.stack([counts, torch.stack(n_cand_l).to(counts.dtype)], dim=1).tolist()  # the one host sync
    flat_all = torch.cat(cand_flat, dim=0)
    results, kept_rows = [], []
    for i in range(num_images):
        c, n_cand = stats[i]
        if n_cand > caps[i]:  # candidate list was truncated: redo this image exactly (rare)
            det, rows_i = _single_image_exact(boxes[i], scores[i], image_shapes[i], score_thresh, nms_thresh, topk_per_image,
                                              rotated)
            results.append(det)
            kept_rows.append(rows_i)
            continue
        sel_i = out_idx[i, :c]
        f = flat_all[sel_i]
        rows = torch.div(f, ncls, rounding_mode="floor")
        results.append(Detections(image_shapes[i], all_boxes[sel_i], scores[i][:, :-1].reshape(-1)[f], f - rows * ncls))
        kept_rows.append(row_maps[i][rows])
    return results, kept_rows


def fast_rcnn_inference_single_image(boxes, scores, image_shape, score_thresh: float, nms_thresh: float,
                                     topk_per_image: int):
    """Single-image form with the reference's signature (fast_rcnn.py:117-124)."""
    res, rows = fast_rcnn_inference([boxes], [scores], [image_shape], score_thresh, nms_thresh, topk_per_image)
    return res[0], rows[0]
