"""Panoptic FPN inference: semantic labels and the thing / stuff combine for all images, on two native entry points.

  * `sem_seg_labels` -- sem_seg_postprocess (modeling/postprocessing.py:77-100) followed by argmax(dim=0), as
    PanopticFPN.inference and SemanticSegmentor use it.  The reference materialises the bilinearly resized C x H x W fp32
    map (230 MB at 54 x 800 x 1333) and reads it back for the argmax; `d2b_sem_seg_labels` evaluates the resize channel by
    channel inside the argmax, one launch for the batch.
  * `combine_semantic_and_instance_outputs` / `..._fixed` -- panoptic_fpn.py:184-269.  The reference walks the instances
    in a Python loop with up to five `.item()` host reads and several full-image launches per instance, then one more host
    read per semantic label.  `d2b_panoptic_combine` does the whole batch in four launches without a host read; the
    reference-shaped wrapper reads the segment table back once to build its dicts.
  * `panoptic_fpn_postprocess` -- the per-image loop of PanopticFPN.inference (panoptic_fpn.py:159-179) for all images.

Instance order: ascending -score, a NaN score last, ties to the lower index (the reference's argsort is not stable).
CPU tensors take `_sem_seg_labels_host` / `_combine_host`, the same computation written with torch ops; run on CUDA
tensors they are the reference the GPU tests compare the kernels against.
"""
import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import torch
from torch.nn import functional as F

from . import _C
from ._C import check, ptr, stream_ptr
from .postprocessing import detector_postprocess

Tensor = torch.Tensor

__all__ = ["sem_seg_labels", "combine_semantic_and_instance_outputs", "combine_semantic_and_instance_outputs_fixed",
           "panoptic_fpn_postprocess", "sem_seg_labels_op", "panoptic_combine_op", "PANOPTIC_MAX_INSTANCES",
           "PANOPTIC_MAX_CLASSES"]

PANOPTIC_MAX_INSTANCES = 4096  # D2B_PANOPTIC_MAX_INSTANCES
PANOPTIC_MAX_CLASSES = 1024    # D2B_PANOPTIC_MAX_CLASSES
STATUS_BAD_LABEL = 1           # D2B_PANOPTIC_STATUS_BAD_LABEL
SEG_FIELDS = 5                 # seg_info columns: id, isthing, category, instance, area


# ---- semantic labels ------------------------------------------------------------------------------------------------
@torch.library.custom_op("d2b200::sem_seg_labels", mutates_args=(), device_types="cuda")
def sem_seg_labels_op(logits: Tensor, image_sizes: List[int], output_sizes: List[int]) -> List[Tensor]:
    """logits [N, C, Hp, Wp] (fp32 / fp16 / bf16); image_sizes / output_sizes: (h, w) pairs flattened, one per image.
    Returns the per-image labels [H, W] int64."""
    _C.require_cuda(logits)
    n = len(image_sizes) // 2
    if logits.dim() != 4 or logits.shape[0] != n or len(output_sizes) != 2 * n:
        raise RuntimeError("sem_seg_labels: logits must be N x C x Hp x Wp with one crop and one output size per image")
    if n > _C.MAX_IMAGES:
        raise RuntimeError("sem_seg_labels: at most %d images per call" % _C.MAX_IMAGES)
    lg = logits if logits.dtype in _C.DTYPE_CODE else logits.to(torch.float32)
    lg = lg.contiguous()
    outs = [torch.empty((output_sizes[2 * i], output_sizes[2 * i + 1]), dtype=torch.int64, device=lg.device)
            for i in range(n)]
    if n:
        d = _C.SemSegImages()
        for i, o in enumerate(outs):
            d.h[i], d.w[i] = image_sizes[2 * i], image_sizes[2 * i + 1]
            d.H[i], d.W[i] = o.shape
            d.labels[i] = o.data_ptr()
        _, c, hp, wp = lg.shape
        with torch.cuda.device(lg.device):
            check(_C.lib().d2b_sem_seg_labels(ptr(lg), _C.DTYPE_CODE[lg.dtype], n, c, hp, wp, C.byref(d),
                                              stream_ptr(lg.device)), "sem_seg_labels")
    return outs


@sem_seg_labels_op.register_fake
def _(logits, image_sizes, output_sizes):
    return [logits.new_empty((output_sizes[2 * i], output_sizes[2 * i + 1]), dtype=torch.int64)
            for i in range(len(output_sizes) // 2)]


def _sem_seg_labels_host(logits: Tensor, image_sizes, output_sizes) -> List[Tensor]:
    """sem_seg_postprocess(...).argmax(0) per image, with the C x H x W map."""
    out = []
    for r, (h, w), (oh, ow) in zip(logits, image_sizes, output_sizes):
        soft = F.interpolate(r[:, :h, :w][None], size=(oh, ow), mode="bilinear", align_corners=False)[0]
        out.append(soft.argmax(dim=0))
    return out


def sem_seg_labels(results: Tensor, image_sizes: Sequence[Tuple[int, int]],
                   output_sizes: Sequence[Tuple[int, int]]) -> List[Tensor]:
    """results [N, C, Hp, Wp] semantic logits; image_sizes[n] = (h, w) the image's crop of the padded logits,
    output_sizes[n] = (H, W).  Returns per image the labels [H, W] int64, equal to
    sem_seg_postprocess(results[n], image_sizes[n], H, W).argmax(0).  On CUDA one launch, without the C x H x W map."""
    image_sizes = [(int(h), int(w)) for h, w in image_sizes]
    output_sizes = [(int(h), int(w)) for h, w in output_sizes]
    if not results.is_cuda:
        return _sem_seg_labels_host(results, image_sizes, output_sizes)
    return sem_seg_labels_op(results, [v for s in image_sizes for v in s], [v for s in output_sizes for v in s])


# ---- combine --------------------------------------------------------------------------------------------------------
@torch.library.custom_op("d2b200::panoptic_combine", mutates_args=(), device_types="cuda")
def panoptic_combine_op(scores: List[Tensor], classes: List[Tensor], masks: List[Tensor], labels: List[Tensor],
                        num_instances: Optional[Tensor], num_classes: int, overlap_threshold: float,
                        stuff_area_thresh: float, instances_score_thresh: float
                        ) -> Tuple[List[Tensor], Tensor, Tensor, Tensor, Tensor]:
    """Per image: scores [R] fp32, classes [R] int64, masks [R, H, W] (nonzero = in), labels [H, W] int64 in
    [0, num_classes); num_instances [N] int64 or None.  Returns (panoptic per image [H, W] int32, num_segments [N] int64,
    seg_info [N, S, 5] int64 (id, isthing, category, instance, area), seg_score [N, S] fp32, status [N] int32), with
    S = max R + num_classes."""
    n = len(labels)
    if not (len(scores) == len(classes) == len(masks) == n):
        raise RuntimeError("panoptic_combine: one scores, classes, masks and labels tensor per image")
    if n > _C.MAX_IMAGES:
        raise RuntimeError("panoptic_combine: at most %d images per call" % _C.MAX_IMAGES)
    _C.require_cuda(*scores, *classes, *masks, *labels, num_instances)
    if n == 0:
        raise RuntimeError("panoptic_combine: no image")
    device = labels[0].device
    d = _C.PanopticImages()
    keep = []  # the converted inputs live until the launches are enqueued
    pans = []
    for i in range(n):
        lab = labels[i]
        if lab.dim() != 2:
            raise RuntimeError("panoptic_combine: labels must be H x W")
        h, w = lab.shape
        m = masks[i]
        r = m.shape[0]
        if m.shape != (r, h, w) or scores[i].shape != (r,) or classes[i].shape != (r,):
            raise RuntimeError("panoptic_combine: image %d: masks must be R x H x W, scores and classes R" % i)
        if r > PANOPTIC_MAX_INSTANCES:
            raise RuntimeError("panoptic_combine: at most %d instances per image" % PANOPTIC_MAX_INSTANCES)
        m = (m if m.dtype == torch.uint8 else (m != 0).to(torch.uint8)).contiguous()
        s = scores[i].to(torch.float32).contiguous()
        c = classes[i].to(torch.int64).contiguous()
        lab = lab.to(torch.int64).contiguous()
        pan = torch.empty((h, w), dtype=torch.int32, device=device)
        keep += [m, s, c, lab]
        pans.append(pan)
        d.R[i], d.H[i], d.W[i] = r, h, w
        d.scores[i], d.classes[i], d.masks[i] = s.data_ptr(), c.data_ptr(), m.data_ptr()
        d.labels[i], d.panoptic[i] = lab.data_ptr(), pan.data_ptr()
    if not 1 <= num_classes <= PANOPTIC_MAX_CLASSES:
        raise RuntimeError("panoptic_combine: 1 <= num_classes <= %d" % PANOPTIC_MAX_CLASSES)
    slots = max(int(m.shape[0]) for m in masks) + num_classes
    cnt = None
    if num_instances is not None:
        if num_instances.shape != (n,):
            raise RuntimeError("panoptic_combine: num_instances must have one count per image")
        cnt = num_instances.to(torch.int64).contiguous()
    num_segments = torch.empty((n,), dtype=torch.int64, device=device)
    seg_info = torch.empty((n, slots, SEG_FIELDS), dtype=torch.int64, device=device)
    seg_score = torch.empty((n, slots), dtype=torch.float32, device=device)
    status = torch.empty((n,), dtype=torch.int32, device=device)
    lib = _C.lib()
    ws_bytes = lib.d2b_panoptic_workspace_bytes(C.byref(d), n, num_classes)
    ws = torch.empty((max(ws_bytes, 1),), dtype=torch.uint8, device=device)
    with torch.cuda.device(device):
        check(lib.d2b_panoptic_combine(C.byref(d), n, num_classes, ptr(cnt), float(overlap_threshold),
                                       float(stuff_area_thresh), float(instances_score_thresh), ptr(num_segments),
                                       ptr(seg_info), ptr(seg_score), ptr(status), ptr(ws), ws_bytes,
                                       stream_ptr(device)), "panoptic_combine")
    return pans, num_segments, seg_info, seg_score, status


@panoptic_combine_op.register_fake
def _(scores, classes, masks, labels, num_instances, num_classes, overlap_threshold, stuff_area_thresh,
      instances_score_thresh):
    n = len(labels)
    slots = max(int(m.shape[0]) for m in masks) + num_classes
    like = labels[0]
    return ([like.new_empty(tuple(lab.shape), dtype=torch.int32) for lab in labels], like.new_empty((n,)),
            like.new_empty((n, slots, SEG_FIELDS)), like.new_empty((n, slots), dtype=torch.float32),
            like.new_empty((n,), dtype=torch.int32))


def combine_semantic_and_instance_outputs_fixed(scores: Sequence[Tensor], classes: Sequence[Tensor],
                                                masks: Sequence[Tensor], labels: Sequence[Tensor], num_classes: int,
                                                overlap_threshold: float = 0.5, stuff_area_thresh: float = 4096,
                                                instances_score_thresh: float = 0.5,
                                                num_instances: Optional[Tensor] = None):
    """Sync-free combine of a batch (CUDA tensors; per-image sequences, or padded batch tensors such as the outputs of
    fast_rcnn_inference_fixed, whose rows at or past num_instances[n] are ignored).  Returns device tensors only:
    (panoptic list of [H, W] int32, num_segments [N] int64, seg_info [N, S, 5] int64 = (id, isthing, category, instance,
    area), seg_score [N, S] fp32, status [N] int32, nonzero when a label is outside [0, num_classes)).  Static shapes: capturable
    in a CUDA graph."""
    return panoptic_combine_op(list(scores), list(classes), list(masks), list(labels), num_instances, int(num_classes),
                               float(overlap_threshold), float(stuff_area_thresh), float(instances_score_thresh))


def _walk_order(scores: Tensor) -> List[int]:
    """Ascending -score, NaN last, ties to the lower index: a stable ascending sort of -score (torch.sort puts NaN last)."""
    return torch.sort(-scores, stable=True).indices.tolist()


def _combine_host(scores: Tensor, classes: Tensor, masks: Tensor, labels: Tensor, overlap_threshold: float,
                  stuff_area_thresh: float, instances_score_thresh: float, count: Optional[int] = None):
    """One image, with torch ops and host reads: returns (panoptic [H, W] int32, records), each record a tuple
    (id, isthing, category, instance, area, score) in id order."""
    r = masks.shape[0] if count is None else max(0, min(int(count), masks.shape[0]))
    panoptic = torch.zeros(labels.shape, dtype=torch.int32, device=labels.device)
    painted = torch.zeros(labels.shape, dtype=torch.bool, device=labels.device)
    records = []
    score_list = scores[:r].tolist()
    for i in _walk_order(scores[:r].to(torch.float32)):
        score = score_list[i]
        if score < instances_score_thresh:
            break
        inside = masks[i] != 0
        area = int(inside.sum().item())
        if area == 0:
            continue
        inter = int((inside & painted).sum().item())
        if inter / area > overlap_threshold:
            continue
        fresh = inside & ~painted
        seg = len(records) + 1
        panoptic[fresh] = seg
        painted |= fresh
        records.append((seg, 1, int(classes[i].item()), i, area - inter, score))
    present = torch.unique(labels).tolist()
    if present and (present[0] < 0):
        raise ValueError("panoptic combine: semantic label %d is negative" % present[0])
    for label in present:
        if label == 0:
            continue
        free = (labels == label) & ~painted
        area = int(free.sum().item())
        if area < stuff_area_thresh:
            continue
        seg = len(records) + 1
        panoptic[free] = seg
        records.append((seg, 0, int(label), -1, area, 0.0))
    return panoptic, records


def _segments_info(records) -> List[Dict]:
    """The reference's segments_info dicts (panoptic_fpn.py:238-266) from (id, isthing, category, instance, area, score)."""
    out = []
    for seg, isthing, category, instance, area, score in records:
        if isthing:
            out.append({"id": seg, "isthing": True, "score": score, "category_id": category, "instance_id": instance})
        else:
            out.append({"id": seg, "isthing": False, "category_id": category, "area": area})
    return out


def _records_from_device(num_segments: Tensor, seg_info: Tensor, seg_score: Tensor, status: Tensor):
    """One host read of the segment table of every image; raises on a label outside [0, C)."""
    host = torch.cat([num_segments.view(-1, 1), status.view(-1, 1).to(torch.int64), seg_info.flatten(1),
                      seg_score.flatten(1).view(torch.int32).to(torch.int64)], dim=1).cpu()
    slots = seg_info.shape[1]
    per_image = []
    for n, row in enumerate(host):
        if row[1].item() & STATUS_BAD_LABEL:
            raise ValueError("panoptic combine: image %d has a semantic label outside [0, num_classes)" % n)
        k = int(row[0])
        info = row[2:2 + slots * SEG_FIELDS].view(slots, SEG_FIELDS)[:k].tolist()
        score = row[2 + slots * SEG_FIELDS:].to(torch.int32).view(torch.float32)[:k].tolist()
        per_image.append([tuple(inf) + (sc,) for inf, sc in zip(info, score)])
    return per_image


def combine_semantic_and_instance_outputs(instance_results, semantic_results: Tensor, overlap_threshold: float,
                                          stuff_area_thresh: float, instances_score_thresh: float,
                                          num_classes: Optional[int] = None):
    """Reference signature and result (panoptic_fpn.py:184-269): instance_results has .scores, .pred_masks [R, H, W] and
    .pred_classes (e.g. postprocessing.PostprocessedDetections); semantic_results [H, W] int64 labels.  Returns
    (panoptic_seg [H, W] int32, segments_info).  CUDA tensors run `d2b_panoptic_combine` and read the segment table back
    once; num_classes bounds the labels (default: the largest label + 1, one more host read).  CPU tensors take the torch
    restatement."""
    scores, masks, classes = instance_results.scores, instance_results.pred_masks, instance_results.pred_classes
    if masks is None:
        masks = semantic_results.new_zeros((0,) + tuple(semantic_results.shape), dtype=torch.uint8)
    if not semantic_results.is_cuda:
        pan, records = _combine_host(scores, classes, masks, semantic_results, overlap_threshold, stuff_area_thresh,
                                     instances_score_thresh)
        return pan, _segments_info(records)
    if num_classes is None:
        num_classes = max(int(semantic_results.max().item()) + 1, 1) if semantic_results.numel() else 1
    pans, *table = combine_semantic_and_instance_outputs_fixed(
        [scores], [classes], [masks], [semantic_results], num_classes, overlap_threshold, stuff_area_thresh,
        instances_score_thresh)
    return pans[0], _segments_info(_records_from_device(*table)[0])


def panoptic_fpn_postprocess(sem_seg_results: Tensor, detections: Sequence, mask_probs: Sequence[Optional[Tensor]],
                             image_sizes: Sequence[Tuple[int, int]], output_sizes: Sequence[Tuple[int, int]],
                             overlap_threshold: float = 0.5, stuff_area_thresh: float = 4096,
                             instances_score_thresh: float = 0.5, mask_threshold: float = 0.5,
                             return_sem_seg: bool = False) -> List[Dict]:
    """The post-processing loop of PanopticFPN.inference (panoptic_fpn.py:159-179) for all images: sem_seg_results
    [N, C, Hp, Wp] logits, detections[n] (`Detections` at image_sizes[n]) with mask_probs[n] [R, 1, M, M] soft masks,
    output_sizes[n] = (height, width).  Per image detector_postprocess, then one sem_seg_labels and one combine for the
    batch and one host read.  Returns per image {"instances", "panoptic_seg": (panoptic_seg, segments_info)}, plus
    "sem_seg" (the C x H x W soft map of sem_seg_postprocess) when return_sem_seg."""
    out_sizes = [(int(h), int(w)) for h, w in output_sizes]
    processed = [detector_postprocess(det, h, w, mask_threshold, pred_masks=mp)
                 for det, mp, (h, w) in zip(detections, mask_probs, out_sizes)]
    labels = sem_seg_labels(sem_seg_results, image_sizes, out_sizes)
    num_classes = sem_seg_results.shape[1]
    masks = [p.pred_masks if p.pred_masks is not None else lab.new_zeros((0,) + tuple(lab.shape), dtype=torch.uint8)
             for p, lab in zip(processed, labels)]
    if sem_seg_results.is_cuda:
        pans, *table = combine_semantic_and_instance_outputs_fixed(
            [p.scores for p in processed], [p.pred_classes for p in processed], masks, labels, num_classes,
            overlap_threshold, stuff_area_thresh, instances_score_thresh)
        records = _records_from_device(*table)
    else:
        pans, records = [], []
        for p, m, lab in zip(processed, masks, labels):
            pan, rec = _combine_host(p.scores, p.pred_classes, m, lab, overlap_threshold, stuff_area_thresh,
                                     instances_score_thresh)
            pans.append(pan)
            records.append(rec)
    results = []
    for n, p in enumerate(processed):
        r = {"instances": p, "panoptic_seg": (pans[n], _segments_info(records[n]))}
        if return_sem_seg:
            h, w = image_sizes[n]
            r["sem_seg"] = F.interpolate(sem_seg_results[n, :, :h, :w][None], size=out_sizes[n], mode="bilinear",
                                         align_corners=False)[0]
        results.append(r)
    return results
