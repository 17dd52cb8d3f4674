"""Plumbing shared by the batched inference post-processors (`proposal_utils` for RPN / RRPN, `fast_rcnn_inference` for
axis-aligned and rotated Fast R-CNN, `dense_inference` for RetinaNet).  Each of them builds candidates for all images, runs
ONE `d2b_nms` over them and hands every image the first k survivors of the score-ordered keep list; what is shared is the
part around the candidate kernel, and the torch-op form of the selection that the host restatements use.

`ops.nms_fixed` is called through the module attribute: the CPU tests replace it with the oracle."""
import torch

from . import ops


def image_hw(image_sizes, device) -> torch.Tensor:
    """[N, 2] float32 (h, w) on `device` from a list of (h, w), or from an [N, 2] tensor (what a CUDA-graph capture needs:
    a list would be copied from the host inside the graph)."""
    if isinstance(image_sizes, torch.Tensor):
        return image_sizes.to(device=device, dtype=torch.float32).contiguous()
    return torch.tensor([[float(h), float(w)] for (h, w) in image_sizes], dtype=torch.float32).to(device)


def topk_levels(proposals, logits, pre_nms_topk: int):
    """The per-level top-k of the objectness logits (proposal_utils.py:84-88, one library `topk` per level) as a filled
    `_C.RpnLevels`.  Returns (levels, t = candidates per image, [k_l], tensors the levels point into: keep them alive
    until the kernels that read them are enqueued)."""
    from . import _C

    if len(proposals) > _C.MAX_LEVELS:
        raise RuntimeError("find_top_rpn_proposals: at most %d feature levels" % _C.MAX_LEVELS)
    lv = _C.RpnLevels()
    lv.num_levels = len(proposals)
    keepalive, ks = [], []
    for l, (p_l, s_l) in enumerate(zip(proposals, logits)):
        k = min(s_l.shape[1], pre_nms_topk)
        top_s, top_i = s_l.float().topk(k, dim=1)
        p_c = p_l.float().contiguous()
        keepalive += [top_s, top_i, p_c]
        lv.proposals[l], lv.topk_idx[l], lv.topk_scores[l] = p_c.data_ptr(), top_i.data_ptr(), top_s.data_ptr()
        lv.A[l], lv.k[l] = p_c.shape[1], k
        ks.append(k)
    return lv, sum(ks), ks, keepalive


def nms_select(nms_boxes, nms_scores, cat_ids, flat_boxes, raw_scores, n: int, t: int, topk: int, nms_thresh: float,
               rotated: bool, max_segment: int):
    """ONE `ops.nms_fixed` over the n * t candidates (category -1 = ignored), then `d2b_rpn_select`: every image
    gets the first `topk` of its survivors.  Returns (out_boxes [n, topk, 4 or 5], out_scores [n, topk], out_index
    [n, topk] into the candidates, counts [n]); rows past counts[i] are zero.  Static shapes: capturable."""
    from . import _C
    from ._C import check, ptr, stream_ptr

    device = flat_boxes.device
    f32 = dict(dtype=torch.float32, device=device)
    i64 = dict(dtype=torch.int64, device=device)
    out_boxes = torch.empty((n, topk, 5 if rotated else 4), **f32)
    out_scores = torch.empty((n, topk), **f32)
    out_index = torch.empty((n, topk), **i64)
    counts = torch.empty((n,), **i64)
    if n * t == 0 or topk == 0:  # the select kernel, which writes every element, does not run
        for x in (out_boxes, out_scores, out_index, counts):
            x.zero_()
        return out_boxes, out_scores, out_index, counts
    keep, num_keep = ops.nms_fixed(nms_boxes, nms_scores, cat_ids, float(nms_thresh), rotated, apply_offsets=False,
                                   max_segment=max_segment)
    flags = _C.SELECT_ROTATED if rotated else 0
    with torch.cuda.device(device):
        check(_C.lib().d2b_rpn_select(ptr(keep), ptr(num_keep), n, t, int(topk), flags, ptr(flat_boxes), ptr(raw_scores),
                                      ptr(cat_ids), ptr(out_boxes), ptr(out_scores), ptr(out_index), ptr(counts),
                                      stream_ptr(device)), "rpn_select")
    return out_boxes, out_scores, out_index, counts


def first_k_per_image(keep, num_keep, img_of, live, n: int, k: int):
    """`d2b_rpn_select` written with torch ops: the first `k` entries of image i in the score-ordered keep list (entries
    past num_keep are padding; candidates with live == False are skipped).  img_of / live: [M] image and liveness of each
    candidate.  Returns (index [n, k] into the candidates, 0 past counts[i]; counts [n])."""
    m = keep.shape[0]
    in_list = torch.arange(m, device=keep.device) < num_keep
    kidx = torch.where(in_list, keep, torch.zeros_like(keep))
    onehot = (img_of[kidx][None, :] == torch.arange(n, device=keep.device)[:, None]) & (in_list & live[kidx])[None, :]
    rank = torch.cumsum(onehot.to(torch.int32), dim=1) - 1
    sel = onehot & (rank < k)
    # scatter without data-dependent shapes: unselected entries are routed to a trash column
    out_idx = torch.zeros((n, k + 1), dtype=torch.int64, device=keep.device)
    col = torch.where(sel, rank.long(), torch.full_like(rank, k, dtype=torch.int64))
    out_idx.scatter_(1, col, kidx[None, :].expand(n, m))
    return out_idx[:, :k], sel.sum(dim=1)
