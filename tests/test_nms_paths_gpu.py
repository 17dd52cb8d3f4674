"""Every code path of d2b_nms (detectron2_b200/csrc/nms.cu) against the CPU oracle, bit-exact keep lists.

The rank kernel has two paths: category ids in [-1, 4096) take the histogram path, any other id (or ids that are not all
in that range) the generic one.  The scan keeps 160 column blocks of a segment in registers and walks the rest with plain
loads; it runs one CTA per segment on at most 2 x SM-count CTAs.  The tests below reach each of these, the max_segment
bound, the score order at NaN / +-0 / +-inf, NaN and infinite coordinates, and the rotated IoU at its geometric edges.
Where scores have no ties the compiled reference CPU ops (torch.ops.detectron2.* on CPU tensors) are a second checker;
their sort is not stable, so they are never used with tied scores.
"""
import numpy as np
import pytest
import torch

from oracle import oracle as orc
from test_oracle_pins import disjoint_boxes, edge_scores, score_order

pytestmark = pytest.mark.gpu
DEV = "cuda"
GENERIC = 5000  # category ids from here take the generic rank path


@pytest.fixture(scope="module")
def L():
    import detectron2_b200.layers as layers

    return layers


@pytest.fixture(scope="module")
def ops():
    from detectron2_b200 import ops as o

    return o


def have_reference():
    return orc.load_reference()


def distinct_scores(g, m):
    return (torch.randperm(m, generator=g).float() + 0.5) / m


def check_fixed(ops, boxes, scores, idxs, thr, rotated, **kw):
    """nms_fixed: keep[:n] is a duplicate-free list of indices in [0, M), the rest is 0.  Returns keep[:n] on the CPU."""
    keep, num = ops.nms_fixed(boxes.to(DEV), scores.to(DEV), None if idxs is None else idxs.to(DEV), thr, rotated, **kw)
    n, keep = int(num.item()), keep.cpu()
    m = boxes.shape[0]
    assert 0 <= n <= m
    k = keep[:n]
    assert ((k >= 0) & (k < m)).all() and k.unique().numel() == n
    assert (keep[n:] == 0).all()
    return k


def per_category_oracle(boxes, scores, idxs, thr, rotated):
    """Per-category loop on raw coordinates; negative ids are ignored.  Kept boxes in the stable global score order."""
    parts = []
    for c in idxs[idxs >= 0].unique():
        cur = torch.nonzero(idxs == c, as_tuple=True)[0]
        fn = orc.nms_rotated if rotated else orc.nms
        parts.append(cur[fn(boxes[cur], scores[cur], thr)])
    ref = torch.cat(parts) if parts else torch.zeros(0, dtype=torch.int64)
    return ref[score_order(scores[ref])]


# ------------------------------------------------------------------------------- score order at NaN / +-0 / +-inf
PATHS = ["nms", "hist", "generic", "rot", "rot_hist", "rot_generic"]


def run_path(L, path, boxes, scores):
    """The public op of `path` on the GPU and the oracle's answer.  Batched paths: two categories, interleaved."""
    m = boxes.shape[0]
    ids = torch.arange(m) % 2 + (GENERIC if path.endswith("generic") else 3)
    b, s, i = boxes.to(DEV), scores.to(DEV), ids.to(DEV)
    if path == "nms":
        return L.nms(b, s, 0.5).cpu(), orc.nms(boxes, scores, 0.5)
    if path == "rot":
        return L.nms_rotated(b, s, 0.5).cpu(), orc.nms_rotated(boxes, scores, 0.5)
    if path.startswith("rot"):
        return L.batched_nms_rotated(b, s, i, 0.5).cpu(), orc.batched_nms_rotated(boxes, scores, ids, 0.5)
    return L.batched_nms(b, s, i, 0.5).cpu(), orc.batched_nms(boxes, scores, ids, 0.5)


@pytest.mark.parametrize("path", PATHS)
def test_score_edges_disjoint_boxes(L, ops, path):
    s = edge_scores()
    m = s.numel()
    boxes = disjoint_boxes(m, path.startswith("rot"))
    got, ref = run_path(L, path, boxes, s)
    order = score_order(s)
    assert torch.equal(ref, order)
    assert torch.equal(got, order), (got.tolist(), order.tolist())
    ids = None if path in ("nms", "rot") else torch.arange(m) % 2 + (GENERIC if path.endswith("generic") else 3)
    assert torch.equal(check_fixed(ops, boxes, s, ids, 0.5, path.startswith("rot")), order)


@pytest.mark.parametrize("path", PATHS)
def test_score_edges_overlapping_boxes(L, ops, path):
    s = torch.cat([edge_scores()] * 4)
    m = s.numel()
    g = torch.Generator().manual_seed(17)
    xy = (torch.rand(m, 2, generator=g) * 40).round()
    boxes = torch.cat([xy, xy + 8 + (torch.rand(m, 2, generator=g) * 16).round()], 1)
    if path.startswith("rot"):
        boxes = torch.cat([(boxes[:, :2] + boxes[:, 2:]) / 2, boxes[:, 2:] - boxes[:, :2],
                           (torch.rand(m, 1, generator=g) * 180 - 90).round()], 1)
    got, ref = run_path(L, path, boxes, s)
    assert 0 < ref.numel() < m
    assert torch.equal(got, ref), (got.tolist(), ref.tolist())
    ids = None if path in ("nms", "rot") else torch.arange(m) % 2 + (GENERIC if path.endswith("generic") else 3)
    check_fixed(ops, boxes, s, ids, 0.5, path.startswith("rot"))


# ------------------------------------------------------------------------------- generic rank path at scale
def clustered_boxes(g, m, size, spread, wmin, wmax):
    """Boxes around m // 8 centres: plenty of overlaps inside a category."""
    base = torch.rand(max(m // 8, 1), 2, generator=g) * size
    ctr = base[torch.randint(0, base.shape[0], (m,), generator=g)] + torch.randn(m, 2, generator=g) * spread
    wh = wmin + torch.rand(m, 2, generator=g) * (wmax - wmin)
    return torch.cat([ctr - wh / 2, ctr + wh / 2], 1)


def test_generic_path_batched_nms_3000(L):
    g = torch.Generator().manual_seed(31)
    m = 3000
    boxes = clustered_boxes(g, m, 600, 6, 10, 80)
    scores = torch.rand(m, generator=g)
    scores[500:600] = scores[:100]  # ties across and inside categories
    idxs = torch.randint(4096, 4200, (m,), generator=g)
    for thr in (0.3, 0.7):
        got = L.batched_nms(boxes.to(DEV), scores.to(DEV), idxs.to(DEV), thr).cpu()
        assert torch.equal(got, orc.batched_nms(boxes, scores, idxs, thr)), thr


@pytest.mark.parametrize("rotated", [False, True])
def test_generic_path_huge_ids_and_ignored_slots(ops, rotated):
    g = torch.Generator().manual_seed(37)
    m = 2500
    boxes = clustered_boxes(g, m, 400, 5, 10, 60)
    if rotated:
        boxes = torch.cat([(boxes[:, :2] + boxes[:, 2:]) / 2, boxes[:, 2:] - boxes[:, :2],
                           torch.rand(m, 1, generator=g) * 180 - 90], 1)
    scores = torch.rand(m, generator=g)
    pool = torch.tensor([4096, 4097, 9000, 2**31 - 2, 2**31 - 1, 2**31, 2**40, 2**40 + 1, 2**62])
    idxs = pool[torch.randint(0, pool.numel(), (m,), generator=g)]
    idxs[torch.rand(m, generator=g) < 0.3] = -1
    got = check_fixed(ops, boxes, scores, idxs, 0.5, rotated, apply_offsets=False)
    assert torch.equal(got, per_category_oracle(boxes, scores, idxs, 0.5, rotated))


def _frcnn_inputs(g, n, r, k):
    """Peaked class scores: a few hundred (row, class) pairs per image pass 0.05, concentrated on 40 classes (the top ones
    included, so image 3's NMS category 3 * (k + 1) + class passes 4096) and on overlapping boxes."""
    boxes, scores = [], []
    classes = torch.cat([torch.tensor([k - 1, k - 2, k - 3]), torch.randint(0, k, (37,), generator=g)])
    for _ in range(n):
        ctr = torch.rand(r // 10, 2, generator=g) * torch.tensor([1000.0, 700.0])
        ctr = ctr[torch.randint(0, r // 10, (r,), generator=g)]
        b = ctr[:, None, :] + torch.randn(r, k, 2, generator=g) * 4
        wh = 30 + torch.rand(r, k, 2, generator=g) * 60
        boxes.append(torch.cat([b - wh / 2, b + wh / 2], 2).reshape(r, 4 * k))
        s = torch.rand(r, k + 1, generator=g) * 0.04
        rows = torch.randint(0, r, (400,), generator=g)
        cls = classes[torch.randint(0, classes.numel(), (400,), generator=g)]
        s[rows, cls] = 0.05 + torch.rand(400, generator=g) * 0.9
        scores.append(s)
    return boxes, scores


def test_fast_rcnn_inference_lvis_size_generic_path():
    """4 images x 1000 proposals x 1203 classes: NMS categories up to 3 * 1204 + 1202 = 4814 (generic path) against the
    per-image reference structure on the histogram path, and against the oracle."""
    from detectron2_b200 import fast_rcnn_inference as fri

    g = torch.Generator().manual_seed(41)
    n, r, k = 4, 1000, 1203
    boxes, scores = _frcnn_inputs(g, n, r, k)
    shapes = [(800, 1067), (768, 1024), (800, 1200), (700, 1000)]
    thr, nms_thr, topk = 0.05, 0.5, 100
    res, rows = fri.fast_rcnn_inference([b.to(DEV) for b in boxes], [s.to(DEV) for s in scores], shapes, thr, nms_thr, topk)
    for i in range(n):
        fg = scores[i][:, :-1]
        filt = (fg > thr).nonzero()
        assert 100 < filt.shape[0] <= 400
        if i == n - 1:
            assert int(filt[:, 1].max()) + i * (k + 1) >= 4096
        ex, ex_rows = fri._single_image_exact(boxes[i].to(DEV), scores[i].to(DEV), shapes[i], thr, nms_thr, topk)
        assert torch.equal(res[i].pred_boxes, ex.pred_boxes), i
        assert torch.equal(res[i].scores, ex.scores) and torch.equal(res[i].pred_classes, ex.pred_classes), i
        assert torch.equal(rows[i], ex_rows), i
        # the oracle: the reference's per-image structure (fast_rcnn.py:117-173) with the CPU batched_nms
        h, w = shapes[i]
        bb = boxes[i].reshape(r, k, 4)
        bb = torch.stack([bb[..., 0].clamp(0, w), bb[..., 1].clamp(0, h), bb[..., 2].clamp(0, w), bb[..., 3].clamp(0, h)], 2)
        cb, cs = bb[fg > thr], fg[fg > thr]
        keep = orc.batched_nms(cb, cs, filt[:, 1], nms_thr)[:topk]
        assert 0 < keep.numel() < filt.shape[0]
        assert torch.equal(res[i].pred_classes.cpu(), filt[keep, 1]), i
        assert torch.equal(rows[i].cpu(), filt[keep, 0]), i
        assert torch.equal(res[i].pred_boxes.cpu(), cb[keep]), i


# ------------------------------------------------------------------------------- scan kernel paths
@pytest.mark.parametrize("m,thrs", [(12000, (0.3, 0.7)), (20000, (0.5,))])
def test_scan_beyond_the_register_window(L, m, thrs):
    """One segment of more than 160 column blocks: the scan's plain-load loop past the prefetched columns."""
    g = torch.Generator().manual_seed(m)
    boxes = clustered_boxes(g, m, 4000, 20, 10, 120)
    scores = torch.rand(m, generator=g)
    for thr in thrs:
        got = L.nms(boxes.to(DEV), scores.to(DEV), thr).cpu()
        ref = orc.nms(boxes, scores, thr)
        assert m // 2 < ref.numel() < m
        assert torch.equal(got, ref), thr


@pytest.mark.parametrize("base", [0, GENERIC])
def test_more_segments_than_scan_ctas(L, base):
    """3000 categories of 1-6 boxes: far more segments than the 2 x SM-count scan CTAs."""
    g = torch.Generator().manual_seed(43)
    sizes = torch.randint(1, 7, (3000,), generator=g)
    idxs = torch.repeat_interleave(torch.arange(3000), sizes)
    m = idxs.numel()
    idxs = idxs[torch.randperm(m, generator=g)] + base
    boxes = clustered_boxes(g, m, 100, 3, 10, 30)
    scores = torch.rand(m, generator=g)
    got = L.batched_nms(boxes.to(DEV), scores.to(DEV), idxs.to(DEV), 0.5).cpu()
    assert torch.equal(got, orc.batched_nms(boxes, scores, idxs, 0.5))


def edge_geometry_boxes(g, m):
    """Integer-grid boxes with exact duplicates, near-duplicates, edge-sharing and corner-touching neighbours."""
    xy = (torch.rand(m, 2, generator=g) * 24).round() * 2
    wh = 2 + (torch.rand(m, 2, generator=g) * 6).round() * 2
    b = torch.cat([xy, xy + wh], 1)
    for i in range(1, m):
        kind = i % 5
        if kind == 1:
            b[i] = b[i - 1]  # identical
        elif kind == 2:
            b[i] = b[i - 1] + torch.tensor([1e-3, 0.0, 1e-3, 0.0])  # near-duplicate
        elif kind == 3:
            w = b[i - 1, 2] - b[i - 1, 0]
            b[i] = b[i - 1] + torch.stack([w, torch.tensor(0.0), w, torch.tensor(0.0)])  # shares an edge
        elif kind == 4:
            b[i] = torch.cat([b[i - 1, 2:], b[i - 1, 2:] + 3])  # touches a corner
    return b


@pytest.mark.parametrize("m", [1, 2, 63, 64, 65, 127, 128, 129])
def test_block_edges_and_thresholds(L, m):
    g = torch.Generator().manual_seed(100 + m)
    boxes = edge_geometry_boxes(g, m)
    rot = torch.cat([(boxes[:, :2] + boxes[:, 2:]) / 2, boxes[:, 2:] - boxes[:, :2], torch.zeros(m, 1)], 1)
    rot[1::7, 4] = 90.0
    scores = torch.rand(m, generator=g)
    scores[3::4] = scores[2::4][: scores[3::4].numel()]  # ties
    idxs = torch.randint(0, 3, (m,), generator=g)
    b, r, s, i = boxes.to(DEV), rot.to(DEV), scores.to(DEV), idxs.to(DEV)
    # at thresholds that IoU 0 passes (rotated 0.0, both -0.1) the reference's one NMS over the offset boxes suppresses
    # across categories as well
    for thr in (-0.1, 0.0, 0.5, 1.0):
        assert torch.equal(L.nms(b, s, thr).cpu(), orc.nms(boxes, scores, thr)), thr
        assert torch.equal(L.batched_nms(b, s, i, thr).cpu(), orc.batched_nms(boxes, scores, idxs, thr)), thr
        assert torch.equal(L.nms_rotated(r, s, thr).cpu(), orc.nms_rotated(rot, scores, thr)), thr
        assert torch.equal(L.batched_nms_rotated(r, s, i, thr).cpu(), orc.batched_nms_rotated(rot, scores, idxs, thr)), thr


# ------------------------------------------------------------------------------- the max_segment bound
@pytest.mark.parametrize("ms", [1, 63, 64, 65, 200])
@pytest.mark.parametrize("offset", [0, 1, 63])
def test_max_segment_bound(ops, ms, offset):
    """A category of exactly max_segment boxes whose first row sits at `offset` inside a 64-box block (the `offset`
    boxes of the single-box categories 0 .. offset-1 come first in the category-major order): exact.  One box more: the
    bound is reported (num_keep == -1)."""
    g = torch.Generator().manual_seed(ms * 100 + offset)
    for n, ok in ((ms, True), (ms + 1, False), (3 * ms + 5, False)):
        idxs = torch.cat([torch.arange(offset), torch.full((n,), offset), torch.full((min(ms, 7),), offset + 1)])
        m = idxs.numel()
        idxs = idxs[torch.randperm(m, generator=g)]
        boxes = clustered_boxes(g, m, 60, 4, 10, 40)
        scores = torch.rand(m, generator=g)
        if ok:
            got = check_fixed(ops, boxes, scores, idxs, 0.5, False, apply_offsets=False, max_segment=ms)
            assert torch.equal(got, per_category_oracle(boxes, scores, idxs, 0.5, False)), n
        else:
            _, num = ops.nms_fixed(boxes.to(DEV), scores.to(DEV), idxs.to(DEV), 0.5, False, apply_offsets=False,
                                   max_segment=ms)
            assert int(num.item()) == -1, n


# ------------------------------------------------------------------------------- rotated NMS at scale
def test_batched_nms_rotated_3000_vs_oracle_and_reference(L):
    g = torch.Generator().manual_seed(47)
    m = 3000
    dets = torch.stack([torch.rand(m, generator=g) * 1024, torch.rand(m, generator=g) * 1024,
                        4 + torch.rand(m, generator=g) * 296, 4 + torch.rand(m, generator=g) * 296,
                        90 - torch.rand(m, generator=g) * 180], 1)  # angles in (-90, 90]
    dets[1000:1500] = dets[:500] + torch.randn(500, 5, generator=g) * torch.tensor([1.0, 1.0, 1.0, 1.0, 2.0])
    dets[:, 2:4].clamp_(min=4)
    scores = distinct_scores(g, m)
    idxs = torch.randint(0, 16, (m,), generator=g)
    thr = 0.5
    got = L.batched_nms_rotated(dets.to(DEV), scores.to(DEV), idxs.to(DEV), thr).cpu()
    ref = orc.batched_nms_rotated(dets, scores, idxs, thr)
    assert torch.equal(got, ref)
    if have_reference():  # the reference's own CPU nms_rotated on the offset boxes of layers/nms.py:137-146
        mx = (torch.max(dets[:, 0], dets[:, 1]) + torch.max(dets[:, 2], dets[:, 3]) / 2).max()
        mn = (torch.min(dets[:, 0], dets[:, 1]) - torch.max(dets[:, 2], dets[:, 3]) / 2).min()
        shifted = dets.clone()
        shifted[:, :2] += (idxs.to(dets) * (mx - mn + 1))[:, None]
        assert torch.equal(got, torch.ops.detectron2.nms_rotated(shifted, scores, thr))


# ------------------------------------------------------------------------------- rotated IoU geometry
def rotated_geometry_cases():
    b = [[50.0, 40.0, 30.0, 12.0, 17.0]]
    pairs = [(b[0], b[0])]  # identical
    for turn in (90.0, 180.0, -180.0, 360.0, 720.0):  # the same box turned
        pairs.append((b[0], b[0][:4] + [b[0][4] + turn]))
    pairs += [
        ([10.0, 10.0, 4.0, 4.0, 0.0], [14.0, 10.0, 4.0, 4.0, 0.0]),  # shared edge
        ([10.0, 10.0, 4.0, 4.0, 0.0], [14.0, 14.0, 4.0, 4.0, 0.0]),  # shared corner
        ([10.0, 10.0, 4.0, 4.0, 45.0], [10.0 + 2 * 2**0.5 * 2, 10.0, 4.0, 4.0, 45.0]),  # corner contact at 45 degrees
        ([20.0, 20.0, 30.0, 30.0, 0.0], [22.0, 19.0, 6.0, 8.0, 30.0]),  # nested
        ([20.0, 20.0, 30.0, 30.0, 45.0], [20.0, 20.0, 10.0, 10.0, -45.0]),  # nested, multiples of 45 degrees
        ([20.0, 20.0, 0.0, 10.0, 0.0], [20.0, 20.0, 10.0, 10.0, 0.0]),  # zero width
        ([20.0, 20.0, 10.0, 0.0, 30.0], [20.0, 20.0, 10.0, 10.0, 0.0]),  # zero height
        ([20.0, 20.0, 1e-7, 1e-7, 0.0], [20.0, 20.0, 1e-7, 1e-7, 0.0]),  # w*h = 1e-14
        ([20.0, 20.0, 1.1e-7, 1e-7, 0.0], [20.0, 20.0, 1.1e-7, 1e-7, 0.0]),  # just above
        ([20.0, 20.0, 0.9e-7, 1e-7, 0.0], [20.0, 20.0, 1e-7, 1e-7, 0.0]),  # just below
        ([100.0, 50.0, 1000.0, 1.0, 0.0], [100.0, 50.0, 1000.0, 1.0, 0.5]),  # aspect ratio 1000
        ([100.0, 50.0, 1000.0, 1.0, 90.0], [100.0, 50.0, 1.0, 1000.0, 0.0]),
        ([12345.5, 54321.25, 40.0, 20.0, 10.0], [12350.0, 54318.0, 40.0, 20.0, 35.0]),  # far from the origin
        ([98765.5, 10000.0, 80.0, 60.0, -30.0], [98760.0, 10010.0, 70.0, 60.0, 15.0]),
    ]
    for a in (45.0, 90.0, 135.0, -45.0, -90.0, 225.0):
        pairs.append(([30.0, 30.0, 20.0, 10.0, a], [32.0, 29.0, 20.0, 10.0, 0.0]))
        pairs.append(([30.0, 30.0, 20.0, 10.0, a], [30.0, 30.0, 20.0, 10.0, a + 45.0]))
    return pairs


def test_rotated_iou_geometry_bit_exact(L):
    pairs = rotated_geometry_cases()
    b1 = torch.tensor([p[0] for p in pairs], dtype=torch.float32)
    b2 = torch.tensor([p[1] for p in pairs], dtype=torch.float32)
    got = L.pairwise_iou_rotated(b1.to(DEV), b2.to(DEV)).cpu()
    ref = orc.box_iou_rotated(b1, b2)
    assert np.array_equal(got.numpy().view(np.uint32), ref.numpy().view(np.uint32))
    assert (got.diagonal()[11:13] == 0).all()  # zero width / height
    if have_reference():
        rr = torch.ops.detectron2.box_iou_rotated(b1, b2)
        assert np.array_equal(got.numpy().view(np.uint32), rr.numpy().view(np.uint32))


# ------------------------------------------------------------------------------- NaN / inf coordinates
def overlapping_pair_sets(g, m, rotated):
    boxes = clustered_boxes(g, m, 50, 2, 20, 30)
    if rotated:
        boxes = torch.cat([(boxes[:, :2] + boxes[:, 2:]) / 2, boxes[:, 2:] - boxes[:, :2], torch.zeros(m, 1)], 1)
    return boxes


@pytest.mark.parametrize("rotated", [False, True])
@pytest.mark.parametrize("value", [float("nan"), float("inf"), float("-inf")])
def test_non_finite_coordinate(L, rotated, value):
    """One non-finite coordinate among overlapping boxes.  NaN: every offset box is NaN in the reference (torch max / min
    propagate it), nothing is suppressed."""
    g = torch.Generator().manual_seed(53)
    m = 40
    boxes = overlapping_pair_sets(g, m, rotated)
    scores = distinct_scores(g, m)
    idxs = torch.randint(0, 3, (m,), generator=g)
    plain = (orc.nms_rotated if rotated else orc.nms)(boxes, scores, 0.5)
    assert plain.numel() < m // 2  # the boxes do overlap
    boxes[7, 2] = value
    fn, ofn = (L.batched_nms_rotated, orc.batched_nms_rotated) if rotated else (L.batched_nms, orc.batched_nms)
    got = fn(boxes.to(DEV), scores.to(DEV), idxs.to(DEV), 0.5).cpu()
    ref = ofn(boxes, scores, idxs, 0.5)
    if value != value:
        assert torch.equal(ref, score_order(scores))
    assert torch.equal(got, ref), (got.tolist(), ref.tolist())
