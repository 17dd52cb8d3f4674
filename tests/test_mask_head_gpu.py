"""Mask R-CNN mask loss (postproc.cu: mask_loss_fwd_kernel / mask_loss_bwd_kernel through mask_head.mask_rcnn_loss) against
the float64 reference of tests/mask_loss_ref.py.

The case table uses dyadic geometry: box corners on multiples of 1/8 pixel, each bin a dyadic multiple of its sampling
grid.  So every target must equal the reference bit for bit.  The per-proposal loss, the batch mean and the gradient must
be within the bounds derived in mask_loss_ref.py.  Off the proposal's class channel the gradient must be exactly 0.
Masks are random bits.  Logits are randn * 4 with 3 % of the entries set to +-30 or +-88.  Every case also runs with fp16
and bf16 logits.  Its loss must then be bitwise the loss of the fp32 run on the up-cast logits, and its gradient that
run's gradient rounded once to the logits' dtype.  tests/test_mask_head_host.py checks on the CPU that each case reaches
the edges listed here.

case          S   C     reaches
inside_s7     7   80    one pass of the 256-thread bin loop; boxes inside the mask; sampling grids 1 to 4 and a count of 9;
                        sub-pixel bins (grid 1 x 1); bins pooled to exactly 0.5 (target 1) and one weight step below 0.5
                        (target 0); six proposals on one mask; classes 0 and C-1; odd H x W
borders_s14   14  80    boxes cut by each image border; two images of different sizes
empty_s16     16  80    exactly 256 bins; boxes entirely outside the mask (all-zero target); zero width and zero height
                        (grid 0); inverted boxes (negative grid before the clamp)
lattice_s28   28  80    three passes plus a ragged fourth; sample rows and columns exactly on -1, 0, H-1 and H
large_s32     32  80    four full passes; boxes 5 to 10 times the mask, grids up to 8 x 6, most samples off the map
thin_s7       7   80    masks of height 1 and of width 1 (the lo >= size - 1 clamp), samples on -1, 0 and 1
agnostic_s28  28  1     mask_index None (one mask per proposal), class-agnostic head; three images, the middle one
                        without proposals
c1203_s14     14  1203  C = 1203 (the backward's grid.y); classes 0, 601 and C-1

Besides the table: a realistic non-dyadic batch (K = 512 on 800 x 1333 masks; targets may differ only next to 0.5),
total == 0, and the properties P1 a proposal's loss and targets are bitwise the same alone and among 500 others, P2 two
runs give the same bits, P3 forward + backward replay from one CUDA graph on new inputs and equal the eager run, P4 a
mask index outside [0, G) gives an all-zero target and a class outside [0, C) no loss and no gradient.  Ground-truth masks
given as bool, as uint8 {0, 1, 255} or as float {0, 0.25, 0.5, 1} are read as `mask != 0`, as BitMasks reads them.
"""
import functools
import math
from collections import namedtuple

import numpy as np
import pytest
import torch

import mask_loss_ref as mr
import roi_align_ref as ra
from test_roi_align_column_walk import sample_pos

pytestmark = pytest.mark.gpu
DEV = "cuda"

# prop: (mask index, start_w, start_h, bin_w, bin_h, class) -- start = the kernel's sw / sh (box corner - 0.5), box side =
# bin * S; mask index and class are unused by a class-agnostic case (proposal k <-> mask k)
Image = namedtuple("Image", "g h w props")
Case = namedtuple("Case", "name s c images agnostic labels")


def _c(name, s, c, images, labels, agnostic=False):
    return Case(name, s, c, [Image(*im) for im in images], agnostic, frozenset(labels))


CASES = [
    _c("inside_s7", 7, 80, [(3, 37, 45, [(1, 2.625, 3, 1, 1, 0), (1, 9.625, 11, 1, 1, 79), (1, 4, 5, 1.5, 2, 5),
                                         (1, 6.5, 2, 3, 3, 42), (1, 1, 1, 0.5, 0.75, 79), (1, 20.25, 7, 0.25, 0.125, 0),
                                         (0, 3, 3, 4, 4, 17), (2, 5, 9, 2, 1, 79)])],
       {"passes1", "inside", "grid9", "subpixel", "half", "below_half", "shared_mask", "class0", "classC-1", "odd_hw"}),
    _c("borders_s14", 14, 80, [(2, 29, 39, [(0, -6, 4, 1, 1, 3), (1, 5, -7.5, 1.5, 1, 0), (1, -3, -3, 0.75, 0.75, 79)]),
                               (2, 25, 21, [(0, 14, 3, 1, 1, 79), (1, 2, 18, 1, 0.75, 8), (1, -4, -4, 3, 3, 0),
                                            (0, 15.5, 19.5, 0.5, 0.5, 2)])],
       {"passes1", "cut_left", "cut_top", "cut_right", "cut_bottom", "image_sizes", "half"}),
    _c("empty_s16", 16, 80, [(2, 33, 31, [(0, 40, 2, 1, 1, 1), (1, 2, -30, 1, 1, 0), (0, 5, 5, 0, 1, 79),
                                          (1, 5, 5, 1, 0, 3), (0, 10, 10, -1, 1, 4), (1, 10, 10, 1, -2, 79),
                                          (0, 3, 4, 1, 1, 0)])],
       {"bins256", "outside", "zero_size", "grid_negative", "inside"}),
    _c("lattice_s28", 28, 80, [(2, 15, 13, [(1, -1.5, -1.5, 1, 1, 0), (1, -1.25, -1.25, 0.5, 0.5, 79),
                                            (1, -2, -2, 2, 2, 6), (1, 3, -1.5, 0.5, 1, 11)])],
       {"passes4_ragged", "pos_-1", "pos_0", "pos_H-1", "pos_H", "half"}),
    _c("large_s32", 32, 80, [(2, 21, 27, [(1, -40, -50, 4, 5, 0), (1, -100, -90, 8, 6, 79), (0, 2, 3, 0.5, 0.5, 7)])],
       {"passes4_full", "large_offmap"}),
    _c("thin_s7", 7, 80, [(3, 1, 19, [(2, -1.5, -2.5, 4, 1, 0), (1, 3.5, -1, 1, 0.25, 79), (0, 2, -0.25, 1, 0.125, 3)]),
                          (2, 23, 1, [(1, -2.5, -1.5, 1, 4, 5), (1, -0.75, 4, 0.25, 1, 79)])],
       {"mask_h1", "mask_w1", "pos_-1", "pos_0", "pos_H-1", "pos_H"}),
    _c("agnostic_s28", 28, 1, [(3, 41, 37, [(0, 2, 3, 1, 1, 0), (0, 5, 6, 0.75, 1.5, 0), (0, -3, 20, 1, 1, 0)]),
                               (0, 30, 30, []),
                               (4, 27, 33, [(0, 1, 1, 0.5, 0.5, 0), (0, 4, 2, 1, 0.75, 0), (0, 20, -5, 1, 1, 0),
                                            (0, -1.5, -1.5, 1, 1, 0)])],
       {"per_proposal_masks", "empty_image_middle", "image_sizes", "passes4_ragged", "pos_-1", "pos_0"}, agnostic=True),
    _c("c1203_s14", 14, 1203, [(2, 31, 29, [(0, 2, 2, 1, 1, 0), (1, 3, 1, 1.5, 1.5, 1202), (1, 5, 4, 0.5, 1, 601),
                                            (0, -2, 10, 1, 1, 1202), (1, 8, 8, 1, 1, 0), (1, 1, 3, 2, 1, 77)])],
       {"C1203", "class0", "classC-1"}),
]
BY_NAME = {c.name: c for c in CASES}
ids = [c.name for c in CASES]
EXTREMES = (30.0, -30.0, 88.0, -88.0)


def case_boxes(case, im):
    """The image's proposal boxes [K, 4] fp32 (exact: corners on multiples of 1/8)."""
    b = np.array([[sx + 0.5, sy + 0.5, sx + bw * case.s + 0.5, sy + bh * case.s + 0.5] for _, sx, sy, bw, bh, _ in im.props],
                 dtype=np.float64).reshape(-1, 4)
    assert (b * 8 == np.round(b * 8)).all() and (b.astype(np.float32) == b).all()
    return b.astype(np.float32)


def _logits(g, k, c, s):
    x = torch.randn(k, c, s, s, generator=g) * 4
    pick = torch.rand(k, c, s, s, generator=g) < 0.03
    ext = torch.tensor(EXTREMES)[torch.randint(0, 4, (k, c, s, s), generator=g)]
    return torch.where(pick, ext, x)


@functools.lru_cache(maxsize=None)
def _inputs(name):
    """Per image: masks [G, H, W] bool, boxes [K, 4], mask_index [K] or None, classes [K] or None (CPU); the logits
    [sum K, C, S, S] fp32; the reference targets per image."""
    case = BY_NAME[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    gts, boxes, midx, cls, refs = [], [], [], [], []
    for im in case.images:
        gts.append(torch.rand(im.g, im.h, im.w, generator=g) < 0.5)
        boxes.append(torch.from_numpy(case_boxes(case, im)))
        midx.append(None if case.agnostic else torch.tensor([p[0] for p in im.props], dtype=torch.int64))
        cls.append(None if case.agnostic else torch.tensor([p[5] for p in im.props], dtype=torch.int64))
        refs.append(mr.targets(gts[-1].numpy(), boxes[-1].numpy(), None if midx[-1] is None else midx[-1].numpy(), case.s))
    total = sum(len(b) for b in boxes)
    return gts, boxes, midx, cls, _logits(g, total, case.c, case.s), refs


def edge_labels(case):
    """Every edge the case reaches, from the fp32 geometry of roi_align_ref.geom and the reference's pooled sums."""
    gts, boxes, midx, cls, logits, refs = _inputs(case.name)
    s, s2 = case.s, case.s * case.s
    out = {"C%d" % case.c}
    npass = -(-s2 // 256)
    out.add("passes1" if s2 < 256 else "bins256" if s2 == 256 else "passes%d_%s" % (npass, "ragged" if s2 % 256 else "full"))
    if case.agnostic and case.c == 1:
        out.add("per_proposal_masks")
    if len(case.images) >= 3 and any(not im.props for im in case.images[1:-1]):
        out.add("empty_image_middle")
    if len({(im.h, im.w) for im in case.images}) > 1:
        out.add("image_sizes")
    for im, gt, b, mi, cl, ref in zip(case.images, gts, boxes, midx, cls, refs):
        if im.h % 2 and im.w % 2:
            out.add("odd_hw")
        if mi is not None and len(mi) and np.bincount(mi.numpy()).max() >= 4:
            out.add("shared_mask")
        if cl is not None:
            out |= {"class0"} if (cl == 0).any() else set()
            out |= {"classC-1"} if (cl == case.c - 1).any() else set()
        for k, R in enumerate(ref.rois):
            out |= _roi_labels(R, gt[k if mi is None else int(mi[k])].numpy(), s)
    cls_all = torch.cat([torch.zeros(len(bb), dtype=torch.int64) if c is None else c for bb, c in zip(boxes, cls)])
    xc = logits[torch.arange(len(cls_all)), cls_all]
    out |= {"logit_%d" % v for v in (30, 88) if (xc == v).any() and (xc == -v).any()}
    return out


def _roi_labels(R, mask, s):
    g, h, w = R.g, R.h, R.w
    out = set()
    if g.count == 0:
        if g.raw_w == 0 or g.raw_h == 0:
            out.add("zero_size")
        if min(math.ceil(g.bin_w), math.ceil(g.bin_h)) < 0:
            out.add("grid_negative")
        return out
    if R.empty:
        return {"outside"}
    ys = [sample_pos(g.start_h, g.bin_h, g.gh, p, i, True) for p in range(s) for i in range(g.gh)]
    xs = [sample_pos(g.start_w, g.bin_w, g.gw, p, i, True) for p in range(s) for i in range(g.gw)]
    if g.count == 9:
        out.add("grid9")
    if min(ys) >= 0 and max(ys) <= h - 1 and min(xs) >= 0 and max(xs) <= w - 1:
        out.add("inside")
    out |= {"cut_left"} if min(xs) < -1 < 0 < max(xs) else set()
    out |= {"cut_top"} if min(ys) < -1 < 0 < max(ys) else set()
    out |= {"cut_right"} if min(xs) < w - 1 < w < max(xs) else set()
    out |= {"cut_bottom"} if min(ys) < h - 1 < h < max(ys) else set()
    if g.gh == g.gw == 1:
        out.add("subpixel")
    on = np.mean([-1 <= y <= h for y in ys]) * np.mean([-1 <= x <= w for x in xs])
    if min(g.gh, g.gw) >= 4 and g.raw_h >= 3 * h and g.raw_w >= 3 * w and on < 0.5:
        out.add("large_offmap")
    if h == 1:
        out.add("mask_h1")
    if w == 1:
        out.add("mask_w1")
    out |= ra.boundary_labels(R, 0, True) - {"sr0"}
    sm, count = mr.pooled_sum(R, mask)
    if (sm == 0.5 * count).any():
        out.add("half")
    for p in range(s):
        for q in range(s):
            wy, wx = [w_ for _, w_ in R.ylists[p] if w_], [w_ for _, w_ in R.xlists[q] if w_]
            if wy and wx and sm[p, q] == 0.5 * count - min(wy) * min(wx):
                out.add("below_half")
    return out


def _dev(ts):
    return [None if t is None else t.to(DEV) for t in ts]


def _fwd_bwd(case, x):
    """mask_rcnn_loss forward + backward of the case's inputs with logits x: (loss, targets, gradient of the logits)."""
    from detectron2_b200.mask_head import mask_rcnn_loss

    gts, boxes, midx, cls = _inputs(case.name)[:4]
    xd = x.to(DEV).requires_grad_(True)
    loss, targets = mask_rcnn_loss(xd, _dev(gts), _dev(boxes), None if case.agnostic else _dev(cls),
                                   None if case.agnostic else _dev(midx))
    loss.backward()
    return loss.detach(), targets, xd.grad


def _check_against_reference(case, x32):
    """fp32 logits x32 (CPU): forward + backward through mask_rcnn_loss, checked against the reference."""
    from detectron2_b200.mask_head import mask_loss_per_roi

    gts, boxes, midx, cls, _, refs = _inputs(case.name)
    loss, targets, grad = _fwd_bwd(case, x32)
    t_ref = np.concatenate([r.t for r in refs])
    assert np.array_equal(targets.cpu().numpy(), t_ref), (case.name, int((targets.cpu().numpy() != t_ref).sum()))
    total, s2 = x32.shape[0], case.s ** 2
    cls_all = None if case.agnostic else torch.cat(cls)
    per_roi, k0 = [], 0
    for gt, b, mi, cl in zip(gts, boxes, midx, cls):
        k = len(b)
        lo, tg = mask_loss_per_roi(x32[k0:k0 + k].to(DEV), gt.to(DEV), b.to(DEV), *_dev([mi, cl]))
        per_roi.append(lo)
        k0 += k
    per_roi = torch.cat(per_roi)
    ref, tol = mr.loss_per_roi(x32.numpy(), t_ref, None if cls_all is None else cls_all.numpy())
    mr.check(per_roi.cpu().numpy(), ref, tol, "%s loss_per_roi" % case.name)
    # the batch mean is the sum of the per-proposal losses over total * S^2, as torch computes it
    assert torch.equal(loss, per_roi.sum() / float(total * s2))
    mean_tol = (tol.sum() + (total + 1) * mr.EPS32 * (ref + tol).sum()) / (total * s2)
    mr.check(loss.item(), ref.sum() / (total * s2), mean_tol, "%s loss" % case.name)
    scale = np.float32(1) / np.float32(total * s2)  # d loss / d loss_per_roi[k], as autograd computes it in fp32
    gref, gtol = mr.grad(x32.numpy(), t_ref, None if cls_all is None else cls_all.numpy(), scale)
    gg = grad.cpu().numpy()
    mr.check(gg, gref, np.broadcast_to(gtol[:, None, None, None], gg.shape), "%s grad" % case.name)
    off = np.ones(gg.shape, bool)
    off[np.arange(total), np.zeros(total, np.int64) if cls_all is None else cls_all.numpy()] = False
    assert (gg[off] == 0).all() and not np.signbit(gg[off]).any()
    assert np.isfinite(gg).all() and math.isfinite(loss.item())
    return loss, targets, grad


@pytest.mark.parametrize("dtype", ["float32", "float16", "bfloat16"])
@pytest.mark.parametrize("name", ids)
def test_mask_loss_case(name, dtype):
    case = BY_NAME[name]
    assert case.labels <= edge_labels(case), case.labels - edge_labels(case)
    x = _inputs(name)[4]
    if dtype == "float32":
        _check_against_reference(case, x)
        return
    dt = getattr(torch, dtype)
    xh = x.to(dt)
    loss32, t32, g32 = _check_against_reference(case, xh.float())
    loss, targets, grad = _fwd_bwd(case, xh)
    assert loss.dtype == torch.float32 and torch.equal(loss, loss32)
    assert torch.equal(targets, t32)
    assert grad.dtype == dt and torch.equal(grad, g32.to(dt))


def test_total_zero():
    """No proposal in the batch: loss 0, no targets, and the (empty) gradient of the logits; zero proposals per image."""
    from detectron2_b200.mask_head import mask_loss_per_roi, mask_rcnn_loss

    x = torch.zeros(0, 80, 28, 28, device=DEV, requires_grad=True)
    gts = [torch.ones(2, 30, 40, dtype=torch.bool, device=DEV), torch.ones(0, 20, 20, dtype=torch.bool, device=DEV)]
    empty = [torch.zeros(0, 4, device=DEV)] * 2
    loss, targets = mask_rcnn_loss(x, gts, empty, [torch.zeros(0, dtype=torch.int64, device=DEV)] * 2)
    assert loss.item() == 0 and targets.shape == (0, 28, 28) and targets.dtype == torch.bool
    loss.backward()
    assert x.grad.shape == x.shape
    lo, tg = mask_loss_per_roi(x.detach(), gts[0], empty[0], None, None)
    assert lo.shape == (0,) and tg.shape == (0, 28, 28)


# ----------------------------------------------------------------------------------------------- realistic batch
def _realistic(g, ks, hw, ng, c):
    """Per image: ng filled ellipses on an H x W mask, K proposals of 10 to 400 px (log-uniform sides) centred within the
    bounding box of their matched ellipse, classes in [0, c)."""
    h, w = hw
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float32), torch.arange(w, dtype=torch.float32), indexing="ij")
    gts, boxes, midx, cls = [], [], [], []
    for k in ks:
        ctr = torch.rand(ng, 2, generator=g) * torch.tensor([w, h])
        rad = 10 + torch.rand(ng, 2, generator=g) * 200
        gts.append(((xx - ctr[:, None, None, 0]) / rad[:, None, None, 0]) ** 2
                   + ((yy - ctr[:, None, None, 1]) / rad[:, None, None, 1]) ** 2 <= 1)
        mi = torch.randint(0, ng, (k,), generator=g)
        side = torch.exp(math.log(10) + torch.rand(k, 2, generator=g) * (math.log(400) - math.log(10)))
        pc = ctr[mi] + (torch.rand(k, 2, generator=g) - 0.5) * 2 * rad[mi]
        boxes.append(torch.cat([pc - side / 2, pc + side / 2], 1))
        midx.append(mi)
        cls.append(torch.randint(0, c, (k,), generator=g))
    return gts, boxes, midx, cls


@functools.lru_cache(maxsize=None)
def realistic_inputs():
    g = torch.Generator().manual_seed(512)
    gts, boxes, midx, cls = _realistic(g, (256, 256), (800, 1333), 6, 80)
    refs = [mr.targets(m.numpy(), b.numpy(), i.numpy(), 28) for m, b, i in zip(gts, boxes, midx)]
    return gts, boxes, midx, cls, _logits(g, 512, 80, 28), refs


def test_realistic_batch():
    """K = 512 non-dyadic proposals of 10-400 px on 800 x 1333 masks, 2 images, C = 80, S = 28.  Targets equal the
    reference except at the few bins whose float64 value is within the bound of 0.5; loss and gradient are checked
    against the reference evaluated on the kernel's own targets."""
    from detectron2_b200.mask_head import mask_loss_per_roi, mask_rcnn_loss

    gts, boxes, midx, cls, x, refs = realistic_inputs()
    xd = x.to(DEV).requires_grad_(True)
    loss, targets = mask_rcnn_loss(xd, _dev(gts), _dev(boxes), _dev(cls), _dev(midx))
    loss.backward()
    t = targets.cpu().numpy()
    t_ref = np.concatenate([r.t for r in refs])
    near = np.concatenate([r.near for r in refs])
    assert not ((t != t_ref) & ~near).any()
    assert near.sum() <= 1e-3 * near.size, near.sum()  # mostly bins with exactly half their samples off the map
    cl = torch.cat(cls).numpy()
    per_roi = torch.cat([mask_loss_per_roi(x[a:a + 256].to(DEV), m.to(DEV), b.to(DEV), i.to(DEV), c.to(DEV))[0]
                         for a, m, b, i, c in zip((0, 256), gts, boxes, midx, cls)])
    ref, tol = mr.loss_per_roi(x.numpy(), t, cl)
    mr.check(per_roi.cpu().numpy(), ref, tol, "realistic loss_per_roi")
    n = 512 * 28 * 28
    mr.check(loss.item(), ref.sum() / n, (tol.sum() + 513 * mr.EPS32 * (ref + tol).sum()) / n, "realistic loss")
    gref, gtol = mr.grad(x.numpy(), t, cl, np.float32(1) / np.float32(n))
    mr.check(xd.grad.cpu().numpy(), gref, gtol[:, None, None, None], "realistic grad")


# ----------------------------------------------------------------------------------------------- properties
def test_p1_proposal_independent_of_k():
    """P1: one CTA per proposal and no reduction across proposals: 16 proposals give the same loss_per_roi and targets
    bits computed alone and among 500 others."""
    from detectron2_b200.mask_head import mask_loss_per_roi

    g = torch.Generator().manual_seed(1)
    (gt,), (b,), (mi,), (cl,) = _realistic(g, (516,), (300, 400), 5, 8)
    x = _logits(g, 516, 8, 28)
    pos = torch.randperm(516, generator=g)[:16]
    gt, b, mi, cl, x = gt.to(DEV), b.to(DEV), mi.to(DEV), cl.to(DEV), x.to(DEV)
    lo_all, tg_all = mask_loss_per_roi(x, gt, b, mi, cl)
    for p in pos.tolist():
        lo, tg = mask_loss_per_roi(x[p:p + 1], gt, b[p:p + 1], mi[p:p + 1], cl[p:p + 1])
        assert torch.equal(lo[0], lo_all[p]) and torch.equal(tg[0], tg_all[p]), p


def test_p2_deterministic():
    """P2: two runs of forward + backward give the same bits."""
    from detectron2_b200.mask_head import mask_rcnn_loss

    gts, boxes, midx, cls, x, _ = realistic_inputs()
    runs = []
    for _ in range(2):
        xd = x.to(DEV).requires_grad_(True)
        loss, targets = mask_rcnn_loss(xd, _dev(gts), _dev(boxes), _dev(cls), _dev(midx))
        loss.backward()
        runs.append((loss.detach(), targets, xd.grad))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_p3_cuda_graph_replay():
    """P3: mask_rcnn_loss forward + backward captured in one CUDA graph, replayed on new logits, boxes, masks, mask indices
    and classes, equals the eager run on the same inputs."""
    from detectron2_b200.mask_head import mask_rcnn_loss

    g = torch.Generator().manual_seed(3)
    ks, hw, ng, c = (64, 48), (200, 300), 4, 80

    def draw():
        gts, boxes, midx, cls = _realistic(g, ks, hw, ng, c)
        return _dev(gts) + _dev(boxes) + _dev(midx) + _dev(cls) + [_logits(g, sum(ks), c, 28).to(DEV)]

    static = draw()
    x = static[-1].clone().requires_grad_(True)

    def step():
        n = len(ks)
        loss, targets = mask_rcnn_loss(x, static[:n], static[n:2 * n], static[3 * n:4 * n], static[2 * n:3 * n])
        loss.backward()
        return loss, targets

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            x.grad = None
            step()
    torch.cuda.current_stream().wait_stream(side)
    x.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, targets = step()
    for _ in range(2):
        new = draw()
        for dst, src in zip(static, new):
            dst.copy_(src)
        with torch.no_grad():
            x.copy_(new[-1])
        graph.replay()
        torch.cuda.synchronize()
        got = (loss.clone(), targets.clone(), x.grad.clone())
        xe = new[-1].clone().requires_grad_(True)
        n = len(ks)
        le, te = mask_rcnn_loss(xe, new[:n], new[n:2 * n], new[3 * n:4 * n], new[2 * n:3 * n])
        le.backward()
        assert torch.equal(got[0], le.detach()) and torch.equal(got[1], te) and torch.equal(got[2], xe.grad)


def test_p4_out_of_range_index_and_class():
    """P4, the library's contract for input the reference would reject: a mask index outside [0, G) gives an all-zero
    target; a class outside [0, C) contributes no loss and no gradient (its targets are still written)."""
    from detectron2_b200.mask_head import mask_loss_per_roi

    g = torch.Generator().manual_seed(4)
    s, c = 14, 3
    gt = torch.rand(2, 25, 23, generator=g) < 0.5
    b = torch.tensor([[2.5, 3.5, 16.5, 17.5]] * 6)
    mi = torch.tensor([0, -1, 2, 7, 1, 1])
    cl = torch.tensor([1, 0, 2, 1, -1, 3])
    x = _logits(g, 6, c, s)
    xd = x.to(DEV).requires_grad_(True)
    lo, tg = mask_loss_per_roi(xd, gt.to(DEV), b.to(DEV), mi.to(DEV), cl.to(DEV))
    ref = mr.targets(gt.numpy(), b.numpy(), mi.numpy(), s)
    assert ref.t[0].any() and not ref.t[1:4].any() and ref.t[4].any()
    assert np.array_equal(tg.cpu().numpy(), ref.t)
    lo.sum().backward()
    lref, ltol = mr.loss_per_roi(x.numpy(), ref.t, cl.numpy())
    mr.check(lo.detach().cpu().numpy(), lref, ltol, "P4 loss_per_roi")
    assert (lo[4:] == 0).all() and lo[:4].gt(0).all()
    assert (xd.grad[4:] == 0).all() and xd.grad[:4].flatten(1).ne(0).any(1).all()


# ----------------------------------------------------------------------------------------------- gt mask dtypes
def encodings(mask, g):
    """The same bitmask as bool, as uint8 with nonzero values 1 / 255, and as float with nonzero values 0.25 / 0.5 / 1."""
    u8 = mask.to(torch.uint8) * torch.tensor([1, 255], dtype=torch.uint8)[torch.randint(0, 2, mask.shape, generator=g)]
    f = mask.float() * torch.tensor([0.25, 0.5, 1.0])[torch.randint(0, 3, mask.shape, generator=g)]
    return {"bool": mask, "uint8": u8, "float": f}


def dtype_case():
    """Dyadic boxes on three random masks: the targets are exact, so every path must give the reference's bits."""
    g = torch.Generator().manual_seed(7)
    gt = torch.rand(3, 33, 37, generator=g) < 0.5
    b = torch.tensor([[2.5, 3.5, 16.5, 17.5], [1.125, 4.5, 8.125, 11.5], [-3.5, 5.5, 38.5, 26.5], [10.5, 0.5, 24.5, 28.5]])
    mi = torch.tensor([0, 2, 1, 2])
    return g, gt, b, mi, mr.targets(gt.numpy(), b.numpy(), mi.numpy(), 14).t


def test_gt_mask_dtypes_read_as_bitmasks():
    """bool, uint8 {0, 1, 255} and float {0, 0.25, 0.5, 1} ground truth give the same targets from mask_loss_per_roi and
    crop_and_resize, equal to the reference's (BitMasks converts with `.to(torch.bool)`: any nonzero value is 1)."""
    from detectron2_b200.mask_head import mask_loss_per_roi
    from detectron2_b200.postprocessing import crop_and_resize

    g, gt, b, mi, t_ref = dtype_case()
    x = torch.zeros(4, 1, 14, 14, device=DEV)
    for name, m in encodings(gt, g).items():
        md = m.to(DEV)
        _, tg = mask_loss_per_roi(x, md, b.to(DEV), mi.to(DEV), None)
        assert np.array_equal(tg.cpu().numpy(), t_ref), name
        cr = crop_and_resize(md[mi.to(DEV)], b.to(DEV), 14)
        assert np.array_equal(cr.cpu().numpy(), t_ref), name
