"""Polygon masks on the GPU (csrc/polygon_masks.cu, the polygon target of postproc.cu's mask loss) bit for bit against the
restatement of pycocotools in tests/polygon_masks_ref.py.

crop cases: COCO-like star polygons of 3 to 300 vertices; overlapping multi-polygon instances (union, not parity) and
self-intersecting polygons; small proposals inside large instances (vertices thousands of lattice units outside the box);
vertices just below 0 and edges on toggle row S; box sides below, at and above 0.1 and w != h; S = 1, 7, 14, 28, 56 and
256; empty instances and mask indices outside [0, G); 1000-vertex polygons.  Full image: 800 x 1333, H = 1, W = 1 and
polygons leaving the image.  Cross-checks: a crop with box [0, 0, S, S] is polygons_to_bitmask(S, S); the fused loss's
targets are the crop's; its loss and gradient are within mask_loss_ref's bounds; fp16 / bf16 logits give the fp32 run's
bits; two runs and a CUDA-graph replay give the eager bits; a multi-image batch equals the per-image calls.
"""
import functools
import math

import numpy as np
import pytest
import torch

import mask_loss_ref as mr
import polygon_masks_ref as pr

pytestmark = pytest.mark.gpu
DEV = "cuda"


def star(rng, n, cx, cy, r0, r1):
    a = np.sort(rng.uniform(0, 2 * np.pi, n))
    r = rng.uniform(r0, r1, n)
    return np.stack([cx + r * np.cos(a), cy + r * np.sin(a)], 1).reshape(-1)


def _scene(seed, n_inst, hw, nv=(3, 300), npoly=(1, 3)):
    """Instances of 1-3 star polygons (3-300 vertices) in an h x w image, some overlapping."""
    rng = np.random.default_rng(seed)
    h, w = hw
    inst = []
    for _ in range(n_inst):
        cx, cy = rng.uniform(0, w), rng.uniform(0, h)
        rad = rng.uniform(5, min(h, w) / 2)
        inst.append([star(rng, int(rng.integers(*nv)), cx + rng.uniform(-rad, rad) / 2, cy + rng.uniform(-rad, rad) / 2,
                          rad * 0.3, rad) for _ in range(int(rng.integers(npoly[0], npoly[1] + 1)))])
    return rng, inst


def _boxes_around(rng, inst, k, lo=2.0, hi=300.0):
    boxes, mi = [], []
    for _ in range(k):
        g = int(rng.integers(0, len(inst)))
        xy = np.concatenate(inst[g]).reshape(-1, 2) if inst[g] else np.zeros((1, 2))
        c = xy[rng.integers(0, len(xy))] + rng.normal(0, 10, 2)
        side = np.exp(rng.uniform(np.log(lo), np.log(hi), 2))
        boxes.append([c[0] - side[0] / 2, c[1] - side[1] / 2, c[0] + side[0] / 2, c[1] + side[1] / 2])
        mi.append(g)
    return np.array(boxes, np.float32), np.array(mi, np.int64)


def _cases():
    """name -> (instances, boxes [K, 4] fp32, mask_index [K], S)."""
    out = {}
    rng, inst = _scene(10, 7, (480, 640))
    b, mi = _boxes_around(rng, inst, 96)
    out["stars_s28"] = (inst, b, mi, 28)
    # union of overlapping polygons, self-intersecting pentagrams
    sq = np.array([0, 0, 20, 0, 20, 20, 0, 20], np.float64)
    penta = np.array([[10 + 9 * math.cos(math.pi / 2 + 4 * math.pi * i / 5), 10 + 9 * math.sin(math.pi / 2 + 4 * math.pi * i / 5)]
                      for i in range(5)]).reshape(-1)
    inst2 = [[sq, sq + 5, sq + 10], [penta], [penta, sq * 0.5 + 5], [sq[::-1].copy()]]
    b2 = np.array([[0, 0, 30, 30], [-1, -1, 21, 21], [2, 3, 17, 19], [0, 0, 20, 20], [4.5, 4.5, 25.5, 25.5]], np.float32)
    out["union_selfintersect_s14"] = (inst2, b2, np.array([0, 1, 2, 3, 0]), 14)
    # small proposals deep inside large instances: vertices far outside the box
    rng, big = _scene(11, 3, (800, 1333), nv=(20, 60))
    big = [[star(rng, 40, 600, 400, 300, 500)], [star(rng, 200, 300, 300, 150, 280), star(rng, 30, 900, 500, 100, 300)]]
    bs = np.array([[598, 398, 600, 401], [600, 400, 600.5, 400.25], [590, 380, 630, 420], [250, 250, 260, 262],
                   [880, 480, 884, 486]], np.float32)
    out["small_in_large_s28"] = (big, bs, np.array([0, 0, 0, 1, 1]), 28)
    # vertices just below 0 (truncation toward zero), edges exactly on toggle rows 0 and S, lattice ties
    tri = np.array([-0.25, -0.05, 7.0, -0.09, 3.5, 7.0])
    edge = np.array([0.0, 0.0, 7.0, 0.0, 7.0, 7.0, 0.0, 7.0])
    tie = np.array([0.3, 0.1, 6.7, 0.1, 6.7, 6.9, 0.3, 6.9])
    bz = np.array([[0, 0, 7, 7], [-0.5, -0.5, 7.5, 7.5], [0.1, 0.1, 6.9, 6.9]], np.float32)
    out["near_zero_row_s_s7"] = ([[tri], [edge], [tie]], np.concatenate([bz, bz, bz]), np.repeat([0, 1, 2], 3), 7)
    # box sides below, at and above 0.1 (S / 0.1 in float64 vs S / w in fp32), w != h
    f01 = float(np.float32(0.1))
    bt = np.array([[5, 5, 5.05, 9], [5, 5, 5 + f01, 5 + f01], [5, 5, 5.2, 5.0999], [5, 5, 5, 5], [5, 5, 9, 5.05],
                   [4.9, 4.9, 5.3, 6.1]], np.float32)
    out["thin_boxes_s14"] = ([[star(np.random.default_rng(1), 12, 5, 5, 0.5, 3)]], bt, np.zeros(6, np.int64), 14)
    for s in (1, 7, 56, 256):
        rng, inst = _scene(20 + s, 5, (300, 400), nv=(3, 80))
        b, mi = _boxes_around(rng, inst, 12, 5, 200)
        out["stars_s%d" % s] = (inst, b, mi, s)
    # empty instances and indices outside [0, G)
    rng, inst = _scene(30, 3, (100, 100))
    inst = [inst[0], [], inst[1], []]
    b, _ = _boxes_around(rng, [inst[0]], 8, 10, 80)
    out["empty_and_bad_index_s28"] = (inst, b, np.array([0, 1, 2, 3, 4, -1, 1 << 40, 2]), 28)
    # LVIS-like thousand-vertex polygons
    rng = np.random.default_rng(40)
    inst = [[star(rng, 1000, 200, 200, 50, 180)], [star(rng, 1500, 150, 260, 20, 120), star(rng, 900, 260, 150, 30, 90)]]
    b, mi = _boxes_around(rng, inst, 24, 10, 300)
    out["lvis_s28"] = (inst, b, mi, 28)
    return out


CASES = _cases()


@functools.lru_cache(maxsize=None)
def _ref(name):
    inst, b, mi, s = CASES[name]
    return pr.crop_and_resize(inst, b, s, mi)


def _pack(instances_per_image):
    from detectron2_b200.polygon_masks import pack_polygons

    return pack_polygons(instances_per_image, DEV)


@pytest.mark.parametrize("name", sorted(CASES))
def test_crop_and_resize(name):
    from detectron2_b200.polygon_masks import polygons_crop_and_resize

    inst, b, mi, s = CASES[name]
    got = polygons_crop_and_resize(_pack([inst]), torch.from_numpy(b).to(DEV), s, torch.from_numpy(mi).to(DEV))
    ref = _ref(name)
    assert got.dtype == torch.bool and got.shape == ref.shape
    bad = got.cpu().numpy() != ref
    assert not bad.any(), (name, np.nonzero(bad.any(axis=(1, 2)))[0].tolist(), int(bad.sum()))
    if name == "empty_and_bad_index_s28":
        assert ref[0].any() and not ref[1].any() and not ref[3:7].any()


def test_crop_k0_and_k_over_65535():
    from detectron2_b200.polygon_masks import polygons_crop_and_resize

    inst, b, mi, s = CASES["stars_s28"]
    pk = _pack([inst])
    assert polygons_crop_and_resize(pk, torch.zeros(0, 4, device=DEV), 28).shape == (0, 28, 28)
    reps = 70000 // len(b) + 1
    got = polygons_crop_and_resize(pk, torch.from_numpy(np.tile(b, (reps, 1))).to(DEV), s,
                                   torch.from_numpy(np.tile(mi, reps)).to(DEV))
    assert got.shape[0] > 65535
    assert np.array_equal(got.cpu().numpy(), np.tile(_ref("stars_s28"), (reps, 1, 1)))


def test_crop_refuses_large_s():
    from detectron2_b200.polygon_masks import polygons_crop_and_resize

    with pytest.raises(RuntimeError):
        polygons_crop_and_resize(_pack([[[np.arange(6.0)]]]), torch.zeros(1, 4, device=DEV), 257)


def test_contracts_for_undefined_input():
    """Non-finite vertex, lattice value outside +-2^30, non-finite box: the polygon adds nothing; polygon offsets out of
    order or past V and instance offsets past P: empty, never an out-of-bounds read."""
    from detectron2_b200.polygon_masks import PackedPolygons, polygons_crop_and_resize, polygons_to_bitmask

    sq = [0.0, 0, 6, 0, 6, 6, 0, 6]
    tri = [1.0, 1, 5, 1, 3, 5]
    coords = np.array(sq + tri + [0, 0, np.nan, 0, 3, 3] + [0, 0, 3e8, 0, 3, 3] + tri, np.float64).reshape(-1, 2)
    # polygons: 0 square, 1 triangle, 2 NaN, 3 huge, 4 triangle; 5 out of order, 6 past V
    poly_start = [0, 4, 7, 10, 13, 16, 10, 40]
    inst_start = [1, 3, 5, 6, 7, 6, 100]
    pk = PackedPolygons(torch.tensor(coords, device=DEV), torch.tensor(poly_start, dtype=torch.int32, device=DEV),
                        torch.tensor(inst_start, dtype=torch.int32, device=DEV), (0, 6))
    # instance 0 = polygons [1, 3): triangle + NaN; 1 = [3, 5): huge + triangle; 2 = [5, 6); 3 = [6, 7); 4 = [7, 6);
    # 5 = [6, 100)
    full = polygons_to_bitmask(pk, 8, 8).cpu().numpy()
    trim = pr.to_bitmask([np.array(tri)], 8, 8)
    assert trim.any()
    assert np.array_equal(full[0], trim) and np.array_equal(full[1], trim) and not full[2:].any()
    b = torch.tensor([[0, 0, 8, 8], [0, 0, 8, 8], [float("nan"), 0, 8, 8], [0, 0, float("inf"), 8]], device=DEV)
    crop = polygons_crop_and_resize(pk, b, 8, torch.tensor([0, 1, 0, 0], device=DEV)).cpu().numpy()
    assert np.array_equal(crop[0], trim) and np.array_equal(crop[1], trim) and not crop[2:].any()


# ------------------------------------------------------------------------------------------------ full image
def test_polygons_to_bitmask_full_image():
    from detectron2_b200.polygon_masks import polygons_to_bitmask

    rng, inst = _scene(50, 7, (800, 1333))
    inst.append([np.array([-50.0, -40, 1400, 300, 700, 900])])  # leaves the image on three sides
    inst.append([])
    got = polygons_to_bitmask(_pack([inst[:4], inst[4:]]), 800, 1333).cpu().numpy()
    for g, polys in enumerate(inst):
        assert np.array_equal(got[g], pr.to_bitmask(polys, 800, 1333)), g


@pytest.mark.parametrize("hw", [(1, 57), (61, 1), (1, 1), (300, 700)])
def test_polygons_to_bitmask_thin(hw):
    from detectron2_b200.polygon_masks import polygons_to_bitmask

    h, w = hw
    rng = np.random.default_rng(h * 1000 + w)
    inst = [[star(rng, 9, w / 2, h / 2, 0.3, max(h, w))], [np.array([-1.0, -1, w + 1, -1, w + 1, h + 1, -1, h + 1])],
            [star(rng, 5, w / 2, h / 2, 0.2, 2), star(rng, 50, 0, 0, 1, max(h, w))]]
    got = polygons_to_bitmask(_pack([inst]), h, w).cpu().numpy()
    for g, polys in enumerate(inst):
        assert np.array_equal(got[g], pr.to_bitmask(polys, h, w)), g


def test_crop_of_unit_box_is_bitmask():
    """crop_and_resize with box [0, 0, S, S] is the identity transform: it equals polygons_to_bitmask(S, S)."""
    from detectron2_b200.polygon_masks import polygons_crop_and_resize, polygons_to_bitmask

    for s in (28, 57):
        _, inst = _scene(60 + s, 6, (s, s), nv=(3, 40))
        pk = _pack([inst])
        crop = polygons_crop_and_resize(pk, torch.tensor([[0.0, 0, s, s]] * 6, device=DEV), s)
        assert torch.equal(crop, polygons_to_bitmask(pk, s, s))


# ------------------------------------------------------------------------------------------------ the fused loss
def _batch(seed, ks=(128, 128), n_inst=7, c=80, s=28):
    rng = np.random.default_rng(seed)
    imgs, boxes, midx, cls = [], [], [], []
    for i, k in enumerate(ks):
        _, inst = _scene(seed * 10 + i, n_inst, (600, 900), nv=(10, 300))
        b, mi = _boxes_around(rng, inst, k, 10, 300)
        mi[::17] = -1  # out of range: all-zero target
        imgs.append(inst)
        boxes.append(torch.from_numpy(b))
        midx.append(torch.from_numpy(mi))
        cls.append(torch.from_numpy(rng.integers(0, c, k)))
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(sum(ks), c, s, s, generator=g) * 4
    return imgs, boxes, midx, cls, x


def _loss(imgs, boxes, midx, cls, x):
    from detectron2_b200.mask_head import mask_rcnn_loss

    xd = x.to(DEV).requires_grad_(True)
    loss, targets = mask_rcnn_loss(xd, _pack(imgs), [b.to(DEV) for b in boxes], [c.to(DEV) for c in cls],
                                   [m.to(DEV) for m in midx])
    loss.backward()
    return loss.detach(), targets, xd.grad


@functools.lru_cache(maxsize=None)
def _loss_case():
    imgs, boxes, midx, cls, x = _batch(7)
    t_ref = np.concatenate([pr.crop_and_resize(inst, b.numpy(), 28, m.numpy()) for inst, b, m in zip(imgs, boxes, midx)])
    return imgs, boxes, midx, cls, x, t_ref


def test_fused_loss_against_reference():
    from detectron2_b200.mask_head import mask_loss_polygons
    from detectron2_b200.polygon_masks import polygons_crop_and_resize

    imgs, boxes, midx, cls, x, t_ref = _loss_case()
    loss, targets, grad = _loss(imgs, boxes, midx, cls, x)
    assert np.array_equal(targets.cpu().numpy(), t_ref)
    # the targets equal crop_and_resize's, image by image
    crops = torch.cat([polygons_crop_and_resize(_pack([inst]), b.to(DEV), 28, m.to(DEV))
                       for inst, b, m in zip(imgs, boxes, midx)])
    assert torch.equal(targets, crops)
    total, s2 = x.shape[0], 28 * 28
    cl = torch.cat(cls).numpy()
    ref, tol = mr.loss_per_roi(x.numpy(), t_ref, cl)
    pk = _pack(imgs)
    from detectron2_b200.polygon_masks import batch_mask_index

    gmi = batch_mask_index(pk, [len(b) for b in boxes], [m.to(DEV) for m in midx], DEV)
    per_roi, _ = mask_loss_polygons(x.to(DEV), pk.coords, pk.poly_start, pk.inst_start, torch.cat(boxes).to(DEV), gmi,
                                    torch.cat(cls).to(DEV))
    mr.check(per_roi.cpu().numpy(), ref, tol, "polygon loss_per_roi")
    assert torch.equal(loss, per_roi.sum() / float(total * s2))
    gref, gtol = mr.grad(x.numpy(), t_ref, cl, np.float32(1) / np.float32(total * s2))
    mr.check(grad.cpu().numpy(), gref, gtol[:, None, None, None], "polygon grad")


@pytest.mark.parametrize("dtype", ["float16", "bfloat16"])
def test_fused_loss_half_logits(dtype):
    imgs, boxes, midx, cls, x, _ = _loss_case()
    xh = x.to(getattr(torch, dtype))
    l32, t32, g32 = _loss(imgs, boxes, midx, cls, xh.float())
    lh, th, gh = _loss(imgs, boxes, midx, cls, xh)
    assert torch.equal(lh, l32) and torch.equal(th, t32) and gh.dtype == xh.dtype and torch.equal(gh, g32.to(xh.dtype))


def test_fused_loss_deterministic_and_per_image():
    """Two runs give the same bits; the batch equals each image run alone."""
    imgs, boxes, midx, cls, x, _ = _loss_case()
    a, b = _loss(imgs, boxes, midx, cls, x), _loss(imgs, boxes, midx, cls, x)
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    from detectron2_b200.mask_head import mask_rcnn_loss

    k0 = 0
    for inst, bx, m, c in zip(imgs, boxes, midx, cls):
        k = len(bx)
        _, tg = mask_rcnn_loss(x[k0:k0 + k].to(DEV), _pack([inst]), [bx.to(DEV)], [c.to(DEV)], [m.to(DEV)])
        assert torch.equal(tg, a[1][k0:k0 + k])
        k0 += k


def test_fused_loss_cuda_graph_replay():
    from detectron2_b200.mask_head import mask_rcnn_loss

    imgs, boxes, midx, cls, x, _ = _loss_case()
    pk = _pack(imgs)
    static_b = [b.to(DEV) for b in boxes]
    static_m = [m.to(DEV) for m in midx]
    static_c = [c.to(DEV) for c in cls]
    xs = x.to(DEV).clone().requires_grad_(True)

    def step():
        loss, targets = mask_rcnn_loss(xs, pk, static_b, static_c, static_m)
        loss.backward()
        return loss, targets

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            xs.grad = None
            step()
    torch.cuda.current_stream().wait_stream(side)
    xs.grad = None
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        loss, targets = step()
    rng = np.random.default_rng(3)
    for _ in range(2):
        nb = [torch.from_numpy(b.numpy() + rng.uniform(-5, 5, b.shape).astype(np.float32)) for b in boxes]
        nx = torch.randn(x.shape) * 4
        for dst, src in zip(static_b, nb):
            dst.copy_(src)
        with torch.no_grad():
            xs.copy_(nx)
        graph.replay()
        torch.cuda.synchronize()
        got = (loss.clone(), targets.clone(), xs.grad.clone())
        le, te, ge = _loss(imgs, nb, midx, cls, nx)
        assert torch.equal(got[0], le) and torch.equal(got[1], te) and torch.equal(got[2], ge)
