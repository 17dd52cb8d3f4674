"""Polygon masks on the CPU: the restatement in tests/polygon_masks_ref.py pinned by checks that do not come from itself,
the kernel's closed-form crossing against the literal walk, the packer, the argument checks of the native entry points
(nothing launched) and the fake kernels."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import polygon_masks_ref as pr


def _bbox(m):
    ys, xs = np.nonzero(m)
    return (0, 0, 0, 0) if len(xs) == 0 else (xs.min(), ys.min(), xs.max() + 1, ys.max() + 1)


@pytest.mark.parametrize("box", [(1, 0, 4, 4), (1, 1, 3, 4), (0, 0, 0, 0)])
def test_reference_known_answers(box):
    """detectron2 tests/structures/test_masks.py:33-40: the rectangle polygon of a box in a 4 x 4 image has that box as its
    mask's bounding box ((0, 0, 0, 0): an empty mask)."""
    x0, y0, x1, y1 = box
    poly = np.array([x0, y0, x1, y0, x1, y1, x0, y1], np.float64)
    m = pr.to_bitmask([poly], 4, 4)
    assert _bbox(m) == box
    assert np.array_equal(pr.fr_poly_literal(poly, 4, 4), m)


def _random_polygon(rng, n, lo, hi):
    return rng.uniform(lo, hi, 2 * n)


def _inside(px, py, P):
    n, c = len(P) // 2, False
    for i in range(n):
        x1, y1, x2, y2 = P[2 * i], P[2 * i + 1], P[(2 * i + 2) % (2 * n)], P[(2 * i + 3) % (2 * n)]
        if (y1 > py) != (y2 > py) and px < x1 + (py - y1) * (x2 - x1) / (y2 - y1):
            c = not c
    return c


def _dist(px, py, P):
    n, best, p = len(P) // 2, math.inf, np.array([px, py])
    for i in range(n):
        a, b = np.array(P[2 * i:2 * i + 2]), np.array([P[(2 * i + 2) % (2 * n)], P[(2 * i + 3) % (2 * n)]])
        t = np.clip(np.dot(p - a, b - a) / max(np.dot(b - a, b - a), 1e-12), 0, 1)
        best = min(best, np.linalg.norm(p - (a + t * (b - a))))
    return best


def test_even_odd_at_pixel_centres():
    """An independent rule: pixel (r, c) is inside when its centre (c + 1/2, r + 1/2) is inside the polygon by the even-odd
    rule.  The rasterizer moves every vertex by at most 0.1 px per axis (rounding to the 1/5 px lattice), so each edge by
    at most sqrt(2) 0.1 < 0.15 px, and the DDA rounds each point to the lattice, at most 0.1 px more across the edge; and a
    pixel belongs to a column's run when its centre row lies past the lattice crossing of the column's centre line.  So every
    pixel whose centre is farther than 0.3 px from every edge must agree."""
    rng = np.random.default_rng(0)
    bad = total = 0
    for _ in range(30):
        P = list(_random_polygon(rng, rng.integers(3, 9), -3, 23))
        m = pr.fr_poly(np.array(P), 20, 20)
        for r in range(20):
            for c in range(20):
                if _dist(c + .5, r + .5, P) > 0.3:
                    total += 1
                    bad += m[r, c] != _inside(c + .5, r + .5, P)
    assert total > 5000 and bad == 0, (bad, total)


def _lattice_polygons(rng, count):
    """Random polygons over three scales, a third snapped to k/5 +- 0.1 (exactly between lattice points), a fifth with a
    repeated vertex (a zero-length edge)."""
    for it in range(count):
        n = int(rng.integers(3, 12))
        sc = float(rng.choice([1, 10, 300]))
        P = rng.uniform(-sc, sc + 28, 2 * n)
        if it % 3 == 0:
            P = np.round(P * 5) / 5 + rng.choice([0, .1, -.1, .3], 2 * n)
        if it % 5 == 0:
            P[2:4] = P[0:2]
        yield P


def test_even_toggle_count_per_column():
    """Every column of every polygon gets an even number of kept pairs (so columns rasterize independently)."""
    rng = np.random.default_rng(1)
    for P in _lattice_polygons(rng, 600):
        L = pr.snap(P)
        c, _ = pr.toggles(*pr.walk(L[0::2], L[1::2]), 28, 28)
        assert (np.bincount(c, minlength=28) % 2 == 0).all(), P


def test_vectorised_walk_equals_literal():
    rng = np.random.default_rng(2)
    for P in _lattice_polygons(rng, 150):
        h, w = int(rng.integers(1, 30)), int(rng.integers(1, 30))
        assert np.array_equal(pr.fr_poly(P, h, w), pr.fr_poly_literal(P, h, w)), (P, h, w)


def _edges(rng):
    yield from [(0, 0, 0, 0), (7, 7, 7, 7), (-3, 4, -3, 4), (2, 2, 3, 2), (12, -5, 12, 50), (-7, -9, -1, -2),
                (-4, 10, 40, 11), (40, 11, -4, 10), (1, 0, 100000, 3), (3, 100000, 1, 0), (-100000, 7, 100000, -3)]
    for _ in range(3000):
        sc = int(rng.choice([5, 40, 200, 5000, 200000]))
        xs, ys, xe, ye = (int(v) for v in rng.integers(-sc, sc + 150, 4))
        if rng.random() < 0.2:
            xe = xs + int(rng.integers(-2, 3))
        if rng.random() < 0.2:
            ye = ys + int(rng.integers(-2, 3))
        yield xs, ys, xe, ye


def test_closed_form_equals_walk():
    """The kernel's per-edge closed form (one toggle per column, located by solving, then checked with the DDA's own
    expression) equals the literal walk's kept pairs on random edges: negative, huge and zero-length ones included."""
    rng = np.random.default_rng(3)
    for e in _edges(rng):
        walked, count = pr.walk_edge_toggles(*e, 30)
        assert all(v == 1 for v in count.values()), e  # at most one toggle per column and edge
        assert pr.closed_form_edge(*e, 0, 29) == walked, e
        assert pr.closed_form_edge(*e, 3, 7) == {c: v for c, v in walked.items() if 3 <= c <= 7}, e


def test_transform_dtypes():
    """rasterize_polygons_within_box: w in fp32, S / w in fp32 at w >= 0.1, else S / 0.1 in float64; float64 polygons."""
    box = np.array([1.25, 2.5, 1.25 + 0.05, 9.0], np.float32)
    (p,) = pr.transform([np.array([2.0, 3.0, 4.0, 5.0, 6.0, 7.0])], box, 28)
    w, h = box[2] - box[0], box[3] - box[1]
    assert p[0] == (2.0 - np.float64(box[0])) * (28 / 0.1)
    assert p[1] == (3.0 - np.float64(box[1])) * np.float64(np.float32(28) / h)


def test_crop_contracts():
    inst = [[np.array([0.0, 0, 8, 0, 8, 8, 0, 8])], []]
    boxes = np.array([[0, 0, 8, 8], [0, 0, 8, 8], [0, 0, 8, 8], [np.nan, 0, 8, 8]], np.float32)
    out = pr.crop_and_resize(inst, boxes, 4, [0, 1, 5, 0])
    assert out[0].all() and not out[1:].any()


def test_packer():
    from detectron2_b200.polygon_masks import pack_polygons

    pk = pack_polygons([[[[0, 0, 4, 0, 4, 4]], []], [[torch.tensor([1.0, 1, 3, 1, 3, 3, 1, 3]), np.arange(6.0)]]], "cpu")
    assert pk.coords.dtype == torch.float64 and pk.coords.shape == (3 + 4 + 3, 2)
    assert pk.poly_start.tolist() == [0, 3, 7, 10] and pk.poly_start.dtype == torch.int32
    assert pk.inst_start.tolist() == [0, 1, 1, 3] and pk.inst_start.dtype == torch.int32
    assert pk.image_start == (0, 2, 3) and pk.num_instances == 3
    empty = pack_polygons([], "cpu")
    assert empty.coords.shape == (0, 2) and empty.inst_start.tolist() == [0] and empty.image_start == (0,)
    for bad in ([1.0, 2, 3, 4], [1.0, 2, 3, 4, 5, 6, 7]):
        with pytest.raises(ValueError, match="Cannot create a polygon from %d coordinates" % len(bad)):
            pack_polygons([[[bad]]], "cpu")


def test_batch_mask_index_stays_in_its_image():
    from detectron2_b200.polygon_masks import PackedPolygons, batch_mask_index

    pk = PackedPolygons(None, None, None, (0, 2, 2, 5))
    mi = batch_mask_index(pk, [3, 1, 4], [torch.tensor([0, 1, 2]), torch.tensor([0]), torch.tensor([-1, 0, 2, 3])], "cpu")
    assert mi.tolist() == [0, 1, -1, -1, -1, 2, 4, -1]
    assert batch_mask_index(pk, [2, 0, 4], None, "cpu").tolist() == [0, 1, 2, 3, 4, -1]
    with pytest.raises(RuntimeError):
        batch_mask_index(pk, [1, 1], None, "cpu")


def test_abi_refusals_without_launch():
    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL = -1
    p = C.c_void_p(16)  # never dereferenced: the checks fail first
    crop = dict(coords=p, V=10, ps=p, P=2, ist=p, G=2, boxes=p, mi=p, K=5, S=28, out=p, stream=None)

    def call_crop(**over):
        return lib.d2b_polygons_crop_and_resize(*dict(crop, **over).values())

    for over in (dict(K=-1), dict(S=0), dict(S=257), dict(V=-1), dict(P=-1), dict(G=-1), dict(boxes=None), dict(out=None),
                 dict(ist=None), dict(ps=None), dict(coords=None)):
        assert call_crop(**over) == EINVAL, over
    assert call_crop(K=0, S=257) == EINVAL  # the shape checks come first
    assert call_crop(K=0, boxes=None, out=None) == 0  # nothing to do, nothing launched

    bm = dict(coords=p, V=10, ps=p, P=2, ist=p, G=2, H=800, W=1333, out=p, stream=None)

    def call_bm(**over):
        return lib.d2b_polygons_to_bitmask(*dict(bm, **over).values())

    for over in (dict(V=-1), dict(P=-1), dict(G=-1), dict(H=0), dict(W=0), dict(H=65536, W=65536), dict(out=None),
                 dict(ist=None), dict(ps=None), dict(coords=None)):
        assert call_bm(**over) == EINVAL, over
    assert call_bm(G=0, out=None, ist=None) == 0

    loss = dict(logits=p, K=5, C=80, S=28, coords=p, V=10, ps=p, P=2, ist=p, G=2, boxes=p, mi=p, cls=p, lo=p, tg=p,
                stream=None)

    def call_loss(**over):
        return lib.d2b_mask_loss_polygons_forward(*dict(loss, **over).values())

    for over in (dict(K=-1), dict(C=0), dict(S=0), dict(S=257), dict(V=-1), dict(P=-1), dict(G=-1), dict(logits=None),
                 dict(boxes=None), dict(lo=None), dict(tg=None), dict(ist=None), dict(ps=None), dict(coords=None)):
        assert call_loss(**over) == EINVAL, over
    assert call_loss(K=0, logits=None, boxes=None, lo=None, tg=None) == 0
    assert call_loss(G=0, ist=None, P=0, ps=None, V=0, coords=None, K=0) == 0


def test_fake_kernels_trace_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    from detectron2_b200 import mask_head, polygon_masks as pm

    with FakeTensorMode():
        pk = pm.PackedPolygons(torch.empty(40, 2, dtype=torch.float64, device="cuda"),
                               torch.empty(5, dtype=torch.int32, device="cuda"),
                               torch.empty(4, dtype=torch.int32, device="cuda"), (0, 3))
        out = pm.polygons_crop_and_resize(pk, torch.empty(7, 4, device="cuda"), 28)
        assert out.shape == (7, 28, 28) and out.dtype == torch.bool
        bm = pm.polygons_to_bitmask(pk, 80, 133)
        assert bm.shape == (3, 80, 133) and bm.dtype == torch.bool
        for dt in (torch.float32, torch.float16, torch.bfloat16):
            x = torch.empty(7, 80, 28, 28, device="cuda", dtype=dt)
            lo, tg = mask_head.mask_loss_polygons(x, pk.coords, pk.poly_start, pk.inst_start,
                                                  torch.empty(7, 4, device="cuda"), None, None)
            assert lo.shape == (7,) and lo.dtype == torch.float32 and tg.shape == (7, 28, 28) and tg.dtype == torch.bool
