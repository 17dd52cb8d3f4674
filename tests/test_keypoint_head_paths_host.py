"""The float64 reference and path model of tests/keypoints_ref.py without a GPU: the reference against the fixture made from
the real detectron2 functions (tests/golden/keypoints.npz), the bicubic bound against PyTorch's CPU resize over a sweep of
map and output sizes, the loss against float64 F.cross_entropy and gradcheck, the launch arithmetic, and the labels of
the GPU cases (tests/test_keypoint_head_paths_gpu.py asserts the labels the kernels' values reach)."""
import math

import pytest
import torch
import torch.nn.functional as F

import keypoints_ref as R
import test_keypoint_head_paths_gpu as G
from test_keypoint_head_host import T as from_np
from test_keypoint_head_host import heatmaps, loss_inputs

F64 = torch.float64


def test_reference_decodes_the_fixture(golden):
    """At the fixture's pixels its fp32 CPU logits lie within the bound, and its positions are the fp32 formula's."""
    d = golden("keypoints")
    maps, rois, xy = heatmaps(d), from_np(d["rois"]), from_np(d["xy_preds"])
    for i in range(len(rois)):
        g = R.roi_geometry(rois[i])
        v, e = R.bicubic(maps[i], g["ho"], g["wo"], any_order=True)
        px, py = R.positions(g)
        ox = (px[None] == xy[i, :, 0:1]).to(torch.uint8).argmax(1)
        oy = (py[None] == xy[i, :, 1:2]).to(torch.uint8).argmax(1)
        assert torch.equal(px[ox], xy[i, :, 0]) and torch.equal(py[oy], xy[i, :, 1]), i
        k = torch.arange(maps.shape[1])
        got = xy[i, :, 2].to(F64)
        assert bool(((got - v[k, oy, ox]).abs() <= e[k, oy, ox]).all()), i
        s, es = R.score(maps[i], xy[i, :, 2])
        assert bool(((xy[i, :, 3].to(F64) - s).abs() <= es + 4 * R.U * s).all()), i


def test_reference_targets_and_loss_match_the_fixture(golden):
    from detectron2_b200 import keypoint_head as kh

    d = golden("keypoints")
    boxes, kps, logits = loss_inputs(d)
    S = int(d["S"])
    targets, valids = [], []
    for i in (0, 2):
        cx, dx = R.exact_cells(kps[i][..., 0], boxes[i][:, None, 0], boxes[i][:, None, 2], S)
        cy, dy = R.exact_cells(kps[i][..., 1], boxes[i][:, None, 1], boxes[i][:, None, 3], S)
        vis = kps[i][..., 2] > 0
        v = (cx >= 0) & (cx < S) & (cy >= 0) & (cy < S) & vis
        dec = (dx & dy) | ~vis
        assert bool(dec.all()), i
        assert torch.equal(v.long(), from_np(d[f"valid{i}"])) and torch.equal(torch.where(v, cy * S + cx, 0),
                                                                              from_np(d[f"target{i}"])), i
    for i in range(3):
        if len(boxes[i]):
            t, v = kh._keypoints_to_heatmap_host(kps[i], boxes[i], S)
            targets.append(t)
            valids.append(v)
    t, v = torch.cat(targets), torch.cat(valids)
    ref = R.LossRef(logits, t, v)
    n = int(v.sum())
    terms, errs = ref.loss[ref.valid], ref.e_loss[ref.valid]
    for norm, key in ((n, "loss_none"), (7.5, "loss_norm")):
        want = float(d[key])
        bound = R.total_bound(terms, errs) / norm * (1 + 2 * R.U) + 2 * R.U * abs(want)
        assert abs(float(terms.sum()) / norm - want) <= bound, key


SWEEP_S = [1, 2, 5, 17, 56, 112, 241]


@pytest.mark.parametrize("S", SWEEP_S)
def test_bound_contains_the_cpu_bicubic(S):
    """PyTorch's CPU resize rounds its own sequence (products and sums separately); the any-order bound holds it at
    every pixel, and axis_taps asserts that the emulated fma was exact for every tap."""
    g = torch.Generator().manual_seed(S)
    m = torch.randn(2, S, S, generator=g) * 3
    m[1, 0, :] = 40.0  # a large border row: cancellation in the taps
    for o in sorted({1, 2, 3, max(S - 1, 1), S, S + 1, 2 * S + 3, 700}):
        for oh, ow in ((o, o), (o, S + 1), (S, o)):
            v, e = R.bicubic(m, oh, ow, any_order=True)
            cpu = F.interpolate(m[None], size=(oh, ow), mode="bicubic", align_corners=False)[0].to(F64)
            bad = (cpu - v).abs() > e
            assert not bool(bad.any()), (S, oh, ow, int(bad.sum()))


def test_taps_restate_the_fp32_source_index():
    idx, t = R.axis_taps(56, 57)
    assert int(idx[0, 0]) == 0 and int(idx[-1, 3]) == 55 and bool(((t >= 0) & (t < 1)).all())
    assert torch.equal(R.axis_taps(17, 34)[1][:4], torch.tensor([0.75, 0.25, 0.75, 0.25], dtype=F64))
    c = R.coeffs_exact(torch.tensor([0.0, 0.3], dtype=F64))
    assert torch.equal(c[0], torch.tensor([0.0, 1.0, 0.0, 0.0], dtype=F64))
    assert abs(float(c[1].sum()) - 1.0) < 1e-15


def test_loss_reference_is_float64_cross_entropy():
    g = torch.Generator().manual_seed(0)
    x = torch.randn(3, 4, 5, 5, generator=g)
    t = torch.randint(0, 25, (3, 4), generator=g)
    v = torch.ones(3, 4, dtype=torch.long)
    v[0, 1] = 0
    ref = R.LossRef(x, t, v)
    ce = F.cross_entropy(x.to(F64).reshape(12, 25), t.reshape(-1), reduction="none")
    keep = v.reshape(-1).bool()
    torch.testing.assert_close(ref.loss[keep], ce[keep], rtol=1e-14, atol=1e-14)
    assert float(ref.loss[~keep].abs().max()) == 0.0 and bool((ref.e_loss[keep] > 0).all())
    gs = torch.rand(3, 4, generator=g)
    xr = x.to(F64).reshape(12, 25).requires_grad_(True)
    (F.cross_entropy(xr, t.reshape(-1), reduction="none") * gs.reshape(-1).to(F64) * keep).sum().backward()
    gr, ge = ref.grad(gs)
    torch.testing.assert_close(gr, xr.grad, rtol=1e-13, atol=1e-15)
    assert bool((ge[keep] > 0).all()) and bool((ge[~keep] == 0).all())

    def f(z):
        return (R._lse(z) - z.gather(1, t.reshape(-1, 1))[:, 0]).sum()

    assert torch.autograd.gradcheck(f, (torch.randn(12, 25, generator=g, dtype=F64, requires_grad=True),))


def test_loss_reference_nonfinite_rules():
    x = torch.zeros(4, 1, 2, 2)
    x[0, 0, 0, 1], x[1, 0, 1, 0], x[2, 0, 0, 0] = math.nan, math.inf, -math.inf
    t = torch.tensor([[0], [0], [0], [1]])
    ref = R.LossRef(x, t, torch.ones(4, 1, dtype=torch.long))
    assert math.isnan(ref.loss[0]) and math.isnan(ref.loss[1]) and ref.loss[2] == math.inf
    assert abs(float(ref.loss[3]) - math.log(4)) < 1e-15
    g, _ = ref.grad(torch.ones(4, 1))
    assert bool(torch.isnan(g[:2]).all())
    # the target on the -inf logit: an infinite loss, p = 0 there and 1/3 at the three others
    torch.testing.assert_close(g[2], torch.tensor([-1.0, 1 / 3, 1 / 3, 1 / 3], dtype=F64), rtol=1e-15, atol=0)


def test_exact_cells_decide_the_boundaries():
    S = 56
    lo, hi = torch.tensor([0.0]), torch.tensor([3.0])
    c = torch.tensor([0.0, 3.0, 1.5, 3.0 * 7 / 56, 3.0 * 7 / 56 + 1e-3, -1.0, math.nan])
    cell, dec = R.exact_cells(c, lo, hi, S)
    assert cell[:3].tolist() == [0, S - 1, 28] and dec[:3].tolist() == [True, True, False]
    assert cell[4].item() == 7 and bool(dec[4]) and bool(dec[5]) and cell[5].item() == -19 and not bool(dec[6])
    _, dec = R.exact_cells(torch.tensor([0.0, 1.0]), torch.tensor([0.0]), torch.tensor([1e-40]), S)
    assert not bool(dec.any())  # subnormal width: the fp32 steps overflow


# ---- the path model ---------------------------------------------------------------------------------------------------
def test_shared_memory_and_tile_arithmetic():
    assert all(R.smem_bytes(s) <= R.SMEM_OPTIN for s in range(1, R.MAX_S + 1))
    assert R.smem_bytes(R.MAX_S) == 232324 and R.SMEM_OPTIN == 232448 and R.smem_bytes(R.MAX_S + 1) > R.SMEM_OPTIN
    assert [s for s in range(1, R.MAX_S + 1) if R.needs_optin(s)] == list(range(111, R.MAX_S + 1))
    assert [R.tiles(n) for n in (1, 4095, 4096, 4097, 8192, 2 ** 32)] == [1, 1, 1, 2, 2, 2 ** 20]
    p = R.decode_paths(torch.tensor([[0.0, 0.0, 1333.0, 800.0]] * 3), 56, 17)
    assert p["tiles"] == [261] * 3 and p["items"] == 3 * 261 * 17 and p["grid"] == 528 and p["per_cta"] == 26
    assert R.decode_paths(torch.zeros(1025, 4), 5, 1)["chunk"] == 2 and R.decode_paths(torch.zeros(2049, 4), 5, 1)["chunk"] == 3
    g = R.roi_geometry(torch.tensor([0.0, 0.0, 65536.0, 65536.0]))
    assert g["ok"] and g["wo"] * g["ho"] == 2 ** 32
    assert not R.roi_geometry(torch.tensor([0.0, 0.0, 65536.0, 65537.0]))["ok"]


@pytest.mark.parametrize("c", G.DECODE, ids=lambda c: c.name)
def test_decode_case_reaches_its_shape_labels(c):
    rois = _rois(c)
    got = R.decode_shape_labels(rois, c.S, c.K, c.dtype) | R.roi_labels(rois)
    assert (c.labels & R.DECODE_SHAPE_LABELS) <= got, (c.name, sorted((c.labels & R.DECODE_SHAPE_LABELS) - got))
    assert c.labels <= R.DECODE_SHAPE_LABELS | R.DECODE_VALUE_LABELS


def _rois(c):
    dev = G.DEV
    G.DEV = torch.device("cpu")
    try:
        return G.decode_inputs(c)[1]
    finally:
        G.DEV = dev


@pytest.mark.parametrize("c", G.LOSS, ids=lambda c: c.name)
def test_loss_case_reaches_its_shape_labels(c):
    got = R.loss_shape_labels(c.N, c.K, c.S, c.dtype)
    assert (c.labels & R.LOSS_SHAPE_LABELS) <= got, (c.name, sorted((c.labels & R.LOSS_SHAPE_LABELS) - got))
    assert c.labels <= R.LOSS_SHAPE_LABELS | R.LOSS_VALUE_LABELS


def test_every_label_is_declared():
    dec = set().union(*(c.labels for c in G.DECODE))
    assert dec == R.DECODE_SHAPE_LABELS | R.DECODE_VALUE_LABELS, sorted((R.DECODE_SHAPE_LABELS | R.DECODE_VALUE_LABELS) ^ dec)
    loss = set().union(*(c.labels for c in G.LOSS))
    assert loss == R.LOSS_SHAPE_LABELS | R.LOSS_VALUE_LABELS, sorted((R.LOSS_SHAPE_LABELS | R.LOSS_VALUE_LABELS) ^ loss)
    assert {1, 2, 5, 17, 112, 241} <= {c.S for c in G.DECODE} and {1, 3, 17} <= {c.K for c in G.DECODE}
    assert {1, 5, 16, 17, 241} <= {c.S for c in G.LOSS}
