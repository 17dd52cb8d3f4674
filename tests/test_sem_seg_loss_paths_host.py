"""The float64 reference and path model of tests/sem_seg_loss_ref.py without a GPU: the reference against the reference
fixture (tests/golden/sem_seg_loss.npz), against the fp32 restatement of detectron2_b200/semantic_seg.py, against float64
F.interpolate + F.cross_entropy where the fp32 scale is exact, and by gradcheck; the backward's region bound over every
stride and map size (the kernel clamps a region to its bound without an error, so a region past it would drop gradient
terms silently); the backward plans' shared memory; and the labels of the GPU cases.

The labels a case's values reach (R.VALUE_LABELS) are asserted by tests/test_sem_seg_loss_paths_gpu.py, which sees the
kernel's own per-pixel values; here every case's shape labels are checked and every label must be declared by a case."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import sem_seg_loss_ref as R
import test_sem_seg_loss_paths_gpu as G
from detectron2_b200 import semantic_seg as S
from sem_seg_ref import CASES, make_case

F64 = torch.float64


def ref_loss(name):
    """(Ref, loss, selection) of a fixture case: the mean, top-k 1.0, or the stable top-k of the float64 values."""
    _, _, _, _, s, ignore, top_k, _, _ = CASES[name]
    logits, targets, weights = make_case(name)
    ref = R.Ref(logits, targets, s, ignore, top_k, weights)
    sel = None
    if ref.mode == "select":
        x = ref.xv.reshape(-1)
        key = torch.where(torch.isnan(x), float("inf"), torch.where(x == 0, 0.0, x))
        sel = torch.zeros(ref.P, dtype=torch.uint8)
        sel[torch.sort(key, descending=True, stable=True).indices[: ref.k]] = 1
        sel = sel.view(targets.shape)
    total, _ = ref.loss_sum(sel)
    div = ref.count if ref.mode == "mean" else ref.k
    return ref, total / div if div else float("nan"), sel, div


@pytest.mark.parametrize("name", list(CASES))
def test_reference_matches_the_fixture_and_the_restatement(name, golden):
    gold = golden("sem_seg_loss")
    ref, loss, sel, div = ref_loss(name)
    want = float(gold[name + "_loss"])
    _, _, _, _, s, ignore, top_k, _, _ = CASES[name]
    logits, targets, weights = make_case(name)
    lg = logits.clone().requires_grad_(True)
    host = S._sem_seg_loss_host(lg, targets, s, ignore, top_k, weights)
    host.backward()
    if name == "all_ignored":
        assert np.isnan(loss) and np.isnan(want) and torch.isnan(host)
        return
    assert abs(loss - want) <= 2e-6 * abs(want), (name, loss, want)
    assert abs(loss - float(host.detach())) <= 2e-6 * abs(loss), name
    g, bound, _ = ref.grad(sel, 1.0 / div)
    scale = float(g.abs().max())
    if name != "const_ties":  # the fixture's topk picks among ties in its own order
        torch.testing.assert_close(g, torch.from_numpy(gold[name + "_grad"]).to(F64), rtol=1e-4, atol=1e-6 * scale)
    torch.testing.assert_close(g, lg.grad.to(F64), rtol=1e-4, atol=1e-6 * scale)
    assert bool((bound >= 0).all()) and float(bound.max()) <= 1e-4 * scale + 1e-7


@pytest.mark.parametrize("stride", [1, 2, 4, 8, 16, 32])
def test_reference_is_float64_interpolate_and_cross_entropy_where_the_scale_is_exact(stride):
    g = torch.Generator().manual_seed(stride)
    n, c, hp, wp = 2, 5, 3, 4
    x = torch.randn(n, c, hp, wp, generator=g, dtype=F64) * 3
    t = torch.randint(0, c, (n, hp * stride, wp * stride), generator=g)
    t[0, 0, :] = 255
    ref = R.Ref(x, t, stride, 255)
    # x is rounded to fp32 by the reference (predictions.float()); compare on the same values
    up = F.interpolate(x.float().to(F64), scale_factor=stride, mode="bilinear", align_corners=False)
    torch.testing.assert_close(ref.v, up, rtol=1e-15, atol=1e-15)
    xr = x.float().to(F64).requires_grad_(True)
    ce = F.cross_entropy(F.interpolate(xr, scale_factor=stride, mode="bilinear", align_corners=False), t,
                         reduction="sum", ignore_index=255)
    ce.backward()
    total, _ = ref.loss_sum()
    assert abs(total - float(ce)) <= 1e-13 * abs(total)
    gr, _, _ = ref.grad(None, 1.0)
    torch.testing.assert_close(gr, xr.grad, rtol=1e-12, atol=1e-14)


def test_odd_stride_taps_use_the_fp32_scale():
    """Stride 3, d = 1: the fp32 index is 1.49e-8, not 0, so row 1 gets a tiny weight; d = 8 is off 2/3 by 1.6e-7."""
    i0, i1, l0, l1 = R.taps(3, 30, 10)
    assert int(i0[1]) == 0 and int(i1[1]) == 1 and 1e-8 < float(l1[1]) < 2e-8
    assert abs(float(l1[8]) - 1 / 3) > 1e-7 and abs(float(l0[8]) - 2 / 3) > 1e-7
    assert int(i0[29]) == int(i1[29]) == 9 and float(l1[29]) > 0  # the last row: both taps on the last logit


def test_autograd_gradients_pass_gradcheck():
    g = torch.Generator().manual_seed(0)
    t = torch.randint(0, 3, (1, 9, 6), generator=g)
    t[0, 0, 0] = 255
    w = torch.rand(1, 9, 6, generator=g, dtype=F64) + 0.5

    def f(x):
        v = R.upsample(x, 3)
        valid = t != 255
        loss = R._lse(v) - v.gather(1, torch.where(valid, t, 0)[:, None])[:, 0]
        return torch.where(valid, loss * w, 0.0).sum()

    x = torch.randn(1, 3, 3, 2, generator=g, dtype=F64, requires_grad=True)
    assert torch.autograd.gradcheck(f, (x,))


def test_positive_infinite_logit_gives_nan_as_log_softmax_does():
    x = torch.tensor([[[[float("inf")]], [[1.0]]]], dtype=F64)
    t = torch.tensor([[[1]]])
    ref = R.Ref(x, t, 1, 255)
    assert torch.isnan(ref.lse).all() and torch.isnan(ref.loss).all()
    assert torch.isnan(F.cross_entropy(x[:, :, 0], t[:, 0], reduction="none")).all()
    g, _, _ = ref.grad(None, 1.0)
    assert torch.isnan(g).all()


# ---- the backward's region bound ------------------------------------------------------------------------------------
MAX_HP = 8192


def region_sweep(stride):
    """(taps monotone, largest true region over every Hp <= MAX_HP and every tile, least spare row count)."""
    T_ = max(2, 32 // stride)
    rb = (T_ + 1) * stride + 2
    # the taps of the largest map; i1 = i0 + 1 before the clamp at the last row, except at stride 1 (a copy: i1 = i0)
    i0, _, _, _ = R.taps(stride, MAX_HP * stride, MAX_HP + 1)
    i0 = i0.numpy()
    i1 = i0 if stride == 1 else i0 + 1
    monotone = bool((np.diff(i0) >= 0).all())
    ys = np.arange(MAX_HP + 1)
    A = np.searchsorted(i1, ys, side="left")      # first row whose i1 >= y (y <= Hp - 1: the clamp does not matter)
    B = np.searchsorted(i0, ys, side="left")      # first row whose i0 >= y
    starts = np.arange(0, MAX_HP, T_)
    inner = starts[starts + T_ <= MAX_HP - 1]
    reg_inner = np.maximum.accumulate(B[inner + T_] - A[inner])  # tiles that end before the last row: Hp-independent
    hps = np.arange(1, MAX_HP + 1)
    n_inner = (hps - 1) // T_
    worst_inner = np.where(n_inner > 0, reg_inner[np.maximum(n_inner - 1, 0)], 0)
    last = hps * stride - A[T_ * n_inner]                          # the last tile runs to the map's last output row
    worst = np.maximum(worst_inner, last)
    return monotone, int(worst.max()), int((rb - worst).min())


@pytest.mark.parametrize("stride", range(1, R.MAX_STRIDE + 1))
def test_every_tile_region_fits_its_bound(stride):
    monotone, worst, spare = region_sweep(stride)
    assert monotone
    # stride 1 copies: a tile's region is its own 32 rows, 3 below the bound of 35
    assert spare == {1: 3, 31: 1}.get(stride, 2), (stride, worst, spare)


def test_region_sweep_agrees_with_a_tile_walk():
    for stride, hp in ((31, 9), (3, 25), (7, 13), (16, 5), (1, 70)):
        T_ = max(2, 32 // stride)
        i0, i1, _, _ = R.taps(stride, hp * stride, hp)
        worst = 0
        for y0 in range(0, hp, T_):
            y1 = min(y0 + T_, hp)
            lo = int(torch.searchsorted(i1, torch.tensor(y0)))
            hi = int(torch.searchsorted(i0, torch.tensor(y1)))
            worst = max(worst, hi - lo)
        assert R.region_spare(stride, hp) == (T_ + 1) * stride + 2 - worst
    assert R.region_spare(31, 9) == 1 and R.region_spare(30, 9) == 2


def test_backward_plans_fit_shared_memory():
    table = {1: (32, 35, 17), 2: (16, 36, 16), 3: (10, 35, 17), 4: (8, 38, 14), 8: (4, 42, 11), 16: (2, 50, 7),
             20: (2, 62, 3), 24: (2, 74, 1), 31: (2, 95, 1), 32: (2, 98, 1)}
    for s, (T_, rb, cc) in table.items():
        b = R.bwd_plan(1000, 1000, 1000, s)
        assert (b["T"], b["RBY"], b["CC"]) == (T_, rb, cc), s
    for s in range(1, R.MAX_STRIDE + 1):
        for c in (1, 2, 7, 133, 100000):
            for hp, wp in ((1, 1), (1, 4096), (4096, 4096), (3, 5)):
                b = R.bwd_plan(c, hp, wp, s)
                assert b["smem"] <= R.SMEM_OPTIN and 1 <= b["CC"] <= c
    assert R.bwd_plan(1000, 1000, 1000, 28)["smem"] > R.SMEM_TWO_PER_SM >= R.bwd_plan(1000, 1000, 1000, 27)["smem"]


# ---- labels -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", G.CASES, ids=lambda c: c.name)
def test_case_reaches_its_shape_labels(c):
    got = R.shape_labels(c.N, c.C, c.Hp, c.Wp, c.stride, c.dtype, c.top_k)
    assert (c.labels & R.SHAPE_LABELS) <= got, (c.name, sorted((c.labels & R.SHAPE_LABELS) - got))
    assert c.labels <= R.SHAPE_LABELS | R.VALUE_LABELS, sorted(c.labels - R.SHAPE_LABELS - R.VALUE_LABELS)


def test_every_label_is_declared():
    declared = set().union(*(c.labels for c in G.CASES))
    assert declared == R.SHAPE_LABELS | R.VALUE_LABELS, sorted((R.SHAPE_LABELS | R.VALUE_LABELS) - declared)
    strides = {c.stride for c in G.CASES}
    assert {1, 2, 3, 5, 7, 8, 13, 16, 20, 24, 31, 32} <= strides
