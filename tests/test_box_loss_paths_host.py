"""CPU checks of tests/box_loss_ref.py: the float64 reference against the fixtures taken from the real reference functions
(tests/golden/losses.npz, the loss cases of tests/golden/fcos.npz) and against torchvision; its autograd gradients by
gradcheck; the path model against the library (workspace sizes, refusals); every case of
tests/test_box_loss_paths_gpu.py reaching the labels it declares, and all of them together reaching every label."""
import ctypes as C

import numpy as np
import pytest
import torch

import box_loss_ref as R
import fcos_ref
import test_box_loss_paths_gpu as G
import test_losses_host as H

F64 = torch.float64

ALL_LABELS = {
    # dense classification
    "vec4", "vec8", "tail_partial", "row_ends_in_vector", "rows_per_vector_gt1", "image_boundary_in_vector",
    "cta_early_break", "empty_level", "labels_i8", "labels_i64", "gamma0", "gamma0_alpha", "gamma2", "gamma_pow",
    "ignored_nan",
    # dense regression
    "sl1_l1", "sl1_quadratic", "sl1_linear", "diff_zero", "giou_inter", "giou_disjoint", "giou_touching", "giou_tie",
    "clamp_equal", "clamp_above", "angle_wrap", "fcos_relu_zero", "fcos_ctr_tie", "status_width", "status_class",
    "status_order", "reg_tail_cta", "finish_multi_pass", "finish_single_pass",
    # Fast R-CNN
    "k1_lt_32", "k1_eq_32", "k1_33", "k1_many_passes", "rows_ragged_cta", "agnostic", "class_specific", "rot5", "giou",
    "background_row", "argmax_tie_across_lanes", "f16", "bf16",
}
SHAPE_LABELS = {"vec4", "vec8", "tail_partial", "row_ends_in_vector", "rows_per_vector_gt1", "image_boundary_in_vector",
                "cta_early_break", "empty_level", "labels_i8", "labels_i64", "gamma0", "gamma0_alpha", "gamma2",
                "gamma_pow", "reg_tail_cta", "finish_multi_pass", "finish_single_pass"}


def _within(got, ref, bound, what):
    got = torch.as_tensor(np.asarray(got)).to(F64).reshape(ref.shape)
    bad = ~((got - ref).abs() <= bound)
    assert not bool(bad.any()), (what, int(bad.sum()), got[bad][:4], ref[bad][:4], bound[bad][:4])


# ---- the reference against the fixtures of the real reference functions ---------------------------------------------
def _golden_dense(z, case):
    lst = lambda k: H._list(z, case, k, "cpu")  # noqa: E731
    rpn = case.startswith("rpn") or case.startswith("rrpn")
    loss_type = R.GIOU if "giou" in case else R.SL1
    anchors, labels, gt = torch.cat(lst("anchors")), torch.stack(lst("labels")), torch.stack(lst("gt"))
    logits, deltas = lst("logits"), lst("deltas")
    n = labels.shape[0]
    beta = float(z[case + "__beta"])
    if rpn:
        w = tuple(z[case + "__weights"].tolist())
        norm = (64.0 * n, 64.0 * n / 2.0)  # batch_size_per_image 64, loss_rpn_loc weighted 2
        keys, pre, grad_pre = ("loss_rpn_cls", "loss_rpn_loc"), case + "__", case
        logits = [x[..., None] for x in logits]
        k, gamma, alpha = 1, 0.0, -1.0
    else:
        w = (1.0, 1.0, 1.0, 1.0)
        nz = float(z[case + "_call0__normalizer"])
        norm = (nz, nz)
        keys, pre, grad_pre = ("loss_cls", "loss_box_reg"), case + "_call0__", case + "_call0"
        k, gamma, alpha = 5, 2.0, 0.25
    gs = [R.f32(1 / norm[0]), R.f32(1 / norm[1]), 0.0]
    ref = R.dense(logits, deltas, [], anchors, gt, labels, k, rpn, gamma, alpha, beta, loss_type, G.SC, w, gs)
    for i, key in enumerate(keys):
        got = float(z[pre + key])
        assert abs(got * norm[i] - ref.sums[i]) <= ref.sum_bounds[i] + 4 * R.U * abs(ref.sums[i]), (case, key)
    want = H._list(z, grad_pre, "grad_logits", "cpu") + H._list(z, grad_pre, "grad_deltas", "cpu")
    for g, rg, b, u in zip(want, ref.grads, ref.bounds, ref.und):
        # the fixture's gradients are torch's fp32 autograd, not the kernel's sequence: its own rounding of each gradient
        # is within the same bound, and the gradient scale 1 / norm is one more rounding
        _within(g.reshape(rg.shape)[~u], rg[~u], 2 * b[~u] + 2 * R.U * rg[~u].abs(), (case, "grad"))


def _golden_frcnn(z, case):
    arr = lambda k: torch.from_numpy(z[case + "__" + k])  # noqa: E731
    scores, deltas, props, gt, cls = arr("scores"), arr("deltas"), arr("props"), arr("gt"), arr("classes")
    loss_type = R.GIOU if "giou" in case else R.SL1
    r = max(len(cls), 1)
    gs = [R.f32(1 / r), R.f32(0.5 / r)]
    ref = R.frcnn(scores, deltas, props, gt, cls, float(z[case + "__beta"]), loss_type, G.SC,
                  tuple(z[case + "__weights"].tolist()), gs)
    for i, (key, scale) in enumerate((("loss_cls", 1.0), ("loss_box_reg", 0.5))):
        got = float(z[case + "__" + key])
        assert abs(got * r / scale - ref.sums[i]) <= ref.sum_bounds[i] + 4 * R.U * abs(ref.sums[i]), (case, key)
    for key, rg, b, u in zip(("grad_scores", "grad_deltas"), ref.grads, ref.bounds, ref.und):
        g = arr(key).to(F64).reshape(rg.shape)
        _within(g[~u], rg[~u], 2 * b[~u] + 2 * R.U * rg[~u].abs(), (case, key))


@pytest.mark.parametrize("case", H.golden_case_names())
def test_reference_reproduces_losses_fixture(case):
    z = H._golden()
    if int(z[case + "__raises"]) or "diou" in case or "ciou" in case:
        pytest.skip("an assertion case, or a loss type without a kernel")
    if case.startswith("frcnn"):
        _golden_frcnn(z, case)
    else:
        _golden_dense(z, case)


@pytest.mark.parametrize("case", ["loss_f32", "loss_f16"])
def test_reference_reproduces_fcos_fixture(case):
    z = fcos_ref.load()
    an = torch.cat(fcos_ref.anchors(z))
    labels, boxes = torch.stack(fcos_ref.lst(z, "a", "labels")), torch.stack(fcos_ref.lst(z, "a", "boxes"))
    logits, deltas = fcos_ref.lst(z, case, "logits"), fcos_ref.lst(z, case, "deltas")
    n = labels.shape[0]
    ctr = [c.reshape(n, -1) for c in fcos_ref.lst(z, case, "ctr")]
    cc = case + "_call0"
    nz = float(z[cc + "__normalizer"])
    gs = [R.f32(1 / nz)] * 3
    ref = R.dense([x.float() for x in logits], [d.float() for d in deltas], [c.float() for c in ctr], an, boxes, labels,
                  fcos_ref.K, False, 2.0, 0.25, 0.0, R.LIN, 0.0, None, gs)
    assert ref.counts[0] == int(z[case + "__num_pos"])
    for i, key in enumerate(("loss_fcos_cls", "loss_fcos_loc", "loss_fcos_ctr")):
        got = float(z[cc + "__" + key])
        assert abs(got * nz - ref.sums[i]) <= ref.sum_bounds[i] + 4 * R.U * abs(ref.sums[i]), key
    if case == "loss_f32":
        want = fcos_ref.lst(z, cc, "grad_logits") + fcos_ref.lst(z, cc, "grad_deltas") + fcos_ref.lst(z, cc, "grad_ctr")
        for g, rg, b, u in zip(want, ref.grads, ref.bounds, ref.und):
            g = g.to(F64).reshape(rg.shape)
            _within(g[~u], rg[~u], 2 * b[~u] + 2 * R.U * rg[~u].abs(), (case, "grad"))


def test_reference_matches_torchvision():
    from torchvision.ops import generalized_box_iou_loss, sigmoid_focal_loss

    g = torch.Generator().manual_seed(0)
    x = torch.randn(5000, generator=g, dtype=F64) * 6
    t = (torch.rand(5000, generator=g) < 0.3).to(F64)
    for gamma, alpha in ((2.0, 0.25), (0.0, -1.0), (0.0, 0.25), (0.5, 0.25), (1.5, -1.0), (3.0, 0.75)):
        a = R.focal_ref(x, t, gamma, alpha).sum()
        b = sigmoid_focal_loss(x, t, alpha=alpha, gamma=gamma, reduction="sum")
        assert torch.allclose(a, b, rtol=1e-13, atol=0), (gamma, alpha)
    b1 = H._boxes(3000, g).to(F64)
    b2 = H._boxes(3000, g).to(F64)
    assert torch.allclose(R.giou_ref(b1, b2).sum(), generalized_box_iou_loss(b1, b2, reduction="sum", eps=1e-7),
                          rtol=1e-13, atol=0)


def test_autograd_gradients_pass_gradcheck():
    """Away from every decision edge: logits off saturation, |diff| away from 0 and beta, no box tie, dw below the clamp."""
    g = torch.Generator().manual_seed(1)
    x = (torch.randn(40, generator=g, dtype=F64) * 3).requires_grad_(True)
    t = (torch.rand(40, generator=g) < 0.4).to(F64)
    for gamma, alpha in ((2.0, 0.25), (0.0, -1.0), (1.5, 0.25), (0.5, -1.0)):
        assert torch.autograd.gradcheck(lambda v: R.focal_ref(v, t, gamma, alpha), (x,))
    d = (torch.rand(30, 4, generator=g, dtype=F64) - 0.5).requires_grad_(True)
    tg = torch.rand(30, 4, generator=g, dtype=F64) * 0.1 + 0.6
    assert torch.autograd.gradcheck(lambda v: R.smooth_l1_ref(v, tg, 0.1), (d,))
    assert torch.autograd.gradcheck(lambda v: R.smooth_l1_ref(v, tg, 0.0), (d,))
    an = H._boxes(30, g).to(F64)
    gt = an + torch.rand(30, 4, generator=g, dtype=F64) * 3 + 0.37
    assert torch.autograd.gradcheck(lambda v: R.giou_ref(R.apply_deltas_ref(v, an, (10.0, 10.0, 5.0, 5.0), G.SC), gt),
                                    (d,))
    dp = (torch.rand(30, 4, generator=g, dtype=F64) + 0.2).requires_grad_(True)
    assert torch.autograd.gradcheck(lambda v: R.giou_ref(R.apply_deltas_linear_ref(v, an), gt), (dp,))
    s = torch.randn(12, 7, generator=g, dtype=F64).requires_grad_(True)
    cls = torch.randint(0, 7, (12,), generator=g)
    assert torch.autograd.gradcheck(lambda v: torch.nn.functional.cross_entropy(v, cls, reduction="none"), (s,))


def test_tracker_is_exact_on_exact_arithmetic_and_bounds_rounding():
    v = lambda *a: torch.tensor(a, dtype=F64)  # noqa: E731
    a, b = R.T(v(1.5, 3.0, 0.1)), R.T(v(0.25, 3.0, 0.2))
    s = a + b
    assert s.e[:2].tolist() == [0.0, 0.0] and s.e[2] > 0      # 0.1 + 0.2 is not an fp32 number
    q = a / b
    assert q.e[:2].tolist() == [0.0, 0.0]                     # 1.5 / 0.25 = 6, 3 / 3 = 1
    assert float((R.T(v(0.0)).exp()).e) == 0.0 and float((R.T(v(1.0)).log()).e) == 0.0
    x32 = torch.tensor([0.1, 1e-3, 7.3], dtype=torch.float32)
    e = R.T(x32.to(F64)).exp()
    assert bool(((torch.exp(x32).to(F64) - torch.exp(x32.to(F64))).abs() <= e.e).all())
    r = R.T(v(180.0, 540.0, -180.0) + 20.0)
    d, und = R.get_deltas_t([R.T(v(0, 0, 0)), R.T(v(0, 0, 0)), R.T(v(1, 1, 1)), R.T(v(1, 1, 1)), R.T(v(20, 20, 20))],
                            [R.T(v(0, 0, 0)), R.T(v(0, 0, 0)), R.T(v(1, 1, 1)), R.T(v(1, 1, 1)), r], [1.0] * 5)
    assert not bool(und.any()) and torch.allclose(d[4].v, v(-np.pi, -np.pi, -np.pi))
    sh, u = R.share(R.T(v(2.0)), R.T(v(2.0)), True)
    assert float(sh) == 0.5 and not bool(u)


# ---- the path model against the library -----------------------------------------------------------------------------
_P, _MIS = 0x1000, 0x1004
EINVAL, EWORKSPACE = -1, -2
SIZEOF_PARTIAL = 48  # float sum[3], int status, long long cnt[4]


def _levels(levels, logits_ptr=_P):
    from detectron2_b200 import _C

    lv = _C.DenseLossLevels()
    lv.num_levels = len(levels)
    for l, r in enumerate(levels):
        lv.R[l], lv.logits[l], lv.deltas[l], lv.ctr[l] = r, (logits_ptr if l == len(levels) - 1 else _P), _P, _P
    return lv


@pytest.mark.parametrize("c", G.DENSE_CASES, ids=lambda c: c.name)
def test_workspace_equals_the_cta_model(c):
    from detectron2_b200 import _C

    lib = _C.lib()
    lv = _levels(c.levels)
    got = lib.d2b_dense_loss_workspace_bytes(C.byref(lv), c.N, c.K, _C.DTYPE_CODE[c.dtype])
    assert got == R.dense_ctas(c.N, c.K, c.levels, R.vec_elems(c.dtype)) * SIZEOF_PARTIAL


def test_frcnn_workspace_equals_the_cta_model():
    from detectron2_b200 import _C

    lib = _C.lib()
    for r in (0, 1, 7, 8, 9, 2051, 100000):
        assert lib.d2b_frcnn_loss_workspace_bytes(r) == R.frcnn_ctas(r) * SIZEOF_PARTIAL


def test_refusals_agree_with_the_library():
    """Every combination of label kind, K, box dim, loss type and logits alignment: the model refuses exactly where the
    library returns EINVAL; an accepted call runs into the empty workspace (EWORKSPACE) before any launch."""
    from detectron2_b200 import _C

    lib = _C.lib()
    w = (C.c_float * 5)(*[1.0] * 5)
    for i8 in (True, False):
        for k in (1, 80):
            for d in (4, 5):
                for lt in (R.SL1, R.GIOU, R.LIN):
                    for ptr in (_P, _MIS):
                        lv = _levels((10, 3), ptr)
                        if lt != R.LIN:
                            for l in range(2):
                                lv.ctr[l] = None
                        rc = lib.d2b_dense_loss_forward(C.byref(lv), 2, k, d, 0, _P, _P, _P, 0 if i8 else 1, 2.0, 0.25,
                                                        0.1, lt, 4.0, None if lt == R.LIN else w, _P, _P, _P, _P, 0,
                                                        None)
                        want = EINVAL if R.dense_refuses(k, d, i8, lt, ptr == _P) else EWORKSPACE
                        assert rc == want, (i8, k, d, lt, ptr, rc)


# ---- coverage -------------------------------------------------------------------------------------------------------
def _host_labels(c):
    shape = R.dense_shape_labels(c.N, c.K, c.levels, c.dtype, c.rpn, c.gamma, c.alpha, c.loss_type)
    if c.big:  # full-size cases: their value labels are checked on the GPU
        return shape | (c.labels - SHAPE_LABELS)
    x = G.build_dense(c)
    w = None if c.loss_type == R.LIN else [1.0] * c.D
    ref = R.dense([t.to(c.dtype) for t in x["logits"]], x["deltas"], x["ctr"], x["anchors"], x["gt"], x["labels"], c.K,
                  c.rpn, c.gamma, c.alpha, c.beta, c.loss_type, G.SC, w, list(c.gs))
    return shape | ref.labels


@pytest.mark.parametrize("c", G.DENSE_CASES, ids=lambda c: c.name)
def test_dense_case_reaches_its_labels(c):
    got = _host_labels(c)
    assert c.labels <= got, (c.name, sorted(c.labels - got))


@pytest.mark.parametrize("c", G.FRCNN_CASES, ids=lambda c: c.name)
def test_frcnn_case_reaches_its_labels(c):
    s, d, p, gt, cls = G.build_frcnn(c)
    ref = R.frcnn(s.to(c.dtype).float(), d.to(c.dtype).float(), p, gt, cls, c.beta, c.loss_type, G.SC, c.weights,
                  list(c.gs))
    got = R.frcnn_shape_labels(c.R, c.K, c.kreg, c.D, c.dtype, c.loss_type) | ref.labels
    assert c.labels <= got, (c.name, sorted(c.labels - got))


def test_every_label_is_declared():
    declared = set().union(*(c.labels for c in G.DENSE_CASES + G.FRCNN_CASES))
    assert declared == ALL_LABELS, (sorted(ALL_LABELS - declared), sorted(declared - ALL_LABELS))
