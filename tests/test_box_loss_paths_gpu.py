"""Box-branch loss kernels (losses.cu) path by path against the float64 reference of tests/box_loss_ref.py.

Each case runs through dense_loss_op / frcnn_loss_op and their backward ops (the raw sums, with grad_sums other than 1) and
asserts: each sum within its derived bound of the float64 sum; the counts and the status exactly; every decided gradient
element within its own bound, which is exactly 0 for the elements the loss does not read (ignored rows' logits, the deltas
of non-positive rows and background proposals, the class-specific columns of other classes); undecided elements a small
share of the case, and none in the cases built on exact edges; fp16 / bf16 gradients equal to the fp32 kernel's gradient
of the same values, rounded once; the path labels the case declares (tests/test_box_loss_paths_host.py checks the labels
of the small cases on the CPU).

case               reaches
rpn_full_*         RPN at 2 x 268 569 anchors, fp32 and bf16: K = 1 vectors of 4 / 8 rows, p6's partial tail, L1
retina_bench       RetinaNet 2 x 201 600 x 80, gamma 2, beta 0.1: many finish passes
retina_k*          K = 3, 7, 13, 1203 on levels of 5, 0, 1 and 13 anchors: rows and images ending inside vectors, CTAs
                   that stop early, an empty level; gamma 0.5, 1.5, 3, 0 with alpha; logits at 0, +-30, +-88, +-100; NaN
                   logits on ignored rows
status_*           a zero-width anchor, a label of K + 1, an unordered GIoU GT
sl1_beta*          beta 0, just below 1e-5, 1e-5 and 1/9 on exact edges: deltas equal to their targets (pinned against the
                   kernel's own difference), |diff| == beta
giou_edges         ties, touching, disjoint and intersecting boxes; dw at and above the clamp
rrpn_wrap          angle differences of +-180, 180 +- 2^-10 and 540
fcos_edges         deltas at and below 0, centerness ties l == r and l == 0
frcnn_*            K = 1, 6, 31, 32, 80, 1203 and R = 1, 7, 9, 2051; agnostic / class-specific / rotated / GIoU; the three
                   cascade weight sets; equal maxima in different lanes, scores at +-1e4, classes -1 and K + 1; fp16, bf16
"""
import math
from collections import namedtuple

import pytest
import torch

import box_loss_ref as R

pytestmark = pytest.mark.gpu
DEV = "cuda"
SC = 4.135166556742356
CLAMP32 = R.f32(SC)

Dense = namedtuple("Dense", "name N K levels dtype rpn gamma alpha beta loss_type D gs exact big labels")
Frcnn = namedtuple("Frcnn", "name R K kreg D dtype beta loss_type weights gs exact labels")


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def grid_anchors(strides, sizes, ratios, hw=(800, 1344)):
    out = []
    for s, sz in zip(strides, sizes):
        h, w = math.ceil(hw[0] / s), math.ceil(hw[1] / s)
        base = []
        for size in sz:
            for r in ratios:
                ww = math.sqrt(size * size / r)
                base.append([-ww / 2, -r * ww / 2, ww / 2, r * ww / 2])
        yy, xx = torch.meshgrid(torch.arange(h) * float(s), torch.arange(w) * float(s), indexing="ij")
        out.append((torch.stack([xx, yy, xx, yy], -1).reshape(-1, 1, 4) + torch.tensor(base)).reshape(-1, 4))
    return out


def dyadic_anchors(n, g, d=4):
    """Corners on multiples of 1/8, sides 2^k: every decode and target of zero deltas is exact in fp32."""
    xy = torch.randint(0, 800, (n, 2), generator=g).float() / 8 * 8 + torch.randint(0, 8, (n, 2), generator=g) / 8
    wh = 2.0 ** torch.randint(2, 8, (n, 2), generator=g).float()
    if d == 5:
        ang = torch.randint(-8, 8, (n, 1), generator=g).float() * 16
        return torch.cat([xy, wh, ang], 1)
    return torch.cat([xy, xy + wh], 1)


def jitter(an, g, scale=0.3):
    """GT boxes near the anchors: targets of moderate size."""
    if an.shape[1] == 5:
        out = an.clone()
        out[:, :2] += (torch.rand(len(an), 2, generator=g) - 0.5) * an[:, 2:4] * scale
        out[:, 2:4] *= torch.exp((torch.rand(len(an), 2, generator=g) - 0.5) * scale)
        out[:, 4] += (torch.rand(len(an), generator=g) - 0.5) * 40
        return out
    w, h = an[:, 2] - an[:, 0], an[:, 3] - an[:, 1]
    j = (torch.rand(len(an), 4, generator=g) - 0.5) * scale * torch.stack([w, h, w, h], 1)
    out = an + j
    out[:, 2:] = torch.maximum(out[:, 2:], out[:, :2] + 1)
    return out


def dense_inputs(c, seed):
    """CPU tensors of a dense case: logits, deltas, ctr, anchors, gt, labels, pin."""
    g = _gen(seed)
    N, K, Dd = c.N, c.K, c.D
    if c.name.startswith("rpn_full"):
        levels = grid_anchors((4, 8, 16, 32, 64), [[32], [64], [128], [256], [512]], (0.5, 1.0, 2.0))
    elif c.name == "retina_bench":
        sizes = [[x, x * 2 ** (1 / 3), x * 2 ** (2 / 3)] for x in (32, 64, 128, 256, 512)]
        levels = grid_anchors((8, 16, 32, 64, 128), sizes, (0.5, 1.0, 2.0))
    else:
        levels = [dyadic_anchors(r, g, Dd) for r in c.levels]
    anchors = torch.cat(levels)
    Rt = len(anchors)
    assert [len(a) for a in levels] == list(c.levels)
    gt = torch.stack([jitter(anchors, g) for _ in range(N)])
    u = torch.rand(N, Rt, generator=g)
    if c.rpn:
        labels = torch.full((N, Rt), -1, dtype=torch.int8)
        labels[u < 0.02 if Rt > 1000 else u < 0.5] = 1
        labels[(u > 0.97) if Rt > 1000 else u > 0.75] = 0
    else:
        labels = torch.randint(0, K, (N, Rt), generator=g)
        labels[u < 0.6] = K
        labels[u < 0.1] = -1
    if c.loss_type == R.LIN:
        pts = torch.cat([anchors[:, :2] + 0.5 * (anchors[:, 2:] - anchors[:, :2])] * 2, 1)
        half = (anchors[:, 2:] - anchors[:, :2]) * 0.5
        lo = pts[:, :2] - half * (1 + 3 * torch.rand(Rt, 2, generator=g))
        hi = pts[:, 2:] + half * (1 + 3 * torch.rand(Rt, 2, generator=g))
        gt = torch.cat([lo, hi], 1).expand(N, Rt, 4).clone()
    logits = [torch.randn(N, len(a), K, generator=g) * 3 - 1 for a in levels]
    deltas = [torch.randn(N, len(a), Dd, generator=g) * 0.4 for a in levels]
    ctr = [torch.randn(N, len(a), generator=g) for a in levels] if c.loss_type == R.LIN else []
    return dict(logits=logits, deltas=deltas, ctr=ctr, anchors=anchors, gt=gt, labels=labels, pin=None)


def edge_inputs(c, seed):
    """Exact edges: dyadic anchors; per image a block of each kind of row (see the module docstring)."""
    x = dense_inputs(c, seed)
    g = _gen(seed + 100)
    an, gt, lab = x["anchors"], x["gt"], x["labels"]
    Rt = len(an)
    N = c.N
    dl = torch.cat(x["deltas"], 1)
    kind = torch.arange(Rt) % 8
    posv = 1 if c.rpn else 0
    lab[:] = posv
    lab[:, kind == 7] = 0 if c.rpn else c.K
    if c.loss_type == R.SL1 and c.D == 4:
        beta = R.f32(c.beta)
        for n in range(N):
            gt[n, kind <= 2] = an[kind <= 2]                  # targets exactly 0
        dl[:, kind == 0] = 0.0                                # diff == 0
        dl[:, kind == 1] = torch.tensor([beta, -beta, beta, -beta])  # |diff| == beta
        dl[:, kind == 2] = torch.tensor([beta / 2, -beta * 2, 0.0, beta * 4])
    elif c.loss_type == R.SL1:  # RRPN: the angle wraps, everything else exact
        for n in range(N):
            gt[n] = an.clone()
            da = torch.tensor([180.0, -180.0, 180.0 + 2 ** -10, 180.0 - 2 ** -10, 540.0, -540.0, 90.0, 0.0])
            gt[n, :, 4] = an[:, 4] + da[kind]
        dl[:] = 0.0
    elif c.loss_type == R.GIOU:
        for n in range(N):
            w = an[:, 2] - an[:, 0]
            h = an[:, 3] - an[:, 1]
            sh = torch.stack([w, h, w, h], 1)
            gt[n] = an + torch.tensor([0.0, 0.0, 0.5, 0.5]) * sh                          # kind 0: x1, y1 ties
            gt[n, kind == 1] = (an + torch.tensor([1.0, 0.25, 2.0, 0.75]) * sh)[kind == 1]  # touching at x2 == x1
            gt[n, kind == 2] = (an + torch.tensor([3.0, 3.0, 4.0, 4.0]) * sh)[kind == 2]    # disjoint
            gt[n, kind == 3] = (an + torch.tensor([0.25, -0.25, 0.5, 1.5]) * sh)[kind == 3]  # inside / across
            gt[n, kind == 4] = (an + torch.tensor([-0.5, -0.5, 0.5, 0.5]) * sh)[kind == 4]  # x2 / y2 ties
            gt[n, kind >= 5] = (an + torch.tensor([0.125, 0.125, 3.0, 3.0]) * sh)[kind >= 5]
        dl[:] = 0.0
        dl[:, kind == 5, 2] = CLAMP32                         # dw exactly at the clamp: passes
        dl[:, kind == 6, 3] = 10.0                            # dh above the clamp: no gradient
    else:  # FCOS
        ctr_ = an[:, :2] + 0.5 * (an[:, 2:] - an[:, :2])
        for n in range(N):
            gt[n, kind == 0] = torch.cat([ctr_ - 8, ctr_ + 8], 1)[kind == 0]                          # l == r, t == b
            gt[n, kind == 1] = torch.cat([ctr_ - torch.tensor([0.0, 8.0]), ctr_ + 16], 1)[kind == 1]  # l == 0
        dl[:] = torch.randint(-2, 6, dl.shape, generator=g).float() / 2   # deltas at 0 and below 0 among others
    x["deltas"] = list(dl.split(list(c.levels), 1))
    x["gt"], x["labels"] = gt, lab
    return x


def _to(x, dtype):
    out = dict(x)
    out["logits"] = [t.to(DEV, dtype) for t in x["logits"]]
    out["deltas"] = [t.to(DEV, dtype) for t in x["deltas"]]
    out["ctr"] = [t.to(DEV, dtype) for t in x["ctr"]]
    for k in ("anchors", "gt", "labels"):
        out[k] = x[k].to(DEV)
    return out


def run_dense(c, x, gs):
    from detectron2_b200 import losses as L

    w = None if c.loss_type == R.LIN else ([1.0] * c.D if c.D == 5 or c.loss_type == R.GIOU else [1.0, 1.0, 1.0, 1.0])
    args = (x["logits"], x["deltas"], x["ctr"], x["anchors"], x["gt"], x["labels"], c.K, c.rpn, c.gamma, c.alpha, c.beta,
            c.loss_type, SC, w)
    sums, counts, status = L.dense_loss_op(*args)
    grads = L.dense_loss_backward_op(*args, torch.tensor(gs, dtype=torch.float32, device=DEV))
    return sums, counts, status, grads, w


def check_grads(got, ref, exact, what):
    n_dec = 0
    for i, (g, rg, b, u) in enumerate(zip(got, ref.grads, ref.bounds, ref.und)):
        g = g.detach().to(torch.float64)
        err = (g - rg).abs()
        bad = ~(err <= b) & ~u
        if bool(bad.any()):
            j = tuple(int(v) for v in torch.nonzero(bad)[0])
            raise AssertionError("%s grad %d: %d elements outside the bound; first %s: got %r ref %r bound %r"
                                 % (what, i, int(bad.sum()), j, float(g[j]), float(rg[j]), float(b[j])))
        n_dec += int((~u).sum())
    if exact:
        assert ref.n_und == 0, (what, ref.n_und)
    else:
        assert ref.n_und <= 0.001 * max(ref.n_dec, 1) + 2, (what, ref.n_und, ref.n_dec)


def check_sums(sums, counts, status, ref, k, what):
    s = sums.double().cpu().tolist()
    for i in range(k):
        assert abs(s[i] - ref.sums[i]) <= ref.sum_bounds[i], (what, i, s[i], ref.sums[i], ref.sum_bounds[i])
    assert counts.cpu().tolist() == ref.counts, (what, counts.cpu().tolist(), ref.counts)
    assert int(status) == ref.status, (what, int(status), ref.status)


def dense_case_labels(c, x, ref):
    return R.dense_shape_labels(c.N, c.K, c.levels, c.dtype, c.rpn, c.gamma, c.alpha, c.loss_type) | ref.labels


def _d(name, N, K, levels, dtype=torch.float32, rpn=False, gamma=2.0, alpha=0.25, beta=0.1, loss_type=R.SL1, D=4,
       gs=(0.37, 2.5, 0.0), exact=False, big=False, labels=()):
    return Dense(name, N, K, tuple(levels), dtype, rpn, gamma, alpha, beta, loss_type, D, gs, exact, big, frozenset(labels))


RPN_LEVELS = (201600, 50400, 12600, 3150, 819)
RETINA_LEVELS = (151200, 37800, 9450, 2457, 693)
SMALL = (5, 0, 1, 13)
DENSE_CASES = [
    _d("rpn_full_f32", 2, 1, RPN_LEVELS, rpn=True, gamma=0.0, alpha=-1.0, beta=0.0, big=True,
       labels={"vec4", "labels_i8", "tail_partial", "rows_per_vector_gt1", "row_ends_in_vector", "gamma0",
               "image_boundary_in_vector", "finish_multi_pass", "sl1_l1", "reg_tail_cta"}),
    _d("rpn_full_bf16", 2, 1, RPN_LEVELS, dtype=torch.bfloat16, rpn=True, gamma=0.0, alpha=-1.0, beta=0.0, big=True,
       gs=(1.0, 0.37, 0.0), labels={"vec8", "labels_i8", "tail_partial", "image_boundary_in_vector", "sl1_l1"}),
    _d("retina_bench", 2, 80, RETINA_LEVELS, big=True,
       labels={"vec4", "labels_i64", "gamma2", "finish_multi_pass", "sl1_quadratic", "sl1_linear"}),
    _d("retina_k3", 2, 3, SMALL, gamma=0.5, gs=(2.5, 0.0, 0.0),
       labels={"rows_per_vector_gt1", "row_ends_in_vector", "image_boundary_in_vector", "tail_partial", "empty_level",
               "cta_early_break", "gamma_pow", "finish_single_pass"}),
    _d("retina_k7_f16", 2, 7, SMALL, dtype=torch.float16, gamma=1.5, gs=(0.37, 2.5, 0.0),
       labels={"vec8", "rows_per_vector_gt1", "row_ends_in_vector", "image_boundary_in_vector", "ignored_nan"}),
    _d("retina_k13", 2, 13, SMALL, gamma=3.0, labels={"row_ends_in_vector", "gamma_pow", "tail_partial"}),
    _d("retina_k1203", 2, 1203, SMALL, gamma=0.0, alpha=0.25, labels={"gamma0_alpha", "row_ends_in_vector"}),
    _d("status_sl1", 2, 5, (40, 9), labels={"status_width", "status_class"}),
    _d("status_giou", 2, 5, (40, 9), loss_type=R.GIOU, labels={"status_order", "giou_inter"}),
    _d("sl1_beta0", 2, 2, (64, 17), beta=0.0, exact=True, labels={"diff_zero", "sl1_l1"}),
    _d("sl1_beta_below", 2, 2, (64, 17), beta=9.999999e-06, exact=True, labels={"diff_zero", "sl1_l1"}),
    _d("sl1_beta_1e5", 2, 2, (64, 17), beta=1e-5, exact=True, labels={"diff_zero", "sl1_quadratic", "sl1_linear"}),
    _d("sl1_beta_ninth", 2, 2, (64, 17), beta=1 / 9, exact=True, gs=(0.0, 0.37, 0.0),
       labels={"diff_zero", "sl1_quadratic", "sl1_linear"}),
    _d("giou_edges", 2, 3, (64, 31), loss_type=R.GIOU, exact=True,
       labels={"giou_inter", "giou_disjoint", "giou_touching", "giou_tie", "clamp_equal", "clamp_above"}),
    _d("rrpn_wrap", 2, 1, (64, 16), rpn=True, gamma=0.0, alpha=-1.0, beta=1 / 9, D=5, exact=True,
       labels={"angle_wrap", "labels_i8", "sl1_linear"}),
    _d("fcos_edges", 2, 4, (64, 29), loss_type=R.LIN, gs=(0.37, 2.5, 0.5), exact=True,
       labels={"fcos_relu_zero", "fcos_ctr_tie", "giou_inter"}),
]
EDGE = {"sl1_beta0", "sl1_beta_below", "sl1_beta_1e5", "sl1_beta_ninth", "giou_edges", "rrpn_wrap", "fcos_edges"}


def build_dense(c, seed=0):
    x = edge_inputs(c, seed) if c.name in EDGE else dense_inputs(c, seed)
    if c.name == "retina_k13":
        vals = torch.tensor([0.0, 30.0, -30.0, 88.0, -88.0, 100.0, -100.0])
        lg = x["logits"][0]
        lg.view(-1)[: lg.numel()] = vals[torch.arange(lg.numel()) % 7]
        x["logits"][3].view(-1)[::5] = vals[torch.arange(x["logits"][3].numel())[::5] % 7]
    if c.name == "retina_k7_f16":
        lab = x["labels"]
        a0 = 0
        for l, r in enumerate(c.levels):
            ign = lab[:, a0:a0 + r] == -1
            x["logits"][l][ign] = float("nan")
            a0 += r
    if c.name == "status_sl1":
        x["labels"][0, 3] = c.K + 1
        x["labels"][:, 7] = c.K           # the zero-width anchor is not regressed
        x["anchors"][7, 2] = x["anchors"][7, 0]
    if c.name == "status_giou":
        p = torch.nonzero(x["labels"][1] < c.K)[0, 0]
        x1, x2 = float(x["gt"][1, p, 0]), float(x["gt"][1, p, 2])
        x["gt"][1, p, 0], x["gt"][1, p, 2] = x2 + 1, x1  # x2 < x1: fvcore's assertion
    return x


def _pin_rows(c, x):
    """sl1 edge cases: rows of kind 3 take the torch restatement's fp32 targets on the same device; a forward with beta 0
    over just those rows then shows the kernel's own difference is exactly 0 on every element."""
    from detectron2_b200 import losses as L

    an = x["anchors"].to(DEV)
    kind = torch.arange(len(an), device=DEV) % 8
    w = [1.0] * c.D
    dl = torch.cat([t.to(DEV) for t in x["deltas"]], 1)
    for n in range(c.N):
        t = L._get_deltas(an, x["gt"][n].to(DEV), w)
        dl[n, kind == 3] = t[kind == 3]
    x["deltas"] = [t.cpu() for t in dl.split(list(c.levels), 1)]
    lab = torch.where((kind == 3).cpu()[None].expand(c.N, -1), x["labels"], torch.full_like(x["labels"], -1))
    y = _to(dict(x, labels=lab), torch.float32)
    sums, _, _ = L.dense_loss_op(y["logits"], y["deltas"], [], y["anchors"], y["gt"], y["labels"], c.K, c.rpn, 0.0, -1.0,
                                 0.0, R.SL1, SC, w)
    assert float(sums[1]) == 0.0
    return (kind == 3)[None, :, None].expand(c.N, -1, c.D).clone()


@pytest.mark.parametrize("c", DENSE_CASES, ids=lambda c: c.name)
def test_dense_case(c):
    x = build_dense(c)
    pin = _pin_rows(c, x) if c.name.startswith("sl1_") else None
    y = _to(x, c.dtype)
    sums, counts, status, grads, w = run_dense(c, y, c.gs)
    if c.dtype != torch.float32:  # the kernel on the same values in fp32; the half gradients are its rounding
        y32 = dict(y, logits=[t.float() for t in y["logits"]], deltas=[t.float() for t in y["deltas"]],
                   ctr=[t.float() for t in y["ctr"]])
        s32, c32, st32, g32, _ = run_dense(c, y32, c.gs)
        for a, b in zip(grads, g32):
            assert a.dtype == c.dtype and torch.equal(a, b.to(c.dtype))
        assert torch.equal(counts, c32) and torch.equal(status, st32)
        sums, grads = s32, g32
        vec_dtype = c.dtype
    else:
        vec_dtype = torch.float32
    ref = R.dense([t.to(vec_dtype) for t in y["logits"]], [t.float() for t in y["deltas"]], [t.float() for t in y["ctr"]],
                  y["anchors"], y["gt"], y["labels"], c.K, c.rpn, c.gamma, c.alpha, c.beta, c.loss_type, SC, w,
                  list(c.gs), pin=pin)
    check_sums(sums, counts, status, ref, 3, c.name)
    check_grads(grads, ref, c.exact, c.name)
    got = dense_case_labels(c, x, ref)
    assert c.labels <= got, (c.name, sorted(c.labels - got))


def test_misaligned_logits_are_relaid_out():
    """A level whose logits sit 4 bytes past a 16-byte boundary: _pred copies it, and the results are identical."""
    c = DENSE_CASES[5]
    x = _to(build_dense(c, seed=3), torch.float32)
    base = torch.empty(x["logits"][3].numel() + 1, device=DEV)
    mis = base[1:].view_as(x["logits"][3])
    mis.copy_(x["logits"][3])
    assert mis.data_ptr() % 16 == 4
    a = run_dense(c, x, c.gs)
    b = run_dense(c, dict(x, logits=x["logits"][:3] + [mis]), c.gs)
    for p, q in zip(a[:3], b[:3]):
        assert torch.equal(p, q)
    assert all(torch.equal(p, q) for p, q in zip(a[3], b[3]))


# ---- Fast R-CNN ---------------------------------------------------------------------------------------------------
CASCADE = ((10.0, 10.0, 5.0, 5.0), (20.0, 20.0, 10.0, 10.0), (30.0, 30.0, 15.0, 15.0))


def _f(name, R_, K, kreg="specific", D=4, dtype=torch.float32, beta=0.0, loss_type=R.SL1, weights=CASCADE[0],
       gs=(0.37, 2.5), exact=False, labels=()):
    kr = 1 if kreg == "agnostic" else K
    return Frcnn(name, R_, K, kr, D, dtype, beta, loss_type, weights, gs, exact, frozenset(labels))


FRCNN_CASES = [
    _f("frcnn_k1_r7", 7, 1, kreg="agnostic", labels={"k1_lt_32", "rows_ragged_cta", "background_row"}),
    _f("frcnn_k6_r9_cascade2", 9, 6, weights=CASCADE[1], beta=0.1, labels={"k1_lt_32", "class_specific"}),
    _f("frcnn_k31_r2051", 2051, 31, gs=(0.0, 1.0), labels={"k1_eq_32", "rows_ragged_cta"}),
    _f("frcnn_k32_r1", 1, 32, kreg="agnostic", labels={"k1_33", "agnostic"}),
    _f("frcnn_k80_r2051_cascade3", 2051, 80, weights=CASCADE[2],
       labels={"argmax_tie_across_lanes", "status_class", "k1_many_passes", "background_row"}),
    _f("frcnn_k1203_r9", 9, 1203, kreg="agnostic", gs=(2.5, 0.37), labels={"k1_many_passes", "agnostic"}),
    _f("frcnn_rot5", 512, 6, D=5, weights=(10.0, 10.0, 5.0, 5.0, 1.0), labels={"rot5"}),
    _f("frcnn_giou", 512, 80, loss_type=R.GIOU, weights=(1.0, 1.0, 1.0, 1.0), labels={"giou"}),
    _f("frcnn_f16", 520, 80, dtype=torch.float16, labels={"f16"}),
    _f("frcnn_bf16", 520, 80, kreg="agnostic", dtype=torch.bfloat16, beta=1 / 9, labels={"bf16"}),
]


def build_frcnn(c, seed=0):
    g = _gen(seed)
    if c.D == 5:
        props = dyadic_anchors(c.R, g, 5)
        props[:, 4] = (torch.rand(c.R, generator=g) - 0.5) * 360
    else:
        props = dyadic_anchors(c.R, g) + torch.rand(c.R, 4, generator=g)
        props[:, 2:] = torch.maximum(props[:, 2:], props[:, :2] + 2)
    gt = jitter(props, g)
    cls = torch.randint(0, c.K, (c.R,), generator=g)
    cls[torch.rand(c.R, generator=g) < 0.5] = c.K
    scores = torch.randn(c.R, c.K + 1, generator=g) * 2
    deltas = torch.randn(c.R, c.kreg * c.D, generator=g) * 0.3
    if c.name == "frcnn_k80_r2051_cascade3":
        scores[:40] = -3.0
        scores[:40, 5] = scores[:40, 6] = 4.0           # equal maxima in lanes 5 and 6
        scores[40:50, 37] = scores[40:50, 70] = 9.0      # ... in lanes 5 and 6 of different passes
        scores[50:60] = scores[50:60].sign() * 1e4      # scores at +-1e4
        scores[60:70, 80] = 1e4                          # argmax the background: false negatives where fg
        cls[70], cls[71] = -1, c.K + 1
    if c.name == "frcnn_k1_r7":
        cls[0], cls[1] = 0, 1
    return scores, deltas, props, gt, cls


def run_frcnn(c, x, gs):
    from detectron2_b200 import losses as L

    scores, deltas, props, gt, cls = x
    sums, counts, status = L.frcnn_loss_op(scores, deltas, props, gt, cls, c.beta, c.loss_type, SC, list(c.weights))
    gsc, gd = L.frcnn_loss_backward_op(scores, deltas, props, gt, cls, c.beta, c.loss_type, SC, list(c.weights),
                                       torch.tensor(gs, dtype=torch.float32, device=DEV))
    return sums, counts, status, [gsc, gd]


@pytest.mark.parametrize("c", FRCNN_CASES, ids=lambda c: c.name)
def test_frcnn_case(c):
    scores, deltas, props, gt, cls = build_frcnn(c)
    x = [scores.to(DEV, c.dtype), deltas.to(DEV, c.dtype), props.to(DEV), gt.to(DEV), cls.to(DEV)]
    sums, counts, status, grads = run_frcnn(c, x, c.gs)
    if c.dtype != torch.float32:
        x32 = [x[0].float(), x[1].float()] + x[2:]
        s32, c32, st32, g32 = run_frcnn(c, x32, c.gs)
        for a, b in zip(grads, g32):
            assert a.dtype == c.dtype and torch.equal(a, b.to(c.dtype))
        assert torch.equal(counts, c32) and torch.equal(status, st32)
        sums, grads = s32, g32
    ref = R.frcnn(x[0].float(), x[1].float(), x[2], x[3], x[4], c.beta, c.loss_type, SC, c.weights, list(c.gs))
    check_sums(sums, counts, status, ref, 2, c.name)
    check_grads(grads, ref, c.exact, c.name)
    got = R.frcnn_shape_labels(c.R, c.K, c.kreg, c.D, c.dtype, c.loss_type) | ref.labels
    assert c.labels <= got, (c.name, sorted(c.labels - got))


# ---- the public wrappers: normalisation -----------------------------------------------------------------------------
def test_wrappers_normalise_the_sums():
    from detectron2_b200 import fcos as FC
    from detectron2_b200 import losses as L

    c = DENSE_CASES[5]  # retina_k13
    x = _to(build_dense(c, seed=7), torch.float32)
    ref = R.dense(x["logits"], x["deltas"], [], x["anchors"], x["gt"], x["labels"], c.K, False, 2.0, 0.25, 0.1, R.SL1,
                  SC, [1.0] * 4, [1.0, 1.0, 0.0])
    levels = list(x["anchors"].split(list(c.levels)))
    losses, num_pos, norm = L.retinanet_losses(levels, x["logits"], list(x["labels"]), x["deltas"], list(x["gt"]),
                                               num_classes=c.K, loss_normalizer=250.0)
    assert num_pos == ref.counts[0] and norm == 250.0 * 0.9 + max(num_pos, 1) * (1 - 0.9)
    for k, i in (("loss_cls", 0), ("loss_box_reg", 1)):
        assert abs(float(losses[k]) * norm - ref.sums[i]) <= ref.sum_bounds[i] + 4 * R.U * abs(ref.sums[i]), k
    c = DENSE_CASES[9]  # sl1_beta0 inputs as an RPN
    x = _to(build_dense(c), torch.float32)
    lab = torch.where(x["labels"] == 0, 1, torch.where(x["labels"] == c.K, 0, -1)).to(torch.int8)
    ref = R.dense([t[..., :1] for t in x["logits"]], x["deltas"], [], x["anchors"], x["gt"], lab, 1, True, 0.0, -1.0,
                  0.0, R.SL1, SC, [1.0] * 4, [1.0, 1.0, 0.0])
    losses, counts = L.rpn_losses(x["anchors"], [t[..., 0] for t in x["logits"]], list(lab), x["deltas"], list(x["gt"]),
                                  batch_size_per_image=256)
    assert counts == {"num_pos_anchors": ref.counts[0], "num_neg_anchors": ref.counts[1]}
    for k, i in (("loss_rpn_cls", 0), ("loss_rpn_loc", 1)):
        assert abs(float(losses[k]) * 512 - ref.sums[i]) <= ref.sum_bounds[i] + 4 * R.U * abs(ref.sums[i]), k
    c = FRCNN_CASES[4]
    scores, deltas, props, gt, cls = [t.to(DEV) for t in build_frcnn(c)]
    cls = torch.where((cls >= 0) & (cls <= c.K), cls, c.K)
    ref = R.frcnn(scores, deltas, props, gt, cls, 0.0, R.SL1, SC, c.weights, [1.0, 1.0])
    losses, stats = L.fast_rcnn_losses(scores, deltas, props, gt, cls, box2box_weights=c.weights)
    assert list(stats.values()) == ref.counts
    for k, i in (("loss_cls", 0), ("loss_box_reg", 1)):
        assert abs(float(losses[k]) * c.R - ref.sums[i]) <= ref.sum_bounds[i] + 4 * R.U * abs(ref.sums[i]), k
    c = DENSE_CASES[15]  # fcos_edges
    x = _to(build_dense(c), torch.float32)
    ref = R.dense(x["logits"], x["deltas"], x["ctr"], x["anchors"], x["gt"], x["labels"], c.K, False, 2.0, 0.25, 0.0,
                  R.LIN, SC, None, [1.0, 1.0, 1.0])
    levels = list(x["anchors"].split(list(c.levels)))
    losses, num_pos, norm = FC.fcos_losses(levels, x["logits"], list(x["labels"]), x["deltas"], list(x["gt"]),
                                           [t[..., None] for t in x["ctr"]], num_classes=c.K)
    assert num_pos == ref.counts[0]
    for k, i in (("loss_fcos_cls", 0), ("loss_fcos_loc", 1), ("loss_fcos_ctr", 2)):
        assert abs(float(losses[k]) * norm - ref.sums[i]) <= ref.sum_bounds[i] + 4 * R.U * abs(ref.sums[i]), k
