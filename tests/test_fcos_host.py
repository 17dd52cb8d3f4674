"""CPU tests of the FCOS surface (detectron2_b200/fcos.py): the torch restatements against the fixture taken from the real
reference methods (tests/golden/make_golden_fcos.py), argument validation of the native entry points, and the fake kernels."""
import ctypes as C

import pytest
import torch

import fcos_ref as R


def test_label_restatement_reproduces_fixture_bit_for_bit():
    from detectron2_b200 import fcos as F

    z = R.load()
    an = R.anchors(z)
    for case in ("a", "nf"):
        labels, boxes = F.fcos_label_anchors(an, R.lst(z, case, "gt"), R.lst(z, case, "cls"), num_classes=R.K)
        R.check_labels(z, case, labels, boxes)
    # the quirks the fixture pins: the first of two tied boxes wins, and a non-finite GT takes every point of its image
    labels = R.lst(z, "nf", "labels")
    assert bool((labels[0] == 2).all()) and bool((labels[1] == 5).all())
    q = R.lst(z, "a", "quality")[0]
    assert float(q[4].max()) == float(q[5].max()) > 0


def test_quality_matrix_restatement_is_the_reference_one():
    from detectron2_b200 import fcos as F

    z = R.load()
    an = torch.cat(R.anchors(z))
    counts = [len(a) for a in R.anchors(z)]
    for case in ("a", "nf"):
        for gt, q in zip(R.lst(z, case, "gt"), R.lst(z, case, "quality")):
            if len(gt):
                assert R.same(F._match_quality_host(an, counts, gt, 1.5), q)


@pytest.mark.parametrize("case", ["loss_f32", "loss_f16", "loss_nan_delta"])
def test_loss_restatement_reproduces_fixture(case):
    z = R.load()
    if case == "loss_f16":  # the reference took the fp32 values of the fp16 predictions
        z = {k: (v.astype("float32") if v.dtype.name == "float16" else v) for k, v in z.items()}
    R.run_loss_case(z, case, "cpu", 1e-6, 1e-6)


def test_ctrness_targets_reproduce_fixture():
    from detectron2_b200 import fcos as F

    z = R.load()
    t = F._ctrness_targets_host(torch.cat(R.anchors(z)), R.lst(z, "a", "boxes"))
    assert R.same(t, R.arr(z, "loss_f32__ctr_targets"))


def test_linear_decode_inverts_get_deltas():
    from detectron2_b200 import fcos as F
    from detectron2_b200.dense_inference import apply_deltas_linear

    an = torch.tensor([[0.0, 0.0, 8.0, 8.0], [16.0, 16.0, 32.0, 32.0]])
    gt = torch.tensor([[1.0, 2.0, 10.0, 7.0], [20.0, 18.0, 30.0, 31.0]])
    assert torch.allclose(apply_deltas_linear(F._get_deltas_linear(an, gt), an), gt)
    assert torch.equal(apply_deltas_linear(torch.tensor([[-1.0, 0.0, -0.5, 0.0]]), an[:1]), torch.tensor([[4.0, 4, 4, 4]]))


def test_fcos_assign_validates_arguments_without_a_gpu():
    from detectron2_b200 import _C

    lib = _C.lib()
    EINVAL = -1
    dummy = C.c_void_p(16)  # never dereferenced: every call below fails its checks first
    lc = (C.c_int * 3)(100, 50, 25)

    def assign(levels=lc, nl=3, N=2, G=5, K=80, **kw):
        a = dict(anchors=dummy, gt=dummy, cnt=dummy, cls=dummy, m=dummy, l=dummy, b=dummy)
        a.update(kw)
        return lib.d2b_fcos_assign(a["anchors"], levels, nl, a["gt"], a["cnt"], N, G, a["cls"], K, 1.5, a["m"], a["l"],
                                   a["b"], None)

    assert assign(nl=0) == EINVAL
    assert assign(nl=_C.MAX_LEVELS + 1) == EINVAL
    assert assign(levels=None) == EINVAL
    assert assign(levels=(C.c_int * 3)(100, -1, 25)) == EINVAL
    assert assign(N=-1) == EINVAL
    assert assign(G=-1) == EINVAL
    assert assign(K=-1) == EINVAL
    assert assign(m=None) == EINVAL
    assert assign(cls=None) == EINVAL  # GT rows need classes
    assert assign(N=0) == 0            # nothing to do: no launch
    assert assign(levels=(C.c_int * 3)(0, 0, 0)) == 0


def test_fake_kernels_trace_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    from detectron2_b200 import _C
    from detectron2_b200 import fcos as F
    from detectron2_b200 import losses as L

    with FakeTensorMode(allow_non_fake_inputs=False):
        dev = torch.device("cuda")
        an = torch.empty((30, 4), device=dev)
        gt = torch.empty((2, 7, 4), device=dev)
        labels, boxes, matches = F.fcos_assign_op(an, [20, 10], gt, torch.empty((2,), dtype=torch.int64, device=dev),
                                                  torch.empty((2, 7), dtype=torch.int64, device=dev), 80, 1.5)
        assert labels.shape == (2, 30) and labels.dtype == torch.int64 and boxes.shape == (2, 30, 4)
        assert matches.shape == (2, 30)
        logits = [torch.empty((2, 20, 80), device=dev), torch.empty((2, 10, 80), device=dev)]
        deltas = [torch.empty((2, 20, 4), device=dev), torch.empty((2, 10, 4), device=dev)]
        ctr = [torch.empty((2, 20, 1), device=dev), torch.empty((2, 10, 1), device=dev)]
        sums, counts, status = L.dense_loss_op(logits, deltas, ctr, an, boxes, labels, 80, False, 2.0, 0.25, 0.0,
                                               _C.LOSS_LINEAR_GIOU, 0.0, None)
        assert sums.shape == (3,) and sums.dtype == torch.float32 and counts.shape == (2,) and counts.dtype == torch.int64
        assert status.shape == () and status.dtype == torch.int32
        grads = L.dense_loss_backward_op(logits, deltas, ctr, an, boxes, labels, 80, False, 2.0, 0.25, 0.0,
                                         _C.LOSS_LINEAR_GIOU, 0.0, None, sums)
        assert [g.shape for g in grads] == [t.shape for t in logits + deltas + ctr]
