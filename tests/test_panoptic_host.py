"""Panoptic FPN inference without a GPU: the torch restatements of detectron2_b200/panoptic.py against the reference
fixture (tests/golden/panoptic.npz, tests/golden/make_golden_panoptic.py), the documented instance order on ties and
NaN scores, the argument checks of d2b_sem_seg_labels / d2b_panoptic_combine (nothing launched), and the fake kernels."""
import ctypes as C

import numpy as np
import pytest
import torch

from detectron2_b200 import _C
from detectron2_b200 import panoptic as P

EINVAL, EWORKSPACE = -1, -2
CONST_CASE = 3  # make_golden_panoptic.py: this case's logits hold a constant patch


def sem_logits(case, i):
    C_, Hp, Wp, _, _, _, _, seed = (int(v) for v in case)
    logits = torch.randn((C_, Hp, Wp), generator=torch.Generator().manual_seed(seed))
    if i == CONST_CASE:
        logits[:, 5:9, 6:12] = 0.125
    return logits


def _scene(gold, name):
    t = lambda k: torch.from_numpy(gold[name + "_" + k])  # noqa: E731
    return t("scores"), t("classes"), t("masks"), t("labels"), gold[name + "_thr"]


def test_sem_seg_labels_restatement_matches_reference(golden):
    gold = golden("panoptic")
    for i in range(5):
        case = gold["sem%d_case" % i]
        _, _, _, h, w, H, W, _ = (int(v) for v in case)
        got = P.sem_seg_labels(sem_logits(case, i)[None], [(h, w)], [(H, W)])[0]
        assert torch.equal(got, torch.from_numpy(gold["sem%d_labels" % i])), i


def test_combine_restatement_matches_reference(golden):
    gold = golden("panoptic")
    assert len(gold["scenes"]) >= 17
    for name in gold["scenes"]:
        scores, classes, masks, labels, (ov, st, sc) = _scene(gold, name)
        inst = type("I", (), dict(scores=scores, pred_classes=classes, pred_masks=masks))
        pan, info = P.combine_semantic_and_instance_outputs(inst, labels, ov, st, sc)
        assert torch.equal(pan, torch.from_numpy(gold[name + "_panoptic"])), name
        want = [tuple(r) for r in gold[name + "_records"].tolist()]
        got = [(d["id"], int(d["isthing"]), d["category_id"], d.get("instance_id", -1), d.get("area", 0)) for d in info]
        assert got == want, name
        assert [d.get("score", 0.0) for d in info] == gold[name + "_record_scores"].tolist(), name
        for d in info:  # the reference's keys per segment kind
            keys = {"id", "isthing", "score", "category_id", "instance_id"} if d["isthing"] else \
                {"id", "isthing", "category_id", "area"}
            assert set(d) == keys


def _stable_order(scores):
    """Explicit restatement of the documented order: finite / infinite scores descending, ties by index, then the NaNs by
    index."""
    s = scores.tolist()
    key = lambda i: (1, 0.0, i) if s[i] != s[i] else (0, -s[i], i)  # noqa: E731
    return sorted(range(len(s)), key=key)


def test_walk_order_ties_and_nan():
    scores = torch.tensor([0.5, float("nan"), 0.9, 0.5, -0.0, 0.0, float("-nan"), 0.9, float("inf"), 0.5])
    assert P._walk_order(scores) == _stable_order(scores)
    g = torch.Generator().manual_seed(0)
    for _ in range(20):
        s = torch.randint(0, 4, (40,), generator=g).float() / 4
        s[torch.rand(40, generator=g) < 0.1] = float("nan")
        assert P._walk_order(s) == _stable_order(s)


def test_combine_tie_and_nan_follow_the_documented_order():
    H, W = 6, 8
    masks = torch.zeros((4, H, W), dtype=torch.uint8)
    masks[:, :, :] = 1  # every instance covers the whole image: only the first walked one paints
    labels = torch.zeros((H, W), dtype=torch.int64)
    for scores, first in ((torch.tensor([0.7, 0.9, 0.9, 0.1]), 1), (torch.tensor([float("nan"), 0.6, 0.6, 0.8]), 3)):
        pan, records = P._combine_host(scores, torch.arange(4), masks, labels, 0.5, 0.0, 0.0)
        assert records[0][3] == first and len(records) == 1 and bool((pan == 1).all())
    # a NaN score never stops the walk; it is walked last
    masks2 = torch.zeros((2, H, W), dtype=torch.uint8)
    masks2[0, :3], masks2[1, 3:] = 1, 1
    _, records = P._combine_host(torch.tensor([float("nan"), 0.9]), torch.arange(2), masks2, labels, 0.5, 0.0, 0.95)
    assert [r[3] for r in records] == []  # 0.9 < 0.95 stops before the NaN
    _, records = P._combine_host(torch.tensor([float("nan"), 0.9]), torch.arange(2), masks2, labels, 0.5, 0.0, 0.5)
    assert [r[3] for r in records] == [1, 0]


def _images(n=2, r=3, h=5, w=7, p=0x1000):
    d = _C.PanopticImages()
    for i in range(n):
        d.R[i], d.H[i], d.W[i] = r, h, w
        d.scores[i] = d.classes[i] = d.masks[i] = d.labels[i] = d.panoptic[i] = p
    return d


def _combine(lib, d, n=2, c=54, ws_bytes=None, **over):
    args = dict(num_instances=None, num_segments=0x2000, seg_info=0x2000, seg_score=0x2000, status=0x2000,
                workspace=0x100000)
    args.update(over)
    ref = C.byref(d) if d is not None else None
    need = lib.d2b_panoptic_workspace_bytes(ref, n, c)
    return lib.d2b_panoptic_combine(ref, n, c, args["num_instances"], 0.5, 4096.0,
                                    0.5, args["num_segments"], args["seg_info"], args["seg_score"], args["status"],
                                    args["workspace"], need if ws_bytes is None else ws_bytes, None)


def test_combine_validates_arguments_in_order_without_a_gpu():
    """Every fault returns before any CUDA call (the pointers are not device memory, so a launch would fail with a CUDA
    error, not a D2B code)."""
    lib = _C.lib()
    d = _images()
    assert _combine(lib, None) == EINVAL
    assert _combine(lib, d, n=-1) == EINVAL
    assert _combine(lib, d, n=_C.MAX_IMAGES + 1) == EINVAL
    assert _combine(lib, d, c=0) == EINVAL
    assert _combine(lib, d, c=P.PANOPTIC_MAX_CLASSES + 1) == EINVAL
    assert _combine(lib, d, n=0, num_segments=None) == 0  # no image: nothing to do, nothing checked further
    for field, value in (("H", 0), ("W", 0), ("R", -1), ("R", P.PANOPTIC_MAX_INSTANCES + 1), ("H", 1 << 16)):
        bad = _images()
        getattr(bad, field)[1] = value
        if field == "H" and value > 1:
            bad.W[1] = 1 << 16  # H * W > INT_MAX
        assert _combine(lib, bad) == EINVAL, (field, value)
    for field in ("labels", "panoptic", "scores", "classes", "masks"):
        bad = _images()
        getattr(bad, field)[0] = None
        assert _combine(lib, bad) == EINVAL, field
    no_inst = _images(r=0)
    no_inst.scores[0] = no_inst.classes[0] = no_inst.masks[0] = None
    assert _combine(lib, no_inst, workspace=None) == EINVAL  # R == 0 needs no instance pointers; workspace is checked
    for name in ("num_segments", "seg_info", "seg_score", "status", "workspace"):
        assert _combine(lib, d, **{name: None}) == EINVAL, name
    assert _combine(lib, d, workspace=0x100010) == EINVAL  # not 256-byte aligned
    assert _combine(lib, d, ws_bytes=lib.d2b_panoptic_workspace_bytes(C.byref(d), 2, 54) - 1) == EWORKSPACE


def test_workspace_query_grows_with_the_scene():
    lib = _C.lib()
    small = lib.d2b_panoptic_workspace_bytes(C.byref(_images(r=1)), 2, 54)
    big = lib.d2b_panoptic_workspace_bytes(C.byref(_images(r=100, h=800, w=1333)), 2, 54)
    assert 0 < small < big
    assert big >= 2 * 100 * 800 * 42 * 4  # the bit rows: R x H x ceil(W / 32) words per image
    assert lib.d2b_panoptic_workspace_bytes(C.byref(_images(r=-1)), 2, 54) == 0
    assert lib.d2b_panoptic_workspace_bytes(None, 2, 54) == 0


def test_sem_seg_labels_validates_arguments_in_order_without_a_gpu():
    lib = _C.lib()

    def call(n=2, dtype=0, c=54, hp=24, wp=40, logits=0x1000, img=True, **over):
        d = _C.SemSegImages()
        for i in range(max(n, 0)):
            if i < _C.MAX_IMAGES:
                d.h[i], d.w[i], d.H[i], d.W[i], d.labels[i] = 20, 30, 40, 50, 0x2000
        for k, (i, v) in over.items():
            getattr(d, k)[i] = v
        return lib.d2b_sem_seg_labels(logits, dtype, n, c, hp, wp, C.byref(d) if img else None, None)

    assert call(img=False) == EINVAL
    assert call(n=-1) == EINVAL and call(n=_C.MAX_IMAGES + 1) == EINVAL
    assert call(dtype=3) == EINVAL and call(c=0) == EINVAL and call(hp=0) == EINVAL and call(wp=0) == EINVAL
    assert call(n=0, logits=None) == 0
    assert call(logits=None) == EINVAL
    for k, v in (("h", 0), ("h", 25), ("w", 0), ("w", 41), ("H", 0), ("W", 0), ("labels", None)):
        assert call(**{k: (1, v)}) == EINVAL, (k, v)
    assert call(H=(1, 1 << 16), W=(1, 1 << 16)) == EINVAL


def test_fake_kernels_trace_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        lg = torch.empty((2, 54, 200, 336), device="cuda")
        labels = P.sem_seg_labels_op(lg, [200, 300, 180, 336], [480, 640, 427, 640])
        assert [tuple(x.shape) for x in labels] == [(480, 640), (427, 640)] and labels[0].dtype == torch.int64
        masks = [torch.empty((5, 480, 640), dtype=torch.uint8, device="cuda"),
                 torch.empty((3, 427, 640), dtype=torch.uint8, device="cuda")]
        scores = [torch.empty((5,), device="cuda"), torch.empty((3,), device="cuda")]
        classes = [torch.empty((5,), dtype=torch.int64, device="cuda"), torch.empty((3,), dtype=torch.int64, device="cuda")]
        pans, nseg, info, sc, status = P.panoptic_combine_op(scores, classes, masks, labels, None, 54, 0.5, 4096.0, 0.5)
        assert [tuple(p.shape) for p in pans] == [(480, 640), (427, 640)] and pans[0].dtype == torch.int32
        assert nseg.shape == (2,) and info.shape == (2, 59, 5) and sc.shape == (2, 59) and status.dtype == torch.int32


def test_cpu_tensors_never_reach_the_kernels():
    with pytest.raises(NotImplementedError):
        P.sem_seg_labels_op(torch.zeros(1, 2, 4, 4), [4, 4], [4, 4])
    m = torch.zeros((1, 4, 4), dtype=torch.uint8)
    with pytest.raises(NotImplementedError):
        P.combine_semantic_and_instance_outputs_fixed([torch.zeros(1)], [torch.zeros(1, dtype=torch.int64)], [m],
                                                      [torch.zeros(4, 4, dtype=torch.int64)], 2)
    np.testing.assert_equal(P._sem_seg_labels_host(torch.zeros(1, 3, 4, 4), [(4, 4)], [(2, 2)])[0].numpy(), 0)
