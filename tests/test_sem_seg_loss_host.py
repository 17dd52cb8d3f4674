"""Semantic segmentation loss without a GPU: the torch restatement of detectron2_b200/semantic_seg.py against the reference
fixture (tests/golden/sem_seg_loss.npz, tests/golden/make_golden_sem_seg.py), the top-k tie rule, the argument checks of
d2b_sem_seg_loss_forward / _backward and the workspace query (nothing launched), and the fake kernels."""
import ctypes as C

import numpy as np
import pytest
import torch

from detectron2_b200 import _C
from detectron2_b200 import semantic_seg as S
from sem_seg_ref import CASES, make_case

EINVAL, EWORKSPACE = -1, -2
MEAN, TOP_K = S.SEMSEG_MEAN, S.SEMSEG_TOP_K


def host_loss(name, logits):
    _, _, _, _, s, ignore, top_k, _, _ = CASES[name]
    _, targets, weights = make_case(name)
    return S._sem_seg_loss_host(logits, targets, s, ignore, top_k, weights)


def test_restatement_matches_reference(golden):
    gold = golden("sem_seg_loss")
    assert list(gold["cases"]) == list(CASES)
    for name in CASES:
        logits = make_case(name)[0].requires_grad_(True)
        loss = host_loss(name, logits)
        loss.backward()
        want = torch.from_numpy(gold[name + "_loss"])
        if name == "all_ignored":  # the reference's NaN and zero gradient
            assert torch.isnan(loss) and torch.isnan(want)
            assert not logits.grad.any()
            continue
        torch.testing.assert_close(loss.detach(), want, rtol=1e-6, atol=0, msg=name)
        if name != "const_ties":  # the reference's topk picks among ties in its own order
            torch.testing.assert_close(logits.grad, torch.from_numpy(gold[name + "_grad"]), rtol=1e-5, atol=1e-8,
                                       msg=name)


def test_top_k_takes_ties_in_ascending_flat_index(golden):
    gold = golden("sem_seg_loss")
    n, c, hp, wp, s, ignore, top_k, _, _ = CASES["const_ties"]
    logits, targets, _ = make_case("const_ties")
    pixel = torch.nn.functional.cross_entropy(torch.full((n, c, hp * s, wp * s), 0.375), targets, reduction="none",
                                              ignore_index=ignore).view(-1)
    k = int(top_k * pixel.numel())
    valid = torch.nonzero(targets.view(-1) != ignore).squeeze(1)
    assert valid.numel() > k and bool((pixel[valid] == pixel[valid[0]]).all())  # every valid pixel ties
    order = torch.sort(pixel, descending=True, stable=True).indices[:k]
    assert torch.equal(order, valid[:k])
    # the tie choice moves the gradient only: the loss is the reference's
    lg = logits.clone().requires_grad_(True)
    loss = S._sem_seg_loss_host(lg, targets, s, ignore, top_k)
    torch.testing.assert_close(loss.detach(), torch.from_numpy(gold["const_ties_loss"]), rtol=1e-6, atol=0)
    # the per-output-pixel gradient is nonzero exactly on the first k valid pixels
    up = torch.nn.functional.interpolate(lg.detach(), scale_factor=s, mode="bilinear", align_corners=False)
    up.requires_grad_(True)
    pix = torch.nn.functional.cross_entropy(up, targets, reduction="none", ignore_index=ignore).view(-1)
    pix[torch.sort(pix.detach(), descending=True, stable=True).indices[:k]].mean().backward()
    hit = up.grad.abs().sum(1).view(-1) > 0
    assert torch.equal(torch.nonzero(hit).squeeze(1), valid[:k])


def test_nan_ranks_above_inf_in_the_restatement():
    pixel = torch.tensor([1.0, float("inf"), float("nan"), 2.0, -0.0, 0.0])
    assert torch.sort(pixel, descending=True, stable=True).indices[:2].tolist() == [2, 1]


def _fwd(lib, **over):
    a = dict(logits=0x1000, dtype=0, N=2, C=19, Hp=8, Wp=10, stride=4, targets=0x1000, ignore=255, reduction=TOP_K,
             top_k=0.2, weights=None, lse=0x1000, selected=0x1000, loss_sum=0x1000, count=0x1000, status=0x1000,
             workspace=0x100000, ws_bytes=None)
    a.update(over)
    need = lib.d2b_sem_seg_loss_workspace_bytes(a["N"], a["C"], a["Hp"], a["Wp"], a["stride"], a["dtype"], a["reduction"],
                                                a["top_k"])
    return lib.d2b_sem_seg_loss_forward(a["logits"], a["dtype"], a["N"], a["C"], a["Hp"], a["Wp"], a["stride"], a["targets"],
                                        a["ignore"], a["reduction"], a["top_k"], a["weights"], a["lse"], a["selected"],
                                        a["loss_sum"], a["count"], a["status"], a["workspace"],
                                        need if a["ws_bytes"] is None else a["ws_bytes"], None)


def _bwd(lib, **over):
    a = dict(logits=0x1000, dtype=0, N=2, C=19, Hp=8, Wp=10, stride=4, targets=0x1000, ignore=255, weights=None,
             selected=None, lse=0x1000, grad_sum=0x1000, grad=0x1000)
    a.update(over)
    return lib.d2b_sem_seg_loss_backward(a["logits"], a["dtype"], a["N"], a["C"], a["Hp"], a["Wp"], a["stride"],
                                         a["targets"], a["ignore"], a["weights"], a["selected"], a["lse"], a["grad_sum"],
                                         a["grad"], None)


# rule 1 of both entry points: shapes and dtype
SHAPE_FAULTS = [dict(N=-1), dict(N=65536), dict(C=0), dict(Hp=0), dict(Wp=0), dict(stride=0),
                dict(stride=S.SEMSEG_MAX_STRIDE + 1), dict(dtype=3), dict(dtype=-1),
                dict(N=64, Hp=2048, Wp=2048, stride=4), dict(C=1 << 16, Hp=1 << 8, Wp=1 << 8, stride=1)]


def test_forward_validates_arguments_in_order_without_a_gpu():
    """Every fault returns before any CUDA call (the pointers are not device memory, so a launch would fail with a CUDA
    error, not a D2B code)."""
    lib = _C.lib()
    for f in SHAPE_FAULTS:
        assert _fwd(lib, **f) == EINVAL, f
    # rule 1: the reduction
    for f in (dict(reduction=2), dict(reduction=-1), dict(reduction=MEAN, weights=0x1000), dict(top_k=float("nan")),
              dict(top_k=-0.01), dict(top_k=1.01)):
        assert _fwd(lib, **f) == EINVAL, f
    # rule 2: outputs and inputs; a rule-2 fault wins over a small workspace (rule 3)
    for f in (dict(loss_sum=None), dict(count=None), dict(status=None), dict(logits=None), dict(targets=None),
              dict(lse=None), dict(selected=None)):
        assert _fwd(lib, **f) == EINVAL, f
        assert _fwd(lib, ws_bytes=0, **f) == EINVAL, f
    # N == 0 needs no input, top-k 1.0 and the mean no selected buffer: these pass rule 2 and stop at rule 3
    for f in (dict(N=0, logits=None, targets=None, lse=None), dict(top_k=1.0, selected=None),
              dict(reduction=MEAN, selected=None)):
        assert _fwd(lib, workspace=None, **f) == EINVAL, f
        assert _fwd(lib, ws_bytes=0, **f) == EWORKSPACE, f
    # rule 3: the workspace
    assert _fwd(lib, workspace=None) == EINVAL
    assert _fwd(lib, workspace=0x100080) == EINVAL  # not 256-byte aligned
    need = lib.d2b_sem_seg_loss_workspace_bytes(2, 19, 8, 10, 4, 0, TOP_K, 0.2)
    assert _fwd(lib, ws_bytes=need - 1) == EWORKSPACE


def test_backward_validates_arguments_in_order_without_a_gpu():
    lib = _C.lib()
    for f in SHAPE_FAULTS:
        assert _bwd(lib, **f) == EINVAL, f
    # rule 2: N == 0 writes nothing and reads no pointer
    assert _bwd(lib, N=0, logits=None, targets=None, lse=None, grad_sum=None, grad=None) == 0
    assert _bwd(lib, N=0, stride=0, logits=None) == EINVAL
    # rule 3
    for f in (dict(logits=None), dict(targets=None), dict(lse=None), dict(grad_sum=None), dict(grad=None)):
        assert _bwd(lib, **f) == EINVAL, f


def test_workspace_query():
    lib = _C.lib()
    q = lib.d2b_sem_seg_loss_workspace_bytes
    for f in SHAPE_FAULTS:
        a = dict(N=2, C=19, Hp=8, Wp=10, stride=4, dtype=0)
        a.update(f)
        assert q(a["N"], a["C"], a["Hp"], a["Wp"], a["stride"], a["dtype"], TOP_K, 0.2) == 0, f
    assert q(2, 19, 8, 10, 4, 0, 2, 0.2) == 0
    assert q(2, 19, 8, 10, 4, 0, TOP_K, 1.5) == 0
    assert q(2, 19, 8, 10, 4, 0, TOP_K, float("nan")) == 0
    pixels = 2 * 32 * 40
    mean, all_, sel = q(2, 19, 8, 10, 4, 0, MEAN, -1.0), q(2, 19, 8, 10, 4, 0, TOP_K, 1.0), q(2, 19, 8, 10, 4, 0, TOP_K, 0.2)
    assert mean >= 256 and mean == all_ and sel >= mean + 4 * pixels
    assert q(0, 19, 8, 10, 4, 0, MEAN, -1.0) >= 256  # the finish alone still gets a workspace
    assert q(2, 19, 8, 10, 4, 0, TOP_K, 0.0) == sel   # k == 0 keeps the selection layout
    big = q(4, 19, 256, 512, 4, 2, TOP_K, 0.2)
    assert big >= 4 * 1024 * 2048 * 4


def test_k_is_pythons_int():
    """The host computes k = int(top_k * numel); the wrappers divide by the same k."""
    for top_k, numel in ((0.2, 2560), (0.2, 4 * 1024 * 2048), (0.3, 10), (0.7, 3), (1e-9, 100)):
        assert int(top_k * numel) == np.int64(np.float64(top_k) * np.float64(numel))


def test_fake_kernels_trace_shapes():
    from torch._subclasses.fake_tensor import FakeTensorMode

    with FakeTensorMode():
        lg = torch.empty((2, 54, 200, 336), device="cuda", dtype=torch.bfloat16)
        tg = torch.empty((2, 800, 1344), dtype=torch.int64, device="cuda")
        loss_sum, count, status, lse, sel = S.sem_seg_loss_op(lg, tg, 4, 255, None, None)
        assert loss_sum.shape == () and loss_sum.dtype == torch.float32 and count.dtype == torch.int64
        assert status.dtype == torch.int32 and lse.shape == (2, 800, 1344) and sel.shape == (0,)
        wt = torch.empty((2, 800, 1344), device="cuda")
        _, _, _, _, sel = S.sem_seg_loss_op(lg, tg, 4, 255, 0.2, wt)
        assert sel.shape == (2, 800, 1344) and sel.dtype == torch.uint8
        _, _, _, _, sel = S.sem_seg_loss_op(lg, tg, 4, 255, 1.0, wt)
        assert sel.shape == (0,)
        g = S.sem_seg_loss_backward_op(lg, tg, 4, 255, wt, sel, lse, loss_sum)
        assert g.shape == lg.shape and g.dtype == torch.bfloat16


def test_cpu_tensors_never_reach_the_kernels(monkeypatch):
    def no_lib():
        raise AssertionError("a CPU tensor reached the native library")

    monkeypatch.setattr(_C, "lib", no_lib)
    logits, targets, weights = make_case("topk02_weights")
    out = S.sem_seg_fpn_losses(logits, targets, 4, 255, 0.5)
    assert set(out) == {"loss_sem_seg"} and torch.isfinite(out["loss_sem_seg"])
    out = S.deeplab_losses(logits, targets, 4, 255, 1.0, "hard_pixel_mining", 0.2, weights)
    assert torch.isfinite(out["loss_sem_seg"])
    with pytest.raises(NotImplementedError):
        S.sem_seg_loss_op(logits, targets, 4, 255, None, None)
    with pytest.raises(ValueError):
        S.deeplab_losses(logits, targets, 4, 255, 1.0, "focal")
    with pytest.raises(ValueError):
        S.deeplab_losses(logits, targets, 4, 255, 1.0, "cross_entropy", weights=weights)


def test_wrappers_match_the_reference_on_cpu(golden):
    gold = golden("sem_seg_loss")
    logits, targets, _ = make_case("fpn_c54")
    out = S.sem_seg_fpn_losses(logits, targets, 4, 255, 0.5)["loss_sem_seg"]
    torch.testing.assert_close(out, torch.from_numpy(gold["fpn_c54_loss"]) * 0.5, rtol=1e-6, atol=0)
    logits, targets, weights = make_case("topk02_weights")
    out = S.deeplab_losses(logits, targets, 4, 255, 1.0, "hard_pixel_mining", 0.2, weights)["loss_sem_seg"]
    torch.testing.assert_close(out, torch.from_numpy(gold["topk02_weights_loss"]), rtol=1e-6, atol=0)
