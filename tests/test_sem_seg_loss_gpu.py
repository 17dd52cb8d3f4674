"""Semantic segmentation loss on the GPU: d2b_sem_seg_loss_forward / _backward against the reference fixture
(tests/golden/sem_seg_loss.npz) and against F.interpolate + F.cross_entropy / DeepLabCE on CUDA (the restatement in
detectron2_b200/semantic_seg.py) at the sizes the heads train at; half-precision logits, reproducibility, CUDA-graph
replay, the top-k tie rule across CTAs, and the bad-label status."""
import pytest
import torch

from detectron2_b200 import semantic_seg as S
from sem_seg_ref import CASES, make_case

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")

# name: (N, C, Hp, Wp, stride, top_k, weights)
SIZES = {
    "panoptic_fpn": (2, 54, 200, 336, 4, None, False),
    "panoptic_deeplab_cityscapes": (4, 19, 256, 512, 4, 0.2, True),
    "panoptic_deeplab_coco": (2, 133, 160, 160, 4, 0.2, True),
    "deeplabv3_stride16": (2, 19, 64, 128, 16, None, False),
    "deeplabv3_stride16_topk": (2, 19, 64, 128, 16, 0.2, False),
}


def make_inputs(n, c, hp, wp, s, with_weights, seed=0, ignore=255, dtype=torch.float32):
    g = torch.Generator(device=DEV).manual_seed(seed)
    h, w = hp * s, wp * s
    logits = (torch.randn((n, c, hp, wp), generator=g, device=DEV) * 3.0).to(dtype)
    targets = torch.randint(0, c, (n, h, w), generator=g, device=DEV)
    targets[torch.rand((n, h, w), generator=g, device=DEV) < 0.1] = ignore
    targets[:, : h // 5, : w // 4] = ignore
    weights = 0.5 + 2.5 * torch.rand((n, h, w), generator=g, device=DEV) if with_weights else None
    return logits, targets, weights


def ours(logits, targets, s, ignore, top_k, weights):
    lg = logits.detach().clone().requires_grad_(True)
    loss, count, status = S.sem_seg_loss_fixed(lg, targets, s, ignore, top_k, weights)
    loss.backward()
    return loss.detach(), lg.grad, count, status


def restated(logits, targets, s, ignore, top_k, weights):
    lg = logits.detach().clone().requires_grad_(True)
    loss = S._sem_seg_loss_host(lg, targets, s, ignore, top_k, weights)
    loss.backward()
    return loss.detach(), lg.grad


def assert_grad_close(got, want, what):
    scale = want.abs().max().item()
    err = (got.float() - want.float()).abs().max().item()
    assert err <= 1e-5 * scale, "%s: max error %g, max |grad| %g" % (what, err, scale)


def test_kernels_match_reference_fixture(golden):
    gold = golden("sem_seg_loss")
    for name in CASES:
        _, _, _, _, s, ignore, top_k, _, _ = CASES[name]
        logits, targets, weights = (None if t is None else t.to(DEV) for t in make_case(name))
        loss, grad, count, status = ours(logits, targets, s, ignore, top_k, weights)
        assert int(status) == 0, name
        assert int(count) == int((targets != ignore).sum()), name
        want = torch.from_numpy(gold[name + "_loss"]).to(DEV)
        if name == "all_ignored":
            assert torch.isnan(loss) and not grad.any()
            continue
        torch.testing.assert_close(loss, want, rtol=1e-5, atol=0, msg=name)
        if name == "const_ties":
            continue  # tied pixels: the documented rule, checked below
        assert_grad_close(grad, torch.from_numpy(gold[name + "_grad"]).to(DEV), name)


@pytest.mark.parametrize("name", list(SIZES))
def test_kernels_match_torch_at_training_sizes(name):
    n, c, hp, wp, s, top_k, with_w = SIZES[name]
    logits, targets, weights = make_inputs(n, c, hp, wp, s, with_w, seed=list(SIZES).index(name))
    loss, grad, count, status = ours(logits, targets, s, 255, top_k, weights)
    want_loss, want_grad = restated(logits, targets, s, 255, top_k, weights)
    assert int(status) == 0 and int(count) == int((targets != 255).sum())
    torch.testing.assert_close(loss, want_loss, rtol=1e-5, atol=0)
    assert_grad_close(grad, want_grad, name)
    if top_k is not None:
        _, _, _, _, sel = S.sem_seg_loss_op(logits, targets, s, 255, top_k, weights)
        assert int(sel.sum()) == int(top_k * targets.numel())


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
@pytest.mark.parametrize("top_k", [None, 0.2])
def test_half_precision_logits_equal_the_fp32_run_of_their_values(dtype, top_k):
    logits, targets, weights = make_inputs(2, 54, 100, 168, 4, top_k is not None, seed=3, dtype=dtype)
    loss, grad, _, _ = ours(logits, targets, 4, 255, top_k, weights)
    loss32, grad32, _, _ = ours(logits.float(), targets, 4, 255, top_k, weights)
    assert grad.dtype == dtype
    assert torch.equal(loss, loss32)
    assert torch.equal(grad, grad32.to(dtype))


@pytest.mark.parametrize("name", ["panoptic_fpn", "panoptic_deeplab_cityscapes"])
def test_two_runs_are_bitwise_identical(name):
    n, c, hp, wp, s, top_k, with_w = SIZES[name]
    logits, targets, weights = make_inputs(n, c, hp, wp, s, with_w, seed=5)
    a = ours(logits, targets, s, 255, top_k, weights)
    b = ours(logits, targets, s, 255, top_k, weights)
    for x, y in zip(a, b):
        assert torch.equal(x, y)


@pytest.mark.parametrize("top_k", [None, 0.2, 1.0])
def test_cuda_graph_replay_on_new_inputs_equals_eager(top_k):
    n, c, hp, wp, s = 2, 19, 64, 96, 4
    with_w = top_k is not None
    logits, targets, weights = make_inputs(n, c, hp, wp, s, with_w, seed=7)
    static_lg = logits.clone().requires_grad_(True)
    static_tg, static_w = targets.clone(), None if weights is None else weights.clone()

    def step():
        loss, count, status = S.sem_seg_loss_fixed(static_lg, static_tg, s, 255, top_k, static_w)
        (grad,) = torch.autograd.grad(loss, static_lg)
        return loss, grad, count, status

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = step()
    new_lg, new_tg, new_w = make_inputs(n, c, hp, wp, s, with_w, seed=8)
    with torch.no_grad():
        static_lg.copy_(new_lg)
        static_tg.copy_(new_tg)
        if static_w is not None:
            static_w.copy_(new_w)
    graph.replay()
    torch.cuda.synchronize()
    want = ours(new_lg, new_tg, s, 255, top_k, new_w)
    for x, y in zip(out, want):
        assert torch.equal(x, y)


def test_top_k_ties_are_taken_in_ascending_flat_index():
    """Constant logits: every valid pixel's loss is log(C), so the k-th largest is tied over ~100 CTAs of pixels."""
    n, c, hp, wp, s = 2, 8, 50, 60, 4
    _, targets, _ = make_inputs(n, c, hp, wp, s, False, seed=9)
    logits = torch.full((n, c, hp, wp), 0.375, device=DEV)
    k = int(0.2 * targets.numel())
    _, _, _, _, sel = S.sem_seg_loss_op(logits, targets, s, 255, 0.2, None)
    valid = torch.nonzero(targets.view(-1) != 255).squeeze(1)
    assert valid.numel() > k
    assert torch.equal(torch.nonzero(sel.view(-1)).squeeze(1), valid[:k])
    loss, grad, _, _ = ours(logits, targets, s, 255, 0.2, None)
    want_loss, want_grad = restated(logits, targets, s, 255, 0.2, None)  # stable sort: the same rule
    torch.testing.assert_close(loss, want_loss, rtol=1e-6, atol=0)
    assert_grad_close(grad, want_grad, "ties")


def test_k_zero_gives_nan_and_a_zero_gradient():
    logits, targets, _ = make_inputs(1, 5, 4, 5, 4, False, seed=10)
    loss, grad, _, _ = ours(logits, targets, 4, 255, 1e-6, None)
    assert torch.isnan(loss) and not grad.any()


def test_bad_label_sets_the_status_and_the_wrappers_raise():
    """Only our kernel sees the bad label: torch's CUDA cross_entropy would assert on the device."""
    logits, targets, weights = make_inputs(2, 19, 16, 20, 4, True, seed=11)
    targets[1, 7, 9] = 19
    _, _, status = S.sem_seg_loss_fixed(logits, targets, 4, 255)
    assert int(status) == S.STATUS_BAD_LABEL
    with pytest.raises(RuntimeError):
        S.sem_seg_fpn_losses(logits, targets, 4, 255, 1.0)
    targets[1, 7, 9] = -3
    with pytest.raises(RuntimeError):
        S.deeplab_losses(logits, targets, 4, 255, 1.0, "hard_pixel_mining", 0.2, weights)


def test_wrappers_return_the_reference_dicts():
    logits, targets, weights = make_inputs(2, 54, 50, 84, 4, True, seed=12)
    got = S.sem_seg_fpn_losses(logits, targets, 4, 255, 0.5)
    want = S._sem_seg_loss_host(logits, targets, 4, 255) * 0.5
    assert set(got) == {"loss_sem_seg"}
    torch.testing.assert_close(got["loss_sem_seg"], want, rtol=1e-5, atol=0)
    got = S.deeplab_losses(logits, targets, 4, 255, 2.0, "hard_pixel_mining", 0.2, weights)
    want = S._sem_seg_loss_host(logits, targets, 4, 255, 0.2, weights) * 2.0
    torch.testing.assert_close(got["loss_sem_seg"], want, rtol=1e-5, atol=0)
    got = S.deeplab_losses(logits, targets, 4, 255, 1.0, "cross_entropy")
    torch.testing.assert_close(got["loss_sem_seg"], S._sem_seg_loss_host(logits, targets, 4, 255), rtol=1e-5, atol=0)
