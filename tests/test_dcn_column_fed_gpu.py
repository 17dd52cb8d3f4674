"""Deformable conv training path with several output-channel tiles: the forward gathers and saves the columns once (tile 0)
and computes the other tiles from them (dcn_fwd_cols_kernel); the weight gradient streams the saved columns.  Compared with
the per-tile gather forward, the re-sampling weight gradient and the oracle, at the R50 res4 / res5 shapes of the benchmark.
Run on an H100: pytest -m gpu."""
import math

import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda"
SHAPES = [(256, 50, 84), (512, 25, 42)]  # res4, res5 of the benchmark (2 images)


def _inputs(c, h, w, mod, seed, dg=1):
    g = torch.Generator().manual_seed(seed)
    n = 2
    x = torch.randn(n, c, h, w, generator=g)
    off = torch.randn(n, 2 * dg * 9, h, w, generator=g) * 2
    mask = torch.sigmoid(torch.randn(n, dg * 9, h, w, generator=g)) if mod else None
    wt = torch.randn(c, c, 3, 3, generator=g) * (1.0 / math.sqrt(c * 9))
    go = torch.randn(n, c, h, w, generator=g)
    return x, off, mask, wt, go


@pytest.fixture(scope="module")
def L():
    import detectron2_b200.layers as layers

    return layers


def _dev(t):
    return None if t is None else t.to(DEV)


def _rel(a, b):
    b = b.detach().float().cpu()
    return (a.detach().float().cpu() - b).abs().max().item() / (b.abs().max().item() + 1e-30)


@pytest.mark.parametrize("c,h,w", SHAPES)
@pytest.mark.parametrize("prec", [1, 2])
@pytest.mark.parametrize("mod", [False, True])
def test_train_forward_matches_gather_forward(c, h, w, prec, mod):
    from detectron2_b200 import ops

    x, off, mask, wt, _ = _inputs(c, h, w, mod, c + h + 7 * prec + mod)
    bias = torch.randn(c, generator=torch.Generator().manual_seed(c)) if mod else None
    args = ([1, 1], [1, 1], [1, 1], 1, 1, prec)
    y_gather = ops.deform_conv_op(_dev(x), _dev(off), _dev(mask), _dev(wt), _dev(bias), *args)
    y_train, _, cols = ops.deform_conv_train_op(_dev(x), _dev(off), _dev(mask), _dev(wt), _dev(bias), *args)
    assert cols.numel() > 0
    # the same bf16 operands on both sides: only the fp32 summation order differs
    assert _rel(y_train, y_gather) <= 1e-5
    if prec == 1 and mod:
        ref = orc.deform_conv_forward(x[:1], off[:1], mask[:1], wt, bias, 1, 1, 1, 1, 1)
        assert _rel(y_train[:1], ref) <= 1e-4


@pytest.mark.parametrize("h,w", [(25, 42), (7, 9)])
def test_fused_train_forward_applies_epilogue_once(L, h, w):
    # 512 channels = 4 output-channel tiles; both maps split the reduction over kernel points, so the partials of the gathering
    # and the column-fed launch meet in one zero-filled output and scale / shift / ReLU run once in the follow-up pass
    from detectron2_b200 import ops

    c = 512
    g = torch.Generator().manual_seed(h)
    x = torch.randn(2, c, h, w, generator=g)
    om = torch.randn(2, 27, h, w, generator=g) * 1.5
    wt = torch.randn(c, c, 3, 3, generator=g) * (1.0 / math.sqrt(c * 9))
    scale, shift = 0.5 + torch.rand(c, generator=g), torch.randn(c, generator=g) * 0.3
    args = (True, [1, 1], [1, 1], [1, 1], 1, 1, 1)
    y_train, _, cols = ops.deform_conv_fused_train_op(_dev(x), _dev(om), _dev(wt), _dev(scale), _dev(shift), *args)
    assert cols.numel() > 0
    ox, oy, m = torch.chunk(_dev(om), 3, dim=1)
    raw = ops.deform_conv_op(_dev(x), torch.cat((ox, oy), 1), m.sigmoid(), _dev(wt), None, [1, 1], [1, 1], [1, 1], 1, 1, 1)
    ref = (raw * _dev(scale)[None, :, None, None] + _dev(shift)[None, :, None, None]).relu()
    assert _rel(y_train, ref) <= 1e-5
    y_gather = ops.deform_conv_fused_op(_dev(x), _dev(om), _dev(wt), _dev(scale), _dev(shift), *args)
    assert _rel(y_train, y_gather) <= 1e-5
    mod = L.DeformBottleneckConv2(c, c, 3, 1, 1, 1, 1, 1, True).to(DEV)
    with torch.no_grad():
        mod.weight.copy_(wt)
        mod.norm_scale.copy_(scale)
        mod.norm_shift.copy_(shift)
    xm = x.to(DEV).requires_grad_(True)
    assert _rel(mod(xm, om.to(DEV)), ref) <= 1e-5


@pytest.mark.parametrize("c,h,w", SHAPES)
@pytest.mark.parametrize("mod", [False, True])
def test_weight_gradient_from_columns_matches_resampling(c, h, w, mod):
    from detectron2_b200 import ops

    x, off, mask, wt, go = _inputs(c, h, w, mod, 3 * c + h + mod)
    args = ([1, 1], [1, 1], [1, 1], 1, 1)
    _, xs, cols = ops.deform_conv_train_op(_dev(x), _dev(off), _dev(mask), _dev(wt), None, *args, 1)
    xk = xs if xs.numel() else _dev(x)
    with_cols = ops.deform_conv_backward_op(xk, _dev(off), _dev(mask), _dev(wt), _dev(go), *args, False, True, True, 1, cols)
    resampled = ops.deform_conv_backward_op(xk, _dev(off), _dev(mask), _dev(wt), _dev(go), *args, False, True, True, 1)
    for name, a, r in zip(["gx", "goff", "gmask", "gw"], with_cols, resampled):
        if r.numel():
            assert _rel(a, r) <= 1e-5, name
    if mod:
        gref = orc.deform_conv_backward(x, off, mask, wt, go, 1, 1, 1, 1, 1, mod)
        assert _rel(with_cols[3], gref[3]) <= 1e-4


def test_training_step_in_cuda_graph():
    # forward (gather + column-fed tiles) and backward (weight gradient from the columns) captured once and replayed
    # on new inputs copied into the captured buffers: same results as the eager calls on those inputs
    from detectron2_b200 import ops

    c, h, w = 512, 25, 42
    args = ([1, 1], [1, 1], [1, 1], 1, 1)

    def step(x, off, mask, wt, go):
        y, xs, cols = ops.deform_conv_train_op(x, off, mask, wt, None, *args, 1)
        gx, goff, gm, gw, _ = ops.deform_conv_backward_op(xs, off, mask, wt, go, *args, False, True, True, 1, cols)
        return y, gx, goff, gm, gw

    static = [_dev(t) for t in _inputs(c, h, w, True, 11)]
    step(*static)  # warm-up: allocations, shared-memory opt-ins
    torch.cuda.synchronize()
    graph, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            outs = step(*static)
    torch.cuda.current_stream().wait_stream(side)
    for seed in (12, 13):
        new = [_dev(t) for t in _inputs(c, h, w, True, seed)]
        for s, t in zip(static, new):
            s.copy_(t)
        graph.replay()
        torch.cuda.synchronize()
        eager = step(*new)
        for name, a, r in zip(["y", "gx", "goff", "gmask", "gw"], outs, eager):
            assert _rel(a, r) <= 1e-5, (seed, name)
