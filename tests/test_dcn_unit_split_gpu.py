"""Deformable conv on the tensor cores with the forward's reduction split by units (64-channel blocks of one kernel point),
so that a CTA's range may begin and end inside a kernel point, and with the data- and weight-gradient kernels of a backward
from saved columns run as one launch.  Every result is compared with the fp32 FFMA path (precision 0).

The shapes are chosen so that the unit ranges cut through kernel points on an H100's 132 SMs: 256 / 512 channels are 4 / 8
blocks per kernel point, and 192 channels give an odd unit count (27 at 3x3, 75 at 5x5), so the last range is short.
Run on an H100: pytest -m gpu."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = 1e-4
# (channels, kernel size, H, W); 2 images each
SHAPES = [(256, 3, 13, 21), (512, 3, 25, 42), (256, 5, 11, 17), (512, 5, 9, 13), (192, 3, 14, 18), (192, 5, 9, 11)]


def _inputs(c, k, h, w, mod, seed):
    g = torch.Generator().manual_seed(seed)
    n, kk = 2, k * k
    x = torch.randn(n, c, h, w, generator=g)
    off = torch.randn(n, 2 * kk, h, w, generator=g) * 2
    mask = torch.sigmoid(torch.randn(n, kk, h, w, generator=g)) if mod else None
    wt = torch.randn(c, c, k, k, generator=g) * (1.0 / math.sqrt(c * kk))
    go = torch.randn(n, c, h, w, generator=g)
    return [None if t is None else t.to(DEV) for t in (x, off, mask, wt, go)]


def _conv(k):
    p = k // 2
    return [1, 1], [p, p], [1, 1], 1, 1


def _rel(a, b):
    b = b.detach().float()
    return (a.detach().float() - b).abs().max().item() / (b.abs().max().item() + 1e-30)


def _check(got, ref, names):
    for name, a, r in zip(names, got, ref):
        assert a.shape == r.shape, name
        if r.numel():
            assert _rel(a, r) <= TOL, (name, _rel(a, r))


@pytest.mark.parametrize("c,k,h,w", SHAPES)
@pytest.mark.parametrize("mod", [False, True])
def test_forward_matches_ffma(c, k, h, w, mod):
    from detectron2_b200 import ops

    x, off, mask, wt, _ = _inputs(c, k, h, w, mod, c + k + h + mod)
    bias = torch.randn(c, generator=torch.Generator().manual_seed(c)).to(DEV) if mod else None
    ref = ops.deform_conv_op(x, off, mask, wt, bias, *_conv(k), 0)
    assert _rel(ops.deform_conv_op(x, off, mask, wt, bias, *_conv(k), 1), ref) <= TOL  # every output-channel tile gathers
    y, _, cols = ops.deform_conv_train_op(x, off, mask, wt, bias, *_conv(k), 1)  # tile 0 gathers, the others read cols
    assert cols.numel() > 0
    assert _rel(y, ref) <= TOL


@pytest.mark.parametrize("c,k,h,w", SHAPES)
@pytest.mark.parametrize("mod", [False, True])
def test_backward_matches_ffma(c, k, h, w, mod):
    # both gradients (one fused launch), the data gradient only and the weight gradient only, all from the saved columns
    from detectron2_b200 import ops

    x, off, mask, wt, go = _inputs(c, k, h, w, mod, 3 * c + k + w + mod)
    _, xs, cols = ops.deform_conv_train_op(x, off, mask, wt, None, *_conv(k), 1)
    xk = xs if xs.numel() else x
    names = ["gx", "goff", "gmask", "gw"]
    ref = ops.deform_conv_backward_op(x, off, mask, wt, go, *_conv(k), False, True, True, 0)[:4]
    both = ops.deform_conv_backward_op(xk, off, mask, wt, go, *_conv(k), False, True, True, 1, cols)[:4]
    _check(both, ref, names)
    data = ops.deform_conv_backward_op(xk, off, mask, wt, go, *_conv(k), False, True, False, 1, cols)[:4]
    assert data[3].numel() == 0
    _check(data[:3], ref[:3], names[:3])
    weight = ops.deform_conv_backward_op(xk, off, mask, wt, go, *_conv(k), False, False, True, 1, cols)[:4]
    assert all(t.numel() == 0 for t in weight[:3])
    _check(weight[3:], ref[3:], names[3:])


@pytest.mark.parametrize("c,k,h,w", [(512, 3, 25, 42), (192, 5, 9, 11)])
def test_fused_offset_mask_matches_ffma(c, k, h, w):
    # offset and mask logits in one tensor, scale / shift / ReLU in the epilogue: forward and backward against the FFMA path
    # on the chunked offset and the sigmoid of the logits
    from detectron2_b200 import ops

    g = torch.Generator().manual_seed(c + k)
    kk = k * k
    x = torch.randn(2, c, h, w, generator=g).to(DEV)
    om = (torch.randn(2, 3 * kk, h, w, generator=g) * 1.5).to(DEV)
    wt = (torch.randn(c, c, k, k, generator=g) * (1.0 / math.sqrt(c * kk))).to(DEV)
    scale, shift = (0.5 + torch.rand(c, generator=g)).to(DEV), (torch.randn(c, generator=g) * 0.3).to(DEV)
    go = torch.randn(2, c, h, w, generator=g).to(DEV)
    conv = _conv(k)
    y, xs, cols = ops.deform_conv_fused_train_op(x, om, wt, scale, shift, True, *conv, 1)
    assert cols.numel() > 0
    off, logit = om[:, : 2 * kk], om[:, 2 * kk:]
    m = logit.sigmoid()
    raw = ops.deform_conv_op(x, off, m, wt, None, *conv, 0)
    pre = raw * scale[None, :, None, None] + shift[None, :, None, None]
    assert _rel(y, pre.relu()) <= TOL
    gx, gom, gw = ops.deform_conv_fused_backward_op(xs if xs.numel() else x, om, wt, scale, True, y, go, *conv, 1, cols)
    gpre = go * (y > 0) * scale[None, :, None, None]  # the ReLU's mask as the kernels read it: from the saved y
    rgx, roff, rm, rgw = ops.deform_conv_backward_op(x, off, m, wt, gpre, *conv, False, True, True, 0)[:4]
    _check([gx, gom, gw], [rgx, torch.cat((roff, rm * m * (1 - m)), 1), rgw], ["gx", "goffset_mask", "gw"])


def test_fused_backward_in_cuda_graph():
    # forward and the one-launch backward captured once and replayed on new inputs copied into the captured buffers: the
    # same results as eager calls on those inputs, and as the FFMA path
    from detectron2_b200 import ops

    c, k, h, w = 512, 3, 25, 42
    conv = _conv(k)

    def step(x, off, mask, wt, go):
        y, xs, cols = ops.deform_conv_train_op(x, off, mask, wt, None, *conv, 1)
        gx, goff, gm, gw, _ = ops.deform_conv_backward_op(xs if xs.numel() else x, off, mask, wt, go, *conv, False, True,
                                                          True, 1, cols)
        return y, gx, goff, gm, gw

    static = _inputs(c, k, h, w, True, 21)
    step(*static)  # warm-up: allocations, shared-memory opt-ins
    torch.cuda.synchronize()
    graph, side = torch.cuda.CUDAGraph(), torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        with torch.cuda.graph(graph, stream=side):
            outs = step(*static)
    torch.cuda.current_stream().wait_stream(side)
    names = ["y", "gx", "goff", "gmask", "gw"]
    for seed in (22, 23):
        new = _inputs(c, k, h, w, True, seed)
        for s, t in zip(static, new):
            s.copy_(t)
        graph.replay()
        torch.cuda.synchronize()
        eager = step(*new)
        for name, a, r in zip(names, outs, eager):
            assert _rel(a, r) <= 1e-5, (seed, name)
        x, off, mask, wt, go = new
        ref = [ops.deform_conv_op(x, off, mask, wt, None, *conv, 0)]
        ref += ops.deform_conv_backward_op(x, off, mask, wt, go, *conv, False, True, True, 0)[:4]
        _check(outs, ref, names)
