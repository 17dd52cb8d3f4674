"""The `detectron2._C`-shaped deform-conv shim (detectron2_b200/_C.py, SURVEY.md 8b "pybind functions").

CPU part: the call protocol of the REAL, unmodified reference autograd Functions `_DeformConv` / `_ModulatedDeformConv`
(detectron2/layers/deform_conv.py:29-184, :205-313) against our signatures.  tests/golden/make_golden.py ran those Functions
with a stand-in `detectron2._C` and recorded every call they make into it (tests/golden/shim_protocol.npz): function, the
positional arguments (scalars as values, tensors as the input they are or as a caller-allocated buffer with its shape and
whether the caller zero-filled it) and which buffers the Functions returned as the output and the gradients.  The test
replays that sequence on stand-ins with EXACTLY the parameter lists of the product's shim functions, backed by the CPU oracle
(torchvision deform_conv2d + autograd), and compares the returned buffers with the reference Functions' recorded results:
argument order (width-first for DCNv1), caller-allocated outputs written in place, gradients accumulated into
zero-initialised buffers.  GPU part: the same protocol, restated call by call, against the real kernels.
"""
import inspect
import json
import math
import os

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SHIM_FUNCTIONS = ("deform_conv_forward", "deform_conv_backward_input", "deform_conv_backward_filter",
                  "modulated_deform_conv_forward", "modulated_deform_conv_backward")


def _plain(t):
    return None if t is None else t.detach().as_subclass(torch.Tensor)


def tv_all(x, off, mask, w, bias, stride, pad, dil, go=None):
    """torchvision deform_conv2d (+ autograd when `go` is given): y, or the gradients of (x, off, mask, w, bias)."""
    import torchvision

    with torch.enable_grad():  # the reference's backward runs under once_differentiable (grad mode off)
        xs = [_plain(t).clone().requires_grad_(True) if t is not None else None for t in (x, off, mask, w, bias)]
        y = torchvision.ops.deform_conv2d(xs[0], xs[1], xs[3], xs[4], stride, pad, dil, xs[2])
        if go is None:
            return y.detach()
        y.backward(_plain(go))
        return [None if t is None else t.grad for t in xs]


def oracle_shim(weight):
    """Stand-ins for the five deform-conv entry points with OUR parameter lists, bodies = the CPU oracle.  `weight` is the
    DCNv1 weight (deform_conv_backward_filter receives only the gradient buffer).  Returns (functions, call log)."""
    from detectron2_b200 import _C as real_shim

    calls = []

    def deform_conv_forward(input, weight, offset, output, columns, ones, kW, kH, dW, dH, padW, padH, dilW, dilH, group,
                            deformable_group, im2col_step):
        calls.append("deform_conv_forward")
        assert (kW, kH) == (weight.shape[3], weight.shape[2]) and group == 1 and deformable_group == 1
        output.copy_(tv_all(input, offset, None, weight, None, (dH, dW), (padH, padW), (dilH, dilW)))
        return 1

    def deform_conv_backward_input(input, offset, gradOutput, gradInput, gradOffset, weight, columns, kW, kH, dW, dH, padW,
                                   padH, dilW, dilH, group, deformable_group, im2col_step):
        calls.append("deform_conv_backward_input")
        assert float(gradInput.abs().sum()) == 0.0 and float(gradOffset.abs().sum()) == 0.0  # zero-initialised by the caller
        g = tv_all(input, offset, None, weight, None, (dH, dW), (padH, padW), (dilH, dilW), gradOutput)
        gradInput.copy_(g[0])
        gradOffset.copy_(g[1])
        return 1

    def deform_conv_backward_filter(input, offset, gradOutput, gradWeight, columns, ones, kW, kH, dW, dH, padW, padH, dilW,
                                    dilH, group, deformable_group, scale, im2col_step):
        calls.append("deform_conv_backward_filter")
        g = tv_all(input, offset, None, _plain(weight), None, (dH, dW), (padH, padW), (dilH, dilW), gradOutput)
        gradWeight.add_(g[3], alpha=scale)
        return 1

    def modulated_deform_conv_forward(input, weight, bias, ones, offset, mask, output, columns, kernel_h, kernel_w, stride_h,
                                      stride_w, pad_h, pad_w, dilation_h, dilation_w, group, deformable_group, with_bias):
        calls.append("modulated_deform_conv_forward")
        output.copy_(tv_all(input, offset, mask, weight, bias if with_bias else None, (stride_h, stride_w), (pad_h, pad_w),
                            (dilation_h, dilation_w)))

    def modulated_deform_conv_backward(input, weight, bias, ones, offset, mask, columns, grad_input, grad_weight, grad_bias,
                                       grad_offset, grad_mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                                       pad_w, dilation_h, dilation_w, group, deformable_group, with_bias):
        calls.append("modulated_deform_conv_backward")
        g = tv_all(input, offset, mask, weight, bias if with_bias else None, (stride_h, stride_w), (pad_h, pad_w),
                   (dilation_h, dilation_w), grad_output)
        grad_input.copy_(g[0])
        grad_offset.copy_(g[1])
        grad_mask.copy_(g[2])
        grad_weight.add_(g[3])
        if with_bias:
            grad_bias.add_(g[4])

    fns = {f.__name__: f for f in (deform_conv_forward, deform_conv_backward_input, deform_conv_backward_filter,
                                   modulated_deform_conv_forward, modulated_deform_conv_backward)}
    for name in SHIM_FUNCTIONS:
        # the oracle-backed stand-in has EXACTLY the parameter list of the product's shim function
        assert list(inspect.signature(fns[name]).parameters) == list(inspect.signature(getattr(real_shim, name)).parameters), name
    return fns, calls


def test_reference_functions_drive_the_shim_signatures(golden):
    d = golden("shim_protocol")
    t = {k: torch.from_numpy(d[k]) for k in ("x", "offset", "mask", "weight", "bias", "grad_output")}
    protocol = json.loads(str(d["protocol"]))
    fns, calls = oracle_shim(t["weight"])
    for phase in protocol:  # DCNv1 through _DeformConv, then DCNv2 through _ModulatedDeformConv
        bufs = {}

        def arg(a):
            if "scalar" in a:
                return a["scalar"]
            if "input" in a:
                return t[a["input"]].clone()
            if a["buffer"] not in bufs:  # first use: the shape the caller allocated, zero-filled only where it zero-filled
                fill = 0.0 if a["zeroed"] else float("nan")
                bufs[a["buffer"]] = torch.full(a["shape"], fill, dtype=torch.float32)
            return bufs[a["buffer"]]

        for call in phase["calls"]:
            fns[call["fn"]](*[arg(a) for a in call["args"]])
        for name, buf in phase["results"].items():
            ref = torch.from_numpy(d["%s_%s" % (phase["name"], name)])
            assert torch.allclose(bufs[buf], ref, atol=1e-5), (phase["name"], name)
    assert calls == list(SHIM_FUNCTIONS)


def test_shim_exports_the_reference_pybind_names():
    # csrc/vision.cpp:86-102
    from detectron2_b200 import _C

    for name in ["get_compiler_version", "get_cuda_version", "has_cuda", "deform_conv_forward", "deform_conv_backward_input",
                 "deform_conv_backward_filter", "modulated_deform_conv_forward", "modulated_deform_conv_backward"]:
        assert callable(getattr(_C, name)), name
    assert len(inspect.signature(_C.deform_conv_forward).parameters) == 17
    assert len(inspect.signature(_C.deform_conv_backward_input).parameters) == 18
    assert len(inspect.signature(_C.deform_conv_backward_filter).parameters) == 18
    assert len(inspect.signature(_C.modulated_deform_conv_forward).parameters) == 19
    assert len(inspect.signature(_C.modulated_deform_conv_backward).parameters) == 24


@pytest.mark.gpu
@pytest.mark.parametrize("c,co,grp", [(8, 12, 1), (128, 128, 1), (64, 64, 4)])
def test_shim_protocol_on_gpu_vs_oracle(c, co, grp):
    """The call sequence of detectron2/layers/deform_conv.py:43-141 (DCNv1) and :205-295 (DCNv2), restated, on the real
    kernels: caller-allocated outputs, zero-initialised gradient buffers, width-first kernel arguments."""
    from detectron2_b200 import _C
    from oracle import oracle as orc

    dev = "cuda"
    g = torch.Generator().manual_seed(c)
    n, h, w = 2, 13, 17
    x = torch.randn(n, c, h, w, generator=g)
    off = torch.randn(n, 18, h, w, generator=g) * 1.5
    mask = torch.sigmoid(torch.randn(n, 9, h, w, generator=g))
    wt = torch.randn(co, c // grp, 3, 3, generator=g) * (1 / math.sqrt(c // grp * 9))
    bias = torch.randn(co, generator=g)
    go = torch.randn(n, co, h, w, generator=g)
    xd, od, md, wd, bd, gd = [t.to(dev) for t in (x, off, mask, wt, bias, go)]
    bufs = [xd.new_empty(0), xd.new_empty(0)]

    def close(a, b, name):
        scale = b.abs().max().item() + 1e-6
        assert (a.cpu() - b).abs().max().item() <= 1e-4 * scale + 1e-5, name

    # ---- DCNv1: forward (deform_conv.py:43-79), backward (:83-141)
    out = xd.new_empty(n, co, h, w)
    _C.deform_conv_forward(xd, wd, od, out, bufs[0], bufs[1], wd.size(3), wd.size(2), 1, 1, 1, 1, 1, 1, grp, 1, 2)
    close(out, orc.deform_conv_forward(x, off, None, wt, None, 1, 1, 1, grp, 1), "y")
    gi, goff, gw = torch.zeros_like(xd), torch.zeros_like(od), torch.zeros_like(wd)
    _C.deform_conv_backward_input(xd, od, gd, gi, goff, wd, bufs[0], wd.size(3), wd.size(2), 1, 1, 1, 1, 1, 1, grp, 1, 2)
    _C.deform_conv_backward_filter(xd, od, gd, gw, bufs[0], bufs[1], wd.size(3), wd.size(2), 1, 1, 1, 1, 1, 1, grp, 1, 1, 2)
    r = orc.deform_conv_backward(x, off, None, wt, go, 1, 1, 1, grp, 1, False)
    close(gi, r[0], "gx"), close(goff, r[1], "goff"), close(gw, r[3], "gw")
    # ---- DCNv2: forward (:205-242), backward (:244-295)
    out = xd.new_empty(n, co, h, w)
    _C.modulated_deform_conv_forward(xd, wd, bd, bufs[0], od, md, out, bufs[1], 3, 3, 1, 1, 1, 1, 1, 1, grp, 1, True)
    close(out, orc.deform_conv_forward(x, off, mask, wt, bias, 1, 1, 1, grp, 1), "y2")
    gi, goff, gm = torch.zeros_like(xd), torch.zeros_like(od), torch.zeros_like(md)
    gw, gb = torch.zeros_like(wd), torch.zeros_like(bd)
    _C.modulated_deform_conv_backward(xd, wd, bd, bufs[0], od, md, bufs[1], gi, gw, gb, goff, gm, gd, 3, 3, 1, 1, 1, 1, 1, 1,
                                      grp, 1, True)
    r = orc.deform_conv_backward(x, off, mask, wt, go, 1, 1, 1, grp, 1, True)
    for a, b, nm in zip((gi, goff, gm, gw, gb), r, ("gx", "goff", "gmask", "gw", "gb")):
        close(a, b, nm)
