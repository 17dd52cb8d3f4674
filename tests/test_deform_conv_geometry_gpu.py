"""Deformable convolution on the tensor-core kernels (deform_conv_tc.cu) at kernel geometries other than a square 3x3 with
padding 1 and dilation 1: the per-axis stride / padding / dilation, the kernel-point -> (row, column) split, the weight
layouts [Cout][Cin/G][kh*kw], the plans and shared-memory budgets that depend on KK = kh * kw, and the unit counts that leave
a macro chunk half empty.  Every case is compared with the CPU oracle (oracle/d2_oracle.c, pinned to torchvision float64 at
these geometries by tests/golden/deform_conv_geometry.npz).  Run on an H100: pytest -m gpu.

Kernels: K1 = gathering forward (dcn_fwd_tc_kernel), K1c = column-fed forward of output-channel tiles 1.. (dcn_fwd_cols_kernel,
training op with more than one 128-wide tile), K2 = backward data, K3 = backward weight re-sampling x, K3c = backward weight
streaming the saved columns; "reduce" = dcn_gw_reduce_tile_kernel for KK <= 9, dcn_gw_reduce_kernel for KK > 9.  Flags are
d2b_deform_conv_tc_shape_supported(forward, backward), asserted on an H100 SXM (132 SMs): for KK > 9 they depend on how the
grid is split, so on the map size and the SM count.

case               flags  reaches
res5_d2_7x9        1 1    K1 split over all 9 kernel points; K1 + K1c (4 tiles); K2; K3 / K3c BN 128; reduce KK <= 9; bf16
res5_d2_13x17      1 1    K1 split over kernel points at 2 pixel tiles; K1 + K1c; K2; K3 / K3c BN 128; reduce KK <= 9
5x5_64             1 1    K1 BN 64; K2 with split macro chunks; K3 / K3c BN 64; reduce KK > 9; bf16
5x5_128            1 1    K1 BN 128; K2 split; K3 / K3c BN 128; reduce KK > 9
7x7_64_16x20       1 1    KK = 49: K1 BN 64 split over kernel points; K2 split; K3 / K3c BN 64; reduce KK > 9
7x7_64to128_16x20  1 1    KK = 49: K1 BN 128 (fits only split over kernel points); K3 / K3c BN 128; reduce KK > 9
7x7_64_42x55       1 0    K1 on the tensor cores; the backward tap table fits only at a deeper split than the grid takes:
                          "auto" runs the FFMA backward, precision 1 raises
1x1_64             1 1    U = 1: one macro chunk with one of its two units filled
1x1_192to128       1 1    U = 3: odd unit count, last macro chunk half filled
1x3_p01, 3x1_p10   1 1    kernel point -> (row, column) with kh != kw; weight layout
3x5_p12_d12        1 1    the same with per-axis padding and dilation; KK = 15 (reduce KK > 9)
s12_d21, s21_d21   1 1    per-axis stride and dilation; one ragged 128-pixel tile
s2_p0_odd          1 1    stride 2, padding 0, odd map: ragged last 128-pixel tile
dg4_3x5            1 1    4 deformable groups of 64 channels: 4 tap tables per CTA; K1 + K1c (2 tiles)
g8_dg2_d2          1 1    super-groups of 2 x 32 channels with 2 deformable groups, dilation 2
lattice_3x3/3x5    1 1    offsets on the half-integer lattice: samples exactly on rows / columns -1, 0, H-1, H and on pixel
                          centres; the strict -1 < h < H rule and no gradient from a sample on -1, in K1 / K2 and FFMA

The 512-channel cases are compared with the oracle on image 0 only (its backward is a scalar loop) and on both images with the
FFMA kernels.
"""
import ctypes as C
import functools
import math
from collections import namedtuple

import pytest
import torch

from oracle import oracle as orc

pytestmark = pytest.mark.gpu
DEV = "cuda"

Case = namedtuple("Case", "name cin cout h w k s p d grp dg mod flags bf16 img0 lattice")


def _c(name, cin, cout, h, w, k, s=(1, 1), p=(0, 0), d=(1, 1), grp=1, dg=1, mod=False, flags=(1, 1), bf16=False, img0=False,
       lattice=False):
    return Case(name, cin, cout, h, w, k, s, p, d, grp, dg, mod, flags, bf16, img0, lattice)


CASES = [
    _c("res5_d2_7x9", 512, 512, 7, 9, (3, 3), p=(2, 2), d=(2, 2), mod=True, bf16=True, img0=True),
    _c("res5_d2_13x17", 512, 512, 13, 17, (3, 3), p=(2, 2), d=(2, 2), mod=True, img0=True),
    _c("5x5_64", 64, 64, 12, 14, (5, 5), p=(2, 2), bf16=True),
    _c("5x5_128", 128, 128, 12, 14, (5, 5), p=(2, 2), mod=True),
    _c("7x7_64_16x20", 64, 64, 16, 20, (7, 7), p=(3, 3), mod=True),
    _c("7x7_64to128_16x20", 64, 128, 16, 20, (7, 7), p=(3, 3)),
    _c("7x7_64_42x55", 64, 64, 42, 55, (7, 7), p=(3, 3), mod=True, flags=(1, 0)),
    _c("1x1_64", 64, 64, 11, 13, (1, 1), mod=True),
    _c("1x1_192to128", 192, 128, 11, 13, (1, 1)),
    _c("1x3_p01", 64, 64, 10, 12, (1, 3), p=(0, 1)),
    _c("3x1_p10", 64, 64, 10, 12, (3, 1), p=(1, 0), mod=True),
    _c("3x5_p12_d12", 64, 128, 11, 15, (3, 5), p=(1, 2), d=(1, 2), mod=True),
    _c("s12_d21", 64, 64, 13, 18, (3, 3), s=(1, 2), p=(2, 1), d=(2, 1)),
    _c("s21_d21", 64, 64, 18, 13, (3, 3), s=(2, 1), p=(2, 1), d=(2, 1), mod=True),
    _c("s2_p0_odd", 128, 128, 27, 31, (3, 3), s=(2, 2)),
    _c("dg4_3x5", 256, 256, 9, 11, (3, 5), p=(1, 2), dg=4, mod=True),
    _c("g8_dg2_d2", 256, 256, 11, 13, (3, 3), p=(2, 2), d=(2, 2), grp=8, dg=2, mod=True),
    _c("lattice_3x3", 64, 64, 10, 12, (3, 3), p=(1, 1), mod=True, lattice=True),
    _c("lattice_3x5", 64, 64, 9, 11, (3, 5), p=(1, 2), lattice=True),
]
BY_NAME = {c.name: c for c in CASES}
ids = [c.name for c in CASES]


def _out_hw(c):
    return tuple((i + 2 * p - (d * (k - 1) + 1)) // s + 1 for i, p, d, k, s in zip((c.h, c.w), c.p, c.d, c.k, c.s))


def _geom(c):
    return list(c.s), list(c.p), list(c.d), c.grp, c.dg


@functools.lru_cache(maxsize=None)
def _inputs(name):
    c = BY_NAME[name]
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    n, (kh, kw), (ho, wo) = 2, c.k, _out_hw(c)
    kk = kh * kw
    x = torch.randn(n, c.cin, c.h, c.w, generator=g)
    if c.lattice:  # multiples of 1/2 in [-3, 3]: sample rows / columns land on -1, 0, H-1, H exactly
        off = torch.randint(-6, 7, (n, 2 * c.dg * kk, ho, wo), generator=g).float() / 2
    else:
        off = torch.randn(n, 2 * c.dg * kk, ho, wo, generator=g) * 2
    mask = torch.sigmoid(torch.randn(n, c.dg * kk, ho, wo, generator=g)) if c.mod else None
    wt = torch.randn(c.cout, c.cin // c.grp, kh, kw, generator=g) * (1.0 / math.sqrt(c.cin // c.grp * kk))
    bias = torch.randn(c.cout, generator=g) if c.mod else None
    go = torch.randn(n, c.cout, ho, wo, generator=g)
    return x, off, mask, wt, bias, go


def _nref(c):
    return 1 if c.img0 else 2


def _go_ref(c):
    """grad_out whose images past those the oracle sees are zero: the weight / bias gradients of the GPU run then equal the
    oracle's."""
    go = _inputs(c.name)[5].clone()
    go[_nref(c):] = 0
    return go


@functools.lru_cache(maxsize=None)
def _oracle(name):
    c = BY_NAME[name]
    x, off, mask, wt, bias, _ = _inputs(name)
    r = slice(0, _nref(c))
    s, p, d = c.s, c.p, c.d
    sm = None if mask is None else mask[r]
    y = orc.deform_conv_forward(x[r], off[r], sm, wt, bias, s, p, d, c.grp, c.dg)
    gr = orc.deform_conv_backward(x[r], off[r], sm, wt, _go_ref(c)[r], s, p, d, c.grp, c.dg, bias is not None)
    return y, gr


def _dev(t):
    return None if t is None else t.to(DEV)


def _close(got, ref, tol, what):
    got = got.detach().float().cpu()
    scale = ref.abs().max().item() + 1e-6
    err = (got - ref).abs().max().item()
    assert err <= tol * scale + 1e-5, (what, err, scale)


def _flags(c):
    from detectron2_b200 import _C

    prm = _C.DcnParams(2, c.cin, c.h, c.w, c.cout, c.k[0], c.k[1], c.s[0], c.s[1], c.p[0], c.p[1], c.d[0], c.d[1], c.grp,
                       c.dg)
    return tuple(_C.lib().d2b_deform_conv_tc_shape_supported(C.byref(prm), b) for b in (0, 1)), prm


def _check_grads(c, gs, ref, tol, what):
    n = _nref(c)
    for name, a, r in zip(["gx", "goff", "gmask", "gw", "gb"], gs, ref):
        if r is None:
            continue
        assert a.numel(), (what, name)
        _close(a[:n] if name in ("gx", "goff", "gmask") else a, r, tol, (what, name))


@pytest.mark.parametrize("name", ids)
def test_forward_vs_oracle(name):
    from detectron2_b200 import ops

    c = BY_NAME[name]
    flags, _ = _flags(c)
    assert flags == c.flags
    x, off, mask, wt, bias, _ = [_dev(t) for t in _inputs(name)]
    ref, _ = _oracle(name)
    n = _nref(c)
    run = lambda prec: ops.deform_conv_op(x, off, mask, wt, bias, *_geom(c), prec)  # noqa: E731
    y0 = run(0)
    _close(y0[:n], ref, 1e-4, "ffma")
    y1 = run(1)
    _close(y1[:n], ref, 1e-4, "bf16x3")
    _close(y1, y0.cpu(), 1e-4, "bf16x3 vs ffma, both images")
    assert torch.allclose(run(-1), y1, rtol=1e-5, atol=1e-5 * ref.abs().max().item())
    if c.bf16:
        _close(run(2)[:n], ref, 2e-2, "bf16")


@pytest.mark.parametrize("name", ids)
def test_backward_vs_oracle(name):
    from detectron2_b200 import ops

    c = BY_NAME[name]
    flags, _ = _flags(c)
    assert flags == c.flags
    x, off, mask, wt, bias, go = [_dev(t) for t in _inputs(name)]
    _, ref = _oracle(name)
    gor = _dev(_go_ref(c))
    run = lambda xx, g, prec: ops.deform_conv_backward_op(xx, off, mask, wt, g, *_geom(c), bias is not None,  # noqa: E731
                                                        True, True, prec)
    _check_grads(c, run(x, gor, 0), ref, 1e-4, "ffma")
    if not flags[1]:
        _check_grads(c, run(x, gor, -1), ref, 1e-4, "auto")
        with pytest.raises(RuntimeError):
            run(x, gor, 1)
        return
    for cl in (False, True):
        xd = x.contiguous(memory_format=torch.channels_last) if cl else x
        gs = run(xd, gor, 1)
        _check_grads(c, gs, ref, 1e-4, ("bf16x3", "channels_last" if cl else "nchw"))
        if cl:
            assert gs[0].is_contiguous(memory_format=torch.channels_last)
    if c.img0:  # both images: the tensor-core gradients against the FFMA ones
        for name_, a, r in zip(["gx", "goff", "gmask", "gw", "gb"], run(x, go, 1), run(x, go, 0)):
            if r.numel():
                _close(a, r.cpu(), 1e-4, ("bf16x3 vs ffma", name_))


@pytest.mark.parametrize("name", ids)
def test_training_op_saved_columns(name):
    # forward that keeps a channels-last copy of x and its sampled columns (K1, plus K1c for the other output-channel tiles),
    # then the backward whose weight gradient streams those columns (K3c)
    from detectron2_b200 import _C, ops

    c = BY_NAME[name]
    flags, prm = _flags(c)
    assert flags == c.flags
    x, off, mask, wt, bias, _ = [_dev(t) for t in _inputs(name)]
    yref, ref = _oracle(name)
    gor = _dev(_go_ref(c))
    n = _nref(c)
    prec = 1 if all(flags) else -1
    y, xs, cols = ops.deform_conv_train_op(x, off, mask, wt, bias, *_geom(c), prec)
    _close(y[:n], yref, 1e-4, "train forward")
    assert cols.numel() == (_C.lib().d2b_deform_conv_cols_bytes(C.byref(prm), 1) if all(flags) else 0)
    if all(flags):
        assert cols.numel() > 0 and xs.is_contiguous(memory_format=torch.channels_last)
    xk = xs if xs.numel() else x
    gs = ops.deform_conv_backward_op(xk, off, mask, wt, gor, *_geom(c), bias is not None, True, True, prec,
                                     cols if cols.numel() else None)
    _check_grads(c, gs, ref, 1e-4, "saved columns")


@pytest.mark.parametrize("h,w", [(7, 9), (13, 17)])
def test_res5_dilated_bottleneck_conv2_fused_vs_unfused(h, w):
    # the reference's res5 with RES5_DILATION = 2: DeformBottleneckBlock conv2 with padding = dilation = 2, stride 1
    import detectron2_b200.layers as L
    from detectron2_b200 import ops

    c = 512
    g = torch.Generator().manual_seed(h * w)
    x = torch.randn(2, c, h, w, generator=g)
    om = torch.randn(2, 27, h, w, generator=g) * 1.5
    wt = torch.randn(c, c, 3, 3, generator=g) * (1.0 / math.sqrt(c * 9))
    scale, shift = 0.5 + torch.rand(c, generator=g), torch.randn(c, generator=g) * 0.3
    go = torch.randn(2, c, h, w, generator=g)
    geom = ([1, 1], [2, 2], [2, 2], 1, 1)
    xu, omu, wu = [t.to(DEV).requires_grad_(True) for t in (x, om, wt)]
    a, b, m = torch.chunk(omu, 3, dim=1)
    yu = ops.deform_conv_op(xu, torch.cat((a, b), 1), m.sigmoid(), wu, None, *geom, 1)
    yu = (yu * _dev(scale)[None, :, None, None] + _dev(shift)[None, :, None, None]).relu()
    yu.backward(go.to(DEV))
    y = ops.deform_conv_fused_op(x.to(DEV), om.to(DEV), wt.to(DEV), _dev(scale), _dev(shift), True, *geom, 1)
    _close(y, yu.detach().cpu(), 1e-5, "fused forward")
    mod = L.DeformBottleneckConv2(c, c, 3, stride=1, padding=2, dilation=2).to(DEV)
    with torch.no_grad():
        mod.weight.copy_(wt)
        mod.norm_scale.copy_(scale)
        mod.norm_shift.copy_(shift)
    xm, omm = x.to(DEV).requires_grad_(True), om.to(DEV).requires_grad_(True)
    ym = mod(xm, omm)  # under autograd: the training op (K1 + K1c with saved columns), backward K2 + K3c
    _close(ym, yu.detach().cpu(), 1e-5, "module forward")
    ym.backward(go.to(DEV))
    for name, t, r in (("gx", xm.grad, xu.grad), ("gom", omm.grad, omu.grad), ("gw", mod.weight.grad, wu.grad)):
        _close(t, r.cpu(), 2e-4, ("module", name))


@pytest.mark.parametrize("name", ["lattice_3x3", "lattice_3x5"])
def test_lattice_samples_on_the_border(name):
    # a sample exactly on row / column -1 or on H / W is outside: no value and no gradient of any kind, in both kernels
    from detectron2_b200 import ops

    c = BY_NAME[name]
    x, off, mask, wt, bias, go = _inputs(name)
    kh, kw = c.k
    ho, wo = _out_hw(c)
    oy, ox = off.view(2, c.dg, kh * kw, 2, ho, wo).unbind(3)
    kp = torch.arange(kh * kw).view(1, 1, -1, 1, 1)
    hs = torch.arange(ho).view(1, 1, 1, -1, 1) * c.s[0] - c.p[0] + (kp // kw) * c.d[0] + oy
    ws = torch.arange(wo).view(1, 1, 1, 1, -1) * c.s[1] - c.p[1] + (kp % kw) * c.d[1] + ox
    on_edge = (hs == -1) | (ws == -1) | (hs == c.h) | (ws == c.w)
    inside = (hs > -1) & (ws > -1) & (hs < c.h) & (ws < c.w)
    assert (hs == -1).any() and (hs == c.h).any() and (ws == -1).any() and (ws == c.w).any()
    assert ((hs == 0) | (hs == c.h - 1)).any() and (inside & (hs.frac() == 0) & (ws.frac() == 0)).any()
    _, ref = _oracle(name)
    edge_off = on_edge.unsqueeze(3).expand(-1, -1, -1, 2, -1, -1).reshape(off.shape)
    assert (ref[1][edge_off] == 0).all()
    for prec in (0, 1):
        gs = ops.deform_conv_backward_op(_dev(x), _dev(off), _dev(mask), _dev(wt), _dev(go), *_geom(c), bias is not None,
                                         True, True, prec)
        assert (gs[1].cpu()[edge_off] == 0).all(), prec
        if mask is not None:
            assert (gs[2].cpu()[on_edge.reshape(mask.shape)] == 0).all(), prec


def test_reference_shim_width_first_arguments():
    # detectron2._C takes DCNv1 arguments width first (kW, kH, dW, dH, padW, padH, dilW, dilH) and DCNv2 arguments height
    # first; every entry point with a different kernel size, stride, padding and dilation per axis
    from detectron2_b200 import _C

    g = torch.Generator().manual_seed(7)
    n, cin, cout, h, w = 2, 64, 64, 13, 17
    kh, kw, sh, sw, ph, pw, dh, dw = 3, 5, 1, 2, 1, 3, 2, 1
    ho, wo = (h + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1, (w + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
    x = torch.randn(n, cin, h, w, generator=g)
    off = torch.randn(n, 2 * kh * kw, ho, wo, generator=g) * 1.5
    mask = torch.sigmoid(torch.randn(n, kh * kw, ho, wo, generator=g))
    wt = torch.randn(cout, cin, kh, kw, generator=g) * (1 / math.sqrt(cin * kh * kw))
    bias = torch.randn(cout, generator=g)
    go = torch.randn(n, cout, ho, wo, generator=g)
    xd, od, md, wd, bd, gd = [t.to(DEV) for t in (x, off, mask, wt, bias, go)]
    bufs = [xd.new_empty(0), xd.new_empty(0)]
    geo = ((sh, sw), (ph, pw), (dh, dw), 1, 1)
    v1 = (kw, kh, sw, sh, pw, ph, dw, dh, 1, 1)
    out = xd.new_empty(n, cout, ho, wo)
    _C.deform_conv_forward(xd, wd, od, out, bufs[0], bufs[1], *v1, 64)
    _close(out, orc.deform_conv_forward(x, off, None, wt, None, *geo), 1e-4, "v1 y")
    gi, goff, gw = torch.zeros_like(xd), torch.zeros_like(od), torch.zeros_like(wd)
    _C.deform_conv_backward_input(xd, od, gd, gi, goff, wd, bufs[0], *v1, 64)
    _C.deform_conv_backward_filter(xd, od, gd, gw, bufs[0], bufs[1], *v1, 1.0, 64)
    r = orc.deform_conv_backward(x, off, None, wt, go, *geo, False)
    _close(gi, r[0], 1e-4, "v1 gx")
    _close(goff, r[1], 1e-4, "v1 goff")
    _close(gw, r[3], 1e-4, "v1 gw")
    v2 = (kh, kw, sh, sw, ph, pw, dh, dw, 1, 1)
    out = xd.new_empty(n, cout, ho, wo)
    _C.modulated_deform_conv_forward(xd, wd, bd, bufs[0], od, md, out, bufs[1], *v2, True)
    _close(out, orc.deform_conv_forward(x, off, mask, wt, bias, *geo), 1e-4, "v2 y")
    gi, goff, gm = torch.zeros_like(xd), torch.zeros_like(od), torch.zeros_like(md)
    gw, gb = torch.zeros_like(wd), torch.zeros_like(bd)
    _C.modulated_deform_conv_backward(xd, wd, bd, bufs[0], od, md, bufs[1], gi, gw, gb, goff, gm, gd, *v2, True)
    r = orc.deform_conv_backward(x, off, mask, wt, go, *geo, True)
    for a, b, nm in zip((gi, goff, gm, gw, gb), r, ("gx", "goff", "gmask", "gw", "gb")):
        _close(a, b, 1e-4, ("v2", nm))
