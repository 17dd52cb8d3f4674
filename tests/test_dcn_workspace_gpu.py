"""Deformable conv on the tensor cores: every call fits in exactly the workspace its size query returns.  Each forward and
backward runs with a workspace of exactly the queried size (256-byte aligned, filled with NaN bytes) followed by a guard
region of known bytes; the guard must be untouched and the results must match a run with a generous zero-filled workspace.
Covered: NCHW and channels-last x, every need_data / need_weight pair, with and without saved columns, a shape whose
forward computes several output-channel tiles from the columns, and a 5x5 kernel (25 kernel points).
Run on an H100: pytest -m gpu."""
import ctypes as C

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
GUARD = 64 * 1024
PRECISION = 1
# (N, Cin, H, W, Cout, k, pad): 192 output channels are three 64-channel tiles, so a forward with saved columns runs the
# column-fed launch; k = 5 has more than 9 kernel points
SHAPES = {"3x3-3tiles": (2, 64, 10, 12, 192, 3, 1), "5x5": (2, 64, 9, 11, 64, 5, 2)}


def _lib():
    from detectron2_b200 import _C

    return _C


def _params(shape):
    n, cin, h, w, cout, k, pad = shape
    return _lib().DcnParams(n, cin, h, w, cout, k, k, 1, 1, pad, pad, 1, 1, 1, 1)


def _inputs(shape, x_nhwc):
    n, cin, h, w, cout, k, _ = shape
    g = torch.Generator().manual_seed(cin + cout + k)
    x = torch.randn(n, cin, h, w, generator=g)
    off = torch.randn(n, 2 * k * k, h, w, generator=g) * 2
    mask = torch.rand(n, k * k, h, w, generator=g)
    wt = torch.randn(cout, cin, k, k, generator=g) * (cin * k * k) ** -0.5
    go = torch.randn(n, cout, h, w, generator=g)
    x = x.to(DEV)
    if x_nhwc:
        x = x.contiguous(memory_format=torch.channels_last)
    return x, off.to(DEV), mask.to(DEV), wt.to(DEV), go.to(DEV)


def _pattern(nbytes):
    return (torch.arange(nbytes, dtype=torch.int64, device=DEV) * 37 % 251 + 1).to(torch.uint8)


def _workspace(nbytes, exact):
    """(workspace, guard): exact -> NaN bytes with a guard region of known bytes right behind them; else zeros, 4x oversized."""
    if not exact:
        return torch.zeros((4 * nbytes + GUARD,), dtype=torch.uint8, device=DEV), None
    buf = torch.empty((nbytes + GUARD,), dtype=torch.uint8, device=DEV)
    assert buf.data_ptr() % 256 == 0 and nbytes % 256 == 0
    buf[:nbytes].fill_(0xFF)
    buf[nbytes:] = _pattern(GUARD)
    return buf, buf[nbytes:]


def _ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def _forward(shape, x_nhwc, with_cols, exact):
    _C = _lib()
    lib, p = _C.lib(), _params(shape)
    x, off, mask, wt, _ = _inputs(shape, x_nhwc)
    flags = _C.DCN_X_NHWC if x_nhwc else 0
    n, _, h, w, cout, _, _ = shape
    out = torch.empty((n, cout, h, w), device=DEV)
    cols = None
    if with_cols:
        cols = torch.zeros((lib.d2b_deform_conv_cols_bytes(C.byref(p), PRECISION),), dtype=torch.uint8, device=DEV)
        assert cols.numel() > 0
    nbytes = lib.d2b_deform_conv_forward_workspace_bytes(C.byref(p), PRECISION, flags)
    ws, guard = _workspace(nbytes, exact)
    _C.check(lib.d2b_deform_conv_forward(_ptr(x), _ptr(off), _ptr(mask), _ptr(wt), None, C.byref(p), PRECISION, flags,
                                         _ptr(out), _ptr(cols), _ptr(ws), nbytes if exact else ws.numel(),
                                         _C.stream_ptr(x.device)),
             "deform_conv_forward")
    torch.cuda.synchronize()
    if guard is not None:
        assert torch.equal(guard, _pattern(GUARD)), "the forward wrote past its queried workspace"
    return out, cols


def _backward(shape, x_nhwc, need_data, need_weight, cols, exact):
    _C = _lib()
    lib, p = _C.lib(), _params(shape)
    x, off, mask, wt, go = _inputs(shape, x_nhwc)
    flags = _C.DCN_X_NHWC if x_nhwc else 0
    gx = torch.empty_like(x) if need_data else None  # channels-last when x is
    goff = torch.empty_like(off) if need_data else None
    gm = torch.empty_like(mask) if need_data else None
    gw = torch.empty_like(wt) if need_weight else None
    nbytes = lib.d2b_deform_conv_backward_workspace_bytes(C.byref(p), PRECISION, flags, need_data, need_weight)
    ws, guard = _workspace(nbytes, exact)
    _C.check(lib.d2b_deform_conv_backward(_ptr(x), _ptr(off), _ptr(mask), _ptr(wt), _ptr(go), C.byref(p), PRECISION, flags,
                                          _ptr(cols), _ptr(gx), _ptr(goff), _ptr(gm), _ptr(gw), None, _ptr(ws),
                                          nbytes if exact else ws.numel(), _C.stream_ptr(x.device)),
             "deform_conv_backward")
    torch.cuda.synchronize()
    if guard is not None:
        assert torch.equal(guard, _pattern(GUARD)), "the backward wrote past its queried workspace"
    return [t for t in (gx, goff, gm, gw) if t is not None]


def _same(a, b):
    # float atomics accumulate in a different order from run to run: equal up to the last bits of the largest element
    torch.testing.assert_close(a, b, rtol=1e-5, atol=1e-5 * b.abs().max().item())


@pytest.mark.parametrize("shape", SHAPES.values(), ids=SHAPES.keys())
@pytest.mark.parametrize("x_nhwc", [0, 1], ids=["nchw", "nhwc"])
@pytest.mark.parametrize("with_cols", [False, True], ids=["gather", "cols"])
def test_forward_fits_queried_workspace(shape, x_nhwc, with_cols):
    out, cols = _forward(shape, x_nhwc, with_cols, exact=True)
    ref, ref_cols = _forward(shape, x_nhwc, with_cols, exact=False)
    _same(out, ref)
    if with_cols:
        assert torch.equal(cols, ref_cols)


@pytest.mark.parametrize("shape", SHAPES.values(), ids=SHAPES.keys())
@pytest.mark.parametrize("x_nhwc", [0, 1], ids=["nchw", "nhwc"])
@pytest.mark.parametrize("need_data,need_weight", [(0, 0), (1, 0), (0, 1), (1, 1)], ids=["none", "data", "weight", "both"])
@pytest.mark.parametrize("with_cols", [False, True], ids=["gather", "cols"])
def test_backward_fits_queried_workspace(shape, x_nhwc, need_data, need_weight, with_cols):
    cols = _forward(shape, x_nhwc, True, exact=False)[1] if with_cols else None
    grads = _backward(shape, x_nhwc, need_data, need_weight, cols, exact=True)
    refs = _backward(shape, x_nhwc, need_data, need_weight, cols, exact=False)
    assert len(grads) == len(refs) == 3 * need_data + need_weight
    for g, r in zip(grads, refs):
        _same(g, r)
