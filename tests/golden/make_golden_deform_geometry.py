"""Generate tests/golden/deform_conv_geometry.npz: deformable convolution at the kernel geometries that
tests/golden/deform_conv.npz (square 3x3 kernels, one stride / padding / dilation for both axes) does not reach --
dilated res5 convs, 5x5, 7x7, 1x1, 1x3 / 3x1 / 3x5 kernels, a different stride, padding or dilation per axis, and several
deformable groups.  Forward and every gradient come from torchvision.ops.deform_conv2d (the reference's backend,
detectron2/layers/deform_conv.py:9,55) under float64 autograd; inputs and outputs are stored as float32.

Run in the authoring container only (needs torchvision and the reference, like make_golden.py):
    python tests/golden/make_golden_deform_geometry.py
It writes only this file.  The offsets are Gaussian, never on the half-integer lattice: where a sample lands exactly on
row or column -1, torchvision returns a non-zero coordinate gradient while the reference's CUDA kernel
(get_coordinate_weight) and this project return 0, so the lattice is tested against the oracle instead.
"""
import os
import sys

import numpy as np
import torch
import torchvision

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (save())

CASES = [
    # n, cin, h, w, cout, kh, kw, sh, sw, ph, pw, dh, dw, groups, dg, modulated, bias (DCNv1 has no bias)
    (2, 8, 7, 9, 8, 3, 3, 1, 1, 2, 2, 2, 2, 1, 1, True, True),     # res5 conv2: padding = dilation = 2
    (1, 6, 9, 11, 8, 5, 5, 1, 1, 2, 2, 1, 1, 1, 1, False, False),  # 5x5
    (1, 4, 8, 9, 6, 7, 7, 1, 1, 3, 3, 1, 1, 1, 1, True, False),   # 7x7 (KK = 49)
    (2, 6, 9, 11, 4, 1, 1, 1, 1, 0, 0, 1, 1, 1, 1, True, True),     # 1x1
    (2, 4, 8, 10, 6, 1, 3, 1, 1, 0, 1, 1, 1, 1, 1, False, False),   # 1x3, padding (0, 1)
    (2, 4, 8, 10, 6, 3, 1, 1, 1, 1, 0, 1, 1, 1, 1, True, False),    # 3x1, padding (1, 0)
    (1, 6, 9, 13, 6, 3, 5, 1, 1, 1, 2, 1, 2, 1, 1, True, True),    # 3x5, padding (1, 2), dilation (1, 2)
    (2, 4, 13, 18, 4, 3, 3, 1, 2, 2, 1, 2, 1, 1, 1, False, False),  # stride (1, 2), dilation (2, 1)
    (2, 4, 18, 13, 4, 3, 3, 2, 1, 2, 1, 2, 1, 1, 1, True, False),   # stride (2, 1), dilation (2, 1)
    (2, 4, 11, 13, 6, 3, 3, 2, 2, 0, 0, 1, 1, 1, 1, False, False),  # stride 2, padding 0, odd map
    (1, 8, 7, 9, 8, 3, 5, 1, 1, 1, 2, 1, 1, 1, 4, True, False),    # 4 deformable groups, 3x5
    (1, 8, 9, 11, 8, 3, 3, 1, 1, 2, 2, 2, 2, 4, 2, True, False),   # 4 groups, 2 deformable groups, dilation 2
]


def gen():
    torch.set_num_threads(1)
    g = torch.Generator().manual_seed(2026)
    out = {"cases": np.asarray([[int(v) for v in c] for c in CASES])}
    for i, (n, cin, h, w, cout, kh, kw, sh, sw, ph, pw, dh, dw, grp, dg, mod, hb) in enumerate(CASES):
        ho = (h + 2 * ph - (dh * (kh - 1) + 1)) // sh + 1
        wo = (w + 2 * pw - (dw * (kw - 1) + 1)) // sw + 1
        x = torch.randn(n, cin, h, w, generator=g)
        off = torch.randn(n, 2 * dg * kh * kw, ho, wo, generator=g) * 1.5
        mask = torch.sigmoid(torch.randn(n, dg * kh * kw, ho, wo, generator=g)) if mod else None
        wt = torch.randn(cout, cin // grp, kh, kw, generator=g) * 0.2
        bias = torch.randn(cout, generator=g) if hb else None
        go = torch.randn(n, cout, ho, wo, generator=g)
        leaf = lambda t: None if t is None else t.double().requires_grad_(True)  # noqa: E731
        xd, od, md, wd, bd = leaf(x), leaf(off), leaf(mask), leaf(wt), leaf(bias)
        y = torchvision.ops.deform_conv2d(xd, od, wd, bd, stride=(sh, sw), padding=(ph, pw), dilation=(dh, dw), mask=md)
        y.backward(go.double())
        f = lambda t: t.detach().float()  # noqa: E731
        out.update({f"x{i}": x, f"off{i}": off, f"w{i}": wt, f"y{i}": f(y), f"go{i}": go,
                    f"gx{i}": f(xd.grad), f"goff{i}": f(od.grad), f"gw{i}": f(wd.grad)})
        if mod:
            out.update({f"mask{i}": mask, f"gmask{i}": f(md.grad)})
        if hb:
            out.update({f"bias{i}": bias, f"gbias{i}": f(bd.grad)})
    mg.save("deform_conv_geometry", **out)


if __name__ == "__main__":
    gen()
