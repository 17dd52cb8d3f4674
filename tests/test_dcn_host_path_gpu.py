"""The host layer of the deformable-conv ops (detectron2_b200/ops.py) pinned by the native calls it makes.  The library
handle is wrapped in a pass-through proxy that records every call that enqueues work on a stream (forward, backward and
layout-change entry points; the host-only shape and size queries are not recorded), and each case of a matrix -- the six
ops through the entry points the layers use, NCHW and channels-last x, fp32 and bf16 x, every precision an op accepts, a
shape the tensor-core kernels take (64 channels) and one they do not (48) -- is compared with its expected trace.
Run on an H100: pytest -m gpu."""
import contextlib

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
GEO = ([1, 1], [1, 1], [1, 1], 1, 1)  # stride, padding, dilation, groups, deformable_groups
# d2b_dcn_params of the two shapes: N, Cin, H, W, Cout, kh, kw, stride, padding, dilation (h, w each), groups, dg
PARAMS = {(2, c, 10, 12, c, 3, 3, 1, 1, 1, 1, 1, 1, 1, 1): "P%d" % c for c in (64, 48)}
_SHORT = {"d2b_deform_conv_forward": "fwd", "d2b_deform_conv_backward": "bwd", "d2b_deform_conv_fused_forward": "ffwd",
          "d2b_deform_conv_fused_backward": "fbwd", "d2b_pyramid_nchw_to_nhwc": "to_nhwc"}


def _describe(name, args):
    """One recorded call: its name, the d2b_dcn_params (or the map size of a layout change), the integer arguments in order
    (fused: relu; then precision, flags, workspace bytes; layout change: n, c, dtype code), and one character per pointer
    argument: x = set, . = NULL.  The last argument, the stream, is left out."""
    words, ptrs = [_SHORT.get(name, name)], ""
    for a in args[:-1]:
        obj = getattr(a, "_obj", None)  # C.byref(struct)
        if obj is not None and type(obj).__name__ == "DcnParams":
            key = tuple(getattr(obj, f) for f, _ in obj._fields_)
            words.append(PARAMS.get(key, str(key)))
        elif obj is not None and type(obj).__name__ == "Pyramid":
            words.append("%dx%d" % (obj.H[0], obj.W[0]))
        elif isinstance(a, int):
            words.append(str(a))
        else:  # None, c_void_p, or the array of destination pointers of the layout change
            ptrs += "." if a is None or getattr(a, "value", 1) is None else "x"
    return " ".join(words + [ptrs])


class _Recorder:
    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if name.endswith(("_bytes", "_supported")):  # host-only queries: free to be reordered or repeated
            return fn

        def call(*args):
            self.calls.append(_describe(name, args))
            return fn(*args)

        return call


@contextlib.contextmanager
def _recording():
    from detectron2_b200 import _C

    lib = _C.lib()
    rec = _Recorder(lib)
    _C._lib = rec
    try:
        yield rec.calls
    finally:
        _C._lib = lib


def _inputs(c, layout, dtype, fused):
    g = torch.Generator().manual_seed(c)
    x = torch.randn(2, c, 10, 12, generator=g).to(DEV, getattr(torch, dtype))
    if layout == "cl":
        x = x.contiguous(memory_format=torch.channels_last)
    off = (torch.randn(2, 27 if fused else 18, 10, 12, generator=g) * 0.5).to(DEV)
    mask = torch.rand(2, 9, 10, 12, generator=g).to(DEV)
    wt = (torch.randn(c, c, 3, 3, generator=g) * 0.05).to(DEV)
    b = torch.randn(c, generator=g).to(DEV)
    return x, off, mask, wt, b


def _run(case):
    """case = kind/shape/layout/dtype/precision -> the recorded calls (+ "raise" when the call raised RuntimeError)."""
    from detectron2_b200 import ops

    kind, shape, layout, dtype, prec = case.split("/")
    prec, fused = int(prec), kind.startswith("fused")
    x, off, mask, wt, b = _inputs(int(shape[1:]), layout, dtype, fused)
    with _recording() as calls:
        try:
            if kind == "plain-infer":
                with torch.no_grad():
                    ops.deform_conv(x, off, mask, wt, b, *GEO, prec)
            elif kind == "plain-train":  # the training op and its autograd backward, every input differentiated
                ins = [t.requires_grad_() for t in (x, off, mask, wt, b)]
                y = ops.deform_conv(*ins, *GEO, prec)
                y.backward(torch.ones_like(y))
            elif kind in ("plain-bwd-data", "plain-bwd-weight"):
                go = torch.ones(x.shape[0], wt.shape[0], 10, 12, device=DEV)
                ops.deform_conv_backward_op(x, off, mask, wt, go, *GEO, True, kind == "plain-bwd-data",
                                            kind == "plain-bwd-weight", prec)
            elif kind == "fused-infer":
                with torch.no_grad():
                    ops.deform_conv_fused(x, off, wt, b.abs(), b, True, *GEO, prec)
            elif kind == "fused-train":
                x, off, wt = (t.requires_grad_() for t in (x, off, wt))
                y = ops.deform_conv_fused(x, off, wt, b.abs(), b, True, *GEO, prec)
                y.backward(torch.ones_like(y))
            elif kind == "fused-infer-grad":  # the inference op called directly on inputs that need a gradient
                x, off, wt = (t.requires_grad_() for t in (x, off, wt))
                y = ops.deform_conv_fused_op(x, off, wt, None, b, False, *GEO, prec)
                y.backward(torch.ones_like(y))
            elif kind == "fused-bwd":
                y = torch.ones(x.shape[0], wt.shape[0], 10, 12, device=DEV)
                ops.deform_conv_fused_backward_op(x, off, wt, b.abs(), True, y, y, *GEO, prec)
            else:
                raise ValueError(kind)
        except RuntimeError:
            calls.append("raise")
        torch.cuda.synchronize()
    return calls


EXPECTED = {  # case -> calls, see _describe
    "fused-bwd/P64/cl/bfloat16/2": ["fbwd 1 P64 2 1 458752 xxxxxx.xxxx"],
    "fused-bwd/P64/nchw/float32/-1": ["fbwd 1 P64 -1 0 581632 xxxxxx.xxxx"],
    "fused-infer-grad/P64/cl/float32/1": ["ffwd 0 P64 1 1 147456 xxx.xx.x", "fbwd 0 P64 1 1 458752 xxx.xx.xxxx"],
    "fused-infer-grad/P64/nchw/float32/-1": ["ffwd 0 P64 1 0 208896 xxx.xx.x", "fbwd 0 P64 1 0 581632 xxx.xx.xxxx"],
    "fused-infer/P48/nchw/float32/-1": ["raise"],
    "fused-infer/P64/cl/bfloat16/-1": ["ffwd 1 P64 1 1 147456 xxxxxx.x"],
    "fused-infer/P64/cl/bfloat16/1": ["ffwd 1 P64 1 1 147456 xxxxxx.x"],
    "fused-infer/P64/cl/bfloat16/2": ["ffwd 1 P64 2 1 147456 xxxxxx.x"],
    "fused-infer/P64/cl/float32/-1": ["ffwd 1 P64 1 1 147456 xxxxxx.x"],
    "fused-infer/P64/cl/float32/1": ["ffwd 1 P64 1 1 147456 xxxxxx.x"],
    "fused-infer/P64/cl/float32/2": ["ffwd 1 P64 2 1 147456 xxxxxx.x"],
    "fused-infer/P64/nchw/bfloat16/-1": ["ffwd 1 P64 1 0 208896 xxxxxx.x"],
    "fused-infer/P64/nchw/bfloat16/1": ["ffwd 1 P64 1 0 208896 xxxxxx.x"],
    "fused-infer/P64/nchw/bfloat16/2": ["ffwd 1 P64 2 0 208896 xxxxxx.x"],
    "fused-infer/P64/nchw/float32/-1": ["ffwd 1 P64 1 0 208896 xxxxxx.x"],
    "fused-infer/P64/nchw/float32/1": ["ffwd 1 P64 1 0 208896 xxxxxx.x"],
    "fused-infer/P64/nchw/float32/2": ["ffwd 1 P64 2 0 208896 xxxxxx.x"],
    "fused-train/P48/cl/float32/1": ["raise"],
    "fused-train/P64/cl/bfloat16/-1": ["ffwd 1 P64 1 1 147456 xxxxxxxx", "fbwd 1 P64 1 1 458752 xxxxxxxxxxx"],
    "fused-train/P64/cl/bfloat16/1": ["ffwd 1 P64 1 1 147456 xxxxxxxx", "fbwd 1 P64 1 1 458752 xxxxxxxxxxx"],
    "fused-train/P64/cl/bfloat16/2": ["ffwd 1 P64 2 1 147456 xxxxxxxx", "fbwd 1 P64 2 1 458752 xxxxxxxxxxx"],
    "fused-train/P64/cl/float32/-1": ["ffwd 1 P64 1 1 147456 xxxxxxxx", "fbwd 1 P64 1 1 458752 xxxxxxxxxxx"],
    "fused-train/P64/cl/float32/1": ["ffwd 1 P64 1 1 147456 xxxxxxxx", "fbwd 1 P64 1 1 458752 xxxxxxxxxxx"],
    "fused-train/P64/cl/float32/2": ["ffwd 1 P64 2 1 147456 xxxxxxxx", "fbwd 1 P64 2 1 458752 xxxxxxxxxxx"],
    "fused-train/P64/nchw/bfloat16/-1": [
        "to_nhwc 10x12 2 64 2 x",
        "ffwd 1 P64 1 1 147456 xxxxxxxx",
        "fbwd 1 P64 1 1 458752 xxxxxxxxxxx",
    ],
    "fused-train/P64/nchw/bfloat16/1": [
        "to_nhwc 10x12 2 64 2 x",
        "ffwd 1 P64 1 1 147456 xxxxxxxx",
        "fbwd 1 P64 1 1 458752 xxxxxxxxxxx",
    ],
    "fused-train/P64/nchw/bfloat16/2": [
        "to_nhwc 10x12 2 64 2 x",
        "ffwd 1 P64 2 1 147456 xxxxxxxx",
        "fbwd 1 P64 2 1 458752 xxxxxxxxxxx",
    ],
    "fused-train/P64/nchw/float32/-1": [
        "to_nhwc 10x12 2 64 0 x",
        "ffwd 1 P64 1 1 147456 xxxxxxxx",
        "fbwd 1 P64 1 1 458752 xxxxxxxxxxx",
    ],
    "fused-train/P64/nchw/float32/1": [
        "to_nhwc 10x12 2 64 0 x",
        "ffwd 1 P64 1 1 147456 xxxxxxxx",
        "fbwd 1 P64 1 1 458752 xxxxxxxxxxx",
    ],
    "fused-train/P64/nchw/float32/2": [
        "to_nhwc 10x12 2 64 0 x",
        "ffwd 1 P64 2 1 147456 xxxxxxxx",
        "fbwd 1 P64 2 1 458752 xxxxxxxxxxx",
    ],
    "plain-bwd-data/P64/cl/bfloat16/2": ["bwd P64 2 1 229376 xxxxx.xxx..x"],
    "plain-bwd-data/P64/nchw/float32/-1": ["bwd P64 -1 0 352256 xxxxx.xxx..x"],
    "plain-bwd-weight/P48/nchw/float32/0": ["bwd P48 0 0 0 xxxxx....xx."],
    "plain-bwd-weight/P64/cl/float32/-1": ["bwd P64 -1 1 229376 xxxxx....xxx"],
    "plain-infer/P48/cl/bfloat16/-1": ["fwd P48 -1 0 0 xxxxxx.."],
    "plain-infer/P48/cl/bfloat16/0": ["fwd P48 0 0 0 xxxxxx.."],
    "plain-infer/P48/cl/float32/-1": ["fwd P48 -1 0 0 xxxxxx.."],
    "plain-infer/P48/cl/float32/0": ["fwd P48 0 0 0 xxxxxx.."],
    "plain-infer/P48/nchw/bfloat16/-1": ["fwd P48 -1 0 0 xxxxxx.."],
    "plain-infer/P48/nchw/bfloat16/0": ["fwd P48 0 0 0 xxxxxx.."],
    "plain-infer/P48/nchw/float32/-1": ["fwd P48 -1 0 0 xxxxxx.."],
    "plain-infer/P48/nchw/float32/0": ["fwd P48 0 0 0 xxxxxx.."],
    "plain-infer/P48/nchw/float32/1": ["fwd P48 1 0 0 xxxxxx..", "raise"],
    "plain-infer/P64/cl/bfloat16/-1": ["fwd P64 -1 1 147456 xxxxxx.x"],
    "plain-infer/P64/cl/bfloat16/0": ["fwd P64 0 0 0 xxxxxx.."],
    "plain-infer/P64/cl/bfloat16/1": ["fwd P64 1 1 147456 xxxxxx.x"],
    "plain-infer/P64/cl/bfloat16/2": ["fwd P64 2 1 147456 xxxxxx.x"],
    "plain-infer/P64/cl/float32/-1": ["fwd P64 -1 1 147456 xxxxxx.x"],
    "plain-infer/P64/cl/float32/0": ["fwd P64 0 0 0 xxxxxx.."],
    "plain-infer/P64/cl/float32/1": ["fwd P64 1 1 147456 xxxxxx.x"],
    "plain-infer/P64/cl/float32/2": ["fwd P64 2 1 147456 xxxxxx.x"],
    "plain-infer/P64/nchw/bfloat16/-1": ["fwd P64 -1 0 208896 xxxxxx.x"],
    "plain-infer/P64/nchw/bfloat16/0": ["fwd P64 0 0 0 xxxxxx.."],
    "plain-infer/P64/nchw/bfloat16/1": ["fwd P64 1 0 208896 xxxxxx.x"],
    "plain-infer/P64/nchw/bfloat16/2": ["fwd P64 2 0 208896 xxxxxx.x"],
    "plain-infer/P64/nchw/float32/-1": ["fwd P64 -1 0 208896 xxxxxx.x"],
    "plain-infer/P64/nchw/float32/0": ["fwd P64 0 0 0 xxxxxx.."],
    "plain-infer/P64/nchw/float32/1": ["fwd P64 1 0 208896 xxxxxx.x"],
    "plain-infer/P64/nchw/float32/2": ["fwd P64 2 0 208896 xxxxxx.x"],
    "plain-train/P48/cl/bfloat16/-1": ["fwd P48 -1 0 0 xxxxxx..", "bwd P48 -1 0 0 xxxxx.xxxxx."],
    "plain-train/P48/cl/bfloat16/0": ["fwd P48 0 0 0 xxxxxx..", "bwd P48 0 0 0 xxxxx.xxxxx."],
    "plain-train/P48/cl/float32/-1": ["fwd P48 -1 0 0 xxxxxx..", "bwd P48 -1 0 0 xxxxx.xxxxx."],
    "plain-train/P48/cl/float32/0": ["fwd P48 0 0 0 xxxxxx..", "bwd P48 0 0 0 xxxxx.xxxxx."],
    "plain-train/P48/nchw/bfloat16/-1": ["fwd P48 -1 0 0 xxxxxx..", "bwd P48 -1 0 0 xxxxx.xxxxx."],
    "plain-train/P48/nchw/bfloat16/0": ["fwd P48 0 0 0 xxxxxx..", "bwd P48 0 0 0 xxxxx.xxxxx."],
    "plain-train/P48/nchw/float32/-1": ["fwd P48 -1 0 0 xxxxxx..", "bwd P48 -1 0 0 xxxxx.xxxxx."],
    "plain-train/P48/nchw/float32/0": ["fwd P48 0 0 0 xxxxxx..", "bwd P48 0 0 0 xxxxx.xxxxx."],
    "plain-train/P64/cl/bfloat16/-1": ["fwd P64 -1 1 147456 xxxxxxxx", "bwd P64 -1 1 458752 xxxxxxxxxxxx"],
    "plain-train/P64/cl/bfloat16/0": ["fwd P64 0 0 0 xxxxxx..", "bwd P64 0 0 0 xxxxx.xxxxx."],
    "plain-train/P64/cl/bfloat16/1": ["fwd P64 1 1 147456 xxxxxxxx", "bwd P64 1 1 458752 xxxxxxxxxxxx"],
    "plain-train/P64/cl/bfloat16/2": ["fwd P64 2 1 147456 xxxxxxxx", "bwd P64 2 1 458752 xxxxxxxxxxxx"],
    "plain-train/P64/cl/float32/-1": ["fwd P64 -1 1 147456 xxxxxxxx", "bwd P64 -1 1 458752 xxxxxxxxxxxx"],
    "plain-train/P64/cl/float32/0": ["fwd P64 0 0 0 xxxxxx..", "bwd P64 0 0 0 xxxxx.xxxxx."],
    "plain-train/P64/cl/float32/1": ["fwd P64 1 1 147456 xxxxxxxx", "bwd P64 1 1 458752 xxxxxxxxxxxx"],
    "plain-train/P64/cl/float32/2": ["fwd P64 2 1 147456 xxxxxxxx", "bwd P64 2 1 458752 xxxxxxxxxxxx"],
    "plain-train/P64/nchw/bfloat16/-1": [
        "to_nhwc 10x12 2 64 2 x",
        "fwd P64 -1 1 147456 xxxxxxxx",
        "bwd P64 -1 1 458752 xxxxxxxxxxxx",
    ],
    "plain-train/P64/nchw/bfloat16/0": ["fwd P64 0 0 0 xxxxxx..", "bwd P64 0 0 0 xxxxx.xxxxx."],
    "plain-train/P64/nchw/bfloat16/1": [
        "to_nhwc 10x12 2 64 2 x",
        "fwd P64 1 1 147456 xxxxxxxx",
        "bwd P64 1 1 458752 xxxxxxxxxxxx",
    ],
    "plain-train/P64/nchw/bfloat16/2": [
        "to_nhwc 10x12 2 64 2 x",
        "fwd P64 2 1 147456 xxxxxxxx",
        "bwd P64 2 1 458752 xxxxxxxxxxxx",
    ],
    "plain-train/P64/nchw/float32/-1": [
        "to_nhwc 10x12 2 64 0 x",
        "fwd P64 -1 1 147456 xxxxxxxx",
        "bwd P64 -1 1 458752 xxxxxxxxxxxx",
    ],
    "plain-train/P64/nchw/float32/0": ["fwd P64 0 0 0 xxxxxx..", "bwd P64 0 0 0 xxxxx.xxxxx."],
    "plain-train/P64/nchw/float32/1": [
        "to_nhwc 10x12 2 64 0 x",
        "fwd P64 1 1 147456 xxxxxxxx",
        "bwd P64 1 1 458752 xxxxxxxxxxxx",
    ],
    "plain-train/P64/nchw/float32/2": [
        "to_nhwc 10x12 2 64 0 x",
        "fwd P64 2 1 147456 xxxxxxxx",
        "bwd P64 2 1 458752 xxxxxxxxxxxx",
    ],
}


@pytest.mark.parametrize("case", sorted(EXPECTED))
def test_native_calls(case):
    assert _run(case) == EXPECTED[case]


def test_fused_ops_refuse_a_weight_that_does_not_match_the_groups():
    """weight.shape[1] must be Cin / groups: the kernels read the weight with that stride, and the C ABI does not receive
    weight.shape[1], so only the host can refuse it -- before any launch."""
    from detectron2_b200 import ops

    x, om, _, _, b = _inputs(64, "nchw", "float32", True)
    wt = torch.randn(64, 64, 3, 3, device=DEV)  # groups = 2 wants [64, 32, 3, 3]
    geo = ([1, 1], [1, 1], [1, 1], 2, 1)
    for op in (ops.deform_conv_fused_op, ops.deform_conv_fused_train_op):
        with _recording() as calls, pytest.raises(RuntimeError, match="weight/groups"):
            op(x, om, wt, b.abs(), b, True, *geo, 1)
        assert calls == [], op
