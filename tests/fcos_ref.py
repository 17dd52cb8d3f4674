"""The FCOS fixture (tests/golden/fcos.npz, from tests/golden/make_golden_fcos.py) and its checks, shared by the CPU tests
of the torch restatement and the GPU tests of the kernels."""
import os

import numpy as np
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "fcos.npz")
K = 6


def load():
    return np.load(GOLDEN)


def arr(z, key, device="cpu"):
    return torch.from_numpy(z[key]).to(device)


def lst(z, case, key, device="cpu"):
    out, i = [], 0
    while "%s__%s%d" % (case, key, i) in z:
        out.append(arr(z, "%s__%s%d" % (case, key, i), device))
        i += 1
    return out


def close(a, b, tol):
    a, b = a.detach().cpu().double(), torch.as_tensor(b).detach().cpu().double()
    if b.numel() == 0:
        return a.numel() == 0
    return float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-12)


def same(a, b):
    """Bitwise equality, NaN == NaN."""
    a, b = a.detach().cpu(), torch.as_tensor(b).detach().cpu()
    return a.shape == b.shape and bool(((a == b) | (a.isnan() & b.isnan())).all())


def anchors(z, device="cpu"):
    return lst(z, "pts", "anchors", device)


def check_labels(z, case, labels, boxes):
    """label_anchors' per-image outputs against the fixture, bit for bit."""
    want_l, want_b = lst(z, case, "labels"), lst(z, case, "boxes")
    assert len(labels) == len(want_l)
    for i, (l, b) in enumerate(zip(labels, boxes)):
        assert same(l, want_l[i]), (case, i)
        assert same(b, want_b[i]), (case, i)


def run_loss_case(z, case, device, tol, grad_tol):
    """FCOS.losses through fcos.fcos_losses on `device` (CPU: the restatement; CUDA: the kernels): losses, the EMA,
    gradients and the assertion against the reference's."""
    import pytest

    from detectron2_b200 import fcos as F

    an = anchors(z, device)
    labels = lst(z, "a", "labels", device)
    boxes = lst(z, "a", "boxes", device)
    # fp16 cases store fp16 predictions; the reference saw their fp32 values
    logits = lst(z, case, "logits", device)
    deltas = lst(z, case, "deltas", device)
    ctr = lst(z, case, "ctr", device)
    if int(z[case + "__raises"]):
        with pytest.raises(AssertionError):
            F.fcos_losses(an, logits, labels, deltas, boxes, ctr, num_classes=K)
        return
    old = None
    for c in range(int(z[case + "__calls"])):
        lx = [t.clone().requires_grad_(True) for t in logits]
        ld = [t.clone().requires_grad_(True) for t in deltas]
        lc = [t.clone().requires_grad_(True) for t in ctr]
        losses, num_pos, old = F.fcos_losses(an, lx, labels, ld, boxes, lc, num_classes=K, loss_normalizer=old)
        cc = "%s_call%d" % (case, c)
        assert num_pos == int(z[case + "__num_pos"])
        assert old == float(z[cc + "__normalizer"])
        for k in ("loss_fcos_cls", "loss_fcos_loc", "loss_fcos_ctr"):
            assert close(losses[k], z[cc + "__" + k], tol), (cc, k, float(losses[k]), float(z[cc + "__" + k]))
        sum(losses.values()).backward()
        for name, got in (("grad_logits", lx), ("grad_deltas", ld), ("grad_ctr", lc)):
            for g, w in zip(got, lst(z, cc, name)):
                assert g.grad.dtype == g.dtype
                assert close(g.grad.float(), w, grad_tol), (cc, name)
