"""Generate tests/golden/sem_seg_loss.npz from the REAL reference losses: SemSegFPNHead.losses
(modeling/meta_arch/semantic_seg.py:255-267, called with a stand-in `self`) and DeepLabCE.forward
(projects/DeepLab/deeplab/loss.py) after the DeepLab heads' F.interpolate, on CPU.

Run in the authoring container only (needs /root/reference, like make_golden_panoptic.py):
    python tests/golden/make_golden_sem_seg.py
It writes only this file: per case the loss and its autograd gradient with respect to the low-res logits (the inputs are
rebuilt from seeds by tests/sem_seg_ref.py).  The reference's semantic_seg.py is loaded with stub modules for the imports
that SemSegFPNHead.losses does not use.
"""
import os
import sys
import types

import numpy as np
import torch
from torch.nn import functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (save())
import make_golden_rotated as mgr  # noqa: E402  (_load())

sys.path.insert(0, os.path.dirname(HERE))
from sem_seg_ref import CASES, make_case  # noqa: E402  (the cases, shared with the tests)

REF = "/root/reference"


def import_reference():
    """semantic_seg.py with stubs for its imports (SemSegFPNHead.losses uses torch.nn.functional only), and loss.py."""
    stub = types.ModuleType
    registry = type("Registry", (), {"__init__": lambda self, name: None,
                                     "register": lambda self, obj=None: (lambda c: c) if obj is None else obj})
    mods = {
        "fvcore": {}, "fvcore.nn": {}, "fvcore.nn.weight_init": {},
        "detectron2": {}, "detectron2.config": {"configurable": lambda f=None, **k: f},
        "detectron2.layers": {"Conv2d": object, "ShapeSpec": object, "get_norm": None},
        "detectron2.structures": {"ImageList": object},
        "detectron2.utils": {}, "detectron2.utils.registry": {"Registry": registry},
        "detectron2.modeling": {}, "detectron2.modeling.backbone": {"Backbone": object, "build_backbone": None},
        "detectron2.modeling.postprocessing": {"sem_seg_postprocess": None},
        "detectron2.modeling.meta_arch": {},
        "detectron2.modeling.meta_arch.build": {"META_ARCH_REGISTRY": registry("META_ARCH")},
    }
    for name, attrs in mods.items():
        m = sys.modules.get(name) or stub(name)
        m.__path__ = getattr(m, "__path__", [])
        m.__dict__.update(attrs)
        sys.modules[name] = m
    sys.modules["fvcore.nn"].weight_init = sys.modules["fvcore.nn.weight_init"]
    ss = mgr._load("detectron2.modeling.meta_arch.semantic_seg", REF + "/detectron2/modeling/meta_arch/semantic_seg.py")
    ce = mgr._load("deeplab_loss", REF + "/projects/DeepLab/deeplab/loss.py")
    return ss.SemSegFPNHead, ce.DeepLabCE


def reference_loss(head, deeplab_ce, name, logits, targets, weights):
    _, _, _, _, s, ignore, top_k, _, _ = CASES[name]
    pred = logits.clone().requires_grad_(True)
    if top_k is None:
        me = types.SimpleNamespace(common_stride=s, ignore_value=ignore, loss_weight=1.0)
        loss = head.losses(me, pred, targets)["loss_sem_seg"]
    else:  # PanopticDeepLabSemSegHead.losses / DeepLabV3PlusHead.losses: interpolate, then DeepLabCE
        up = F.interpolate(pred, scale_factor=s, mode="bilinear", align_corners=False)
        loss = deeplab_ce(ignore_label=ignore, top_k_percent_pixels=top_k)(up, targets, weights)
    loss.backward()
    return loss.detach(), pred.grad


def main():
    torch.set_num_threads(1)
    head, deeplab_ce = import_reference()
    out = {}
    for name in CASES:
        logits, targets, weights = make_case(name)
        loss, grad = reference_loss(head, deeplab_ce, name, logits, targets, weights)
        out[name + "_loss"], out[name + "_grad"] = loss, grad
    out["cases"] = np.asarray(list(CASES))
    mg.save("sem_seg_loss", **out)


if __name__ == "__main__":
    main()
