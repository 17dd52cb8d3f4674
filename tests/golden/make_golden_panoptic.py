"""Generate tests/golden/panoptic.npz from the REAL reference functions: combine_semantic_and_instance_outputs
(modeling/meta_arch/panoptic_fpn.py:184-269) and sem_seg_postprocess (modeling/postprocessing.py:77-100) + argmax(0).

Run in the authoring container only (needs /root/reference, like make_golden_matching.py):
    python tests/golden/make_golden_panoptic.py
It writes only this file.  The combine scenes are built by `scenes()` below and stored whole (they are small); the
semantic logits are regenerated from the stored seeds with a CPU torch.Generator (`sem_logits()`, mirrored by
tests/test_panoptic_host.py).  Scores avoid exact ties: the reference's unstable argsort decides those.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (save())
import make_golden_matching as mgm  # noqa: E402
import make_golden_rotated as mgr  # noqa: E402

REF = "/root/reference/detectron2"
# (C, Hp, Wp, crop h, crop w, out H, out W, seed): up-sampled, down-sampled, same size, odd crops, C = 1
SEM_CASES = [(54, 24, 40, 20, 33, 45, 61, 11), (54, 24, 40, 24, 40, 13, 17, 12), (54, 24, 40, 19, 31, 19, 31, 13),
             (54, 24, 40, 17, 29, 31, 7, 14), (1, 8, 8, 7, 5, 9, 11, 15)]
# (name, overlap_threshold, stuff_area_thresh, instances_score_thresh) per scene below
THRESHOLDS = {"default": (0.5, 4096.0, 0.5), "stuff0": (0.5, 0.0, 0.5), "stuff8": (0.5, 8.0, 0.5),
              "overlap1": (1.0, 0.0, 0.5), "score03": (0.5, 0.0, 0.3)}


def sem_logits(C, Hp, Wp, seed):
    return torch.randn((C, Hp, Wp), generator=torch.Generator().manual_seed(seed))


def _rect(H, W, y0, y1, x0, x1, value=1):
    m = torch.zeros((H, W), dtype=torch.uint8)
    m[y0:y1, x0:x1] = value
    return m


def _random_scene(g, H, W, R, C):
    masks = torch.zeros((R, H, W), dtype=torch.uint8)
    for i in range(R):
        y0, x0 = int(torch.randint(0, H, (1,), generator=g)), int(torch.randint(0, W, (1,), generator=g))
        y1 = y0 + 1 + int(torch.randint(0, max(H - y0, 1), (1,), generator=g))
        x1 = x0 + 1 + int(torch.randint(0, max(W - x0, 1), (1,), generator=g))
        masks[i, y0:y1, x0:x1] = 1 if i % 3 else 255  # any nonzero byte is "in"
        masks[i] &= (torch.rand((H, W), generator=g) < 0.9).to(torch.uint8) * 255  # ragged edges
    scores = torch.randperm(1000, generator=g)[:R].float() / 1000.0 * 0.9 + 0.05  # distinct
    classes = torch.randint(0, 80, (R,), generator=g)
    labels = torch.randint(0, C, (H, W), generator=g)
    return scores, classes, masks, labels


def scenes():
    """(name, thresholds key, scores, classes, masks, labels)."""
    g = torch.Generator().manual_seed(2026)
    out = []
    # overlap ratio exactly at the threshold (kept: > is strict) and just above it
    H, W = 16, 33
    a = _rect(H, W, 0, 4, 0, 33)                                  # 132 px
    b = _rect(H, W, 2, 6, 0, 33)                                  # 132 px, 66 of them under a: ratio 0.5, kept
    c = _rect(H, W, 5, 8, 0, 33)                                  # 99 px, 33 under b: 1/3, kept
    d = _rect(H, W, 7, 9, 0, 33)                                  # 66 px, 33 under c: exactly 0.5, kept
    e = _rect(H, W, 8, 10, 0, 33)
    e[9, 0] = 0                                                   # 65 px, 33 under d: 33/65 just above 0.5, skipped
    labels = torch.zeros((H, W), dtype=torch.int64)
    labels[10:, :20], labels[10:, 20:] = 3, 7
    labels[0, 0] = 5                                              # present only under an instance
    out.append(("overlap_edge", "stuff0", torch.tensor([0.9, 0.8, 0.7, 0.6, 0.55]), torch.tensor([1, 2, 3, 4, 5]),
                torch.stack([a, b, c, d, e]), labels))
    out.append(("overlap_edge_stuff8", "stuff8", out[-1][2], out[-1][3], out[-1][4], labels))
    # a score exactly at the threshold (walked), one below it (stops the walk), a zero-area mask, masks holding 255
    m = torch.stack([_rect(H, W, 0, 3, 0, 10, 255), _rect(H, W, 3, 6, 0, 10), torch.zeros((H, W), dtype=torch.uint8),
                     _rect(H, W, 6, 9, 0, 10), _rect(H, W, 9, 12, 0, 10)])
    out.append(("score_at_threshold", "stuff0", torch.tensor([0.5, 0.95, 0.7, 0.45, 0.6]), torch.tensor([0, 1, 2, 3, 4]),
                m, torch.randint(0, 54, (H, W), generator=g)))
    # threshold 0.3 (not representable): fp32 scores on both sides of it
    above = torch.tensor(0.3, dtype=torch.float32)                # 0.30000001192... > 0.3
    below = torch.nextafter(above, torch.tensor(0.0))             # 0.29999998... < 0.3
    out.append(("score_03", "score03", torch.stack([above, torch.tensor(0.8), below, torch.tensor(0.2)]),
                torch.tensor([5, 6, 7, 8]), m[[0, 1, 3, 4]], torch.randint(0, 54, (H, W), generator=g)))
    # overlap_threshold 1.0: a fully covered instance is kept, paints nothing and consumes an id
    out.append(("overlap_one", "overlap1", torch.tensor([0.9, 0.8, 0.7]), torch.tensor([1, 2, 3]),
                torch.stack([_rect(H, W, 0, 8, 0, 20), _rect(H, W, 2, 5, 3, 9), _rect(H, W, 6, 12, 10, 30)]),
                torch.randint(0, 5, (H, W), generator=g)))
    # label 0 only; no instances
    out.append(("label0_only", "stuff0", torch.tensor([0.9]), torch.tensor([3]), _rect(H, W, 1, 4, 1, 4)[None],
                torch.zeros((H, W), dtype=torch.int64)))
    out.append(("no_instances", "stuff8", torch.zeros(0), torch.zeros(0, dtype=torch.int64),
                torch.zeros((0, H, W), dtype=torch.uint8), torch.randint(0, 54, (H, W), generator=g)))
    # widths around the 32-pixel words, C = 1 and C = 54
    for W2, C in ((1, 54), (31, 54), (32, 1), (33, 54), (1333, 54)):
        H2 = 40 if W2 < 100 else 9
        s, cl, mk, lb = _random_scene(g, H2, W2, 12, C)
        out.append(("width%d_c%d" % (W2, C), "default" if W2 == 1333 else "stuff8", s, cl, mk, lb))
        out.append(("width%d_c%d_stuff0" % (W2, C), "stuff0", s, cl, mk, lb))
    return out


def import_reference():
    mgm.import_reference()
    pkg = "detectron2.modeling"
    for name in (pkg, pkg + ".meta_arch"):
        if name not in sys.modules:
            m = types.ModuleType(name)
            m.__path__ = []
            sys.modules[name] = m
    pp = mgr._load(pkg + ".postprocessing", REF + "/modeling/postprocessing.py")
    for name, attrs in ((".meta_arch.build", {"META_ARCH_REGISTRY": types.SimpleNamespace(register=lambda: (lambda c: c))}),
                        (".meta_arch.rcnn", {"GeneralizedRCNN": type("GeneralizedRCNN", (), {})}),
                        (".meta_arch.semantic_seg", {"build_sem_seg_head": None})):
        m = types.ModuleType(pkg + name)
        m.__dict__.update(attrs)
        sys.modules[pkg + name] = m
    sys.modules.setdefault("detectron2.config", types.ModuleType("detectron2.config")).configurable = lambda f=None, **k: f
    pf = mgr._load(pkg + ".meta_arch.panoptic_fpn", REF + "/modeling/meta_arch/panoptic_fpn.py")
    return pp, pf


def main():
    torch.set_num_threads(1)
    pp, pf = import_reference()
    out = {}
    for i, (C, Hp, Wp, h, w, H, W, seed) in enumerate(SEM_CASES):
        logits = sem_logits(C, Hp, Wp, seed)
        if i == 3:
            logits[:, 5:9, 6:12] = 0.125  # constant logits: every channel ties, label 0
        out["sem%d_case" % i] = np.asarray([C, Hp, Wp, h, w, H, W, seed])
        out["sem%d_labels" % i] = pp.sem_seg_postprocess(logits, (h, w), H, W).argmax(dim=0)
    names = []
    for name, thr, scores, classes, masks, labels in scenes():
        ov, st, sc = THRESHOLDS[thr]
        inst = types.SimpleNamespace(scores=scores.clone(), pred_classes=classes.clone(), pred_masks=masks.clone())
        pan, info = pf.combine_semantic_and_instance_outputs(inst, labels.clone(), ov, st, sc)
        rec = [(d["id"], int(d["isthing"]), d["category_id"], d.get("instance_id", -1), d.get("area", 0),
                d.get("score", 0.0)) for d in info]
        names.append(name)
        out[name + "_thr"] = np.asarray([ov, st, sc])
        out[name + "_scores"], out[name + "_classes"], out[name + "_masks"] = scores, classes, masks
        out[name + "_labels"], out[name + "_panoptic"] = labels, pan
        out[name + "_records"] = np.asarray([r[:5] for r in rec], dtype=np.int64).reshape(-1, 5)
        out[name + "_record_scores"] = np.asarray([r[5] for r in rec], dtype=np.float64)
    out["scenes"] = np.asarray(names)
    mg.save("panoptic", **out)


if __name__ == "__main__":
    main()
