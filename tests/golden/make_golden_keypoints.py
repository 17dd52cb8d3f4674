"""Generate tests/golden/keypoints.npz from the REAL reference functions: heatmaps_to_keypoints and Keypoints.to_heatmap
(detectron2/structures/keypoints.py:105-235), keypoint_rcnn_loss (modeling/roi_heads/keypoint_head.py:40-96, with the
event-storage stub of make_golden_matching.py) and the keypoint branch of detector_postprocess
(modeling/postprocessing.py:70-72).

Run in the authoring container only (needs /root/reference, like make_golden_matching.py):
    python tests/golden/make_golden_keypoints.py
It writes only this file.  The heatmaps and logits are not stored: they are regenerated from the stored seeds with a CPU
torch.Generator (`heatmaps()` / `loss_logits()` below, mirrored by tests/test_keypoint_head_host.py).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (save())
import make_golden_matching as mgm  # noqa: E402
import make_golden_rotated as mgr  # noqa: E402

REF = "/root/reference/detectron2"
K, S = 17, 56
MAPS_SEED, LOGITS_SEED = 31, 37
CONST_ROI, CONST_VALUE = 3, 0.25  # every map of this ROI is constant: the argmax tie rule picks the first pixel


def heatmaps(r):
    maps = torch.randn((r, K, S, S), generator=torch.Generator().manual_seed(MAPS_SEED))
    maps[CONST_ROI] = CONST_VALUE
    return maps


def loss_logits(n):
    return torch.randn((n, K, S, S), generator=torch.Generator().manual_seed(LOGITS_SEED))


def inference_rois(g):
    special = torch.tensor([
        [10.3, 20.7, 55.9, 99.2],      # sub-pixel edges
        [8.0, 8.0, 64.0, 64.0],        # integer edges, ceil(w) = ceil(h) = S: PyTorch's same-size copy
        [3.0, 4.0, 3.5, 90.0],         # narrower than 1 px: w clamped to 1
        [0.0, 0.0, 40.0, 28.0],        # the constant maps (CONST_ROI)
        [5.2, 5.1, 5.4, 5.9],          # smaller than 1 px both ways
        [12.5, 7.25, 612.0, 431.75],   # much larger than the map
        [100.0, 50.0, 100.0, 50.0],    # empty box
    ])
    side = torch.exp(torch.empty(8, 2).uniform_(np.log(2.0), np.log(300.0), generator=g))
    ctr = torch.rand(8, 2, generator=g) * 400
    rand = torch.cat([ctr - side / 2, ctr + side / 2], dim=1)
    return torch.cat([special, rand])


def loss_inputs(g):
    """Three images: 5 proposals, none, 4 proposals whose keypoints are all invisible or outside (no valid keypoint)."""
    boxes0 = torch.tensor([[10.0, 20.0, 66.0, 76.0], [0.5, 0.25, 30.75, 90.5], [100.0, 100.0, 101.0, 180.0],
                           [40.0, 40.0, 140.0, 60.0], [7.3, 9.1, 8.0, 9.9]])
    kp0 = torch.empty(5, K, 3)
    for i, b in enumerate(boxes0):
        w, h = b[2] - b[0], b[3] - b[1]
        kp0[i, :, 0] = b[0] + (torch.rand(K, generator=g) * 1.4 - 0.2) * w  # some outside the box
        kp0[i, :, 1] = b[1] + (torch.rand(K, generator=g) * 1.4 - 0.2) * h
        kp0[i, :, 2] = torch.randint(0, 3, (K,), generator=g).float()  # v = 0 / 1 / 2
        kp0[i, :3, 2] = 2.0
        kp0[i, 0, 0], kp0[i, 1, 1] = b[2], b[3]  # exactly on x2, exactly on y2
        kp0[i, 2, 0], kp0[i, 2, 1] = b[0], b[1]  # exactly on (x1, y1)
    boxes2 = torch.tensor([[0.0, 0.0, 20.0, 20.0], [5.0, 5.0, 50.0, 30.0], [1.0, 2.0, 3.0, 4.0], [9.0, 9.0, 90.0, 90.0]])
    kp2 = torch.cat([torch.rand(4, K, 2, generator=g) * 20, torch.zeros(4, K, 1)], dim=2)  # invisible
    kp2[3, :, 0], kp2[3, :, 2] = 95.0, 2.0  # visible, outside
    return [boxes0, torch.zeros(0, 4), boxes2], [kp0, torch.zeros(0, K, 3), kp2]


def main():
    torch.set_num_threads(1)
    mgm.import_reference()
    kh = mgr._load("ref_keypoint_head", REF + "/modeling/roi_heads/keypoint_head.py")
    pp = mgr._load("ref_postprocessing", REF + "/modeling/postprocessing.py")
    from detectron2.structures import Boxes, Instances, Keypoints, heatmaps_to_keypoints

    g = torch.Generator().manual_seed(2025)
    out = {"K": np.asarray(K), "S": np.asarray(S), "maps_seed": np.asarray(MAPS_SEED),
           "logits_seed": np.asarray(LOGITS_SEED), "const_roi": np.asarray(CONST_ROI), "const_value": np.asarray(CONST_VALUE)}

    # inference
    rois = inference_rois(g)
    maps = heatmaps(len(rois))
    out["rois"] = rois
    out["xy_preds"] = heatmaps_to_keypoints(maps, rois)

    # training targets and loss
    boxes, kps = loss_inputs(g)
    n = sum(len(b) for b in boxes)
    logits = loss_logits(n)
    inst = []
    for i, (b, kp) in enumerate(zip(boxes, kps)):
        out[f"boxes{i}"], out[f"kps{i}"] = b, kp
        it = Instances((800, 1333), proposal_boxes=Boxes(b.clone()), gt_keypoints=Keypoints(kp.clone()))
        inst.append(it)
        if len(b):
            t, v = Keypoints(kp.clone()).to_heatmap(b.clone(), S)
            out[f"target{i}"], out[f"valid{i}"] = t, v
    out["loss_none"] = kh.keypoint_rcnn_loss(logits.clone(), inst, None)
    out["loss_norm"] = kh.keypoint_rcnn_loss(logits.clone(), inst, 7.5)
    n2 = len(boxes[2])
    out["loss_no_valid"] = kh.keypoint_rcnn_loss(logits[n - n2:].clone(), [inst[2]], None)

    # detector_postprocess with keypoints: boxes partly outside the image, some empty after clipping
    h, w, oh, ow = 60, 90, 97, 141
    pb = torch.cat([torch.rand(9, 2, generator=g) * torch.tensor([w, h]), torch.zeros(9, 2)], dim=1)
    pb[:, 2:] = pb[:, :2] + torch.rand(9, 2, generator=g) * 40
    pb[2] = torch.tensor([95.0, 10.0, 120.0, 30.0])  # right of the image: empty after clipping
    pb[5] = torch.tensor([10.0, -30.0, 40.0, -2.0])  # above the image: empty after clipping
    pk = torch.cat([torch.rand(9, K, 2, generator=g) * torch.tensor([w, h]), torch.rand(9, K, 1, generator=g)], dim=2)
    scores, classes = torch.rand(9, generator=g), torch.randint(0, 3, (9,), generator=g)
    res = pp.detector_postprocess(Instances((h, w), pred_boxes=Boxes(pb.clone()), scores=scores.clone(),
                                            pred_classes=classes.clone(), pred_keypoints=pk.clone()), oh, ow)
    out.update(pp_hw=np.asarray([h, w, oh, ow]), pp_boxes=pb, pp_keypoints=pk, pp_scores=scores, pp_classes=classes,
               pp_out_boxes=res.pred_boxes.tensor, pp_out_keypoints=res.pred_keypoints)
    mg.save("keypoints", **out)


if __name__ == "__main__":
    main()
