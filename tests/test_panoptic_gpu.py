"""Panoptic FPN inference on the GPU: d2b_panoptic_combine against the reference fixture and against the torch restatement
on CUDA (realistic scenes: masks pasted by d2b_paste_masks from random boxes), the num_instances padding, reproducibility,
d2b_sem_seg_labels against F.interpolate + argmax on CUDA, a CUDA-graph capture of the pair, and panoptic_fpn_postprocess
against the reference-shaped composition."""
import pytest
import torch
from torch.nn import functional as F

from detectron2_b200 import panoptic as P
from detectron2_b200.fast_rcnn_inference import Detections
from detectron2_b200.layers import paste_masks_in_image
from detectron2_b200.postprocessing import detector_postprocess

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
C54 = 54


def _records(num_segments, seg_info, seg_score, n):
    k = int(num_segments[n])
    return [tuple(r) + (s,) for r, s in zip(seg_info[n, :k].tolist(), seg_score[n, :k].tolist())]


def _assert_same(scores, classes, masks, labels, thr, num_classes=C54, counts=None):
    """The kernel against the restatement on the same CUDA tensors: panoptic bit-exact, identical segment records."""
    pans, nseg, info, sc, status = P.combine_semantic_and_instance_outputs_fixed(
        scores, classes, masks, labels, num_classes, *thr, num_instances=counts)
    assert int(status.abs().sum()) == 0
    for n in range(len(labels)):
        cnt = None if counts is None else int(counts[n])
        want_pan, want = P._combine_host(scores[n], classes[n], masks[n], labels[n], *thr, count=cnt)
        assert torch.equal(pans[n], want_pan), n
        assert _records(nseg, info, sc, n) == want, n
        slots = info.shape[1]
        assert int(info[n, int(nseg[n]):].abs().sum()) == 0 and slots == max(m.shape[0] for m in masks) + num_classes
    return pans, nseg, info, sc


def test_combine_matches_reference_fixture(golden):
    gold = golden("panoptic")
    for name in gold["scenes"]:
        t = lambda k: torch.from_numpy(gold[name + "_" + k]).to(DEV)  # noqa: E731
        ov, st, sct = gold[name + "_thr"].tolist()
        labels = t("labels")
        inst = type("I", (), dict(scores=t("scores"), pred_classes=t("classes"), pred_masks=t("masks")))
        pan, info = P.combine_semantic_and_instance_outputs(inst, labels, ov, st, sct, num_classes=C54)
        assert torch.equal(pan.cpu(), torch.from_numpy(gold[name + "_panoptic"])), name
        got = [(d["id"], int(d["isthing"]), d["category_id"], d.get("instance_id", -1), d.get("area", 0)) for d in info]
        assert got == [tuple(r) for r in gold[name + "_records"].tolist()], name
        assert [d.get("score", 0.0) for d in info] == gold[name + "_record_scores"].tolist(), name


def _scene(g, h, w, r, num_classes=C54):
    """Masks pasted from random boxes by d2b_paste_masks, distinct random scores, blocky semantic labels."""
    ctr = torch.rand(r, 2, generator=g) * torch.tensor([w, h])
    wh = 4 + torch.rand(r, 2, generator=g) ** 2 * torch.tensor([w, h]) * 0.6
    boxes = torch.cat([ctr - wh / 2, ctr + wh / 2], 1).to(DEV)
    soft = torch.rand(r, 28, 28, generator=g).to(DEV)
    masks = paste_masks_in_image(soft, boxes, (h, w), 0.5)
    scores = (torch.randperm(100000, generator=g)[:r].float() / 100000.0).to(DEV)
    classes = torch.randint(0, 80, (r,), generator=g).to(DEV)
    coarse = torch.randint(0, num_classes, (1, 1, (h + 31) // 32, (w + 31) // 32), generator=g).float()
    labels = F.interpolate(coarse, size=(h, w), mode="nearest")[0, 0].long().to(DEV)
    return scores, classes, masks, labels


THRESHOLDS = [(0.5, 4096.0, 0.5), (0.3, 0.0, 0.1), (0.8, 500.0, 0.7), (1.0, 64.0, 0.0)]


@pytest.mark.parametrize("thr", THRESHOLDS)
def test_combine_matches_restatement_on_realistic_scenes(thr):
    g = torch.Generator().manual_seed(7)
    sizes = [(480, 640), (427, 640), (800, 1333), (1024, 2048)]
    parts = [_scene(g, h, w, 100) for h, w in sizes]
    _assert_same(*[list(x) for x in zip(*parts)], thr)


@pytest.mark.parametrize("thr", THRESHOLDS[:2])
def test_combine_small_and_large_instance_counts(thr):
    g = torch.Generator().manual_seed(8)
    parts = [_scene(g, 480, 640, 0), _scene(g, 427, 640, 1), _scene(g, 333, 517, 1), _scene(g, 64, 33, 0)]
    _assert_same(*[list(x) for x in zip(*parts)], thr)
    _assert_same(*[[x] for x in _scene(g, 480, 640, 1000)], thr)


def test_num_instances_padding_agrees_with_unpadded_inputs():
    g = torch.Generator().manual_seed(9)
    parts = [_scene(g, 427, 640, 60), _scene(g, 480, 640, 100), _scene(g, 200, 301, 0)]
    counts = torch.tensor([37, 100, 0], device=DEV)
    cut = [[x[:c] for x in p[:3]] + [p[3]] for p, c in zip(parts, counts.tolist())]
    pans, nseg, info, sc, status = P.combine_semantic_and_instance_outputs_fixed(
        *[list(x) for x in zip(*parts)], C54, num_instances=counts)
    pans2, nseg2, info2, sc2, _ = P.combine_semantic_and_instance_outputs_fixed(*[list(x) for x in zip(*cut)], C54)
    for n in range(3):
        assert torch.equal(pans[n], pans2[n])
        assert _records(nseg, info, sc, n) == _records(nseg2, info2, sc2, n)
    _assert_same(*[list(x) for x in zip(*parts)], (0.5, 4096.0, 0.5), counts=counts)


def test_repeated_runs_are_bitwise_identical():
    g = torch.Generator().manual_seed(10)
    inputs = [list(x) for x in zip(*[_scene(g, 800, 1333, 100), _scene(g, 480, 640, 100)])]
    first = P.combine_semantic_and_instance_outputs_fixed(*inputs, C54, 0.5, 0.0, 0.3)
    for _ in range(3):
        again = P.combine_semantic_and_instance_outputs_fixed(*inputs, C54, 0.5, 0.0, 0.3)
        assert all(torch.equal(a, b) for a, b in zip(first[0], again[0]))
        assert all(torch.equal(a, b) for a, b in zip(first[1:], again[1:]))


def test_bad_label_raises():
    g = torch.Generator().manual_seed(11)
    s, c, m, lab = _scene(g, 40, 50, 3)
    lab[3, 7] = C54
    inst = type("I", (), dict(scores=s, pred_classes=c, pred_masks=m))
    with pytest.raises(ValueError):
        P.combine_semantic_and_instance_outputs(inst, lab, 0.5, 0.0, 0.5, num_classes=C54)


def _sem_reference(logits, crops, outs):
    return [F.interpolate(r[:, :h, :w][None], size=o, mode="bilinear", align_corners=False)[0].argmax(0)
            for r, (h, w), o in zip(logits, crops, outs)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_sem_seg_labels_match_interpolate_argmax(dtype):
    g = torch.Generator().manual_seed(12)
    logits = (torch.randn(5, C54, 100, 168, generator=g) * 3).to(DEV, dtype)
    logits[1, :, 10:30, 20:50] = 0.5      # constant logits: every channel ties, label 0
    logits[2, 7, 40:44, 60:64] = float("nan")
    logits[2, 9, 41:45, 61:66] = float("nan")
    logits[3, 3, :, :] = -0.0
    logits[3, 4, :, :] = 0.0
    logits[3, :3] = -1.0
    logits[3, 5:] = -2.0
    crops = [(100, 168), (93, 151), (77, 131), (100, 168), (51, 97)]
    outs = [(800, 1344), (427, 640), (77, 131), (100, 168), (33, 41)]  # up, up (odd crop), same size, same, down
    got = P.sem_seg_labels(logits, crops, outs)
    for n, (a, b) in enumerate(zip(got, _sem_reference(logits, crops, outs))):
        assert torch.equal(a, b), (dtype, n, int((a != b).sum()))
    one = P.sem_seg_labels(logits[:1, :1], [(60, 70)], [(123, 45)])[0]  # C = 1
    assert int(one.abs().sum()) == 0


def test_graph_capture_replays_on_new_inputs():
    g = torch.Generator().manual_seed(13)
    crops, outs = [(200, 334), (180, 320)], [(480, 640), (427, 640)]
    logits = torch.randn(2, C54, 200, 336, generator=g).to(DEV)
    parts = [_scene(g, h, w, 50) for h, w in outs]
    scores, classes, masks, _ = [list(x) for x in zip(*parts)]
    counts = torch.tensor([50, 31], device=DEV)

    def step():
        labels = P.sem_seg_labels(logits, crops, outs)
        return P.combine_semantic_and_instance_outputs_fixed(scores, classes, masks, labels, C54, 0.5, 256.0, 0.2,
                                                             num_instances=counts)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = step()
    for seed in (14, 15):
        g2 = torch.Generator().manual_seed(seed)
        logits.copy_(torch.randn(logits.shape, generator=g2).to(DEV))
        for n, (h, w) in enumerate(outs):
            s, c, m, _ = _scene(g2, h, w, 50)
            scores[n].copy_(s), classes[n].copy_(c), masks[n].copy_(m)
        counts.copy_(torch.tensor([17, 50], device=DEV))
        graph.replay()
        eager = step()
        assert all(torch.equal(a, b) for a, b in zip(captured[0], eager[0]))
        assert all(torch.equal(a, b) for a, b in zip(captured[1:], eager[1:]))


def test_panoptic_fpn_postprocess_matches_the_reference_composition():
    g = torch.Generator().manual_seed(16)
    image_sizes, output_sizes = [(512, 683), (480, 640), (600, 400)], [(480, 640), (427, 640), (800, 533)]
    logits = torch.randn(3, C54, 152, 176, generator=g).to(DEV)  # the padded semantic head output (stride 4)
    logits = F.interpolate(logits, scale_factor=4, mode="bilinear", align_corners=False)[:, :, :608, :704]
    dets, probs = [], []
    for (h, w), r in zip(image_sizes, (40, 0, 100)):
        ctr = torch.rand(r, 2, generator=g) * torch.tensor([w, h])
        wh = 8 + torch.rand(r, 2, generator=g) * 200
        boxes = torch.cat([ctr - wh / 2, ctr + wh / 2], 1).to(DEV)
        dets.append(Detections((h, w), boxes, torch.rand(r, generator=g).to(DEV),
                               torch.randint(0, 80, (r,), generator=g).to(DEV)))
        probs.append(torch.rand(r, 1, 28, 28, generator=g).to(DEV))
    got = P.panoptic_fpn_postprocess(logits, dets, probs, image_sizes, output_sizes, return_sem_seg=True)
    for n, ((h, w), (oh, ow)) in enumerate(zip(image_sizes, output_sizes)):
        sem = F.interpolate(logits[n, :, :h, :w][None], size=(oh, ow), mode="bilinear", align_corners=False)[0]
        det = detector_postprocess(dets[n], oh, ow, pred_masks=probs[n])
        pan, records = P._combine_host(det.scores, det.pred_classes, det.pred_masks, sem.argmax(0), 0.5, 4096, 0.5)
        assert torch.equal(got[n]["sem_seg"], sem)
        assert torch.equal(got[n]["instances"].pred_masks, det.pred_masks)
        assert torch.equal(got[n]["panoptic_seg"][0], pan)
        assert got[n]["panoptic_seg"][1] == P._segments_info(records)
