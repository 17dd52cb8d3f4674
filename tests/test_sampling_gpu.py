"""d2b_sample_labels on the GPU: bit-exact against the numpy restatement (tests/sampling_ref.py) at the RPN and ROI-head
sizes, against the reference's subsample_labels on CUDA where the two must agree, the sampling law over 4 096 identical
images, and the sync-free training-target chains (matching -> sampling -> pooler -> loss) eagerly under the sync debug
mode and replayed in one CUDA graph."""
import numpy as np
import pytest
import torch

import sampling_ref as sr

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def _seed(s: int) -> torch.Tensor:
    return torch.tensor([s], dtype=torch.int64, device=DEV)


def _boxes(g, k, w=1344.0, h=800.0, lo=16.0, hi=512.0):
    ctr = torch.rand(k, 2, generator=g) * torch.tensor([w, h])
    wh = lo + torch.rand(k, 2, generator=g) * (hi - lo)
    return torch.cat([ctr - wh / 2, ctr + wh / 2], 1)


def _rboxes(g, k, w=1344.0, h=800.0):
    ctr = torch.rand(k, 2, generator=g) * torch.tensor([w, h])
    wh = 16 + torch.rand(k, 2, generator=g) * 300
    return torch.cat([ctr, wh, (torch.rand(k, 1, generator=g) - 0.5) * 180], 1)


def _sample(labels, num_samples, frac, bg, seed):
    from detectron2_b200 import ops
    from detectron2_b200.sampling import max_positive

    return ops.sample_labels_op(labels, num_samples, max_positive(num_samples, frac), bg, _seed(seed), True, True)


def _check_exact(labels, num_samples, frac, bg, seed):
    from detectron2_b200.sampling import max_positive, subsample_labels_fixed

    out_labels, sampled, num_pos, num_neg = _sample(labels, num_samples, frac, bg, seed)
    ref_s, ref_p, ref_n, ref_l = sr.subsample(labels.cpu().numpy(), num_samples, max_positive(num_samples, frac), bg, seed)
    assert np.array_equal(num_pos.cpu().numpy(), ref_p) and np.array_equal(num_neg.cpu().numpy(), ref_n)
    assert np.array_equal(sampled.cpu().numpy(), ref_s)
    assert np.array_equal(out_labels.cpu().numpy(), ref_l)
    # either output form alone gives the same sample
    s2, p2, n2 = subsample_labels_fixed(labels, num_samples, frac, bg, seed=_seed(seed))
    assert torch.equal(s2, sampled) and torch.equal(p2, num_pos) and torch.equal(n2, num_neg)
    from detectron2_b200 import ops

    l3 = ops.sample_labels_op(labels, num_samples, max_positive(num_samples, frac), bg, _seed(seed), True, False)[0]
    assert torch.equal(l3, out_labels)
    return sampled, num_pos, num_neg


def _check_against_reference(labels, sampled, num_pos, num_neg, num_samples, frac, bg):
    """The reference's subsample_labels on CUDA: the same counts; the same positive SET when every positive is taken;
    ours distinct, of the right set, fg before bg, -1 padding."""
    from detectron2_b200.matching import subsample_labels

    max_pos = int(num_samples * frac)
    for n in range(labels.shape[0]):
        lab = labels[n]
        pos, neg = subsample_labels(lab, num_samples, frac, bg)
        kp, kn = int(num_pos[n]), int(num_neg[n])
        assert (kp, kn) == (pos.numel(), neg.numel())
        s = sampled[n].cpu()
        fg, bgs, pad = s[:kp], s[kp:kp + kn], s[kp + kn:]
        lc = lab.cpu().to(torch.int64)
        assert bool(((lc[fg] != -1) & (lc[fg] != bg)).all()) and bool((lc[bgs] == bg).all()) and bool((pad == -1).all())
        assert len(set(s[:kp + kn].tolist())) == kp + kn
        npos = int(((lc != -1) & (lc != bg)).sum())
        if npos <= max_pos:
            assert set(fg.tolist()) == set(pos.cpu().tolist())


def test_rpn_size_from_match_boxes():
    """2 x 268 569 anchors labelled by match_boxes_fixed (int8), 256 per image, half positive."""
    from detectron2_b200 import matching as mt

    g = torch.Generator().manual_seed(0)
    anchors = _boxes(g, 268569).to(DEV)
    gt = torch.stack([_boxes(g, 7, lo=64, hi=400), _boxes(g, 7, lo=64, hi=400)]).to(DEV)
    count = torch.tensor([7, 3], device=DEV)
    _, labels, _, _, _ = mt.match_boxes_fixed(gt, count, anchors, mt.Matcher([0.3, 0.7], [0, -1, 1], True))
    assert labels.dtype == torch.int8 and int((labels == 1).sum()) > 0
    for seed in (0, 12345, -7):
        sampled, p, n = _check_exact(labels, 256, 0.5, 0, seed)
    _check_against_reference(labels, sampled, p, n, 256, 0.5, 0)


@pytest.mark.parametrize("rotated", [False, True])
def test_roi_size_from_match_boxes(rotated):
    """2 x (2000 + G) proposals ++ GT with 80 classes (int64, bg_label 80), 512 per image, a quarter foreground."""
    from detectron2_b200 import matching as mt

    g = torch.Generator().manual_seed(1)
    mk = _rboxes if rotated else _boxes
    props = torch.stack([mk(g, 2000), mk(g, 2000)]).to(DEV)
    gt = torch.stack([mk(g, 40), mk(g, 40)]).to(DEV)
    gcount = torch.tensor([40, 13], device=DEV)
    pcount = torch.tensor([2000, 1777], device=DEV)
    gcls = torch.randint(0, 80, (2, 40), generator=g).to(DEV)
    _, _, _, classes, _ = mt.match_boxes_fixed(gt, gcount, props, mt.Matcher([0.5], [0, 1], False), pred_count=pcount,
                                               append_gt=True, gt_classes=gcls, num_classes=80)
    sampled, p, n = _check_exact(classes, 512, 0.25, 80, 99)
    _check_against_reference(classes, sampled, p, n, 512, 0.25, 80)


CASES = [  # N, P, dtype, bg_label, num_samples, positive_fraction, P(pos), P(neg)
    (1, 1000, torch.int8, 0, 256, 0.5, 0.05, 0.9),
    (3, 4099, torch.int64, 80, 512, 0.25, 0.3, 0.5),
    (16, 777, torch.int64, 5, 64, 0.29, 0.1, 0.3),
    (5, 8193, torch.int8, 2, 100, 0.29, 0.6, 0.3),
    (2, 300, torch.int64, 3, 512, 0.5, 0.2, 0.2),  # fewer candidates than num_samples
    (4, 2000, torch.int8, 0, 0, 0.5, 0.3, 0.3),    # num_samples 0
    (2, 0, torch.int64, 0, 16, 0.5, 0.3, 0.3),     # no candidates at all
]


@pytest.mark.parametrize("case", CASES, ids=[f"N{c[0]}-P{c[1]}-{str(c[2])[6:]}-bg{c[3]}-S{c[4]}" for c in CASES])
def test_random_labels_bit_exact(case):
    n, p, dtype, bg, ns, frac, ppos, pneg = case
    g = torch.Generator().manual_seed(n * 1000 + p)
    u = torch.rand(n, p, generator=g)
    fg = torch.randint(0, 80, (n, p), generator=g)
    fg = torch.where(fg == bg, fg + 1, fg) if dtype == torch.int64 else torch.where(fg % 2 == 0, 1, 3) if bg == 2 else \
        torch.ones_like(fg)
    labels = torch.where(u < ppos, fg, torch.where(u < ppos + pneg, torch.full_like(fg, bg), torch.full_like(fg, -1)))
    labels = labels.to(dtype).to(DEV)
    for seed in (3, 2**62 + 17):
        sampled, np_, nn_ = _check_exact(labels, ns, frac, bg, seed)
    if p:
        _check_against_reference(labels, sampled, np_, nn_, ns, frac, bg)


def test_threshold_bin_overflow_is_refined_exactly():
    """3 M candidates per image: the smallest keys' top-digit bin holds more candidates than its buffer, so the kernel
    refines it by the next key digits (image 0: negatives, image 1: positives)."""
    p = 3_000_000
    labels = torch.zeros((2, p), dtype=torch.int8)
    labels[1] = 1
    labels[0, ::1000] = 1
    labels[1, ::997] = 0
    labels[:, 5::7919] = -1
    _check_exact(labels.to(DEV), 512, 0.5, 0, 2024)
    # every candidate positive and a sample of the whole image
    _check_exact(torch.ones((1, p), dtype=torch.int8, device=DEV), 8192, 1.0, 0, 5)


def test_law_over_identical_images():
    """4 096 identical images in one launch (P = 64, 10 positives, 54 negatives, at most 4 positives of 8): each positive's
    inclusion and first-slot frequencies stay within 5 binomial standard deviations."""
    from detectron2_b200.sampling import subsample_labels_fixed

    n = 4096
    row = torch.zeros(64, dtype=torch.int64)
    pos = torch.arange(3, 63, 6)  # 10 positives spread over the row
    row[pos] = 1
    labels = row.repeat(n, 1).to(DEV)
    sampled, num_pos, num_neg = subsample_labels_fixed(labels, 8, 0.5, 0, seed=_seed(77))
    assert bool((num_pos == 4).all()) and bool((num_neg == 4).all())
    fg = sampled[:, :4].cpu()
    for i in pos.tolist():
        inc = int((fg == i).any(dim=1).sum())
        first = int((fg[:, 0] == i).sum())
        for count, prob in ((inc, 0.4), (first, 0.1)):
            mean, sd = n * prob, (n * prob * (1 - prob)) ** 0.5
            assert abs(count - mean) <= 5 * sd, (i, count, mean)
    # the images draw different samples
    assert len({tuple(r) for r in fg.tolist()}) > n // 2


def _rpn_inputs(g, n=2, a=268569):
    anchors = _boxes(g, a).to(DEV)
    gt = torch.stack([_boxes(g, 9, lo=64, hi=400) for _ in range(n)]).to(DEV)
    count = torch.tensor([9, 4][:n], device=DEV)
    logits = [torch.randn(n, a, generator=g).to(DEV)]
    deltas = [(torch.randn(n, a, 4, generator=g) * 0.1).to(DEV)]
    return anchors, gt, count, logits, deltas


def _rpn_chain(anchors, gt, count, logits, deltas, seed):
    from detectron2_b200 import losses, matching as mt

    labels, boxes = mt.rpn_label_and_sample_anchors_fixed(anchors, gt, count, mt.Matcher([0.3, 0.7], [0, -1, 1], True),
                                                          256, 0.5, seed=seed)
    l, num_pos, num_neg, status = losses.rpn_losses_fixed(anchors, logits, labels, deltas, boxes, batch_size_per_image=256)
    return labels, l["loss_rpn_cls"], l["loss_rpn_loc"], num_pos, num_neg, status


def _roi_inputs(g, n=2, pmax=2000, gmax=20, c=16, k=80):
    props = torch.stack([_boxes(g, pmax) for _ in range(n)]).to(DEV)
    gt = torch.stack([_boxes(g, gmax, lo=64, hi=400) for _ in range(n)]).to(DEV)
    gcount = torch.tensor([gmax, gmax // 2][:n], device=DEV)
    gcls = torch.randint(0, k, (n, gmax), generator=g).to(DEV)
    feats = [torch.randn(n, c, 200 // s, 336 // s, generator=g).to(DEV).requires_grad_(True) for s in (1, 2, 4, 8)]
    w_cls = (torch.randn(c * 49, k + 1, generator=g) * 0.01).to(DEV)
    w_box = (torch.randn(c * 49, 4 * k, generator=g) * 0.01).to(DEV)
    return props, gt, gcount, gcls, feats, w_cls, w_box


def _roi_chain(props, pcount, gt, gcount, gcls, feats, w_cls, w_box, seed, b=512):
    from detectron2_b200 import losses, matching as mt
    from detectron2_b200.poolers import ROIPooler

    out = mt.label_and_sample_proposals_fixed(props, pcount, gt, gcount, gcls, mt.Matcher([0.5], [0, 1], False), 80, b,
                                              0.25, seed=seed)
    sampled, cls, _, pboxes, gboxes, num_fg, num_bg = out
    pooler = ROIPooler(7, [1 / 4, 1 / 8, 1 / 16, 1 / 32], 0, "ROIAlignV2")
    pooled = pooler(feats, list(pboxes.unbind(0)))
    x = pooled.flatten(1)
    l, counts, status = losses.fast_rcnn_losses_fixed(x @ w_cls, x @ w_box, pboxes.reshape(-1, 4), gboxes.reshape(-1, 4),
                                                      cls.reshape(-1))
    return sampled, pooled, l["loss_cls"], l["loss_box_reg"], num_fg, num_bg, status


def test_chains_run_without_host_sync():
    g = torch.Generator().manual_seed(5)
    rpn = _rpn_inputs(g)
    roi = _roi_inputs(g)
    props, gt, gcount, gcls, feats, w_cls, w_box = roi
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        r = _rpn_chain(*rpn, None)  # seed drawn from torch's CUDA generator
        o = _roi_chain(props, None, gt, gcount, gcls, feats, w_cls, w_box, None)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    labels, cls_loss, loc_loss, num_pos, num_neg, status = r
    assert int(status) == 0 and torch.isfinite(cls_loss) and torch.isfinite(loc_loss)
    # the loss counts the sampled anchors of the batch: 1 -> positive, 0 -> negative, at most 256 per image
    assert int((labels == 1).sum()) == int(num_pos) > 0 and int((labels == 0).sum()) == int(num_neg)
    assert bool(((labels >= 0).sum(1) <= 256).all()) and bool(((labels == 1).sum(1) <= 128).all())
    sampled, pooled, lc, lb, num_fg, num_bg, st = o
    assert bool((num_fg + num_bg == 512).all()) and int(st) == 0 and torch.isfinite(lc) and torch.isfinite(lb)
    # torch.manual_seed governs the default seed
    torch.manual_seed(11)
    a = _rpn_chain(*rpn, None)[0]
    torch.manual_seed(11)
    assert torch.equal(_rpn_chain(*rpn, None)[0], a)


def test_chains_in_one_cuda_graph():
    """match -> sample -> loss (RPN) and match -> sample -> pooler -> loss (ROI heads) captured in one graph; the seed
    tensor is refilled before each replay, and each replay equals the eager run with that seed."""
    g = torch.Generator().manual_seed(6)
    rpn = _rpn_inputs(g)
    props, gt, gcount, gcls, feats, w_cls, w_box = _roi_inputs(g)
    pcount = torch.tensor([2000, 1500], device=DEV)
    seed = _seed(0)

    def step():
        return _rpn_chain(*rpn, seed) + _roi_chain(props, pcount, gt, gcount, gcls, feats, w_cls, w_box, seed)

    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            step()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.no_grad():
        with torch.cuda.graph(graph):
            outs = step()
    results = {}
    for s in (1, 2, 1):
        seed.fill_(s)
        graph.replay()
        torch.cuda.synchronize()
        with torch.no_grad():
            eager = step()
        for x, y in zip(outs, eager):
            assert torch.equal(x, y)
        results.setdefault(s, [o.clone() for o in outs])
    assert not torch.equal(results[1][0], results[2][0])  # RPN labels
    assert not torch.equal(results[1][6], results[2][6])  # ROI sampled indices
    for x, y in zip(results[1], [o for o in outs]):
        assert torch.equal(x, y)


def test_padded_roi_rows_pool_to_zero_without_gradient():
    """Few proposals: the sample is padded.  Padding rows have index / class / match -1, NaN boxes that pool to zeros,
    and the feature gradient equals that of the valid rows alone."""
    from detectron2_b200 import matching as mt
    from detectron2_b200.poolers import ROIPooler

    g = torch.Generator().manual_seed(7)
    props, gt, gcount, gcls, feats, _, _ = _roi_inputs(g, pmax=60, gmax=6)
    pcount = torch.tensor([60, 25], device=DEV)
    sampled, cls, match, pboxes, gboxes, num_fg, num_bg = mt.label_and_sample_proposals_fixed(
        props, pcount, gt, gcount, gcls, mt.Matcher([0.5], [0, 1], False), 80, 512, 0.25, seed=_seed(3))
    valid = sampled >= 0
    assert torch.equal(valid.sum(1), num_fg + num_bg) and int(valid.sum()) < valid.numel()
    assert bool((cls[~valid] == -1).all()) and bool((match[~valid] == -1).all()) and bool(pboxes[~valid].isnan().all())
    assert bool((cls[valid] >= 0).all()) and bool((gboxes[~valid] == 0).all())
    # fg rows first: classes < 80 in [0, num_fg), background after
    for n in range(2):
        f = int(num_fg[n])
        assert bool((cls[n, :f] < 80).all()) and bool((cls[n, f:int(num_fg[n] + num_bg[n])] == 80).all())
    # the sampled rows are the proposals ++ GT rows they index
    for n in range(2):
        rows = torch.cat([props[n, :int(pcount[n])], gt[n]])
        idx = sampled[n][valid[n]]
        assert torch.equal(pboxes[n][valid[n]], rows[idx])
    pooler = ROIPooler(7, [1 / 4, 1 / 8, 1 / 16, 1 / 32], 0, "ROIAlignV2")
    pooled = pooler(feats, list(pboxes.unbind(0)))
    flat_valid = valid.reshape(-1)
    assert bool((pooled[~flat_valid] == 0).all())
    pooled.sum().backward()
    grads = [f.grad.clone() for f in feats]
    for f in feats:
        f.grad = None
    pooler(feats, [pboxes[n][valid[n]] for n in range(2)]).sum().backward()
    for a, b in zip(grads, feats):
        assert torch.allclose(a, b.grad, rtol=1e-5, atol=1e-5)
