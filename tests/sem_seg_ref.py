"""The semantic segmentation loss cases of tests/golden/sem_seg_loss.npz: inputs rebuilt from seeds on the CPU (shared by
tests/golden/make_golden_sem_seg.py and the tests)."""
import torch

# name: (N, C, Hp, Wp, stride, ignore, top_k (None = CrossEntropyLoss mean), weights, seed)
CASES = {
    "fpn_c54": (2, 54, 10, 13, 4, 255, None, False, 1),       # 255-ignored regions, image 1 fully ignored
    "all_ignored": (2, 5, 4, 5, 4, 255, None, False, 2),
    "c1": (1, 1, 5, 6, 4, 255, None, False, 3),
    "c19_stride16": (1, 19, 3, 4, 16, 255, None, False, 4),
    "odd": (2, 7, 7, 9, 4, 255, None, False, 5),
    "odd_stride3": (1, 7, 5, 7, 3, 255, None, False, 6),
    "stride1": (2, 4, 9, 11, 1, 255, None, False, 7),
    "ignore_m1": (2, 6, 6, 8, 4, -1, None, False, 8),
    "topk02": (2, 19, 8, 10, 4, 255, 0.2, False, 9),
    "topk02_weights": (2, 19, 8, 10, 4, 255, 0.2, True, 10),
    "topk1": (2, 19, 8, 10, 4, 255, 1.0, False, 11),
    "topk1_weights": (2, 19, 8, 10, 4, -1, 1.0, True, 12),
    "const_ties": (2, 8, 6, 7, 4, 255, 0.2, False, 13),       # constant logits: every valid pixel ties at log(C)
}


def make_case(name):
    """(logits, targets, weights) of a case, built on the CPU from its seed."""
    n, c, hp, wp, s, ignore, top_k, has_w, seed = CASES[name]
    g = torch.Generator().manual_seed(seed)
    h, w = hp * s, wp * s
    logits = torch.randn((n, c, hp, wp), generator=g) * 2.0
    if name == "const_ties":
        logits.fill_(0.375)
    targets = torch.randint(0, c, (n, h, w), generator=g)
    if name != "c1":
        targets[torch.rand((n, h, w), generator=g) < 0.15] = ignore  # scattered ignored pixels
    targets[:, : h // 4, : w // 3] = ignore                          # an ignored region
    if name == "fpn_c54":
        targets[1] = ignore
    if name == "all_ignored":
        targets.fill_(ignore)
    weights = (0.5 + 2.5 * torch.rand((n, h, w), generator=g)) if has_w else None
    return logits, targets, weights
