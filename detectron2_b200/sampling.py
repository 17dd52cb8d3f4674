"""Sampling of the training labels: subsample_labels (modeling/sampling.py:9-54) for all images at once.

The reference samples one image at a time: two `nonzero` host syncs and two `torch.randperm` calls per image (over the
~268 k negatives of an RPN image), then the gathers.  `subsample_labels_fixed` runs ONE `d2b_sample_labels` for the
batch (five launches, no host read): every candidate gets a SplitMix64 key derived from one device seed, and the sample is
the k smallest-key positives and negatives, each in ascending key order.  That is the reference's law -- a uniform random
subset in uniform random order, with the reference's counts -- but not torch.randperm's random stream.  The seed is drawn
from torch's CUDA generator on the labels' device, so `torch.manual_seed` governs the sample, and a CUDA-graph replay
draws a fresh one.  CUDA tensors only, like `matching.match_boxes_fixed`; `matching.subsample_labels` stays the
reference's own code, seed-exact with it.
"""
from typing import Optional

import torch

from . import ops

__all__ = ["subsample_labels_fixed", "draw_seed"]


def draw_seed(device) -> torch.Tensor:
    """A fresh [1] int64 seed on `device` from torch's current CUDA generator (no host read; graph-replay safe)."""
    return torch.empty((1,), dtype=torch.int64, device=device).random_()


def max_positive(num_samples: int, positive_fraction: float) -> int:
    """sampling.py:41: int(num_samples * positive_fraction) in Python float arithmetic (int(100 * 0.29) == 28)."""
    return int(num_samples * positive_fraction)


def sample_labels(labels: torch.Tensor, num_samples: int, positive_fraction: float, bg_label: int, *,
                  seed: Optional[torch.Tensor] = None, rpn_labels: bool = False):
    """d2b200::sample_labels with the reference's count rule and a default seed.  rpn_labels: return the RPN label map
    (1 / 0 / -1, rpn.py:296-303) instead of the index list."""
    if labels.dim() != 2:
        raise ValueError("sample_labels: labels must be [N, P]")
    if seed is None:
        seed = draw_seed(labels.device)
    out_labels, sampled, num_pos, num_neg = ops.sample_labels_op(
        labels, int(num_samples), max_positive(num_samples, positive_fraction), int(bg_label), seed, rpn_labels,
        not rpn_labels)
    return (out_labels if rpn_labels else sampled), num_pos, num_neg


def subsample_labels_fixed(labels: torch.Tensor, num_samples: int, positive_fraction: float, bg_label: int, *,
                           seed: Optional[torch.Tensor] = None):
    """subsample_labels for all images: labels [N, P] (int8 or int64; -1 ignored, bg_label negative, anything else
    positive).  Returns (sampled [N, num_samples] int64: each image's positive indices, then its negative ones, then -1
    padding; num_pos [N], num_neg [N] int64 device counts, those of the reference).  seed: [1] int64 device tensor (None:
    drawn from torch's CUDA generator).  No host read: capturable in a CUDA graph."""
    return sample_labels(labels, num_samples, positive_fraction, bg_label, seed=seed)
