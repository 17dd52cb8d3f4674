"""ROIPooler -- the multi-level pooler of detectron2/modeling/poolers.py:114-263, as ONE kernel launch.

The reference assigns every box to an FPN level in Python (assign_boxes_to_levels, poolers.py:23-59) and then, per
level, runs nonzero (host sync) -> gather -> ROIAlign -> index_put_.  Here level assignment happens inside the
RoIAlign kernel (one CTA per RoI picks its level's feature map), so a pooler call is a single launch with no host
synchronisation, for the forward and for the backward.
"""
import math
from typing import List

import torch
from torch import nn

from . import ops
from .layers import ROIAlignRotated

__all__ = ["ROIPooler", "assign_boxes_to_levels", "convert_boxes_to_pooler_format", "pyramid_to_channels_last"]

pyramid_to_channels_last = ops.pyramid_to_channels_last


def _tensor_of(b):
    return b if isinstance(b, torch.Tensor) else b.tensor


def assign_boxes_to_levels(box_lists, min_level: int, max_level: int, canonical_box_size: int, canonical_level: int):
    """Host-side restatement of poolers.py:23-59 for callers that want the assignment vector itself.  Boxes are (x1, y1, x2, y2)
    or rotated (cx, cy, w, h, angle), whose area is w*h (RotatedBoxes.area, structures/rotated_boxes.py:236-245)."""
    boxes = torch.cat([_tensor_of(b) for b in box_lists], dim=0)
    if boxes.shape[1] == 5:
        sizes = torch.sqrt(boxes[:, 2] * boxes[:, 3])
    else:
        sizes = torch.sqrt((boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1]))
    lv = torch.floor(canonical_level + torch.log2(sizes / canonical_box_size + 1e-8))
    return torch.clamp(lv, min=min_level, max=max_level).to(torch.int64) - min_level


def convert_boxes_to_pooler_format(box_lists):
    """list of per-image (L_i, 4|5) boxes -> (M, 5|6) with the batch index in column 0 (poolers.py:72-98)."""
    tensors = [_tensor_of(b) for b in box_lists]
    # batch-index column built from host-side lengths: no repeat_interleave / device sync (cf. poolers.py:64-69)
    cols = [torch.cat([t.new_full((t.shape[0], 1), float(i)), t], dim=1) for i, t in enumerate(tensors)]
    return cols[0] if len(cols) == 1 else torch.cat(cols, dim=0)


class ROIPooler(nn.Module):
    def __init__(self, output_size, scales, sampling_ratio, pooler_type, canonical_box_size=224, canonical_level=4):
        """Same constructor as the reference (poolers.py:120-204).  pooler_type: "ROIAlign" (aligned=False),
        "ROIAlignV2" (aligned=True) or "ROIAlignRotated"; "ROIPool" is not on the hot path and not provided."""
        super().__init__()
        if isinstance(output_size, int):
            output_size = (output_size, output_size)
        assert len(output_size) == 2 and isinstance(output_size[0], int) and isinstance(output_size[1], int)
        self.output_size = output_size
        self.scales = [float(s) for s in scales]
        self.sampling_ratio = sampling_ratio
        if pooler_type not in ("ROIAlign", "ROIAlignV2", "ROIAlignRotated"):
            raise ValueError("Unknown pooler type: {}".format(pooler_type))
        self.pooler_type = pooler_type
        min_level = -(math.log2(scales[0]))
        max_level = -(math.log2(scales[-1]))
        assert math.isclose(min_level, int(min_level)) and math.isclose(max_level, int(max_level)), \
            "Featuremap stride is not power of 2!"
        self.min_level, self.max_level = int(min_level), int(max_level)
        assert len(scales) == self.max_level - self.min_level + 1, \
            "[ROIPooler] Sizes of input featuremaps do not form a pyramid!"
        assert 0 <= self.min_level <= self.max_level
        assert canonical_box_size > 0
        self.canonical_level = canonical_level
        self.canonical_box_size = canonical_box_size
        if pooler_type == "ROIAlignRotated":
            self.level_poolers = nn.ModuleList(
                ROIAlignRotated(output_size, spatial_scale=s, sampling_ratio=sampling_ratio) for s in scales)

    def forward(self, x: List[torch.Tensor], box_lists):
        assert isinstance(x, list) and isinstance(box_lists, list), "Arguments to pooler must be lists"
        assert len(x) == len(self.scales)
        assert len(box_lists) == x[0].size(0)
        if len(box_lists) == 0:
            return x[0].new_zeros((0, x[0].shape[1]) + tuple(self.output_size))
        rois = convert_boxes_to_pooler_format(box_lists)
        if self.pooler_type == "ROIAlignRotated":
            return self._forward_rotated(x, box_lists, rois)
        return ops.roi_pooler_op(list(x), rois, self.scales, self.output_size[0], self.output_size[1],
                                 int(self.sampling_ratio), self.pooler_type == "ROIAlignV2", self.min_level,
                                 self.max_level, self.canonical_level, float(self.canonical_box_size))

    def _forward_rotated(self, x, box_lists, rois):
        # one level: the ROIAlignRotated layer, as in the reference (poolers.py:245-246); several: one fused launch per
        # direction, the level of each rotated box (area = w*h, RotatedBoxes.area) picked in-kernel
        if len(self.scales) == 1:
            return self.level_poolers[0](x[0], rois)
        return ops.roi_pooler_rotated_op(list(x), rois, self.scales, self.output_size[0], self.output_size[1],
                                         int(self.sampling_ratio), self.min_level, self.max_level, self.canonical_level,
                                         float(self.canonical_box_size))
