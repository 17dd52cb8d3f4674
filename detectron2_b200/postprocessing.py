"""Mask target generation and detection post-processing around the RoIAlign / paste kernels (SURVEY 8f-4):

  * `crop_and_resize`      -- `BitMasks.crop_and_resize` (detectron2/structures/masks.py:193-224): Mask R-CNN training
                              targets, RoIAlign of every ground-truth bitmask with its own box, thresholded at 0.5;
  * `detector_postprocess` -- `detector_postprocess` (detectron2/modeling/postprocessing.py:9-74): boxes rescaled to the
                              output resolution, clipped, empty ones dropped, soft masks pasted into the output image.

Both are host glue over `layers.ROIAlign` / `layers.paste_masks_in_image` with the reference's expression order; the
containers (`Instances`, `Boxes`, `ROIMasks`) are out of scope, so tensors and the small `Detections` record are used.
"""
from typing import Optional, Tuple

import torch

from .fast_rcnn_inference import Detections
from .layers import ROIAlign, paste_masks_in_image

__all__ = ["crop_and_resize", "detector_postprocess", "PostprocessedDetections"]


def crop_and_resize(bit_masks: torch.Tensor, boxes: torch.Tensor, mask_size: int) -> torch.Tensor:
    """bit_masks (N, H, W) bool / uint8 / float, boxes (N, 4) -> (N, mask_size, mask_size) bool (masks.py:193-224)."""
    assert len(boxes) == len(bit_masks), "{} != {}".format(len(boxes), len(bit_masks))
    device = bit_masks.device
    batch_inds = torch.arange(len(boxes), device=device).to(dtype=boxes.dtype)[:, None]
    rois = torch.cat([batch_inds, boxes.to(device=device)], dim=1)  # N x 5: every mask is pooled with its own box
    masks = (bit_masks != 0).to(dtype=torch.float32)  # BitMasks stores `tensor.to(torch.bool)`: any nonzero value is 1
    output = ROIAlign((mask_size, mask_size), 1.0, 0, aligned=True).forward(masks[:, None, :, :], rois).squeeze(1)
    return output >= 0.5


class PostprocessedDetections(Detections):
    """`Detections` plus the optional full-resolution masks and rescaled keypoints `detector_postprocess` produces."""

    def __init__(self, image_size, pred_boxes, scores, pred_classes, pred_masks: Optional[torch.Tensor] = None,
                 pred_keypoints: Optional[torch.Tensor] = None):
        super().__init__(image_size, pred_boxes, scores, pred_classes)
        self.pred_masks = pred_masks
        self.pred_keypoints = pred_keypoints


def detector_postprocess(results: Detections, output_height: int, output_width: int, mask_threshold: float = 0.5,
                         pred_masks: Optional[torch.Tensor] = None,
                         pred_keypoints: Optional[torch.Tensor] = None) -> PostprocessedDetections:
    """results: detections at the resolution the detector saw (`results.image_size`); pred_masks: optional
    (N, 1, M, M) or (N, M, M) soft masks of the mask head; pred_keypoints: optional (N, K, 3) keypoints (x, y, score) of the
    keypoint head.  Returns the detections at (output_height, output_width):
    boxes scaled (Boxes.scale, boxes.py:271-276), clipped (Boxes.clip, :183-197), empty boxes removed
    (Boxes.nonempty, :199-213; the one data-dependent shape, as in the reference), masks pasted
    (ROIMasks.to_bitmasks -> paste_masks_in_image, masks.py:522-539) and keypoint x / y scaled (postprocessing.py:70-72)."""
    scale_x, scale_y = output_width / results.image_size[1], output_height / results.image_size[0]
    boxes = results.pred_boxes.clone()
    boxes[:, 0::2] *= scale_x
    boxes[:, 1::2] *= scale_y
    assert torch.isfinite(boxes).all(), "Box tensor contains infinite or NaN!"
    x1 = boxes[:, 0].clamp(min=0, max=output_width)
    y1 = boxes[:, 1].clamp(min=0, max=output_height)
    x2 = boxes[:, 2].clamp(min=0, max=output_width)
    y2 = boxes[:, 3].clamp(min=0, max=output_height)
    boxes = torch.stack((x1, y1, x2, y2), dim=-1)
    keep = ((boxes[:, 2] - boxes[:, 0]) > 0.0) & ((boxes[:, 3] - boxes[:, 1]) > 0.0)
    boxes = boxes[keep]
    masks = None
    if pred_masks is not None:
        soft = pred_masks[:, 0, :, :] if pred_masks.dim() == 4 else pred_masks
        masks = paste_masks_in_image(soft[keep], boxes, (output_height, output_width), threshold=mask_threshold)
    keypoints = None
    if pred_keypoints is not None:
        keypoints = pred_keypoints[keep]
        keypoints[:, :, 0] *= scale_x
        keypoints[:, :, 1] *= scale_y
    return PostprocessedDetections((output_height, output_width), boxes, results.scores[keep], results.pred_classes[keep],
                                   masks, keypoints)
