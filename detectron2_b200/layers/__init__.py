"""Hot-path subset of `detectron2.layers` (detectron2/layers/__init__.py:2-24), H100-native.

Only the operators that sit on custom kernels are provided; plain-PyTorch helpers of the reference package
(norm layers, wrappers, losses, ...) are out of scope (SURVEY.md section 8).
"""
from .deform_conv import DeformBottleneckConv2, DeformConv, ModulatedDeformConv, deform_conv, modulated_deform_conv
from .mask_ops import paste_masks_in_image, paste_masks_in_image_packed, unpack_mask_bits
from .nms import batched_nms, batched_nms_fixed, batched_nms_images_fixed, batched_nms_rotated, nms, nms_rotated
from .roi_align import ROIAlign, roi_align
from .roi_align_rotated import ROIAlignRotated, roi_align_rotated
from .rotated_boxes import pairwise_iou_rotated

__all__ = [k for k in globals().keys() if not k.startswith("_")]
