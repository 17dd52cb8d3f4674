"""ctypes binding of libd2b200.so -- the C-ABI drop-in boundary declared in include/d2b200.h.

This module plays the role of ``detectron2._C`` (csrc/vision.cpp:81-113) for the hot path: it is the only place
where the Python host touches native code.  There is NO CPU fallback: if the library is missing or a tensor is not
on a CUDA device the call raises.
"""
import ctypes as C
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libd2b200.so")

_lib = None

D2B_ERRORS = {-1: "invalid argument", -2: "workspace too small", -3: "unsupported configuration"}


class DcnParams(C.Structure):
    _fields_ = [(n, C.c_int) for n in ("N", "Cin", "H", "W", "Cout", "kh", "kw", "stride_h", "stride_w", "pad_h",
                                        "pad_w", "dil_h", "dil_w", "groups", "deformable_groups")]


MAX_LEVELS = 8
MAX_IMAGES = 64  # D2B_MAX_IMAGES
ABI_VERSION = 7  # include/d2b200.h D2B_ABI_VERSION
DCN_X_NHWC = 1   # D2B_DCN_X_NHWC
ROI_ROTATED, ROI_BACKWARD, ROI_NHWC = 1, 2, 4  # D2B_ROI_ROTATED / D2B_ROI_BACKWARD / D2B_ROI_NHWC
DTYPE_CODE = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}  # D2B_F32 / D2B_F16 / D2B_BF16
MATCH_ROTATED, MATCH_LOW_QUALITY, MATCH_APPEND_GT = 1, 2, 4  # D2B_MATCH_*
MATCH_MAX_THRESHOLDS = 8  # D2B_MATCH_MAX_THRESHOLDS
SELECT_ROTATED, SELECT_SEG_PER_IMAGE, SELECT_NO_OFFSETS, SELECT_LINEAR = 1, 2, 4, 8  # D2B_SELECT_*


class Pyramid(C.Structure):
    _fields_ = [("num_levels", C.c_int), ("feat", C.c_void_p * MAX_LEVELS), ("grad", C.c_void_p * MAX_LEVELS),
                ("H", C.c_int * MAX_LEVELS), ("W", C.c_int * MAX_LEVELS), ("scale", C.c_float * MAX_LEVELS),
                ("min_level", C.c_int), ("max_level", C.c_int), ("canonical_level", C.c_int),
                ("canonical_box_size", C.c_float), ("level_rois", C.c_void_p)]


class RpnLevels(C.Structure):
    _fields_ = [("num_levels", C.c_int), ("proposals", C.c_void_p * MAX_LEVELS), ("topk_idx", C.c_void_p * MAX_LEVELS),
                ("topk_scores", C.c_void_p * MAX_LEVELS), ("A", C.c_int * MAX_LEVELS), ("k", C.c_int * MAX_LEVELS)]


class DenseLevels(C.Structure):
    _fields_ = [("num_levels", C.c_int), ("anchors", C.c_void_p * MAX_LEVELS), ("deltas", C.c_void_p * MAX_LEVELS),
                ("topk_idx", C.c_void_p * MAX_LEVELS), ("topk_scores", C.c_void_p * MAX_LEVELS),
                ("R", C.c_int * MAX_LEVELS), ("k", C.c_int * MAX_LEVELS)]


LABELS_I8, LABELS_I64 = 0, 1  # D2B_LABELS_*
SAMPLE_MAX_SAMPLES = 8192  # D2B_SAMPLE_MAX_SAMPLES
POLYGON_MAX_S = 256  # D2B_POLYGON_MAX_S
LOSS_STATUS_INVALID_BOX, LOSS_STATUS_INVALID_CLASS, LOSS_STATUS_INVALID_BOX_ORDER = 1, 2, 4  # D2B_LOSS_STATUS_*
LOSS_TYPES = {"smooth_l1": 0, "giou": 1}  # D2B_LOSS_SMOOTH_L1 / D2B_LOSS_GIOU: the box_reg_loss_type values with a kernel
LOSS_LINEAR_GIOU = 2  # D2B_LOSS_LINEAR_GIOU: FCOS, dense only


class DenseLossLevels(C.Structure):
    _fields_ = [("num_levels", C.c_int), ("logits", C.c_void_p * MAX_LEVELS), ("deltas", C.c_void_p * MAX_LEVELS),
                ("grad_logits", C.c_void_p * MAX_LEVELS), ("grad_deltas", C.c_void_p * MAX_LEVELS),
                ("ctr", C.c_void_p * MAX_LEVELS), ("grad_ctr", C.c_void_p * MAX_LEVELS), ("R", C.c_int * MAX_LEVELS)]


class SemSegImages(C.Structure):
    _fields_ = [("h", C.c_int * MAX_IMAGES), ("w", C.c_int * MAX_IMAGES), ("H", C.c_int * MAX_IMAGES),
                ("W", C.c_int * MAX_IMAGES), ("labels", C.c_void_p * MAX_IMAGES)]


class PanopticImages(C.Structure):
    _fields_ = [("R", C.c_int * MAX_IMAGES), ("H", C.c_int * MAX_IMAGES), ("W", C.c_int * MAX_IMAGES),
                ("scores", C.c_void_p * MAX_IMAGES), ("classes", C.c_void_p * MAX_IMAGES),
                ("masks", C.c_void_p * MAX_IMAGES), ("labels", C.c_void_p * MAX_IMAGES),
                ("panoptic", C.c_void_p * MAX_IMAGES)]


def _declare(lib):
    vp, f32p, i64p, u8p = C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p
    i, f, d, sz, i64 = C.c_int, C.c_float, C.c_double, C.c_size_t, C.c_int64
    sig = {
        "d2b_abi_version": (i, []),
        "d2b_cuda_version": (i, []),
        "d2b_arch": (C.c_char_p, []),
        "d2b_roi_pooler_forward": (i, [C.POINTER(Pyramid), i, i, f32p, i, i, i, i, i, i, vp, i, vp]),
        "d2b_roi_pooler_backward": (i, [C.POINTER(Pyramid), i, i, vp, i, f32p, i, i, i, i, i, i, vp]),
        "d2b_pyramid_nchw_to_nhwc": (i, [C.POINTER(Pyramid), i, i, C.POINTER(C.c_void_p), i, vp]),
        "d2b_pyramid_nhwc_to_nchw": (i, [C.POINTER(Pyramid), i, i, C.POINTER(C.c_void_p), i, vp]),
        "d2b_roi_pooler_nhwc_supported": (i, [C.POINTER(Pyramid), i, i, i, i]),
        "d2b_nms_workspace_bytes": (sz, [i64, i, i64]),
        "d2b_nms": (i, [f32p, f32p, i64p, i64, d, i, i64, i64p, i64p, vp, sz, vp]),
        "d2b_rpn_prepare": (i, [C.POINTER(RpnLevels), i, f32p, f, i, f32p, f32p, f32p, f32p, i64p, vp, vp]),
        "d2b_rpn_select": (i, [i64p, i64p, i, i, i, i, f32p, f32p, i64p, f32p, f32p, i64p, i64p, vp]),
        "d2b_frcnn_prepare": (i, [f32p, f32p, C.POINTER(C.c_int), i, i, i, f32p, f, i, i, f32p, f32p, f32p, f32p, i64p, i64p,
                                  i64p, i64p, vp]),
        "d2b_dense_prepare": (i, [C.POINTER(DenseLevels), i, i, C.POINTER(C.c_float), f, i, f32p, f32p, f32p, f32p, i64p,
                                  i64p, vp]),
        "d2b_mask_loss_forward": (i, [f32p, i, i, i, u8p, i, i, i, f32p, i64p, i64p, f32p, u8p, vp]),
        "d2b_mask_loss_backward": (i, [f32p, i, i, i, u8p, i64p, f32p, f32p, vp]),
        "d2b_polygons_crop_and_resize": (i, [vp, i, vp, i, vp, i, f32p, i64p, i, i, u8p, vp]),
        "d2b_polygons_to_bitmask": (i, [vp, i, vp, i, vp, i, i, i, u8p, vp]),
        "d2b_mask_loss_polygons_forward": (i, [f32p, i, i, i, vp, i, vp, i, vp, i, f32p, i64p, i64p, f32p, u8p, vp]),
        "d2b_keypoints_workspace_bytes": (sz, [i, i]),
        "d2b_keypoints_from_heatmaps": (i, [f32p, i, i, i, f32p, f32p, vp, sz, vp]),
        "d2b_keypoint_loss_forward": (i, [vp, i, i, i, i, f32p, f32p, i64p, u8p, f32p, i64p, vp]),
        "d2b_keypoint_loss_backward": (i, [vp, i, i, i, i, i64p, u8p, f32p, vp, vp]),
        "d2b_dense_loss_workspace_bytes": (sz, [C.POINTER(DenseLossLevels), i, i, i]),
        "d2b_dense_loss_forward": (i, [C.POINTER(DenseLossLevels), i, i, i, i, f32p, f32p, vp, i, f, f, f, i, f,
                                       C.POINTER(C.c_float), f32p, i64p, vp, vp, sz, vp]),
        "d2b_dense_loss_backward": (i, [C.POINTER(DenseLossLevels), i, i, i, i, f32p, f32p, vp, i, f, f, f, i, f,
                                        C.POINTER(C.c_float), f32p, vp]),
        "d2b_frcnn_loss_workspace_bytes": (sz, [i]),
        "d2b_frcnn_loss_forward": (i, [vp, vp, i, i, i, i, i, f32p, f32p, i64p, f, i, f, C.POINTER(C.c_float), f32p, i64p, vp,
                                       vp, sz, vp]),
        "d2b_frcnn_loss_backward": (i, [vp, vp, i, i, i, i, i, f32p, f32p, i64p, f, i, f, C.POINTER(C.c_float), f32p, vp, vp,
                                        vp]),
        "d2b_box_iou_rotated": (i, [f32p, i64, f32p, i64, f32p, vp]),
        "d2b_match_workspace_bytes": (sz, [i, i, i]),
        "d2b_match_boxes": (i, [f32p, i64p, i, i, f32p, i64, i64p, i, C.POINTER(C.c_double), i, C.POINTER(C.c_int), i, f32p, d,
                                i64p, i64, i64p, vp, f32p, i64p, vp, vp, sz, vp]),
        "d2b_fcos_assign": (i, [f32p, C.POINTER(C.c_int), i, f32p, i64p, i, i, i64p, i64, d, i64p, i64p, f32p, vp]),
        "d2b_sample_labels_workspace_bytes": (sz, [i, i, i]),
        "d2b_sample_labels": (i, [vp, i, i, i, i64, i, i, vp, vp, i64p, i64p, i64p, vp, sz, vp]),
        "d2b_deform_conv_tc_shape_supported": (i, [C.POINTER(DcnParams), i]),
        "d2b_deform_conv_forward_workspace_bytes": (sz, [C.POINTER(DcnParams), i, i]),
        "d2b_deform_conv_cols_bytes": (sz, [C.POINTER(DcnParams), i]),
        "d2b_deform_conv_forward": (i, [f32p, f32p, f32p, f32p, f32p, C.POINTER(DcnParams), i, i, f32p, vp, vp, sz, vp]),
        "d2b_deform_conv_backward_workspace_bytes": (sz, [C.POINTER(DcnParams), i, i, i, i]),
        "d2b_deform_conv_backward": (i, [f32p, f32p, f32p, f32p, f32p, C.POINTER(DcnParams), i, i, vp, f32p, f32p, f32p,
                                         f32p, f32p, vp, sz, vp]),
        "d2b_deform_conv_fused_forward": (i, [f32p, f32p, f32p, f32p, f32p, i, C.POINTER(DcnParams), i, i, f32p, vp, vp, sz,
                                              vp]),
        "d2b_deform_conv_fused_backward": (i, [f32p, f32p, f32p, f32p, i, f32p, f32p, C.POINTER(DcnParams), i, i, vp, f32p,
                                               f32p, f32p, vp, sz, vp]),
        "d2b_sem_seg_labels": (i, [vp, i, i, i, i, i, C.POINTER(SemSegImages), vp]),
        "d2b_panoptic_workspace_bytes": (sz, [C.POINTER(PanopticImages), i, i]),
        "d2b_panoptic_combine": (i, [C.POINTER(PanopticImages), i, i, i64p, d, d, d, i64p, i64p, f32p, vp, vp, sz, vp]),
        "d2b_sem_seg_loss_workspace_bytes": (sz, [i, i, i, i, i, i, i, d]),
        "d2b_sem_seg_loss_forward": (i, [vp, i, i, i, i, i, i, i64p, i64, i, d, f32p, f32p, u8p, f32p, i64p, vp, vp, sz,
                                         vp]),
        "d2b_sem_seg_loss_backward": (i, [vp, i, i, i, i, i, i, i64p, i64, f32p, u8p, f32p, f32p, vp, vp]),
        "d2b_paste_masks": (i, [f32p, f32p, i, i, i, i, f, u8p, vp]),
        "d2b_paste_masks_packed": (i, [f32p, f32p, i, i, i, i, f, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)  # AttributeError here == symbol missing from the .so
        fn.restype = res
        fn.argtypes = args
    return sig


EXPORTED = None


def lib():
    """Load (once) and return the native library.  Raises if it cannot be loaded -- never falls back."""
    global _lib, EXPORTED
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "detectron2_b200: native library %s is missing. Build it with `python -m detectron2_b200.build` "
                "(or __graft_entry__.build()). There is no CPU / PyTorch fallback for these ops." % LIB_PATH)
        l = C.CDLL(LIB_PATH)
        EXPORTED = _declare(l)
        if l.d2b_abi_version() != ABI_VERSION:
            raise RuntimeError("libd2b200.so ABI version mismatch")
        _lib = l
    return _lib


def check(rc, what):
    if rc == 0:
        return
    if rc < 0:
        raise RuntimeError("%s: %s (d2b error %d)" % (what, D2B_ERRORS.get(rc, "error"), rc))
    raise RuntimeError("%s: CUDA error %d" % (what, rc))


def stream_ptr(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise NotImplementedError("detectron2_b200 ops run on CUDA tensors only (no CPU fallback)")


# --- detectron2._C-shaped helpers (csrc/vision.cpp:86-88) -----------------------------------------
def get_cuda_version():
    v = lib().d2b_cuda_version()
    return "CUDA %d.%d" % (v // 1000, (v % 1000) // 10)


def has_cuda():
    return True


def get_compiler_version():
    return "nvcc (sm_90a)"


# --- the five pybind deform-conv entry points of detectron2._C (csrc/vision.cpp:90-102, deform_conv.h:116-375) -----------
# Same positional signatures and the same in-place contract: outputs are CALLER-ALLOCATED tensors written in place
# (detectron2/layers/deform_conv.py:43-45,97-98,121,219,250-254); `columns` / `ones` are scratch tensors of the reference's
# im2col design that a fused implementation has no use for.  With this module bound as `detectron2._C`, the reference's own
# `_DeformConv` / `_ModulatedDeformConv` autograd Functions run unchanged on our kernels (INTEGRATION.md).
# Note the reference's argument order for DCNv1: kW, kH, dW, dH, padW, padH, dilW, dilH (width first, deform_conv.py:69-76).
DCN_PRECISION = -1  # -1 auto (bf16x3 wgmma when the shape is taken, else fp32 FFMA); see include/d2b200.h


def _into(dst, src):
    if dst.shape != src.shape:
        dst.resize_(src.shape)  # the reference resizes its outputs as well (deform_conv_cuda.cu:340-344)
    dst.copy_(src)


def deform_conv_forward(input, weight, offset, output, columns, ones, kW, kH, dW, dH, padW, padH, dilW, dilH, group,
                        deformable_group, im2col_step):
    from . import ops

    if weight.shape[3] != kW or weight.shape[2] != kH:
        raise RuntimeError("deform_conv_forward: kernel size does not match the weight tensor")
    y = ops.deform_conv_op(input, offset, None, weight, None, [dH, dW], [padH, padW], [dilH, dilW], group, deformable_group,
                           DCN_PRECISION)
    _into(output, y)
    return 1


def deform_conv_backward_input(input, offset, gradOutput, gradInput, gradOffset, weight, columns, kW, kH, dW, dH, padW,
                               padH, dilW, dilH, group, deformable_group, im2col_step):
    from . import ops

    gx, go, _, _, _ = ops.deform_conv_backward_op(input, offset, None, weight, gradOutput, [dH, dW], [padH, padW],
                                                  [dilH, dilW], group, deformable_group, False, True, False, DCN_PRECISION)
    _into(gradInput, gx)
    _into(gradOffset, go)
    return 1


def deform_conv_backward_filter(input, offset, gradOutput, gradWeight, columns, ones, kW, kH, dW, dH, padW, padH, dilW,
                                dilH, group, deformable_group, scale, im2col_step):
    from . import ops

    _, _, _, gw, _ = ops.deform_conv_backward_op(input, offset, None, gradWeight.new_empty(gradWeight.shape), gradOutput,
                                                 [dH, dW], [padH, padW], [dilH, dilW], group, deformable_group, False,
                                                 False, True, DCN_PRECISION)
    gradWeight.add_(gw, alpha=float(scale))  # the reference accumulates scale * dW into the caller's buffer
    return 1


def modulated_deform_conv_forward(input, weight, bias, ones, offset, mask, output, columns, kernel_h, kernel_w, stride_h,
                                  stride_w, pad_h, pad_w, dilation_h, dilation_w, group, deformable_group, with_bias):
    from . import ops

    y = ops.deform_conv_op(input, offset, mask, weight, bias if with_bias else None, [stride_h, stride_w], [pad_h, pad_w],
                           [dilation_h, dilation_w], group, deformable_group, DCN_PRECISION)
    _into(output, y)


def modulated_deform_conv_backward(input, weight, bias, ones, offset, mask, columns, grad_input, grad_weight, grad_bias,
                                   grad_offset, grad_mask, grad_output, kernel_h, kernel_w, stride_h, stride_w, pad_h,
                                   pad_w, dilation_h, dilation_w, group, deformable_group, with_bias):
    from . import ops

    gx, go, gm, gw, gb = ops.deform_conv_backward_op(input, offset, mask, weight, grad_output, [stride_h, stride_w],
                                                     [pad_h, pad_w], [dilation_h, dilation_w], group, deformable_group,
                                                     bool(with_bias), True, True, DCN_PRECISION)
    _into(grad_input, gx)
    _into(grad_offset, go)
    _into(grad_mask, gm)
    grad_weight.add_(gw)  # accumulated into the caller's zero-initialised buffers (deform_conv_cuda.cu:1196-1203)
    if with_bias:
        grad_bias.add_(gb)
