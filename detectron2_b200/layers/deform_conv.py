"""DeformConv / ModulatedDeformConv -- same surface as detectron2/layers/deform_conv.py:16-502.

Parameter names/shapes (`weight`, `bias`) match the reference so checkpoints load unchanged.  The functional forms
`deform_conv` / `modulated_deform_conv` keep the reference's positional signatures (:16-28, :187-201).
"""
import math

import torch
from torch import nn
from torch.nn.modules.utils import _pair

from .. import ops

# -1 = auto: bf16x3 operand split on wgmma when the tensor-core kernel takes the shape, else fp32 FFMA (both are
# fp32-class, <= 1e-4 rel);  0 = fp32 FFMA;  1 = bf16x3 wgmma;  2 = plain bf16 wgmma (autocast-style operands).
DEFAULT_PRECISION = -1


def deform_conv(input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1,
                im2col_step=64):
    """DCNv1 (`_DeformConv.apply`).  `im2col_step` is accepted for signature compatibility; the fused kernels
    have no column buffer, so it has no effect."""
    if input is not None and input.dim() != 4:
        raise ValueError("Expected 4D tensor as input, got {}D tensor instead.".format(input.dim()))
    if not input.is_cuda:
        raise NotImplementedError("Deformable Conv is not supported on CPUs!")
    return ops.deform_conv(input, offset, None, weight, None, list(_pair(stride)), list(_pair(padding)),
                           list(_pair(dilation)), groups, deformable_groups, DEFAULT_PRECISION)


def modulated_deform_conv(input, offset, mask, weight, bias=None, stride=1, padding=0, dilation=1, groups=1,
                          deformable_groups=1):
    """DCNv2 (`_ModulatedDeformConv.apply`)."""
    if not input.is_cuda:
        raise NotImplementedError("Deformable Conv is not supported on CPUs!")
    return ops.deform_conv(input, offset, mask, weight, bias, list(_pair(stride)), list(_pair(padding)),
                           list(_pair(dilation)), groups, deformable_groups, DEFAULT_PRECISION)


def _empty_output(x, weight, padding, dilation, kernel_size, stride):
    # deform_conv.py:370-382: keep shape arithmetic alive for empty batches
    shape = [(i + 2 * p - (di * (k - 1) + 1)) // s + 1
             for i, p, di, k, s in zip(x.shape[-2:], padding, dilation, kernel_size, stride)]
    return x.new_empty([x.shape[0], weight.shape[0]] + shape) + 0 * x.sum()


class DeformConv(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=False, norm=None, activation=None):
        super().__init__()
        assert not bias
        assert in_channels % groups == 0, "in_channels {} cannot be divisible by groups {}".format(in_channels, groups)
        assert out_channels % groups == 0, "out_channels {} cannot be divisible by groups {}".format(out_channels,
                                                                                                      groups)
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride = _pair(stride)
        self.padding = _pair(padding)
        self.dilation = _pair(dilation)
        self.groups = groups
        self.deformable_groups = deformable_groups
        self.norm = norm
        self.activation = activation
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // self.groups, *self.kernel_size))
        self.bias = None
        nn.init.kaiming_uniform_(self.weight, nonlinearity="relu")

    def forward(self, x, offset):
        if x.numel() == 0:
            return _empty_output(x, self.weight, self.padding, self.dilation, self.kernel_size, self.stride)
        x = deform_conv(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups,
                        self.deformable_groups)
        if self.norm is not None:
            x = self.norm(x)
        if self.activation is not None:
            x = self.activation(x)
        return x

    def extra_repr(self):
        return ("in_channels={}, out_channels={}, kernel_size={}, stride={}, padding={}, dilation={}, groups={}, "
                "deformable_groups={}, bias=False").format(self.in_channels, self.out_channels, self.kernel_size,
                                                           self.stride, self.padding, self.dilation, self.groups,
                                                           self.deformable_groups)


class ModulatedDeformConv(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=True, norm=None, activation=None):
        super().__init__()
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.kernel_size = _pair(kernel_size)
        self.stride = stride
        self.padding = padding
        self.dilation = dilation
        self.groups = groups
        self.deformable_groups = deformable_groups
        self.with_bias = bias
        self.norm = norm
        self.activation = activation
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        if bias:
            self.bias = nn.Parameter(torch.Tensor(out_channels))
        else:
            self.bias = None
        nn.init.kaiming_uniform_(self.weight, nonlinearity="relu")
        if self.bias is not None:
            nn.init.constant_(self.bias, 0)

    def forward(self, x, offset, mask):
        if x.numel() == 0:
            return _empty_output(x, self.weight, _pair(self.padding), _pair(self.dilation), self.kernel_size,
                                 _pair(self.stride))
        x = modulated_deform_conv(x, offset, mask, self.weight, self.bias, self.stride, self.padding, self.dilation,
                                  self.groups, self.deformable_groups)
        if self.norm is not None:
            x = self.norm(x)
        if self.activation is not None:
            x = self.activation(x)
        return x

    def extra_repr(self):
        return ("in_channels={}, out_channels={}, kernel_size={}, stride={}, padding={}, dilation={}, groups={}, "
                "deformable_groups={}, bias={}").format(self.in_channels, self.out_channels, self.kernel_size,
                                                        self.stride, self.padding, self.dilation, self.groups,
                                                        self.deformable_groups, self.with_bias)


class DeformBottleneckConv2(nn.Module):
    """conv2 of the reference's DeformBottleneckBlock with modulated deformable convolution, as ONE op
    (detectron2/modeling/backbone/resnet.py:291-318): takes the raw output of `conv2_offset` (27 channels for a 3x3
    kernel), applies chunk / cat / sigmoid, the ModulatedDeformConv, its norm (FrozenBatchNorm folded into a per-channel
    scale and shift) and the ReLU that follows.  `weight` keeps the reference's name / shape, so `conv2.weight` of a
    checkpoint loads unchanged; `norm_scale` / `norm_shift` are buffers (call `load_frozen_bn` with the norm's tensors)."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, dilation=1, groups=1,
                 deformable_groups=1, relu=True):
        super().__init__()
        self.kernel_size = _pair(kernel_size)
        self.stride, self.padding, self.dilation = _pair(stride), _pair(padding), _pair(dilation)
        self.groups, self.deformable_groups, self.relu = groups, deformable_groups, relu
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        nn.init.kaiming_uniform_(self.weight, nonlinearity="relu")
        self.register_buffer("norm_scale", torch.ones(out_channels))
        self.register_buffer("norm_shift", torch.zeros(out_channels))

    def load_frozen_bn(self, weight, bias, running_mean, running_var, eps=1e-5):
        """Fold FrozenBatchNorm2d (layers/batch_norm.py:50-58): y = x * scale + shift."""
        scale = weight * (running_var + eps).rsqrt()
        self.norm_scale.copy_(scale)
        self.norm_shift.copy_(bias - running_mean * scale)

    def forward(self, x, offset_mask):
        return ops.deform_conv_fused(x, offset_mask, self.weight, self.norm_scale, self.norm_shift, self.relu,
                                     list(self.stride), list(self.padding), list(self.dilation), self.groups,
                                     self.deformable_groups, DEFAULT_PRECISION if DEFAULT_PRECISION != 0 else 1)
