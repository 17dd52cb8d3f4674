// Host entry points of the tensor-core deformable convolution (deform_conv_tc.cu) that the public entry points in
// deform_conv.cu dispatch to.  Library-internal: not exported from libd2b200.so.  Whether the kernels take a shape is the
// public d2b_deform_conv_tc_shape_supported; the sizes below are 0 when they do not.
#pragma once
#include <stddef.h>

#include "../../include/d2b200.h"

size_t d2b_deform_conv_tc_fwd_workspace(const d2b_dcn_params* p, int precision, int x_nhwc);
size_t d2b_deform_conv_tc_bwd_workspace(const d2b_dcn_params* p, int precision, int x_nhwc, int need_data, int need_weight);
size_t d2b_deform_conv_tc_cols_bytes(const d2b_dcn_params* p, int precision);

int d2b_deform_conv_forward_tc(const float* x, const float* offset, const float* mask, const float* weight,
                               const float* scale, const float* shift, int relu, const d2b_dcn_params* p, int precision,
                               int tcflags, float* out, void* cols, void* workspace, size_t workspace_bytes, void* stream);
int d2b_deform_conv_backward_tc(const float* x, const float* offset, const float* mask, const float* weight,
                                const float* grad_out, const float* scale, const float* y_saved, int relu,
                                const d2b_dcn_params* p, int precision, int tcflags, const void* cols, float* grad_x,
                                float* grad_offset, float* grad_mask, float* grad_weight, void* workspace,
                                size_t workspace_bytes, void* stream);
