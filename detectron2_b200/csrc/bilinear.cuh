// PyTorch's CUDA upsample_bilinear2d taps (align_corners = false), shared by the kernels that evaluate the resize on the
// fly instead of storing it (panoptic.cu, sem_seg_loss.cu).  Files that include this header are compiled with -fmad=false:
// the one fused multiply-add of the source index is written as __fmaf_rn, where PyTorch's sm_90 build contracts it.
#pragma once
#include <cuda_runtime.h>

// area_pixel_compute_source_index(scale, d, align_corners = false, cubic = false): max(scale * (d + 0.5) - 0.5, 0)
__device__ __forceinline__ float src_index(float scale, int d) {
  const float r = __fmaf_rn(scale, __fadd_rn((float)d, 0.5f), -0.5f);
  return r < 0.f ? 0.f : r;
}

struct Tap {
  int i0, i1;      // source index and its neighbour (clamped at the crop's last row / column)
  float l0, l1;    // weights of i0 and i1
};

__device__ __forceinline__ Tap make_tap(float scale, int d, int in_size) {
  const float r = src_index(scale, d);
  Tap t;
  t.i0 = (int)r;
  t.i1 = t.i0 + (t.i0 < in_size - 1 ? 1 : 0);
  t.l1 = __fsub_rn(r, (float)t.i0);
  t.l0 = __fsub_rn(1.f, t.l1);
  return t;
}
