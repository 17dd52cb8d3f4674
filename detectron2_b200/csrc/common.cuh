// Shared helpers for the sm_90a kernels behind include/d2b200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "../../include/d2b200.h"

#define D2B_API extern "C" __attribute__((visibility("default")))

#define D2B_CHECK_LAUNCH()                               \
  do {                                                   \
    cudaError_t e__ = cudaGetLastError();                \
    if (e__ != cudaSuccess) return (int)e__;             \
  } while (0)

#define D2B_CUDA(expr)                                   \
  do {                                                   \
    cudaError_t e__ = (expr);                            \
    if (e__ != cudaSuccess) return (int)e__;             \
  } while (0)

__host__ __device__ static inline int d2b_cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// SM count of the current device (132 on an H100 SXM, 114 on an H100 PCIe): grid sizing in waves.  Queried once per device
// ordinal and cached, so it costs no CUDA call inside a graph capture after the first eager call (abi.cu).
int d2b_num_sms();

// up to D2B_MAX_ZERO device buffers zero-filled by one launch (abi.cu); null / empty entries are skipped
#define D2B_MAX_ZERO 8
int d2b_zero_buffers(void* const* ptrs, const size_t* bytes, int n, cudaStream_t stream);

// Kernels that need more than 48 KB of dynamic shared memory must opt in once PER DEVICE.  The opt-in is remembered per
// call site and device ordinal (lock-free bit mask), raised to the device maximum so that it covers every launch
// configuration, and therefore never runs inside a CUDA-graph capture after the first eager call on that device.
#define D2B_ALLOW_BIG_SMEM(kernel)                                                                              \
  do {                                                                                                          \
    static std::atomic<unsigned long long> done__{0ull};                                                        \
    int dev__ = 0;                                                                                              \
    cudaError_t e__ = cudaGetDevice(&dev__);                                                                    \
    if (e__ != cudaSuccess) return (int)e__;                                                                    \
    const unsigned long long bit__ = 1ull << (dev__ & 63);                                                      \
    if (!(done__.load(std::memory_order_acquire) & bit__)) {                                                    \
      cudaFuncAttributes fa__;                                                                                  \
      e__ = cudaFuncGetAttributes(&fa__, kernel);                                                               \
      if (e__ != cudaSuccess) return (int)e__;                                                                  \
      e__ = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,                           \
                                 227 * 1024 - (int)fa__.sharedSizeBytes); /* static + dynamic <= 227 KB */      \
      if (e__ != cudaSuccess) return (int)e__;                                                                  \
      done__.fetch_or(bit__, std::memory_order_release);                                                        \
    }                                                                                                           \
  } while (0)
