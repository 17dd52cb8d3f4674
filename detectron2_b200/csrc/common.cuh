// Shared helpers for the sm_90a kernels behind include/d2b200.h.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
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

// Element type of an ABI dtype code (D2B_F32 / D2B_F16 / D2B_BF16): half-precision tensors are read and written in place,
// with fp32 arithmetic, instead of a separate cast pass per tensor.  ld(const T*) reads through the read-only data cache;
// ld(T) widens a value already in registers.
template <int DT>
struct Elem;
template <>
struct Elem<D2B_F32> {
  using T = float;
  static __device__ __forceinline__ float ld(const T* __restrict__ p) { return __ldg(p); }
  static __device__ __forceinline__ float ld(T v) { return v; }
  static __device__ __forceinline__ T st(float v) { return v; }
};
template <>
struct Elem<D2B_F16> {
  using T = __half;
  static __device__ __forceinline__ float ld(const T* __restrict__ p) { return __half2float(__ldg(p)); }
  static __device__ __forceinline__ float ld(T v) { return __half2float(v); }
  static __device__ __forceinline__ T st(float v) { return __float2half_rn(v); }
};
template <>
struct Elem<D2B_BF16> {
  using T = __nv_bfloat16;
  static __device__ __forceinline__ float ld(const T* __restrict__ p) { return __bfloat162float(__ldg(p)); }
  static __device__ __forceinline__ float ld(T v) { return __bfloat162float(v); }
  static __device__ __forceinline__ T st(float v) { return __float2bfloat16_rn(v); }
};

// Exclusive prefix sum of one value per thread over the CTA (shuffle scan inside the warps); `total` receives the sum
// over the CTA.  warp_tot: 32 elements of shared memory.  blockDim.x <= 1024, multiple of 32; every thread calls it.
// Barriers: the one inside separates the warp totals' writes from their reads.  Nothing follows the reads, so a caller
// that writes warp_tot again -- a second call included -- puts a __syncthreads() between this call and that write.
template <class T>
__device__ __forceinline__ T block_exclusive_scan(T v, T* __restrict__ warp_tot, T& total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  T inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  if (lane == 31) warp_tot[warp] = inc;
  __syncthreads();
  const T wt = lane < nwarps ? warp_tot[lane] : T(0);
  T winc = wt;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const T t = __shfl_up_sync(0xffffffffu, winc, o);
    if (lane >= o) winc += t;
  }
  total = __shfl_sync(0xffffffffu, winc, 31);
  const T wbase = __shfl_sync(0xffffffffu, winc, warp) - __shfl_sync(0xffffffffu, wt, warp);
  return wbase + inc - v;
}

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
