// Micro-benchmarks that bound the gather / scatter kernels (run on an H100; built by tools/build_microbench.sh):
//   gather : random 256-byte runs (16 lanes x LDG.128, the channels-last tap pattern) out of an L2-resident buffer
//   red    : red.global.add.f32 (scalar) vs red.global.add.v4.f32 with the same addressing
// Prints GB/s of useful bytes and giga-operations/s.  Results are quoted in DESIGN.md next to the kernels they bound.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

__device__ __forceinline__ uint32_t hash32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}

// every half-warp reads `iters` x 8 random 256-byte runs; 8 loads in flight per lane
__global__ void gather_kernel(const float4* __restrict__ buf, uint32_t nruns, int iters, float4* __restrict__ sink) {
  const uint32_t hw = (blockIdx.x * blockDim.x + threadIdx.x) >> 4, q = threadIdx.x & 15;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int it = 0; it < iters; ++it) {
    float4 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const uint32_t run = hash32(hw * 7919u + (uint32_t)(it * 8 + j) * 104729u) % nruns;
      v[j] = __ldg(buf + (size_t)run * 16 + q);
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { acc.x += v[j].x; acc.y += v[j].y; acc.z += v[j].z; acc.w += v[j].w; }
  }
  if (acc.x == 123.456f) sink[0] = acc;
}

template <int VEC>
__global__ void red_kernel(float* __restrict__ buf, uint32_t nruns, int iters) {
  const uint32_t hw = (blockIdx.x * blockDim.x + threadIdx.x) >> 4, q = threadIdx.x & 15;
  for (int it = 0; it < iters; ++it) {
    const uint32_t run = hash32(hw * 7919u + (uint32_t)it * 104729u) % nruns;
    float* p = buf + (size_t)run * 64 + q * 4;
    if (VEC == 4) {
      asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(1.f), "f"(2.f), "f"(3.f), "f"(4.f) : "memory");
    } else {
#pragma unroll
      for (int e = 0; e < 4; ++e) asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p + e), "f"(1.f) : "memory");
    }
  }
}

static float time_ms(cudaEvent_t a, cudaEvent_t b) {
  float ms;
  cudaEventElapsedTime(&ms, a, b);
  return ms;
}

int main() {
  cudaEvent_t a, b;
  cudaEventCreate(&a);
  cudaEventCreate(&b);
  const size_t sizes_mb[3] = {17, 68, 400};
  for (int si = 0; si < 3; ++si) {
    const size_t bytes = sizes_mb[si] << 20;
    float* buf;
    cudaMalloc(&buf, bytes);
    cudaMemset(buf, 0, bytes);
    const uint32_t nruns = (uint32_t)(bytes / 256);
    const int blocks = 132 * 8, threads = 512, iters = 64;
    const double halfwarps = (double)blocks * threads / 16;
    // gather
    gather_kernel<<<blocks, threads>>>((const float4*)buf, nruns, iters, (float4*)buf);
    cudaEventRecord(a);
    gather_kernel<<<blocks, threads>>>((const float4*)buf, nruns, iters, (float4*)buf);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    double ms = time_ms(a, b);
    printf("gather  %4zu MB buffer: %8.1f GB/s (256-byte runs, %.3f ms)\n", sizes_mb[si], halfwarps * iters * 8 * 256 / ms / 1e6, ms);
    // red v4
    red_kernel<4><<<blocks, threads>>>(buf, nruns, iters);
    cudaEventRecord(a);
    red_kernel<4><<<blocks, threads>>>(buf, nruns, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    ms = time_ms(a, b);
    printf("red.v4  %4zu MB buffer: %8.1f GB/s  %7.2f Gred/s (%.3f ms)\n", sizes_mb[si], halfwarps * iters * 256 / ms / 1e6,
           halfwarps * iters * 16 / ms / 1e6, ms);
    red_kernel<1><<<blocks, threads>>>(buf, nruns, iters);
    cudaEventRecord(a);
    red_kernel<1><<<blocks, threads>>>(buf, nruns, iters);
    cudaEventRecord(b);
    cudaEventSynchronize(b);
    ms = time_ms(a, b);
    printf("red.f32 %4zu MB buffer: %8.1f GB/s  %7.2f Gred/s (%.3f ms)\n", sizes_mb[si], halfwarps * iters * 256 / ms / 1e6,
           halfwarps * iters * 64 / ms / 1e6, ms);
    cudaFree(buf);
  }
  cudaError_t e = cudaDeviceSynchronize();
  printf("status: %s\n", cudaGetErrorString(e));
  return e != cudaSuccess;
}
