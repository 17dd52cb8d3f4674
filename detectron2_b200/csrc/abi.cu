// ABI bookkeeping entry points of libd2b200.so (include/d2b200.h).
#include "common.cuh"

D2B_API int d2b_abi_version(void) { return D2B_ABI_VERSION; }
D2B_API int d2b_cuda_version(void) { return CUDART_VERSION; }
D2B_API const char* d2b_arch(void) { return "sm_90a"; }

// ---- several buffers zero-filled by ONE launch (gradient outputs of a backward call): a cudaMemsetAsync per buffer costs a
// graph node / launch each, and most of these buffers are a few KB.  16-byte stores where alignment allows.
namespace {
struct ZeroList {
  int n;
  void* p[D2B_MAX_ZERO];
  size_t bytes[D2B_MAX_ZERO];
  size_t blk0[D2B_MAX_ZERO + 1];  // first block of every buffer (prefix over ceil(bytes / 16 KB))
};
constexpr size_t kZeroChunk = 16384;

__global__ void __launch_bounds__(256) zero_buffers_kernel(const ZeroList z) {
  int i = 0;
  while (i + 1 < z.n && blockIdx.x >= z.blk0[i + 1]) ++i;
  const size_t off = (blockIdx.x - z.blk0[i]) * kZeroChunk;
  const size_t len = min(kZeroChunk, z.bytes[i] - off);
  char* base = (char*)z.p[i] + off;
  if ((reinterpret_cast<uintptr_t>(base) & 15) == 0) {
    uint4* q = reinterpret_cast<uint4*>(base);
    for (size_t e = threadIdx.x; e < len / 16; e += 256) q[e] = make_uint4(0u, 0u, 0u, 0u);
    for (size_t e = (len / 16) * 16 + threadIdx.x; e < len; e += 256) base[e] = 0;
  } else {
    for (size_t e = threadIdx.x; e < len; e += 256) base[e] = 0;
  }
}
}  // namespace

int d2b_num_sms() {
  static std::atomic<int> cached[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;  // the launch that follows reports the error
  int n = cached[dev].load(std::memory_order_relaxed);
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
    cached[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

int d2b_zero_buffers(void* const* ptrs, const size_t* bytes, int n, cudaStream_t stream) {
  ZeroList z = {};
  size_t blocks = 0;
  for (int i = 0; i < n && z.n < D2B_MAX_ZERO; ++i) {
    if (!ptrs[i] || !bytes[i]) continue;
    z.p[z.n] = ptrs[i];
    z.bytes[z.n] = bytes[i];
    z.blk0[z.n] = blocks;
    blocks += (bytes[i] + kZeroChunk - 1) / kZeroChunk;
    ++z.n;
  }
  z.blk0[z.n] = blocks;
  if (z.n == 0) return D2B_OK;
  if (blocks > 0x7fffffffULL) return D2B_EUNSUPPORTED;
  zero_buffers_kernel<<<(unsigned)blocks, 256, 0, stream>>>(z);
  D2B_CHECK_LAUNCH();
  return D2B_OK;
}
