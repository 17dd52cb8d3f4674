// PTX wrappers shared by the wgmma / bulk-copy kernels (sm_90a).
//
//   mbarrier            producer/consumer rings (generic and async-proxy arrivals)
//   cp.async.bulk       TMA engine, linear form: one instruction moves a whole pre-tiled operand block
//                       global -> shared and completes on an mbarrier (SASS: UBLKCP)
//   wgmma.*             warpgroup MMA from shared-memory descriptors into register accumulators (SASS: HGMMA)
//   red.global.v4.f32   128-bit vector reduction to global memory (SASS: REDG.E.ADD.F32x4)
#pragma once
#include <cuda_bf16.h>
#include <stdint.h>

namespace d2b_tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// ------------------------------------------------------------------------------------------------ mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_init_fence() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded wait: a protocol bug must surface as a launch failure (trap -> cudaErrorLaunchFailure), never as a hung GPU.
__device__ __forceinline__ uint64_t global_timer_ns() {
  uint64_t t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const uint64_t t0 = global_timer_ns();
  for (uint32_t spin = 1;; ++spin) {
    if (mbar_try_wait(bar, parity)) return;
    if ((spin & 1023u) == 0 && global_timer_ns() - t0 > 2000000000ull) __trap();  // 2 s: far beyond any legitimate wait
  }
}

// ------------------------------------------------------------------------------------------------ proxies / fences
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// ------------------------------------------------------------------------------------------------ bulk copy (TMA, linear)
// size % 16 == 0, both addresses 16-byte aligned; completes `bytes` on `bar` (pair with mbar_arrive_expect_tx)
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gmem_src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(smem_dst)),
               "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// shared -> global, tracked by the thread's bulk async-group (commit, then wait for the reads of the source to finish
// before the shared-memory tile is reused)
__device__ __forceinline__ void bulk_s2g(void* gmem_dst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem_dst), "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ------------------------------------------------------------------------------------------------ wgmma
// Shared-memory matrix descriptor (sm_90), 128-byte swizzle.
//   K-major  tile [rows][64 bf16]: rows 128 B apart, 8-row atoms `sbo` bytes apart (1024 when rows are dense)
//   MN-major tile [k rows][64 bf16 of M/N]: 8-k-row atoms `sbo` bytes apart, 64-element M/N blocks `lbo` bytes apart
__device__ __forceinline__ uint64_t wgmma_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFF);
  d |= (uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16;
  d |= (uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32;
  d |= (uint64_t)1 << 62;  // SWIZZLE_128B
  return d;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(kPending) : "memory"); }

// One warpgroup: D[64 x N] (+)= A[64 x 16] . B[16 x N], bf16 operands from shared memory, fp32 accumulator in registers
// (N / 2 per thread: element (16 w + l / 4 + 8 h, 8 j + 2 (l % 4) + e) of warp w, lane l is acc[4 j + 2 h + e]).
// kTransA: A is MN-major (M contiguous); B is always K-major.
template <int N, int kTransA>
struct Wgmma;

template <int kTransA>
struct Wgmma<8, kTransA> {
  __device__ __forceinline__ static void mma(float (&d)[4], uint64_t a, uint64_t b, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %4, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, %5, %6, p, 1, 1, %7, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "r"(accumulate), "l"(a), "l"(b), "n"(kTransA));
  }
};
template <int kTransA>
struct Wgmma<16, kTransA> {
  __device__ __forceinline__ static void mma(float (&d)[8], uint64_t a, uint64_t b, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %8, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %9, %10, p, 1, 1, %11, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "r"(accumulate), "l"(a), "l"(b), "n"(kTransA));
  }
};
template <int kTransA>
struct Wgmma<32, kTransA> {
  __device__ __forceinline__ static void mma(float (&d)[16], uint64_t a, uint64_t b, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %16, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %17, %18, p, 1, 1, %19, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "r"(accumulate), "l"(a), "l"(b), "n"(kTransA));
  }
};
template <int kTransA>
struct Wgmma<64, kTransA> {
  __device__ __forceinline__ static void mma(float (&d)[32], uint64_t a, uint64_t b, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %32, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %33, %34, p, 1, 1, %35, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "r"(accumulate), "l"(a), "l"(b), "n"(kTransA));
  }
};
template <int kTransA>
struct Wgmma<128, kTransA> {
  __device__ __forceinline__ static void mma(float (&d)[64], uint64_t a, uint64_t b, int accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %64, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %65, %66, p, 1, 1, %67, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(accumulate), "l"(a), "l"(b), "n"(kTransA));
  }
};

// Register budget of the calling warpgroup (every warp of it executes the instruction): the TMA / saver warpgroup gives
// registers back so that the four worker warpgroups can hold accumulators and gather state without spilling.
template <int kRegs>
__device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kRegs)); }
template <int kRegs>
__device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kRegs)); }

// ------------------------------------------------------------------------------------------------ misc
__device__ __forceinline__ void red_add_v4(float* p, float a, float b, float c, float d) {
  asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(a), "f"(b), "f"(c), "f"(d) : "memory");
}
__device__ __forceinline__ void red_add_v2(float* p, float a, float b) {
  asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(a), "f"(b) : "memory");
}
__device__ __forceinline__ void red_add(float* p, float a) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(a) : "memory");
}
__device__ __forceinline__ uint32_t pack_bf16(float a, float b) {  // a -> low half
  __nv_bfloat162 v = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&v);
}
// x = hi + lo with hi, lo bf16 (lo = rn(x - hi)): three bf16 MMAs hi*hi + hi*lo + lo*hi keep ~16 mantissa bits per product
__device__ __forceinline__ void split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  hi = pack_bf16(a, b);                                   // one F2FP for both values
  const float ha = __uint_as_float(hi << 16), hb = __uint_as_float(hi & 0xffff0000u);
  lo = pack_bf16(a - ha, b - hb);
}
__device__ __forceinline__ void split4(const float (&v)[4], uint2& hi, uint2& lo) {
  split2(v[0], v[1], hi.x, lo.x);
  split2(v[2], v[3], hi.y, lo.y);
}
// Pairs of fp32 lanes: the gather / scatter loops are written over channel pairs (one FFMA per lane on sm_90)
struct F2 {
  float x, y;
};
__device__ __forceinline__ F2 f2_pack(float a, float b) { return F2{a, b}; }
__device__ __forceinline__ void f2_unpack(F2 p, float& a, float& b) {
  a = p.x;
  b = p.y;
}
__device__ __forceinline__ F2 f2_fma(F2 w, F2 v, F2 c) { return F2{__fmaf_rn(w.x, v.x, c.x), __fmaf_rn(w.y, v.y, c.y)}; }
__device__ __forceinline__ F2 f2_mul(F2 a, F2 b) { return F2{__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 f2_add(F2 a, F2 b) { return F2{__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)}; }
__device__ __forceinline__ F2 f2_sub(F2 a, F2 b) { return F2{__fsub_rn(a.x, b.x), __fsub_rn(a.y, b.y)}; }
__device__ __forceinline__ void red_add_v4(float* p, F2 ab, F2 cd) {
  float a, b, c, d;
  f2_unpack(ab, a, b);
  f2_unpack(cd, c, d);
  red_add_v4(p, a, b, c, d);
}
// predicated form: one instruction slot, no branch around it
__device__ __forceinline__ void red_add_v4_if(int pred, float* p, F2 ab, F2 cd) {
  float a, b, c, d;
  f2_unpack(ab, a, b);
  f2_unpack(cd, c, d);
  asm volatile(
      "{\n\t.reg .pred q;\n\tsetp.ne.b32 q, %5, 0;\n\t@q red.global.add.v4.f32 [%0], {%1, %2, %3, %4};\n\t}" ::"l"(p),
      "f"(a), "f"(b), "f"(c), "f"(d), "r"(pred)
      : "memory");
}

// byte offset of the 16-byte chunk `c16` of row `r` inside a 128-byte-swizzled tile of 128-byte rows
__device__ __forceinline__ uint32_t swz128(uint32_t r, uint32_t c16) { return r * 128u + ((c16 ^ (r & 7u)) << 4); }

}  // namespace d2b_tc
