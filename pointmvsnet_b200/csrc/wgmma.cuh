// Hopper warpgroup MMA (wgmma, kind tf32) and mbarrier primitives shared by the two tensor-core GEMMs
// (gemm_tc.cu, gemm_ws.cu).  Operands are read from shared memory in the K-major SWIZZLE_128B layout: a row of 32 fp32
// (128 bytes) per matrix row, 16-byte piece p of row r stored at piece p ^ (r & 7) inside 8-row, 1024-byte atoms.
#pragma once
#include <stdint.h>

namespace pmvs {
namespace wg {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done = 0;
  while (!done) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  }
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// generic-proxy shared-memory stores -> visible to the tensor core's async proxy
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// byte offset of 16-byte piece `pc` of row `r` inside a K-major SWIZZLE_128B plane
__device__ __forceinline__ int swz128(int r, int pc) { return (r >> 3) * 1024 + (r & 7) * 128 + ((pc ^ (r & 7)) << 4); }

// K-major SWIZZLE_128B shared-memory matrix descriptor: start address >> 4 in bits [0,14), leading byte offset
// (unused for swizzled K-major) = 1 in [16,30), stride byte offset = 1024 B (one 8-row atom) >> 4 in [32,46),
// layout 1 (128-byte swizzle) in [62,64).  A k-step of 8 fp32 advances the start address by 32 bytes.
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}

__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// keeps the compiler from moving accumulator reads above the wait
template <int R>
__device__ __forceinline__ void fence_regs(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64, N] (+)= A[64, 8] * B[N, 8]^T, issued by the 128 threads of a warpgroup.  Thread t = 32 * w + l holds
// d[4 * i + {0, 1}] = D[16 * w + l / 4][8 * i + 2 * (l % 4) + {0, 1}] and d[4 * i + {2, 3}] = the same columns of row + 8.
template <int N>
__device__ __forceinline__ void mma_tf32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void mma_tf32<16>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7}, "
      "%8, %9, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void mma_tf32<32>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "%16, %17, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void mma_tf32<64>(float* d, uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "%32, %33, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate));
}

// D[64, N] (+)= A * B^T issued as N / BLK instructions of shape m64n(BLK)k8 (BLK = 16, 32 or 64; BLK rows of B are
// BLK * 128 bytes apart, a multiple of the 1024-byte swizzle atom).  PTX orders the accumulator accesses of
// wgmma.mma_async instructions only when they have the same shape, so every instruction that a kernel issues into one
// accumulator between two fences must use the same BLK.
template <int N, int BLK>
__device__ __forceinline__ void mma_tile(float* d, uint32_t a_addr, uint32_t b_addr, uint32_t accumulate) {
  static_assert(N % BLK == 0 && (BLK == 16 || BLK == 32 || BLK == 64), "block shape");
#pragma unroll
  for (int nb = 0; nb < N / BLK; ++nb)
    mma_tf32<BLK>(d + (BLK / 2) * nb, make_desc(a_addr), make_desc(b_addr + nb * BLK * 128), accumulate);
}

}  // namespace wg
}  // namespace pmvs
