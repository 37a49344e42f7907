// Hopper warpgroup MMA (wgmma, kind tf32) and mbarrier primitives shared by the tensor-core GEMMs
// (gemm_tc.cu, gemm_ws.cu) and the fused fetch + first contraction (fetch.cu).  Operands are read from shared memory in the K-major SWIZZLE_128B layout: a row of 32 fp32
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
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// TMA: the box of a 3-D tensor map at (c0, c1, c2) -> shared memory, completion counted in bytes on `bar`
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const void* tmap, int c0, int c1, int c2, uint32_t bar) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
      ::"r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
      : "memory");
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

// ---- A operand in registers -------------------------------------------------------------------------------------
// Thread t = 32 * w + l of the warpgroup holds a[0..3] = A[16 w + l / 4][l % 4], A[16 w + l / 4 + 8][l % 4],
// A[16 w + l / 4][l % 4 + 4], A[16 w + l / 4 + 8][l % 4 + 4] (tf32 bit patterns).  The registers are read
// asynchronously: they must not change before the instruction's group has been waited for.
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R>
__device__ __forceinline__ void fence_regs(uint32_t (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

template <int N>
__device__ __forceinline__ void mma_tf32_ra(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void mma_tf32_ra<16>(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %13, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7}, "
      "{%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void mma_tf32_ra<32>(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %21, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
      "{%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
template <>
__device__ __forceinline__ void mma_tf32_ra<64>(float* d, const uint32_t* a, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
      "{%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]),
        "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]),
        "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]),
        "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]),
        "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate));
}
// mma_tile with the A fragment in registers
template <int N, int BLK>
__device__ __forceinline__ void mma_tile_ra(float* d, const uint32_t* a, uint32_t b_addr, uint32_t accumulate) {
  static_assert(N % BLK == 0 && (BLK == 16 || BLK == 32 || BLK == 64), "block shape");
#pragma unroll
  for (int nb = 0; nb < N / BLK; ++nb) mma_tf32_ra<BLK>(d + (BLK / 2) * nb, a, make_desc(b_addr + nb * BLK * 128), accumulate);
}

// ---- 3xTF32 with stationary weight planes (gemm_tma_kernel in gemm_ws.cu, fetch_gemm_kernel in fetch.cu) ----------
// hi = the 10 explicit mantissa bits the tensor core reads, lo = x - hi (exact)
__device__ __forceinline__ float tf32_hi(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }

// W [cout, K] -> shared memory at `planes` as the B operand: per 32-column chunk c of K, rows [0, cout) hold W_hi and
// rows [cout, 2 cout) W_lo, K-major SWIZZLE_128B (chunk c starts 2 * cout * 128 bytes after chunk c - 1), zero beyond K.
// Thread `t` of `nthreads` writes its share; the caller fences (fence_proxy_async) and synchronises.
template <int COUT>
__device__ __forceinline__ void store_weight_planes(uint32_t planes, const float* __restrict__ w, int K, int t,
                                                    int nthreads) {
  const int nch = (K + 31) / 32;
  for (int e = t; e < COUT * nch * 8; e += nthreads) {
    const int n = e / (nch * 8), rem = e - n * (nch * 8), c = rem >> 3, pc = rem & 7;
    const int k0 = c * 32 + pc * 4;  // K is a multiple of 8: a 16-byte piece is all inside or all padding
    const float4 v = k0 < K ? __ldg(reinterpret_cast<const float4*>(w + (size_t)n * K + k0)) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 hi, lo;
    hi.x = tf32_hi(v.x); hi.y = tf32_hi(v.y); hi.z = tf32_hi(v.z); hi.w = tf32_hi(v.w);
    lo.x = __fsub_rn(v.x, hi.x); lo.y = __fsub_rn(v.y, hi.y); lo.z = __fsub_rn(v.z, hi.z); lo.w = __fsub_rn(v.w, hi.w);
    const uint32_t dst = planes + c * (2 * COUT * 128) + swz128(n, pc);
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(hi.x), "f"(hi.y), "f"(hi.z), "f"(hi.w) : "memory");
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + COUT * 128), "f"(lo.x), "f"(lo.y), "f"(lo.z), "f"(lo.w)
                 : "memory");
  }
}

// One 32-column chunk c of a 64-row tile, issued by a warpgroup: the thread reads its A fragments (rows r, r + 8 and
// columns 8 j + q (+ 4) of k-step j, r = 16 * (warp % 4) + lane / 4, q = lane % 4) from the K-major SWIZZLE_128B
// box at `st` = box + r * 128 + q * 4 (fx = (r & 7) << 4), applies relu(fma(x, A, B)) when IN_BN (bn = the chunk's
// [A x 8 | B x 8] of this lane % 4), splits hi / lo and issues the chunk's KSTEPS k-steps against the weight planes at
// w_hi as one wgmma group, then waits for it: the next chunk rewrites fh / fl.
template <int COUT, bool IN_BN, int KSTEPS>
__device__ __forceinline__ void mma_chunk_3xtf32(float* acc, uint32_t (&fh)[16], uint32_t (&fl)[16], uint32_t st,
                                                 uint32_t fx, const float* bn, uint32_t w_hi, int c) {
  constexpr bool STACKED = COUT <= 64;
  constexpr int BLK = COUT < 64 ? COUT : 64;  // one wgmma shape for every product into this accumulator
  float bA[8], bB[8];
  if (IN_BN) {
    const float4* t4 = reinterpret_cast<const float4*>(bn);
    const float4 a0 = t4[0], a1 = t4[1], b0 = t4[2], b1 = t4[3];
    bA[0] = a0.x; bA[1] = a0.y; bA[2] = a0.z; bA[3] = a0.w; bA[4] = a1.x; bA[5] = a1.y; bA[6] = a1.z; bA[7] = a1.w;
    bB[0] = b0.x; bB[1] = b0.y; bB[2] = b0.z; bB[3] = b0.w; bB[4] = b1.x; bB[5] = b1.y; bB[6] = b1.z; bB[7] = b1.w;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (j < KSTEPS) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const uint32_t addr = st + ((uint32_t)((2 * j + h) << 4) ^ fx);
        float v[2];
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v[0]) : "r"(addr) : "memory");
        asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v[1]) : "r"(addr + 1024) : "memory");
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float x = v[e];
          if (IN_BN) x = fmaxf(fmaf(x, bA[2 * j + h], bB[2 * j + h]), 0.f);
          const float hi = tf32_hi(x);
          fh[4 * j + 2 * h + e] = __float_as_uint(hi);
          fl[4 * j + 2 * h + e] = __float_as_uint(__fsub_rn(x, hi));
        }
      }
    }
  }
  fence();
  const uint32_t w_lo = w_hi + COUT * 128;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (j < KSTEPS) {
      const uint32_t first = (c | j) != 0 ? 1u : 0u;
      if (STACKED) {
        mma_tile_ra<2 * COUT, BLK>(acc, &fh[4 * j], w_hi + j * 32, first);
        mma_tile_ra<COUT, BLK>(acc + COUT / 2, &fl[4 * j], w_hi + j * 32, 1u);
      } else {
        mma_tile_ra<COUT, BLK>(acc, &fl[4 * j], w_hi + j * 32, first);
        mma_tile_ra<COUT, BLK>(acc, &fh[4 * j], w_lo + j * 32, 1u);
        mma_tile_ra<COUT, BLK>(acc, &fh[4 * j], w_hi + j * 32, 1u);
      }
    }
  }
  commit();
  // A second fragment buffer (wait_group 1) does not fit: ptxas then serialises every wgmma for lack of registers.
  wait<0>();
  fence_regs(fh);
  fence_regs(fl);
}

}  // namespace wg
}  // namespace pmvs
