// Warpgroup-MMA (wgmma) GEMM for the per-point contractions of EdgeConv / flow_mlp:
//   Y[r, 0:N] = f(X[r, 0:K]) * W[0:N, 0:K]^T        r = points (rows), fp32 in / fp32 out
// (reference: nn.Conv1d 1x1 in networks.py:13-14,22-23,51-52 and nn/conv.py:21-30 followed by
// train-mode BatchNorm + ReLU, which is fused here as the INPUT transform of the next layer).
//
// The contraction is memory/latency bound (25 FLOP/B), so the kernel is organised for bytes in
// flight rather than for MMA throughput: one CTA (256 threads = two warpgroups) owns one 128-row
// tile, uses ~40-70 KB of shared memory, and 3-4 CTAs are resident per SM, each in a different
// phase (load / MMA / epilogue).  Per 32-column K chunk:
//   all threads : coalesced 128-bit loads of the X slab (128 x 32 fp32) and of the W slab
//                 (N x 32) into registers - issued BEFORE waiting for the previous chunk's MMA
//   all threads : fused BatchNorm+ReLU, TF32 hi/lo split, stores in the K-major SWIZZLE_128B
//                 layout, fence.proxy.async, __syncthreads
//   warpgroup w : wgmma.mma_async m64nNk8 tf32 x ksteps on rows [64 w, 64 w + 64), commit, wait
// Epilogue: the fp32 accumulator fragments go from registers through shared memory to
// coalesced stores; per-column sum / sum-of-squares (BN statistics of the next layer) reduced in fp64.
//
// Precision: tf32 operands have a 10-bit mantissa.  NSPLIT = 3 runs the error-
// compensated product A*B ~= Alo*Bhi + Ahi*Blo + Ahi*Bhi ("3xTF32", residuals exact in fp32),
// which keeps fp32-level accuracy (measured in tests/test_gpu_parity.py); NSPLIT = 1 is plain TF32.
#include <algorithm>

#include "common.cuh"
#include "wgmma.cuh"

namespace pmvs {

namespace tc {

using namespace wg;

constexpr int BM = 128;            // rows per tile: two warpgroups x wgmma M = 64
constexpr int KC = 32;             // fp32 columns per K chunk == one 128-byte swizzle row
constexpr int NUM_THREADS = 256;
constexpr int A_PLANE_BYTES = BM * KC * 4;  // 16 KB

// TF32 split: hi keeps the 10 explicit mantissa bits the tensor core reads, lo = x - hi (exact)
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
  lo = __fsub_rn(x, hi);
}
__device__ __forceinline__ void store_planes(unsigned char* hi_plane, size_t lo_off, int off, float4 v, bool split) {
  if (split) {
    float4 hi, lo;
    split_tf32(v.x, hi.x, lo.x); split_tf32(v.y, hi.y, lo.y);
    split_tf32(v.z, hi.z, lo.z); split_tf32(v.w, hi.w, lo.w);
    *reinterpret_cast<float4*>(hi_plane + off) = hi;
    *reinterpret_cast<float4*>(hi_plane + lo_off + off) = lo;
  } else {
    *reinterpret_cast<float4*>(hi_plane + off) = v;
  }
}

template <int N_OUT, int NSPLIT>
struct Smem {
  static constexpr int NPL = NSPLIT == 3 ? 2 : 1;          // planes (hi [, lo])
  static constexpr int B_PLANE_BYTES = N_OUT * KC * 4;     // one K chunk of W, one plane
  static constexpr int D_PITCH = N_OUT + 4;                // floats
  static constexpr int AB_BYTES = NPL * (A_PLANE_BYTES + B_PLANE_BYTES);
  static constexpr int D_BYTES = BM * D_PITCH * 4;
  static constexpr int MAIN_BYTES = AB_BYTES > D_BYTES ? AB_BYTES : D_BYTES;  // D staging aliases A/B
  static constexpr int TOTAL = 1024 /*align slack*/ + MAIN_BYTES + 4 * 224 * 4 /*BN coeffs*/;
};

template <int N_OUT, int NSPLIT>
__global__ void __launch_bounds__(NUM_THREADS) gemm_tc_kernel(const GemmArgs a) {
  using S = Smem<N_OUT, NSPLIT>;
  constexpr int NPL = S::NPL;
  constexpr bool SPLIT = NSPLIT == 3;
  // 3xTF32 with N <= 64 stacks [Bhi ; Blo] into one N' = 2N operand: A_hi * [Bhi;Blo] is ONE MMA that
  // reads A_hi once (accumulator columns [0,N) = Ahi*Bhi, [N,2N) = Ahi*Blo), and A_lo * B_hi
  // accumulates into [N,2N); the epilogue adds the two halves, so the small terms are summed apart
  // from the large one.  N = 128 keeps one accumulator (64 registers a thread).
  constexpr bool STACKED = SPLIT && N_OUT <= 64;
  constexpr int ACC_COLS = STACKED ? 2 * N_OUT : N_OUT;
  constexpr int ACC_REGS = ACC_COLS / 2;              // accumulator registers per thread (64 rows x ACC_COLS / 128 threads)
  constexpr int BLK = N_OUT < 64 ? N_OUT : 64;        // one wgmma shape for every product into this accumulator (wgmma.cuh)
  constexpr int A_LD = BM * 8 / NUM_THREADS;          // float4 loads per thread per chunk (4)
  constexpr int B_LD = (N_OUT * 8 + NUM_THREADS - 1) / NUM_THREADS;
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sA = smem;                                  // [plane][128 x 128 B swizzled]
  unsigned char* sB = sA + NPL * A_PLANE_BYTES;              // [plane][N_OUT x 128 B swizzled]
  float* sD = (float*)smem;                                  // epilogue staging (aliases sA/sB)
  float* sBN = (float*)(smem + S::MAIN_BYTES);               // mean, istd, gamma, beta  x 224

  const int K = a.cin;
  const int nch = (K + KC - 1) / KC;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wgi = warp >> 2;  // warpgroup: rows [64 * wgi, 64 * wgi + 64) of the tile
  const int g = blockIdx.y;
  const int row0 = blockIdx.x * BM;
  const int rows_valid = min(BM, a.rows_per_group - row0);
  const size_t grow0 = (size_t)g * a.rows_per_group + row0;
  const bool in_bn = a.in_stats != nullptr;

  if (in_bn) {
    const double* s = a.in_stats + (size_t)g * 2 * K;
    for (int c = tid; c < K; c += NUM_THREADS) {
      BnCoef k = bn_coef(s[c], s[K + c], a.in_count, a.eps);
      sBN[c] = k.mean;
      sBN[224 + c] = k.invstd;
      sBN[448 + c] = a.in_gamma[c];
      sBN[672 + c] = a.in_beta[c];
    }
  }

  // global -> register staging of one K chunk (A: 4 float4 per thread, B: B_LD float4 per thread)
  const int pc = tid & 7;                       // 16-byte piece inside the 128-byte row
  const int arow = tid >> 3;                    // 0..31 ; rows arow + 32*i
  auto load_chunk = [&](int c, float4 (&xa)[A_LD], float4 (&xb)[B_LD]) {
    const int k0 = c * KC + pc * 4;
    const bool kvalid = k0 < K;
#pragma unroll
    for (int i = 0; i < A_LD; ++i) {
      const int r = arow + 32 * i;
      xa[i] = (kvalid && r < rows_valid) ? ldg4(a.x + (grow0 + r) * a.ldx + k0) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) {
      const int n = arow + 32 * i;
      xb[i] = (kvalid && n < N_OUT) ? ldg4(a.w + (size_t)n * K + k0) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_chunk = [&](int c, const float4 (&xa)[A_LD], const float4 (&xb)[B_LD]) {
    const int k0 = c * KC + pc * 4;
    const bool kvalid = k0 < K;
#pragma unroll
    for (int i = 0; i < A_LD; ++i) {
      const int r = arow + 32 * i;
      float4 v = xa[i];
      if (in_bn && kvalid && r < rows_valid) {
        v.x = fmaxf(bn_apply(v.x, sBN[k0 + 0], sBN[224 + k0 + 0], sBN[448 + k0 + 0], sBN[672 + k0 + 0]), 0.f);
        v.y = fmaxf(bn_apply(v.y, sBN[k0 + 1], sBN[224 + k0 + 1], sBN[448 + k0 + 1], sBN[672 + k0 + 1]), 0.f);
        v.z = fmaxf(bn_apply(v.z, sBN[k0 + 2], sBN[224 + k0 + 2], sBN[448 + k0 + 2], sBN[672 + k0 + 2]), 0.f);
        v.w = fmaxf(bn_apply(v.w, sBN[k0 + 3], sBN[224 + k0 + 3], sBN[448 + k0 + 3], sBN[672 + k0 + 3]), 0.f);
      }
      const int off = swz128(r, pc);
      store_planes(sA, A_PLANE_BYTES, off, v, SPLIT);
    }
#pragma unroll
    for (int i = 0; i < B_LD; ++i) {
      const int n = arow + 32 * i;
      if (n < N_OUT) {
        const int off = swz128(n, pc);
        store_planes(sB, S::B_PLANE_BYTES, off, xb[i], SPLIT);
      }
    }
  };

  float4 xa[A_LD], xb[B_LD];
  load_chunk(0, xa, xb);
  __syncthreads();   // BN coefficients visible
  float acc[ACC_REGS];
  const uint32_t a_hi = smem_u32(sA) + wgi * 64 * 128, a_lo = a_hi + A_PLANE_BYTES;
  const uint32_t b_hi = smem_u32(sB), b_lo = b_hi + S::B_PLANE_BYTES;

  for (int c = 0; c < nch; ++c) {
    store_chunk(c, xa, xb);
    fence_proxy_async();   // generic-proxy stores -> visible to the tensor core's async proxy
    __syncthreads();
    if (c + 1 < nch) load_chunk(c + 1, xa, xb);   // in flight while the tensor core works
    const int ksteps = min(KC, K - c * KC) / 8;
    fence();
    for (int j = 0; j < ksteps; ++j) {
      const uint32_t first = (c == 0 && j == 0) ? 0u : 1u;
      if (STACKED) {
        // B planes are contiguous in shared memory: rows [0,N) = Bhi, [N,2N) = Blo
        mma_tile<2 * N_OUT, BLK>(acc, a_hi + j * 32, b_hi + j * 32, first);
        mma_tile<N_OUT, BLK>(acc + N_OUT / 2, a_lo + j * 32, b_hi + j * 32, 1u);
      } else if (SPLIT) {
        mma_tile<N_OUT, BLK>(acc, a_lo + j * 32, b_hi + j * 32, first);
        mma_tile<N_OUT, BLK>(acc, a_hi + j * 32, b_lo + j * 32, 1u);
        mma_tile<N_OUT, BLK>(acc, a_hi + j * 32, b_hi + j * 32, 1u);
      } else {
        mma_tile<N_OUT, BLK>(acc, a_hi + j * 32, b_hi + j * 32, first);
      }
    }
    commit();
    wait_all();
    fence_regs(acc);
    __syncthreads();   // both warpgroups have consumed this chunk's shared memory
  }

  // ---- epilogue: accumulator fragments -> shared (aliases the operand buffers) -> global --------
  {
    const int row = wgi * 64 + (warp & 3) * 16 + (lane >> 2);
    const int col = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < N_OUT / 8; ++i) {
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) v[e] = STACKED ? acc[4 * i + e] + acc[N_OUT / 2 + 4 * i + e] : acc[4 * i + e];
      *reinterpret_cast<float2*>(sD + row * S::D_PITCH + 8 * i + col) = make_float2(v[0], v[1]);
      *reinterpret_cast<float2*>(sD + (row + 8) * S::D_PITCH + 8 * i + col) = make_float2(v[2], v[3]);
    }
  }
  __syncthreads();
  constexpr int C4 = N_OUT / 4;
  for (int e = tid; e < BM * C4; e += NUM_THREADS) {
    const int r = e / C4, c4 = e - r * C4;
    if (r < rows_valid)
      st4(a.y + (grow0 + r) * a.ldy + c4 * 4, *reinterpret_cast<const float4*>(sD + r * S::D_PITCH + c4 * 4));
  }
  if (a.out_stats != nullptr) {
    // column statistics: thread -> (column, row part); 4 independent accumulators per sum
    constexpr int PARTS = NUM_THREADS / N_OUT;
    constexpr int RPP = BM / PARTS;
    const int col = tid % N_OUT, part = tid / N_OUT;
    float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
    const int r0 = part * RPP;
    const float* colp = sD + col;
#pragma unroll 4
    for (int r = 0; r < RPP; r += 4) {
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int rr = r0 + r + u;
        const float v = rr < rows_valid ? colp[rr * S::D_PITCH] : 0.f;
        s1[u] += v;
        s2[u] = fmaf(v, v, s2[u]);
      }
    }
    // combine the row parts in shared memory (the BN-coefficient area is free now): one fp64
    // atomic per column and statistic per CTA
    __syncthreads();   // every thread has finished reading sD / sBN
    float* red = sBN;  // [2][PARTS][N_OUT] floats <= 2 * 256
    red[part * N_OUT + col] = (s1[0] + s1[1]) + (s1[2] + s1[3]);
    red[NUM_THREADS + part * N_OUT + col] = (s2[0] + s2[1]) + (s2[2] + s2[3]);
    __syncthreads();
    if (tid < 2 * N_OUT) {
      const int which = tid / N_OUT, c = tid - which * N_OUT;
      double t = 0.0;
#pragma unroll
      for (int pp = 0; pp < PARTS; ++pp) t += (double)red[which * NUM_THREADS + pp * N_OUT + c];
      atomicAdd(a.out_stats + (size_t)g * 2 * a.cout + which * a.cout + c, t);
    }
  }
}

static int g_mode = 3;  // 0: SIMT fp32 GEMM, 1: TF32 tensor cores, 3: 3xTF32 tensor cores (default)

template <int N_OUT, int NSPLIT>
static int launch_one(const GemmArgs& a, cudaStream_t st, const char* name) {
  using S = Smem<N_OUT, NSPLIT>;
  static unsigned long long smem_done = 0;  // per device: the attribute belongs to the device's context
  PMVS_TRY((ensure_dyn_smem(gemm_tc_kernel<N_OUT, NSPLIT>, S::TOTAL, smem_done, "gemm_tc")));
  dim3 grid(cdiv(a.rows_per_group, BM), a.groups);
  prof_begin(name, st);
  gemm_tc_kernel<N_OUT, NSPLIT><<<grid, NUM_THREADS, S::TOTAL, st>>>(a);
  return check_launch("gemm_tc_kernel", st);
}

}  // namespace tc

// returns -1 if the tensor-core path does not apply (caller falls back to the SIMT kernel)
int launch_gemm_tc(const GemmArgs& a, cudaStream_t st, const char* name) {
  if (tc::g_mode == 0) return -1;
  if (a.cin % 8 != 0 || a.cin > 224 || a.ldx % 4 != 0 || a.ldy % 4 != 0 || a.groups > 65535) return -1;
  if (((uintptr_t)a.x & 15) || ((uintptr_t)a.y & 15) || ((uintptr_t)a.w & 15)) return -1;
  const bool x3 = tc::g_mode == 3;
  switch (a.cout) {
    case 16: return x3 ? tc::launch_one<16, 3>(a, st, name) : tc::launch_one<16, 1>(a, st, name);
    case 64: return x3 ? tc::launch_one<64, 3>(a, st, name) : tc::launch_one<64, 1>(a, st, name);
    case 128: return x3 ? tc::launch_one<128, 3>(a, st, name) : tc::launch_one<128, 1>(a, st, name);
  }
  return -1;
}

}  // namespace pmvs

extern "C" int pmvs_set_gemm_mode(int mode) {
  if (mode != 0 && mode != 1 && mode != 3) {
    pmvs::set_error("set_gemm_mode: mode must be 0 (SIMT fp32), 1 (TF32) or 3 (3xTF32)");
    return PMVS_ERR_ARG;
  }
  pmvs::tc::g_mode = mode;
  return PMVS_OK;
}
extern "C" int pmvs_get_gemm_mode(void) { return pmvs::tc::g_mode; }
