// Warpgroup-MMA GEMM, second generation: persistent, warp-specialised, WEIGHTS STATIONARY IN SHARED MEMORY.
//
//   Y[r, 0:cout] = f(X[r, 0:K]) * W[0:cout, 0:K]^T       r = points, fp32 in / fp32 out (3xTF32)
// (reference: the 1x1 nn.Conv1d of networks.py:13-14,22-23,51-52 and nn/conv.py:21-30, followed by
// train-mode BatchNorm + ReLU, which is fused here as the INPUT transform of the next layer).
//
// Why this shape.  The round-1 kernel (gemm_tc.cu) re-loads and re-splits the weight slab for every 128-row tile
// and one CTA per tile serialises load -> convert -> MMA -> epilogue.  Here
//   * the CTA is persistent: the TF32 planes [W_hi ; W_lo] of the whole weight matrix are written to shared memory
//     once per CTA (K-major SWIZZLE_128B, one 32-column chunk after the other) and stay there as the B operand of
//     every tile; cout <= 64 stacks the two planes into one N' = 2 cout operand, so X_hi is read once per k-step
//     (accumulator columns [0,cout) = X_hi*W_hi, [cout,2cout) = X_hi*W_lo + X_lo*W_hi; the epilogue adds the halves).
//   * warp-specialised: 8 producer warps (coalesced 128-bit global loads several chunks ahead -> fused input
//     BatchNorm+ReLU -> TF32 hi/lo split -> K-major SWIZZLE_128B stores into an mbarrier ring of 128-point operand
//     stages) and two consumer warpgroups (wgmma.mma_async m64nNk8 on rows [64 w, 64 w + 64) of the stage, accumulator
//     in registers, epilogue straight from the fragments).  The producers run ahead of the consumers' epilogue by
//     the depth of the ring, so the global loads never stop.
//   * the BatchNorm statistics of the outputs (per-channel sum / sum of squares) are reduced per warp and tile in
//     fp32 (shuffles), combined over the warps in fp64 (shared-memory atomics), carried by one thread per statistic,
//     and leave the CTA as one fp64 atomic per statistic and group.
// Precision: as gemm_tc.cu - hi = the 10 explicit mantissa bits the tensor core reads, lo = x - hi (exact).
#include <algorithm>
#include <type_traits>

#include "common.cuh"
#include "tensor_map.cuh"
#include "wgmma.cuh"

namespace pmvs {

namespace ws {

using namespace wg;

constexpr int NT = 128;                       // points per tile: two consumer warpgroups x wgmma M = 64
constexpr int KC = 32;                        // fp32 K columns per chunk == one 128-byte swizzle row
constexpr int PLANE_BYTES = NT * KC * 4;      // 16 KB
constexpr int STAGE_BYTES = 2 * PLANE_BYTES;  // X_hi, X_lo
// Warp roles: warps [0, 8) = two consumer warpgroups, warps [8, 16) = producers.  512 threads leave 128 registers a
// thread, which the 64 accumulator registers of a consumer need.
constexpr int CONS_WARPS = 8, CONS_THREADS = CONS_WARPS * 32;
constexpr int PROD_WARPS = 8, PROD_WARP0 = CONS_WARPS, PROD_THREADS = PROD_WARPS * 32;
constexpr int THREADS = CONS_THREADS + PROD_THREADS;
constexpr int A_LD = NT * 8 / PROD_THREADS;   // 16-byte pieces per producer thread and chunk (4)
static_assert(A_LD * PROD_THREADS == NT * 8, "the producers share a chunk evenly");
constexpr int MAXK = 224;
constexpr int SMEM_MAX = 227 * 1024;          // shared memory a block may use on sm_90

// Shared-memory layout.  ASYNC = 0: the producers prefetch through registers (4 chunks ahead) into an NSTAGES-stage
// operand ring.  ASYNC = N > 0: the raw fp32 chunks travel global -> shared memory with cp.async (LDGSTS, no registers
// held) into an N-stage staging ring, N - 1 chunks ahead; the producer converts its own pieces from there into the
// operand ring.  16 KB per staging stage, 32 KB per operand stage (X_hi | X_lo).  The weight planes follow
// (2 * cout * 128 bytes per K chunk, sized at launch), then the small tables at TAIL.
template <int ASYNC, int NSTAGES>
struct Layout {
  static constexpr int NST = NSTAGES;  // operand stages
  static constexpr int RING = 0;
  static constexpr int STAGING = RING + NST * STAGE_BYTES;
  static constexpr int W = STAGING + ASYNC * PLANE_BYTES;
};
__host__ __device__ constexpr int weight_bytes(int cout, int nch) { return nch * 2 * cout * 128; }
// after the weights: input BatchNorm tables (2 x MAXK floats), the output-statistics scratch (2 x cout doubles), the mbarriers
constexpr int TAIL_BN = 0, TAIL_RED = TAIL_BN + 2 * MAXK * 4;
__host__ __device__ constexpr int tail_bar(int cout) { return TAIL_RED + 2 * cout * 8; }
__host__ __device__ constexpr int tail_bytes(int cout) { return tail_bar(cout) + 128; }

__device__ __forceinline__ void sts128(uint32_t addr, float4 v) {
  asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr) : "memory");
  return v;
}

struct TileRange {
  int first, count;
};
__device__ __forceinline__ TileRange my_tiles(int total) {
  // contiguous, balanced: CTA b owns [b*total/G, (b+1)*total/G)
  const long long G = gridDim.x, b = blockIdx.x;
  const int lo = (int)(b * total / G), hi = (int)((b + 1) * total / G);
  return TileRange{lo, hi - lo};
}

template <int COUT, bool IN_BN, int ASYNC, int NSTAGES>
__global__ void __launch_bounds__(THREADS, 1) gemm_ws_kernel(const GemmArgs a) {
  using LY = Layout<ASYNC, NSTAGES>;
  constexpr int STAGES = LY::NST;
  constexpr int SM_RING = LY::RING, SM_STAGING = LY::STAGING, SM_W = LY::W;
  constexpr int PF = ASYNC > 0 ? ASYNC - 1 : 4;  // chunks of global loads in flight per producer thread
  constexpr bool STACKED = COUT <= 64;
  constexpr int W_CHUNK = 2 * COUT * 128;        // [W_hi ; W_lo] of one K chunk
  extern __shared__ __align__(1024) unsigned char smem[];  // SWIZZLE_128B operands need 1024-byte alignment
  const uint32_t smem_base = smem_u32(smem);

  const int K = a.cin;
  const int nch = (K + KC - 1) / KC;
  // the warp index through a shuffle: the compiler then knows the role branches below are warp-uniform
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int tpg = (a.rows_per_group + NT - 1) / NT;  // tiles per group
  const TileRange tr = my_tiles(a.groups * tpg);

  unsigned char* tail = smem + SM_W + weight_bytes(COUT, nch);
  float* sBN = (float*)(tail + TAIL_BN);      // input BatchNorm as one FMA per element: A = istd * gamma | B = beta - mean * A, x MAXK
  double* sRed = (double*)(tail + TAIL_RED);  // per-tile sums of the outputs: [sum(COUT) | sumsq(COUT)]
  // bars: full[STAGES] (one arrival per producer warp), empty[STAGES] (one per consumer warp)
  const uint32_t bar0 = smem_u32(tail + tail_bar(COUT));
  auto bar_full = [&](int s) { return bar0 + 8u * (uint32_t)s; };
  auto bar_empty = [&](int s) { return bar0 + 8u * (uint32_t)(STAGES + s); };

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(bar_full(s), PROD_WARPS);
      mbar_init(bar_empty(s), CONS_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = tid; i < 2 * COUT; i += THREADS) sRed[i] = 0.0;
  // ---- weights -> shared memory (B operand), once per CTA: chunk c = rows [0,COUT) W_hi | rows [COUT,2 COUT) W_lo ----
  for (int e = tid; e < COUT * nch * 8; e += THREADS) {
    const int n = e / (nch * 8), rem = e - n * (nch * 8), c = rem >> 3, pc = rem & 7;
    const int k0 = c * KC + pc * 4;  // K is a multiple of 8: a 16-byte piece is all inside or all padding
    const float4 v = k0 < K ? ldg4(a.w + (size_t)n * K + k0) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 hi, lo;
    hi.x = tf32_hi(v.x); hi.y = tf32_hi(v.y); hi.z = tf32_hi(v.z); hi.w = tf32_hi(v.w);
    lo.x = __fsub_rn(v.x, hi.x); lo.y = __fsub_rn(v.y, hi.y); lo.z = __fsub_rn(v.z, hi.z); lo.w = __fsub_rn(v.w, hi.w);
    const uint32_t dst = smem_base + SM_W + c * W_CHUNK + swz128(n, pc);
    sts128(dst, hi);
    sts128(dst + COUT * 128, lo);
  }
  fence_proxy_async();  // the weight planes are read by the tensor core's async proxy
  __syncthreads();

  if (warp >= PROD_WARP0) {
    // =============================== producers ==========================================================
    const int ptid = tid - PROD_WARP0 * 32;
    const int pc = ptid & 7;     // 16-byte piece inside the 128-byte row
    const int prow = ptid >> 3;  // first row of this thread; rows prow + ROWS_STEP * i
    constexpr int ROWS_STEP = PROD_THREADS / 8;
    const int total = tr.count * nch;
    int cur_g = -1;
    float4 buf[ASYNC > 0 ? 1 : PF + 1][A_LD];
    // byte offsets of this thread's pieces inside a K-major SWIZZLE_128B plane (the same for every chunk)
    int soff[A_LD];
#pragma unroll
    for (int i = 0; i < A_LD; ++i) {
      const int r = prow + ROWS_STEP * i;
      soff[i] = swz128(r, pc);
    }

    // (tile, chunk) cursors of the load stream and of the store stream: both walk items 0, 1, 2, .. in order, so
    // they advance incrementally (no integer divisions / 64-bit multiplies on the per-chunk path)
    struct Cursor {
      int g, row0, c;
      const float* ptr;  // load stream only: this thread's first piece of the current chunk
    };
    Cursor ci, cp;
    {
      const int t0 = tr.first;
      ci.g = t0 / tpg; ci.row0 = (t0 - ci.g * tpg) * NT; ci.c = 0;
      ci.ptr = a.x + ((size_t)ci.g * a.rows_per_group + ci.row0 + prow) * a.ldx + pc * 4;
      cp = ci;
    }
    const bool last_kvalid = (nch - 1) * KC + pc * 4 < K;  // K % 32 != 0: the last chunk is partly padding
    const size_t tile_step = (size_t)NT * a.ldx - (size_t)(nch - 1) * KC;
    int n_issued = 0;
    auto issue = [&](float4 (&xa)[A_LD]) {
      const int rows_valid = a.rows_per_group - ci.row0;  // >= NT except in the last tile of a group
      const bool kvalid = ci.c != nch - 1 || last_kvalid;
#pragma unroll
      for (int i = 0; i < A_LD; ++i) {
        const int r = prow + ROWS_STEP * i;
        const bool ok = kvalid && r < rows_valid;
        if (ASYNC > 0) {
          // 16 bytes global -> this thread's own slot of the staging stage; src-size 0 zero-fills (padding rows / columns)
          const uint32_t dst = smem_base + SM_STAGING + (n_issued % (ASYNC > 0 ? ASYNC : 1)) * PLANE_BYTES + (ptid + PROD_THREADS * i) * 16;
          const float* src = ok ? ci.ptr + (size_t)(ROWS_STEP * i) * a.ldx : a.x;
          asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
        } else {
          xa[i] = ok ? ldg4(ci.ptr + (size_t)(ROWS_STEP * i) * a.ldx) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
      }
      ++n_issued;
      if (++ci.c == nch) {
        ci.c = 0;
        ci.row0 += NT;
        ci.ptr += tile_step;
        if (ci.row0 >= a.rows_per_group) {  // next group: its rows follow the previous group's (ragged tail skipped)
          ci.row0 = 0;
          ++ci.g;
          ci.ptr = a.x + ((size_t)ci.g * a.rows_per_group + prow) * a.ldx + pc * 4;
        }
      } else {
        ci.ptr += KC;
      }
    };
    auto advance = [&](Cursor& cu) {
      if (++cu.c == nch) {
        cu.c = 0;
        cu.row0 += NT;
        if (cu.row0 >= a.rows_per_group) {
          cu.row0 = 0;
          ++cu.g;
        }
      }
    };
    auto put = [&](const float4 (&xa)[A_LD], int n) {
      const int k0 = cp.c * KC + pc * 4;
      if (IN_BN) {
        const int g = cp.g;
        if (g != cur_g) {  // uniform over all producer threads: they walk the same item sequence
          named_bar_sync(1, PROD_THREADS);
          const double* s = a.in_stats + (size_t)g * 2 * K;
          for (int cc = ptid; cc < K; cc += PROD_THREADS) {
            const BnCoef k = bn_coef(s[cc], s[K + cc], a.in_count, a.eps);
            // the same coefficient form as the EdgeConv apply kernels (edge_tile.cu): relu(fma(x, A, B))
            const float A = __fmul_rn(k.invstd, a.in_gamma[cc]);
            sBN[cc] = A;
            sBN[MAXK + cc] = fmaf(-k.mean, A, a.in_beta[cc]);
          }
          named_bar_sync(1, PROD_THREADS);
          cur_g = g;
        }
      }
      const int stage = n % STAGES;
      mbar_wait(bar_empty(stage), (uint32_t)(((n / STAGES) & 1) ^ 1));
      const uint32_t hi_plane = smem_base + SM_RING + stage * STAGE_BYTES;
      if (ASYNC > 0) {
        // every call is preceded by exactly one commit (possibly of an empty group), so "at most PF groups pending"
        // means the group of chunk n has landed; the thread reads back only what it copied itself
        asm volatile("cp.async.wait_group %0;" ::"n"(PF) : "memory");
      }
#pragma unroll
      for (int i = 0; i < A_LD; ++i) {
        float4 v = ASYNC > 0 ? lds128(smem_base + SM_STAGING + (n % (ASYNC > 0 ? ASYNC : 1)) * PLANE_BYTES + (ptid + PROD_THREADS * i) * 16)
                             : xa[i];
        if (IN_BN) {
          // rows / columns beyond the valid range were loaded as zeros and must stay zero
          const int r = prow + ROWS_STEP * i;
          if (k0 < K && r < a.rows_per_group - cp.row0) {
            // k0 is a multiple of 4 and the two tables start MAXK floats apart: two 128-bit loads
            const float4 A4 = *reinterpret_cast<const float4*>(&sBN[k0]);
            const float4 B4 = *reinterpret_cast<const float4*>(&sBN[MAXK + k0]);
            v.x = fmaxf(fmaf(v.x, A4.x, B4.x), 0.f);
            v.y = fmaxf(fmaf(v.y, A4.y, B4.y), 0.f);
            v.z = fmaxf(fmaf(v.z, A4.z, B4.z), 0.f);
            v.w = fmaxf(fmaf(v.w, A4.w, B4.w), 0.f);
          }
        }
        float4 hi, lo;
        hi.x = tf32_hi(v.x); hi.y = tf32_hi(v.y); hi.z = tf32_hi(v.z); hi.w = tf32_hi(v.w);
        lo.x = __fsub_rn(v.x, hi.x); lo.y = __fsub_rn(v.y, hi.y); lo.z = __fsub_rn(v.z, hi.z); lo.w = __fsub_rn(v.w, hi.w);
        sts128(hi_plane + soff[i], hi);
        sts128(hi_plane + PLANE_BYTES + soff[i], lo);
      }
      fence_proxy_async();  // these generic-proxy stores are read by the consumers' wgmma (async proxy)
      __syncwarp();
      if (lane == 0) mbar_arrive(bar_full(stage));
      advance(cp);
    };

    // PF chunks (PF x 16 KB per SM) of loads in flight while one is converted and stored: at ~2 us of loaded
    // DRAM latency the SM's share of the HBM bandwidth needs ~100 KB in flight
    if (ASYNC > 0) {
      for (int i = 0; i < PF; ++i) {
        if (i < total) issue(buf[0]);
        asm volatile("cp.async.commit_group;" ::: "memory");
      }
      for (int m = 0; m < total; ++m) {
        if (m + PF < total) issue(buf[0]);
        asm volatile("cp.async.commit_group;" ::: "memory");
        put(buf[0], m);
      }
    } else {
#pragma unroll
      for (int i = 0; i < PF; ++i)
        if (i < total) issue(buf[i]);
      for (int n = 0; n < total; n += PF + 1) {
#pragma unroll
        for (int u = 0; u <= PF; ++u) {
          const int m = n + u;
          if (m < total) {
            if (m + PF < total) issue(buf[ASYNC > 0 ? 0 : (u + PF) % (PF + 1)]);
            put(buf[ASYNC > 0 ? 0 : u], m);
          }
        }
      }
    }
  } else {
    // =============================== consumers: MMA + epilogue ==========================================
    const int wgi = warp >> 2;                                   // warpgroup: rows [64 wgi, 64 wgi + 64) of a tile
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2);   // this thread's fragment rows: frow, frow + 8
    const int fcol = 2 * (lane & 3);                             // fragment columns 8 i + fcol + {0, 1}
    constexpr int ACC_REGS = (STACKED ? 2 * COUT : COUT) / 2;
    constexpr int BLK = COUT < 64 ? COUT : 64;  // one wgmma shape for every product into this accumulator (wgmma.cuh)
    float acc[ACC_REGS];
    const uint32_t w_base = smem_base + SM_W;
    // output statistics: thread t < 2 COUT carries statistic t ([sum | sumsq] x COUT) of the current group in fp64
    double racc = 0.0;
    int acc_g = -1;
    auto flush = [&]() {
      if (a.out_stats != nullptr && acc_g >= 0 && tid < 2 * COUT) atomicAdd(a.out_stats + (size_t)acc_g * 2 * a.cout + tid, racc);
      racc = 0.0;
    };
    int n = 0;
    for (int it = 0; it < tr.count; ++it) {
      const int t = tr.first + it;
      const int g = t / tpg, row0 = (t - g * tpg) * NT;
      const int rows_valid = min(NT, a.rows_per_group - row0);
      const size_t grow0 = (size_t)g * a.rows_per_group + row0;
      if (g != acc_g) {
        flush();
        acc_g = g;
      }
      for (int c = 0; c < nch; ++c, ++n) {
        const int stage = n % STAGES;
        mbar_wait(bar_full(stage), (uint32_t)((n / STAGES) & 1));
        const uint32_t x_hi = smem_base + SM_RING + stage * STAGE_BYTES + wgi * 64 * 128, x_lo = x_hi + PLANE_BYTES;
        const uint32_t w_hi = w_base + c * W_CHUNK, w_lo = w_hi + COUT * 128;
        const int ksteps = min(KC, K - c * KC) / 8;
        fence();
        for (int j = 0; j < ksteps; ++j) {
          const uint32_t first = (c | j) != 0 ? 1u : 0u;
          if (STACKED) {
            mma_tile<2 * COUT, BLK>(acc, x_hi + j * 32, w_hi + j * 32, first);
            mma_tile<COUT, BLK>(acc + COUT / 2, x_lo + j * 32, w_hi + j * 32, 1u);
          } else {
            mma_tile<COUT, BLK>(acc, x_lo + j * 32, w_hi + j * 32, first);
            mma_tile<COUT, BLK>(acc, x_hi + j * 32, w_lo + j * 32, 1u);
            mma_tile<COUT, BLK>(acc, x_hi + j * 32, w_hi + j * 32, 1u);
          }
        }
        commit();
        wait_all();
        fence_regs(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty(stage));  // this warp's MMAs have consumed the stage
      }
      // ---- epilogue from the fragments: a warp's store instruction writes 32-byte runs of 8 rows ----
      const bool ok0 = frow < rows_valid, ok1 = frow + 8 < rows_valid;
      float* y0 = a.y + (grow0 + frow) * a.ldy + fcol;
      float* y1 = y0 + (size_t)8 * a.ldy;
#pragma unroll
      for (int i = 0; i < COUT / 8; ++i) {
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = STACKED ? acc[4 * i + e] + acc[COUT / 2 + 4 * i + e] : acc[4 * i + e];
        if (ok0) *reinterpret_cast<float2*>(y0 + 8 * i) = make_float2(v[0], v[1]);
        if (ok1) *reinterpret_cast<float2*>(y1 + 8 * i) = make_float2(v[2], v[3]);
        if (a.out_stats != nullptr) {
          if (!ok0) v[0] = v[1] = 0.f;
          if (!ok1) v[2] = v[3] = 0.f;
          float s[4] = {v[0] + v[2], v[1] + v[3], fmaf(v[0], v[0], v[2] * v[2]), fmaf(v[1], v[1], v[3] * v[3])};
#pragma unroll
          for (int e = 0; e < 4; ++e) {  // the 8 lanes with the same lane % 4 hold the same columns
            s[e] += __shfl_xor_sync(0xffffffffu, s[e], 4);
            s[e] += __shfl_xor_sync(0xffffffffu, s[e], 8);
            s[e] += __shfl_xor_sync(0xffffffffu, s[e], 16);
          }
          if (lane < 4) {  // fp64 from here on: the order in which the 8 warps arrive does not show in the fp32 results
            atomicAdd(&sRed[8 * i + fcol], (double)s[0]);
            atomicAdd(&sRed[8 * i + fcol + 1], (double)s[1]);
            atomicAdd(&sRed[COUT + 8 * i + fcol], (double)s[2]);
            atomicAdd(&sRed[COUT + 8 * i + fcol + 1], (double)s[3]);
          }
        }
      }
      if (a.out_stats != nullptr) {
        named_bar_sync(2, CONS_THREADS);  // every consumer warp has added this tile's sums
        if (tid < 2 * COUT) {
          racc += sRed[tid];
          sRed[tid] = 0.0;
        }
        named_bar_sync(2, CONS_THREADS);  // cleared before the next tile's sums arrive
      }
    }
    flush();
  }
}

// Ring depths by K: <ASYNC staging stages, operand stages> of the cp.async form and of the register-prefetch form
constexpr int DEEP_K = 160;
template <int ASYNC, int NSTAGES>
constexpr int smem_bytes(int cout, int cin) {
  return Layout<ASYNC, NSTAGES>::W + weight_bytes(cout, (cin + KC - 1) / KC) + tail_bytes(cout);
}
constexpr bool fits(int cin, int cout) {
  return cin <= DEEP_K ? (smem_bytes<4, 2>(cout, cin) <= SMEM_MAX && smem_bytes<0, 4>(cout, cin) <= SMEM_MAX)
                       : (smem_bytes<3, 2>(cout, cin) <= SMEM_MAX && smem_bytes<0, 3>(cout, cin) <= SMEM_MAX);
}
// The six contractions of a PointFlow iteration must stay on this kernel: growing the tail tables or the rings, or a
// static __shared__ variable in the kernel (which would also break the 1024-byte alignment the swizzled planes need:
// the dynamic window is 1024-aligned only while it starts the block's shared memory), shows up here, not as a
// silently slower pass.  224 -> 64 leaves 128 bytes.
static_assert(fits(136, 64) && fits(32, 64) && fits(64, 128) && fits(224, 64) && fits(64, 64) && fits(64, 16),
              "a hot-path GEMM shape no longer fits the shared memory of gemm_ws_kernel");

template <int COUT, bool IN_BN, int ASYNC, int NSTAGES>
static int launch_pf(const GemmArgs& a, cudaStream_t st, const char* name) {
  const int smem_total = smem_bytes<ASYNC, NSTAGES>(COUT, a.cin);
  if (smem_total > SMEM_MAX) return -1;  // the weight planes of this shape do not fit beside the rings
  static unsigned long long smem_done = 0;
  PMVS_TRY((ensure_dyn_smem(gemm_ws_kernel<COUT, IN_BN, ASYNC, NSTAGES>, SMEM_MAX, smem_done, "gemm_ws")));
  const long long tiles = (long long)a.groups * cdiv(a.rows_per_group, NT);
  const int grid = (int)std::min<long long>(tiles, sm_count());
  prof_begin(name, st);
  gemm_ws_kernel<COUT, IN_BN, ASYNC, NSTAGES><<<grid, THREADS, smem_total, st>>>(a);
  return check_launch("gemm_ws_kernel", st);
}
// =============================== PMVS_OPT_GEMM = 3: TMA producer, register-A wgmma, ping-pong consumers ===========
// The same weight planes and the same products as above, with a different path for X:
//   * each consumer warpgroup owns every other 64-point tile of the CTA's range (ping-pong: one warpgroup's epilogue
//     overlaps the other's MMAs) and has its own producer warp, ring and full / empty barriers.  One thread of the
//     producer warp loads 64-row x 32-column boxes of X with the TMA (3-D tensor map (cin, rows, groups),
//     SWIZZLE_128B; the ragged rows of a group and the K padding arrive as zeros) into the warpgroup's ring of 8 KB
//     stages, completing on expect_tx barriers.  The two rings share the shared memory the weight planes leave (6 + 6
//     stages for 224 -> 64).  A stage is only ever filled for and read by one warpgroup, in order, so a parity wait
//     can never see the phase of another warpgroup's item, whatever order the TMA boxes complete in;
//   * per chunk a consumer reads its wgmma A fragments straight from the swizzled stage (4 LDS.32 per k-step,
//     conflict-free), applies the input BatchNorm+ReLU, splits hi / lo in registers and issues the chunk's MMAs as
//     one wgmma group (the k-step count is a template parameter, so no branch separates them).  It waits for the
//     group, then hands the stage back and the next chunk rewrites the fragments; the other warpgroup's MMAs and the
//     producers' loads continue meanwhile.
// No shared-memory copy of the converted operands exists any more: per 224 -> 64 chunk of 64 points, shared memory
// carries the 8 KB the TMA writes, the 8 KB read into the fragments and the weight reads of the MMAs.
// Every output element goes through the same instruction sequence as under option 2, so Y is identical; the output
// statistics are summed in another order (fp64 per warpgroup and group instead of per CTA and tile).
namespace tma {
constexpr int NT = 64;                              // points per tile = one warpgroup's wgmma M
constexpr int STAGE_BYTES = NT * KC * 4;            // one TMA box, 8 KB
constexpr int CONS_THREADS = 256;                   // two consumer warpgroups
constexpr int THREADS = CONS_THREADS + 64;          // + one producer warp per warpgroup (168 registers a thread)
constexpr int MAX_STAGES = 32, MIN_STAGES = 8;      // both rings together; each warpgroup gets half
constexpr int BN_FLOATS = (MAXK / KC) * 4 * 16;     // per warpgroup: [chunk][lane % 4][A x 8 | B x 8]
// after the ring: BatchNorm tables and output sums of each warpgroup, then the full / empty barriers
constexpr int TAIL_BN = 0, TAIL_RED = TAIL_BN + 2 * BN_FLOATS * 4;
__host__ __device__ constexpr int tail_bar(int cout) { return TAIL_RED + 2 * 2 * cout * 8; }
__host__ __device__ constexpr int tail_bytes(int cout) { return tail_bar(cout) + 2 * MAX_STAGES * 8; }
__host__ __device__ constexpr int stages_for(int cin, int cout) {
  return (SMEM_MAX - weight_bytes(cout, (cin + KC - 1) / KC) - tail_bytes(cout)) / STAGE_BYTES < MAX_STAGES
             ? (SMEM_MAX - weight_bytes(cout, (cin + KC - 1) / KC) - tail_bytes(cout)) / STAGE_BYTES
             : MAX_STAGES;
}
}  // namespace tma

// one round of a reduce-scatter over lanes l, l ^ m: the lane keeps the half of its N values selected by lane bit m and
// adds the partner's copy of that half (the sum of the pair is the one a butterfly step computes)
template <int N>
__device__ __forceinline__ void reduce_scatter_round(float* sv, int lane, int m) {
  const bool up = (lane & m) != 0;
#pragma unroll
  for (int k = 0; k < N / 2; ++k) {
    const float keep = up ? sv[k + N / 2] : sv[k], send = up ? sv[k] : sv[k + N / 2];
    sv[k] = keep + __shfl_xor_sync(0xffffffffu, send, m);
  }
}

template <int COUT, bool IN_BN>
__global__ void __launch_bounds__(tma::THREADS, 1) gemm_tma_kernel(const __grid_constant__ CUtensorMap tmx,
                                                                   const GemmArgs a, const int wstages) {
  constexpr int NT = tma::NT, STAGE_BYTES = tma::STAGE_BYTES, CONS_THREADS = tma::CONS_THREADS;
  constexpr int MAX_STAGES = tma::MAX_STAGES, BN_FLOATS = tma::BN_FLOATS, TAIL_BN = tma::TAIL_BN, TAIL_RED = tma::TAIL_RED;
  constexpr bool STACKED = COUT <= 64;
  constexpr int W_CHUNK = 2 * COUT * 128;
  constexpr int ACC_REGS = (STACKED ? 2 * COUT : COUT) / 2;
  extern __shared__ __align__(1024) unsigned char smem[];
  const uint32_t smem_base = smem_u32(smem);

  const int K = a.cin;
  const int nch = (K + KC - 1) / KC;
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const int tpg = (a.rows_per_group + NT - 1) / NT;
  const TileRange tr = my_tiles(a.groups * tpg);
  // [weights | ring of warpgroup 0 | ring of warpgroup 1 | tail], each 1024-byte aligned
  unsigned char* tail = smem + weight_bytes(COUT, nch) + 2 * wstages * STAGE_BYTES;
  const uint32_t bar0 = smem_u32(tail + tma::tail_bar(COUT));
  // barriers of stage s of warpgroup w's ring: full (one arrival + the TMA bytes), empty (one arrival per consumer warp)
  auto bar_full = [&](int w, int s) { return bar0 + 8u * (uint32_t)(w * (MAX_STAGES / 2) + s); };
  auto bar_empty = [&](int w, int s) { return bar0 + 8u * (uint32_t)(MAX_STAGES + w * (MAX_STAGES / 2) + s); };

  if (tid == 0) {
    for (int w = 0; w < 2; ++w)
      for (int s = 0; s < wstages; ++s) {
        mbar_init(bar_full(w, s), 1);
        mbar_init(bar_empty(w, s), 4);
      }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= CONS_THREADS / 32) {
    // =============================== producers: one thread per warpgroup, TMA ==================================
    // They start while the consumers are still writing the weight planes.
    const int w = warp - CONS_THREADS / 32;
    if (lane == 0) {
      const uint32_t ring = smem_base + weight_bytes(COUT, nch) + w * wstages * STAGE_BYTES;
      int stage = 0;
      uint32_t phase = 0;
      for (int i = w; i < tr.count; i += 2) {
        const int t = tr.first + i, g = t / tpg, row0 = (t - g * tpg) * NT;
        for (int c = 0; c < nch; ++c) {
          mbar_wait(bar_empty(w, stage), phase ^ 1u);
          mbar_arrive_expect_tx(bar_full(w, stage), STAGE_BYTES);
          tma_load_3d(ring + stage * STAGE_BYTES, &tmx, c * KC, row0, g, bar_full(w, stage));
          if (++stage == wstages) {
            stage = 0;
            phase ^= 1u;
          }
        }
      }
    }
    return;
  }

  // =============================== consumers ==========================================================
  const int wgi = warp >> 2, wtid = tid & 127;
  const uint32_t ring = smem_base + weight_bytes(COUT, nch) + wgi * wstages * STAGE_BYTES;
  float* sBN = (float*)(tail + TAIL_BN) + wgi * BN_FLOATS;
  double* sRed = (double*)(tail + TAIL_RED) + wgi * 2 * COUT;  // this warpgroup's [sum(COUT) | sumsq(COUT)] of a group
  for (int i = wtid; i < 2 * COUT; i += 128) sRed[i] = 0.0;
  // weights -> shared memory (B operand), as in gemm_ws_kernel
  store_weight_planes<COUT>(smem_base, a.w, K, tid, CONS_THREADS);
  fence_proxy_async();
  named_bar_sync(1, CONS_THREADS);

  // this thread's A elements: rows r, r + 8 of the warpgroup's tile, columns 8 j + q (+ 4) of k-step j; in the
  // swizzled box the 16-byte piece p of row r sits at piece p ^ (r & 7), and row r + 8 is 1024 bytes further
  const int r = (warp & 3) * 16 + (lane >> 2), q = lane & 3;
  const uint32_t fbase = r * 128 + q * 4, fx = (r & 7) << 4;
  const int frow = r, fcol = 2 * q;  // accumulator fragment: rows frow, frow + 8, columns 8 i + fcol + {0, 1}
  const uint32_t w_base = smem_base;
  float acc[ACC_REGS];
  uint32_t fh[16], fl[16];  // [4 j + e]: the hi / lo A fragments of the k-steps of a chunk
  const uint32_t wg_bar = 2 + wgi;

  // Output statistics.  Per tile, a warp's fp32 sums over its 16 rows are reduce-scattered over the 8 lanes that
  // hold the same columns (the same pairings, lane ^ 4, then ^ 8, then ^ 16, as the butterfly of gemm_ws_kernel, so
  // the same fp32 values), after which lane l owns NV statistics and adds them to fp64 registers.  The 4 warps meet
  // in shared memory once per group.  Statistic of value k = 4 i + e (e: sum col, sum col + 1, sumsq col, sumsq col + 1
  // of col = 8 i + fcol): lane l owns k = kofs + j, j < NV.
  // cout = 128 runs this in two passes of 64 columns (i += 8 h), which keeps it within 168 registers.
  constexpr int HC = COUT < 64 ? COUT : 64, NH = COUT / HC;
  constexpr int NV = HC / 16;  // (HC / 8) x 4 values per lane, / 8 lanes
  const int kofs = ((lane >> 2) & 1) * (8 * NV / 2) + ((lane >> 3) & 1) * (8 * NV / 4) + ((lane >> 4) & 1) * (8 * NV / 8);
  double racc[NH][NV];
#pragma unroll
  for (int h = 0; h < NH; ++h)
#pragma unroll
    for (int j = 0; j < NV; ++j) racc[h][j] = 0.0;
  auto flush = [&](int g) {  // the warpgroup's sums of group g -> global memory, once per statistic
    if (a.out_stats == nullptr) return;
#pragma unroll
    for (int h = 0; h < NH; ++h)
#pragma unroll
      for (int j = 0; j < NV; ++j) {
        const int k = kofs + j, i = (k >> 2) + h * (HC / 8), e = k & 3;
        atomicAdd(&sRed[(e >> 1) * COUT + 8 * i + fcol + (e & 1)], racc[h][j]);
        racc[h][j] = 0.0;
      }
    named_bar_sync(wg_bar, 128);
    for (int s = wtid; s < 2 * COUT; s += 128) {
      atomicAdd(a.out_stats + (size_t)g * 2 * a.cout + s, sRed[s]);
      sRed[s] = 0.0;
    }
  };

  // chunk c of the current tile (item m of this warpgroup's ring) with KSTEPS k-steps
  auto chunk = [&](auto KSTEPS, int c, int m) {
    constexpr int ksteps = decltype(KSTEPS)::value;
    const int stage = m % wstages;
    mbar_wait(bar_full(wgi, stage), (uint32_t)((m / wstages) & 1));
    mma_chunk_3xtf32<COUT, IN_BN, ksteps>(acc, fh, fl, ring + stage * STAGE_BYTES + fbase, fx, sBN + (c * 4 + q) * 16,
                                          w_base + c * W_CHUNK, c);
    // The stage goes back to the producer only now.  Released straight after the loads, the arrive was scheduled
    // ahead of the loads' results and the TMA could overwrite data that had not been read yet.  The fragments went
    // through the MMAs just waited for, so every value read from the stage has arrived.
    __syncwarp();
    if (lane == 0) mbar_arrive(bar_empty(wgi, stage));
  };
  // only the last chunk of a K that is not a multiple of 32 (136: one k-step) has fewer than 4 k-steps
  auto chunk_ks = [&](int c, int m) {
    switch (min(KC, K - c * KC) / 8) {
      case 4: chunk(std::integral_constant<int, 4>(), c, m); break;
      case 3: chunk(std::integral_constant<int, 3>(), c, m); break;
      case 2: chunk(std::integral_constant<int, 2>(), c, m); break;
      default: chunk(std::integral_constant<int, 1>(), c, m); break;
    }
  };

  int cur_g = -1;
  for (int i = wgi; i < tr.count; i += 2) {
    const int t = tr.first + i;
    const int g = t / tpg, row0 = (t - g * tpg) * NT;
    const int rows_valid = min(NT, a.rows_per_group - row0);
    const size_t grow0 = (size_t)g * a.rows_per_group + row0;
    if (g != cur_g) {
      named_bar_sync(wg_bar, 128);  // the warpgroup is done with the previous group's tables and sums
      if (cur_g >= 0) flush(cur_g);
      if (IN_BN) {
        // relu(fma(x, A, B)) coefficients as in gemm_ws_kernel, laid out per (chunk, lane % 4); zero beyond K
        const double* s = a.in_stats + (size_t)g * 2 * K;
        for (int e = wtid; e < nch * 64; e += 128) {
          const int c = e >> 6, qq = (e >> 4) & 3, k = e & 15, jh = k & 7;
          const int col = c * KC + 8 * (jh >> 1) + qq + 4 * (jh & 1);
          float val = 0.f;
          if (col < K) {
            const BnCoef bc = bn_coef(s[col], s[K + col], a.in_count, a.eps);
            const float A = __fmul_rn(bc.invstd, a.in_gamma[col]);
            val = k < 8 ? A : fmaf(-bc.mean, A, a.in_beta[col]);
          }
          sBN[e] = val;
        }
      }
      named_bar_sync(wg_bar, 128);
      cur_g = g;
    }
    const int m0 = (i >> 1) * nch;  // this warpgroup's ring items of the tile
    for (int c = 0; c < nch; ++c) chunk_ks(c, m0 + c);
    fence_regs(acc);
    // ---- epilogue from the fragments, as in gemm_ws_kernel ----
    const bool ok0 = frow < rows_valid, ok1 = frow + 8 < rows_valid;
    float* y0 = a.y + (grow0 + frow) * a.ldy + fcol;
    float* y1 = y0 + (size_t)8 * a.ldy;
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      float sv[HC / 2];  // this thread's per-tile sums of columns [64 h, 64 h + HC): k = 4 (i - 8 h) + e
#pragma unroll
      for (int il = 0; il < HC / 8; ++il) {
        const int ii = h * (HC / 8) + il;
        float v[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) v[e] = STACKED ? acc[4 * ii + e] + acc[COUT / 2 + 4 * ii + e] : acc[4 * ii + e];
        if (ok0) *reinterpret_cast<float2*>(y0 + 8 * ii) = make_float2(v[0], v[1]);
        if (ok1) *reinterpret_cast<float2*>(y1 + 8 * ii) = make_float2(v[2], v[3]);
        if (!ok0) v[0] = v[1] = 0.f;
        if (!ok1) v[2] = v[3] = 0.f;
        sv[4 * il + 0] = v[0] + v[2];
        sv[4 * il + 1] = v[1] + v[3];
        sv[4 * il + 2] = fmaf(v[0], v[0], v[2] * v[2]);
        sv[4 * il + 3] = fmaf(v[1], v[1], v[3] * v[3]);
      }
      if (a.out_stats != nullptr) {
        // reduce-scatter: in each round a lane keeps the half of its values selected by one lane bit and adds the
        // partner's copy of that half
        reduce_scatter_round<HC / 2>(sv, lane, 4);
        reduce_scatter_round<HC / 4>(sv, lane, 8);
        reduce_scatter_round<HC / 8>(sv, lane, 16);
#pragma unroll
        for (int j = 0; j < NV; ++j) racc[h][j] += (double)sv[j];
      }
    }
  }
  if (cur_g >= 0) flush(cur_g);
}

// Ring depth of the six contractions of a PointFlow iteration: growing the tail tables or the weight planes, or a
// static __shared__ variable (which would also break the 1024-byte alignment of the swizzled planes), shows up here,
// not as a silently shallower ring.  224 -> 64 gets 6 + 6 stages.
static_assert(tma::stages_for(136, 64) >= tma::MIN_STAGES && tma::stages_for(32, 64) >= tma::MIN_STAGES &&
                  tma::stages_for(64, 128) >= tma::MIN_STAGES && tma::stages_for(224, 64) >= tma::MIN_STAGES &&
                  tma::stages_for(64, 64) >= tma::MIN_STAGES && tma::stages_for(64, 16) >= tma::MIN_STAGES,
              "a hot-path GEMM shape no longer gets the minimum ring depth of gemm_tma_kernel");

// -1: this shape or argument set does not suit the kernel (the caller uses option 2, or reports an error under
// PMVS_OPT_GEMM_STRICT)
template <int COUT, bool IN_BN>
static int launch_tma(const GemmArgs& a, cudaStream_t st, const char* name) {
  const int stages = tma::stages_for(a.cin, COUT);
  if (stages < tma::MIN_STAGES) return -1;
  const int wstages = stages / 2;
  const unsigned long long row_bytes = (unsigned long long)a.ldx * 4, group_bytes = row_bytes * a.rows_per_group;
  if (group_bytes >= (1ull << 40) || (unsigned long long)a.groups > 0xffffffffull) return -1;
  EncodeTiledFn enc = encode_tiled_fn();
  if (enc == nullptr) return -1;
  // X as (cin, rows_per_group, groups): columns >= cin and rows >= rows_per_group of a box read as zeros
  CUtensorMap tm;
  const cuuint64_t gdim[3] = {(cuuint64_t)a.cin, (cuuint64_t)a.rows_per_group, (cuuint64_t)a.groups};
  const cuuint64_t gstr[2] = {row_bytes, group_bytes};
  const cuuint32_t box[3] = {KC, tma::NT, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  if (enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(a.x), gdim, gstr, box, estr,
          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
    return -1;
  const int smem_total = weight_bytes(COUT, cdiv(a.cin, KC)) + 2 * wstages * tma::STAGE_BYTES + tma::tail_bytes(COUT);
  static unsigned long long smem_done = 0;
  PMVS_TRY((ensure_dyn_smem(gemm_tma_kernel<COUT, IN_BN>, SMEM_MAX, smem_done, "gemm_tma")));
  const long long tiles = (long long)a.groups * cdiv(a.rows_per_group, tma::NT);
  const int grid = (int)std::min<long long>(tiles, sm_count());
  prof_begin(name, st);
  gemm_tma_kernel<COUT, IN_BN><<<grid, tma::THREADS, smem_total, st>>>(tm, a, wstages);
  return check_launch("gemm_tma_kernel", st);
}

template <int COUT, bool IN_BN>
static int launch_one(const GemmArgs& a, cudaStream_t st, const char* name) {
  if (opt(OPT_GEMM) == 3) {
    const int rc = launch_tma<COUT, IN_BN>(a, st, name);
    if (rc >= 0 || opt(OPT_GEMM_STRICT)) return rc;
  }
  // The weight planes take 2 * cout * 128 bytes per 32-column chunk of K (112 KB for 224 -> 64), the rings get the
  // rest of the 227 KB: deeper rings for the shapes with K <= 160.
  const bool deep = a.cin <= DEEP_K;
  if (opt(OPT_GEMM) == 1)  // register prefetch, 4 chunks in flight
    return deep ? launch_pf<COUT, IN_BN, 0, 4>(a, st, name) : launch_pf<COUT, IN_BN, 0, 3>(a, st, name);
  // cp.async staging, 3 or 2 chunks (48 / 32 KB) in flight, 2 operand stages
  return deep ? launch_pf<COUT, IN_BN, 4, 2>(a, st, name) : launch_pf<COUT, IN_BN, 3, 2>(a, st, name);
}

}  // namespace ws

static int launch_gemm_ws_any(const GemmArgs& a, cudaStream_t st, const char* name) {
  if (a.cin % 8 != 0 || a.cin > ws::MAXK || a.ldx % 4 != 0 || a.ldy % 2 != 0 || a.groups <= 0 || a.rows_per_group <= 0) return -1;
  if (((uintptr_t)a.x & 15) || ((uintptr_t)a.w & 15) || ((uintptr_t)a.y & 7)) return -1;
  if ((long long)a.groups * cdiv(a.rows_per_group, ws::NT) >= (1ll << 31) / ws::MAXK) return -1;
  const bool bn = a.in_stats != nullptr;
  switch (a.cout) {
    case 16: return bn ? ws::launch_one<16, true>(a, st, name) : ws::launch_one<16, false>(a, st, name);
    case 32: return bn ? ws::launch_one<32, true>(a, st, name) : ws::launch_one<32, false>(a, st, name);
    case 64: return bn ? ws::launch_one<64, true>(a, st, name) : ws::launch_one<64, false>(a, st, name);
    case 128: return bn ? ws::launch_one<128, true>(a, st, name) : ws::launch_one<128, false>(a, st, name);
  }
  return -1;
}

bool gemm_in_bn_fma_form(const GemmArgs& a) {
  if (opt(OPT_GEMM) == 0 || pmvs_get_gemm_mode() != 3) return false;  // launch_gemm's dispatch
  if (a.cin % 8 != 0 || a.cin > ws::MAXK || a.ldx % 4 != 0 || a.ldy % 2 != 0 || a.groups <= 0 || a.rows_per_group <= 0) return false;
  if (((uintptr_t)a.x & 15) || ((uintptr_t)a.w & 15) || ((uintptr_t)a.y & 7)) return false;
  if ((long long)a.groups * cdiv(a.rows_per_group, ws::NT) >= (1ll << 31) / ws::MAXK) return false;
  return a.cout == 16 || a.cout == 32 || a.cout == 64 || a.cout == 128;
}

// returns -1 when this path does not apply (caller falls back to gemm_tc / SIMT); under PMVS_OPT_GEMM = 3 with
// PMVS_OPT_GEMM_STRICT = 1 a launch that gemm_tma_kernel does not take is an error instead
int launch_gemm_ws(const GemmArgs& a, cudaStream_t st, const char* name) {
  const int rc = launch_gemm_ws_any(a, st, name);
  if (rc < 0 && opt(OPT_GEMM) == 3 && opt(OPT_GEMM_STRICT)) {
    set_error("gemm: gemm_tma_kernel does not take cin %d, cout %d, ldx %d, %d groups of %d rows (strict mode)", a.cin,
              a.cout, a.ldx, a.groups, a.rows_per_group);
    return PMVS_ERR_ARG;
  }
  return rc;
}

}  // namespace pmvs
