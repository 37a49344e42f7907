// PointFlow with running-statistics BatchNorm (pmvs_flow_shape.bn_eval = 1, the reference under model.eval()).
//
// With the running statistics every point's result depends on that point alone, so two things the batch-statistics
// path cannot do become possible:
//   * the BatchNorm coefficients are known before any layer runs: flow_eval_coef_kernel writes the EdgeConv tile
//     table (edge_tile.cu) and flow_mlp's table from the running statistics, and the statistics launches, their fp64
//     sums and the running-statistics update disappear;
//   * flow_mlp (224 -> 64 -> 64 -> 16 -> 1, model.py:40-43,220) and the flow head (model.py:220-227) run as one
//     kernel: flow_mlp_head_eval_kernel reads the concatenated EdgeConv output once and keeps h0, h1 and h2 in
//     registers.
//
// flow_mlp_head_eval_kernel.  A work unit is 64 pixels of one cloud: the cloud's rows are m * P + pixel (hypothesis
// slowest), so the unit is 5 blocks of 64 contiguous rows, each one wgmma M-tile.  Per block a consumer warpgroup
//   1. contracts ecat [64, 224] with W0 chunk by chunk from a TMA-fed ring (3-D tensor map (224, P, 5 * clouds),
//      SWIZZLE_128B; pixels >= P arrive as zeros), exactly as gemm_tma_kernel does (mma_chunk_3xtf32);
//   2. applies relu(fma(h, A, B)) to the accumulator and feeds it straight back as the register A operand of the next
//      contraction.  An accumulator thread holds columns 2q, 2q + 1 of each 8-column block, an A fragment thread holds
//      k positions q, q + 4: the weight planes of W1 and W2 are stored with their K columns permuted to match
//      (position p of a block holds column 2p for p < 4, 2(p - 4) + 1 otherwise), so no shuffle is needed;
//   3. does the 16 -> 1 projection with a 4-lane reduction and keeps the raw value of its two rows.
// After the fifth block the warpgroup holds all five hypotheses of its 64 pixels and finishes them with the flow
// head's own code (flow_head_store).  Every product is 3xTF32 (hi * hi + hi * lo + lo * hi), as in the
// batch-statistics path.
// The KEEP variant (pmvs_point_flow_eval_keep) also stores each block's accumulators h0, h1, h2 (pre-BatchNorm, the
// values the fma above reads) and the raw outputs for the backward; its arithmetic is the same instruction for
// instruction, so depth and prob are the same bits.
// Shared memory: the hi / lo planes of the three weight matrices (152 KB), a 4-stage ring of 8 KB boxes per
// warpgroup, the coefficient tables and the barriers.
#include <algorithm>

#include "common.cuh"
#include "tensor_map.cuh"
#include "wgmma.cuh"

namespace pmvs {

namespace {

using namespace wg;

constexpr int FE_NT = 64;                        // rows per block = pixels per unit = wgmma M
constexpr int FE_KC = 32;                        // fp32 K columns per ring stage (one 128-byte swizzle row)
constexpr int FE_STAGE = FE_NT * FE_KC * 4;      // 8 KB
constexpr int FE_CONS = 256;                     // two consumer warpgroups
constexpr int FE_THREADS = FE_CONS + 64;         // + one producer warp per warpgroup
constexpr int FE_K0 = 224, FE_NCH0 = FE_K0 / FE_KC;
constexpr int FE_W0 = FE_NCH0 * 2 * 64 * 128;    // [W0_hi ; W0_lo] per chunk, 112 KB
constexpr int FE_W1 = 2 * 2 * 64 * 128;          // W1 (K = 64, permuted), 32 KB
constexpr int FE_W2 = 2 * 2 * 16 * 128;          // W2 (K = 64, permuted), 8 KB
constexpr int FE_RING = FE_W0 + FE_W1 + FE_W2;
constexpr int FE_WSTAGES = 4;                    // ring stages per warpgroup
constexpr int FE_TAB = FE_RING + 2 * FE_WSTAGES * FE_STAGE;
constexpr int FE_TAB_FLOATS = FLOW_EVAL_MLP_COEF + 16;  // + w3
constexpr int FE_BARS = FE_TAB + FE_TAB_FLOATS * 4;
constexpr int FE_SMEM = FE_BARS + 2 * 2 * FE_WSTAGES * 8;
static_assert(FE_RING % 1024 == 0 && FE_BARS % 8 == 0, "swizzled planes and stages need 1024-byte alignment");
static_assert(FE_SMEM <= 227 * 1024, "flow_mlp_head_eval_kernel: shared memory");

// W [COUT, K] -> B-operand planes as store_weight_planes (wgmma.cuh), with the K columns of each 8-column block in the
// order of the accumulator fragments: position p holds column 2p (p < 4) or 2(p - 4) + 1.  K % 32 == 0.
template <int COUT>
__device__ __forceinline__ void store_weight_planes_paired(uint32_t planes, const float* __restrict__ w, int K, int t,
                                                           int nthreads) {
  const int nch = K / 32;
  for (int e = t; e < COUT * nch * 8; e += nthreads) {
    const int n = e / (nch * 8), rem = e - n * (nch * 8), c = rem >> 3, pc = rem & 7;
    // piece pc = positions 4 pc .. 4 pc + 3 of the chunk = half (pc & 1) of 8-column block pc / 2
    const float* src = w + (size_t)n * K + c * 32 + (pc >> 1) * 8 + (pc & 1);
    const float v[4] = {__ldg(src), __ldg(src + 2), __ldg(src + 4), __ldg(src + 6)};
    float hi[4], lo[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      hi[i] = tf32_hi(v[i]);
      lo[i] = __fsub_rn(v[i], hi[i]);
    }
    const uint32_t dst = planes + c * (2 * COUT * 128) + swz128(n, pc);
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst), "f"(hi[0]), "f"(hi[1]), "f"(hi[2]), "f"(hi[3]) : "memory");
    asm volatile("st.shared.v4.f32 [%0], {%1, %2, %3, %4};" ::"r"(dst + COUT * 128), "f"(lo[0]), "f"(lo[1]), "f"(lo[2]), "f"(lo[3])
                 : "memory");
  }
}

// Columns [32 half, 32 half + 32) of the accumulator of a 64-row tile (STACKED: acc[k] + acc[4 NB + k] are the 8 NB
// output columns, as in gemm_tma_kernel's epilogue; else acc[k]) -> relu(fma(y, A, B)) -> hi / lo register A fragments
// of the 4 k-steps of the next contraction's K chunk `half`
template <int NB, bool STACKED>
__device__ __forceinline__ void bn_relu_fragments(const float* acc, int half, const float* A, const float* B, int q,
                                                  uint32_t (&fh)[16], uint32_t (&fl)[16]) {
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int i = 4 * half + j;
    const int c0 = 8 * i + 2 * q;
    float x[4];
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int col = c0 + (e & 1);
      const float y = STACKED ? acc[4 * i + e] + acc[4 * NB + 4 * i + e] : acc[4 * i + e];
      x[e] = fmaxf(fmaf(y, A[col], B[col]), 0.f);
    }
    // fragment order: (row r, position q), (row r + 8, position q), (row r, q + 4), (row r + 8, q + 4)
    const float a[4] = {x[0], x[2], x[1], x[3]};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float hi = tf32_hi(a[e]);
      fh[4 * j + e] = __float_as_uint(hi);
      fl[4 * j + e] = __float_as_uint(__fsub_rn(a[e], hi));
    }
  }
}

// KEEP: columns [0, 8 NB) of the accumulator of this thread's rows r, r + 8 (the values bn_relu_fragments reads) ->
// rows row0 + r, row0 + r + 8 of h [., 8 NB], rows at or past `valid` skipped
template <int NB, bool STACKED>
__device__ __forceinline__ void keep_acc(const float* acc, float* __restrict__ h, long long row0, int r, int q,
                                         int valid) {
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int rr = r + 8 * half;
    if (rr >= valid) continue;
    float* dst = h + (size_t)(row0 + rr) * (8 * NB) + 2 * q;
#pragma unroll
    for (int i = 0; i < NB; ++i) {
      const int e = 2 * half;
      const float y0 = STACKED ? acc[4 * i + e] + acc[4 * NB + 4 * i + e] : acc[4 * i + e];
      const float y1 = STACKED ? acc[4 * i + e + 1] + acc[4 * NB + 4 * i + e + 1] : acc[4 * i + e + 1];
      *reinterpret_cast<float2*>(dst + 8 * i) = make_float2(y0, y1);
    }
  }
}

template <bool KEEP>
__global__ void __launch_bounds__(FE_THREADS, 1) flow_mlp_head_eval_kernel(const __grid_constant__ CUtensorMap tm,
                                                                           const FlowEvalArgs a) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const uint32_t sb = smem_u32(smem);
  const int tid = threadIdx.x, warp = __shfl_sync(0xffffffffu, tid >> 5, 0), lane = tid & 31;
  const HeadArgs& h = a.head;
  const int P = (h.h / h.ratio) * (h.w / h.ratio);
  const int upc = (P + FE_NT - 1) / FE_NT;  // units per cloud
  // contiguous, balanced range of units per CTA; its two warpgroups take every other unit
  const long long total = (long long)h.S * h.B * upc;
  const int u_lo = (int)(blockIdx.x * total / gridDim.x), u_hi = (int)((blockIdx.x + 1) * total / gridDim.x);
  float* tab = reinterpret_cast<float*>(smem + FE_TAB);
  const uint32_t bar0 = sb + FE_BARS;
  auto bar_full = [&](int w, int s) { return bar0 + 8u * (uint32_t)(w * FE_WSTAGES + s); };
  auto bar_empty = [&](int w, int s) { return bar0 + 8u * (uint32_t)((2 + w) * FE_WSTAGES + s); };

  if (tid == 0) {
    for (int w = 0; w < 2; ++w)
      for (int s = 0; s < FE_WSTAGES; ++s) {
        mbar_init(bar_full(w, s), 1);
        mbar_init(bar_empty(w, s), 4);
      }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= FE_CONS / 32) {
    // producers: one thread per warpgroup streams its units' 5 x 7 boxes of ecat, in the order they are consumed
    const int w = warp - FE_CONS / 32;
    if (lane == 0) {
      const uint32_t ring = sb + FE_RING + w * FE_WSTAGES * FE_STAGE;
      int stage = 0;
      uint32_t phase = 0;
      for (int u = u_lo + w; u < u_hi; u += 2) {
        const int cloud = u / upc, pix0 = (u - cloud * upc) * FE_NT;
        for (int m = 0; m < PMVS_NUM_HYP; ++m)
          for (int c = 0; c < FE_NCH0; ++c) {
            mbar_wait(bar_empty(w, stage), phase ^ 1u);
            mbar_arrive_expect_tx(bar_full(w, stage), FE_STAGE);
            tma_load_3d(ring + stage * FE_STAGE, &tm, c * FE_KC, pix0, cloud * PMVS_NUM_HYP + m, bar_full(w, stage));
            if (++stage == FE_WSTAGES) {
              stage = 0;
              phase ^= 1u;
            }
          }
      }
    }
    return;
  }

  // =============================== consumers ==========================================================
  const uint32_t w0 = sb, w1 = sb + FE_W0, w2 = sb + FE_W0 + FE_W1;
  store_weight_planes<64>(w0, a.w[0], FE_K0, tid, FE_CONS);
  store_weight_planes_paired<64>(w1, a.w[1], 64, tid, FE_CONS);
  store_weight_planes_paired<16>(w2, a.w[2], 64, tid, FE_CONS);
  for (int i = tid; i < FLOW_EVAL_MLP_COEF; i += FE_CONS) tab[i] = a.mlp_coef[i];
  if (tid < 16) tab[FLOW_EVAL_MLP_COEF + tid] = h.w3[tid];
  fence_proxy_async();
  named_bar_sync(1, FE_CONS);
  const float *A0 = tab, *B0 = tab + 64, *A1 = tab + 128, *B1 = tab + 192, *A2 = tab + 256, *B2 = tab + 272;
  const float* W3 = tab + FLOW_EVAL_MLP_COEF;

  const int wgi = warp >> 2;
  const uint32_t ring = sb + FE_RING + wgi * FE_WSTAGES * FE_STAGE;
  // this thread's rows r, r + 8 of a block; A fragments at columns 8 j + q (+ 4), accumulator columns 8 i + 2q (+ 1)
  const int r = (warp & 3) * 16 + (lane >> 2), q = lane & 3;
  const uint32_t fbase = r * 128 + q * 4, fx = (r & 7) << 4;
  int n = 0;  // ring items consumed by this warpgroup
  for (int u = u_lo + wgi; u < u_hi; u += 2) {
    const int cloud = u / upc, pix0 = (u - cloud * upc) * FE_NT;
    float raw[PMVS_NUM_HYP];  // lane q = 0: row r, q = 1: row r + 8 (the lane that finishes it)
    const int valid = P - pix0;  // rows of the block inside the cloud
#pragma unroll 1
    for (int m = 0; m < PMVS_NUM_HYP; ++m) {
      const long long row0 = (long long)cloud * PMVS_NUM_HYP * P + (long long)m * P + pix0;
      // h0 = ecat * W0^T
      float acc0[64];
      {
        uint32_t fh[16], fl[16];
#pragma unroll 1
        for (int c = 0; c < FE_NCH0; ++c, ++n) {
          const int stage = n % FE_WSTAGES;
          mbar_wait(bar_full(wgi, stage), (uint32_t)((n / FE_WSTAGES) & 1));
          mma_chunk_3xtf32<64, false, 4>(acc0, fh, fl, ring + stage * FE_STAGE + fbase, fx, nullptr,
                                         w0 + c * (2 * 64 * 128), c);
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_empty(wgi, stage));
        }
      }
      fence_regs(acc0);
      if constexpr (KEEP) keep_acc<8, true>(acc0, a.keep_h[0], row0, r, q, valid);
      // Layers 1 and 2 accumulate the three products in one accumulator (small terms first), not stacked as layer 0:
      // with the A operand in registers stacking saves no shared-memory reads, and it would cost 40 registers.  They
      // run one 32-column K chunk at a time, so that the fragments of only one chunk are live.
      uint32_t fh[16], fl[16];
      // h1 = relu(BN(h0)) * W1^T
      float acc1[32];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        bn_relu_fragments<8, true>(acc0, c, A0, B0, q, fh, fl);
        fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t b = w1 + c * (2 * 64 * 128) + j * 32;
          mma_tile_ra<64, 64>(acc1, &fl[4 * j], b, (c | j) != 0 ? 1u : 0u);
          mma_tile_ra<64, 64>(acc1, &fh[4 * j], b + 64 * 128, 1u);
          mma_tile_ra<64, 64>(acc1, &fh[4 * j], b, 1u);
        }
        commit();
        wait<0>();
        fence_regs(fh);
        fence_regs(fl);
      }
      fence_regs(acc1);
      if constexpr (KEEP) keep_acc<8, false>(acc1, a.keep_h[1], row0, r, q, valid);
      // h2 = relu(BN(h1)) * W2^T
      float acc2[8];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        bn_relu_fragments<8, false>(acc1, c, A1, B1, q, fh, fl);
        fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t b = w2 + c * (2 * 16 * 128) + j * 32;
          mma_tile_ra<16, 16>(acc2, &fl[4 * j], b, (c | j) != 0 ? 1u : 0u);
          mma_tile_ra<16, 16>(acc2, &fh[4 * j], b + 16 * 128, 1u);
          mma_tile_ra<16, 16>(acc2, &fh[4 * j], b, 1u);
        }
        commit();
        wait<0>();
        fence_regs(fh);
        fence_regs(fl);
      }
      fence_regs(acc2);
      if constexpr (KEEP) keep_acc<2, false>(acc2, a.keep_h[2], row0, r, q, valid);
      // raw = relu(BN(h2)) * w3^T: this thread's 4 columns, then the 4 lanes of the row
      float s0 = 0.f, s1 = 0.f;
#pragma unroll
      for (int i = 0; i < 2; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int col = 8 * i + 2 * q + (e & 1);
          const float x = fmaxf(fmaf(acc2[4 * i + e], A2[col], B2[col]), 0.f);
          if (e < 2) s0 = fmaf(x, W3[col], s0);
          else s1 = fmaf(x, W3[col], s1);
        }
      s0 += __shfl_xor_sync(0xffffffffu, s0, 1);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 1);
      s0 += __shfl_xor_sync(0xffffffffu, s0, 2);
      s1 += __shfl_xor_sync(0xffffffffu, s1, 2);
      // a register array indexed by the (not unrolled) m would live in local memory
#pragma unroll
      for (int mm = 0; mm < PMVS_NUM_HYP; ++mm)
        if (mm == m) raw[mm] = q == 0 ? s0 : s1;
    }
    // lane q = 0 finishes row r, lane q = 1 row r + 8
    const int pp = pix0 + r + 8 * q;
    if (q < 2 && pp < P) {
      flow_head_store(h, raw, cloud / h.B, cloud % h.B, pp);
      if constexpr (KEEP) {
#pragma unroll
        for (int m = 0; m < PMVS_NUM_HYP; ++m) a.keep_raw[(size_t)cloud * PMVS_NUM_HYP * P + (size_t)m * P + pp] = raw[m];
      }
    }
  }
}

__global__ void flow_eval_coef_kernel(const pmvs_flow_weights w, int S, float* __restrict__ ec_coef,
                                      float* __restrict__ mlp_coef, float* __restrict__ run_copy) {
  const int g = blockIdx.x;
  const float eps = w.eps;
  auto istd = [&](float rv) { return (float)(1.0 / sqrt((double)rv + (double)eps)); };
  for (int l = 0; l < 3; ++l) {
    const int C = flow_ec_cout(l);
    const bool central = l > 0;  // EdgeConv: channels [0, C) central, [C, 2C) neighbour; EdgeConvNoC: neighbour only
    float* cg = ec_coef + flow_ec_coef_offset(l, S, g);
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
      // the same forms as the statistics kernel's table (edge_tile.cu)
      const int gn = central ? C + c : c;
      const float A = istd(w.ec_run_var[l][gn]) * w.ec_gamma[l][gn];
      cg[c] = A;
      cg[C + c] = fmaf(-w.ec_run_mean[l][gn], A, w.ec_beta[l][gn]);
      if (central) {
        cg[2 * C + c] = w.ec_run_mean[l][c];
        cg[3 * C + c] = istd(w.ec_run_var[l][c]);
        cg[4 * C + c] = w.ec_gamma[l][c];
        cg[5 * C + c] = w.ec_beta[l][c];
      }
    }
  }
  if (g == 0) {
    for (int l = 0; l < 3; ++l) {
      const int C = flow_mlp_cout(l);
      float* t = mlp_coef + flow_mlp_coef_offset(l);
      for (int c = threadIdx.x; c < C; c += blockDim.x) {
        // as gemm_tma_kernel's input BatchNorm table
        const float A = __fmul_rn(istd(w.mlp_run_var[l][c]), w.mlp_gamma[l][c]);
        t[c] = A;
        t[C + c] = fmaf(-w.mlp_run_mean[l][c], A, w.mlp_beta[l][c]);
      }
    }
    if (run_copy != nullptr)
      for (int l = 0; l < 6; ++l) {
        const int C = flow_eval_run_channels(l);
        const float* rm = l < 3 ? w.ec_run_mean[l] : w.mlp_run_mean[l - 3];
        const float* rv = l < 3 ? w.ec_run_var[l] : w.mlp_run_var[l - 3];
        float* o = run_copy + flow_eval_run_offset(l);
        for (int c = threadIdx.x; c < C; c += blockDim.x) {
          o[c] = rm[c];
          o[C + c] = rv[c];
        }
      }
  }
}

}  // namespace

int launch_flow_eval_coef(const pmvs_flow_weights& w, int S, float* ec_coef, float* mlp_coef, float* run_copy,
                          cudaStream_t st) {
  for (int l = 0; l < 3; ++l)
    PMVS_REQUIRE(w.ec_run_mean[l] && w.ec_run_var[l] && w.mlp_run_mean[l] && w.mlp_run_var[l] && w.ec_gamma[l] &&
                     w.ec_beta[l] && w.mlp_gamma[l] && w.mlp_beta[l],
                 "point_flow: bn_eval = 1 needs the running mean and variance of all six BatchNorm layers");
  PMVS_REQUIRE(S > 0 && S <= 65535 && ec_coef && mlp_coef, "flow_eval_coef: bad arguments");
  prof_begin("flow_eval_coef", st);
  flow_eval_coef_kernel<<<S, 64, 0, st>>>(w, S, ec_coef, mlp_coef, run_copy);
  return check_launch("flow_eval_coef_kernel", st);
}

int launch_flow_mlp_head_eval(const FlowEvalArgs& a, cudaStream_t st) {
  const HeadArgs& h = a.head;
  PMVS_REQUIRE(a.ecat && a.w[0] && a.w[1] && a.w[2] && a.mlp_coef && h.w3 && h.depth_prev && h.interval && h.depth_out,
               "flow_mlp_head_eval: NULL pointer");
  PMVS_REQUIRE(((uintptr_t)a.ecat & 15) == 0, "flow_mlp_head_eval: ecat must be 16-byte aligned");
  // the KEEP variant writes all four; a partial set is a caller error, not a silent plain launch
  const int kept = (a.keep_h[0] != nullptr) + (a.keep_h[1] != nullptr) + (a.keep_h[2] != nullptr) +
                   (a.keep_raw != nullptr);
  PMVS_REQUIRE(kept == 0 || kept == 4, "flow_mlp_head_eval: keep_h[0..2] and keep_raw must all be set or all be NULL");
  const bool keep = kept == 4;
  PMVS_REQUIRE(h.B > 0 && h.S > 0 && h.ratio > 0 && h.h % h.ratio == 0 && h.w % h.ratio == 0,
               "flow_mlp_head_eval: bad shape");
  const long long P = (long long)(h.h / h.ratio) * (h.w / h.ratio);
  const long long layers = (long long)h.S * h.B * PMVS_NUM_HYP;
  const long long units = (long long)h.S * h.B * cdiv(P, FE_NT);
  PMVS_REQUIRE(units < (1ll << 31) / 4 && layers < (1ll << 31) && P * FE_K0 * 4 < (1ll << 40),
               "flow_mlp_head_eval: problem too large");
  EncodeTiledFn enc = encode_tiled_fn();
  if (enc == nullptr) {
    set_error("flow_mlp_head_eval: cuTensorMapEncodeTiled is not available from this driver");
    return PMVS_ERR_CUDA;
  }
  // ecat as (224 columns, P pixels, 5 * clouds hypothesis layers): a box is 32 columns x 64 pixels of one layer
  CUtensorMap tm;
  const cuuint64_t gdim[3] = {(cuuint64_t)FE_K0, (cuuint64_t)P, (cuuint64_t)layers};
  const cuuint64_t gstr[2] = {(cuuint64_t)FE_K0 * 4, (cuuint64_t)P * FE_K0 * 4};
  const cuuint32_t box[3] = {FE_KC, FE_NT, 1};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult rc = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<float*>(a.ecat), gdim, gstr, box, estr,
                          CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                          CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) {
    set_error("flow_mlp_head_eval: cuTensorMapEncodeTiled failed (%d) for %lld pixels", (int)rc, P);
    return PMVS_ERR_CUDA;
  }
  const int grid = (int)std::min<long long>(units, sm_count());
  if (keep) {
    static unsigned long long smem_keep = 0;
    PMVS_TRY(ensure_dyn_smem(flow_mlp_head_eval_kernel<true>, FE_SMEM, smem_keep, "flow_mlp_head_eval_keep"));
    prof_begin("flow_mlp_head_eval_keep", st);
    flow_mlp_head_eval_kernel<true><<<grid, FE_THREADS, FE_SMEM, st>>>(tm, a);
    return check_launch("flow_mlp_head_eval_kernel<KEEP>", st);
  }
  static unsigned long long smem_done = 0;
  PMVS_TRY(ensure_dyn_smem(flow_mlp_head_eval_kernel<false>, FE_SMEM, smem_done, "flow_mlp_head_eval"));
  prof_begin("flow_mlp_head_eval", st);
  flow_mlp_head_eval_kernel<false><<<grid, FE_THREADS, FE_SMEM, st>>>(tm, a);
  return check_launch("flow_mlp_head_eval_kernel", st);
}

}  // namespace pmvs
