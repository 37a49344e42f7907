// EdgeConv statistics / apply of the fused path with the neighbour rows gathered from SHARED memory.
//
// Reference: networks.py:18-45,56-81 (gather the conv2 output by kNN index, [central | neighbour -
// central], BatchNorm2d with batch statistics over (B, N, K), ReLU, mean over K) on the structured
// clouds of model.py:236-255, whose neighbours all lie in the 5x5x5 window of torch_utils.py:16-61.
//
// A CTA owns a tile of TX x TY pixels x the 5 hypothesis layers of one sub-cloud.  The `edge` half of
// the rows of the tile plus its 2-pixel halo - a [5][TY+4][TX+4][32-channel] box of the points-major
// matrix LE[R, 2*cout] seen as the 4-D tensor (channel, x, y, cloud*5 + layer) - arrives with ONE
// cp.async.bulk.tensor.4d (TMA, SASS UTMALDG) completing on an mbarrier; coordinates outside the
// grid are zero-filled by the TMA unit.  Neighbour k of a point is then one LDS.128 at
// base(point) + 128 * code, the 16-bit code being what the kNN kernel emits instead of 4/8-byte row indices:
// the row offset (dd+2)*96 + (dh+2)*12 + (dw+2) inside this very tile geometry (knn3d.cu knn_code16) - no
// look-up table, one shift-add per gather.  A pick that lies OUTSIDE the grid (the zero-vector candidates
// of torch_utils.py:44, whose clamped / row-wrapped linear index aliases some other row, :51-59; 0.04 % of
// the picks) carries bit 15 + the candidate id and is fetched from global memory at exactly that aliased row.  Several CTAs are resident per SM, so one CTA's TMA wait overlaps the others' math.
//
// Arithmetic is edge_kernel's (edgeconv.cu), on fp32 pairs (FFMA2 / FADD2): statistics d = e - l,
// s1 += d, s2 = fma(d, d, s2); apply fma(e, A, c0) with A = istd * gamma, c0 = beta - (mean + l) * A.
// The statistics of the central half come from the GEMM epilogue (per-column sums of LE).
#include <algorithm>

#include "common.cuh"
#include "tensor_map.cuh"

namespace pmvs {

namespace {

constexpr int ET_THREADS = 256;
constexpr int ET_WARPS = ET_THREADS / 32;
constexpr int ET_CP = 32;            // channels per slab = one 128-byte row of the halo tile
constexpr int ET_LPP = ET_CP / 4;    // 8 lanes per point
constexpr int ET_PPW = 32 / ET_LPP;  // 4 points per warp step

__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

template <int TX, int TY>
struct TileGeom {
  static constexpr int HX = TX + 4, HY = TY + 4;
  static constexpr int ROWS = PMVS_NUM_HYP * HY * HX;
  static constexpr int NPTS = PMVS_NUM_HYP * TY * TX;
  static constexpr int BYTES = ROWS * ET_CP * 4;
  static constexpr int SMEM = BYTES;
};

// per (layer, group) BatchNorm coefficients, written once by the LAST statistics CTA of the group and read by
// every apply CTA: [A | B | kM | kI | kG | kBt] x COUT floats
//   neighbour half: A = istd * gamma, B = beta - mean * A      (apply: fma(e, A, B - l * A))
//   central half (concat_central): mean, istd, gamma, beta     (apply: ATen's ((x - mean) * istd) * gamma + beta)
constexpr int ET_COEF = 6;

template <int COUT, bool APPLY, int TX, int TY>
__global__ void __launch_bounds__(ET_THREADS, 3) edge_tile_kernel(const __grid_constant__ CUtensorMap tm,
                                                                   const EdgeTileArgs a) {
  using G = TileGeom<TX, TY>;
  static_assert(COUT % ET_CP == 0, "edge_tile: channels must be a multiple of 32");
  static_assert(G::NPTS % (ET_WARPS * ET_PPW) == 0, "edge_tile: every thread owns NPTS / 32 points");
  constexpr int LD = 2 * COUT;
  constexpr int SLABS = COUT / ET_CP;
  constexpr int STEPS = G::NPTS / (ET_WARPS * ET_PPW);  // points per thread
  static_assert(G::HX == 12 && G::HY == 8, "the kNN kernel's 16-bit codes are row offsets of a 12 x 8 x 5 halo tile");
  extern __shared__ __align__(128) float halo[];  // [ROWS][32], filled by the TMA
  __shared__ __align__(8) unsigned long long bar;
  __shared__ float part[APPLY ? 1 : ET_WARPS][APPLY ? 1 : 2 * ET_CP];
  __shared__ __align__(16) float coef[APPLY ? ET_COEF * COUT : 4];
  __shared__ int s_last;

  const int g = blockIdx.z;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane / ET_LPP, cl = (lane % ET_LPP) * 4;
  const int gh = a.gh, gw = a.gw;
  const int tiles_x = (gw + TX - 1) / TX, tiles_per_cloud = tiles_x * ((gh + TY - 1) / TY);
  const int tiles_per_group = tiles_per_cloud * a.clouds_per_group;
  const int HW = gh * gw, N = PMVS_NUM_HYP * HW;
  const int rows_per_group = a.clouds_per_group * N;
  const unsigned bar_addr = smem_u32(&bar);

  if (tid == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bar_addr));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (APPLY) {
    const float* cg = a.coef + (size_t)g * ET_COEF * COUT;
    for (int c = tid; c < ET_COEF * COUT; c += ET_THREADS) coef[c] = __ldg(cg + c);
  }
  // A warp step covers one hypothesis layer of the tile (TX * TY = 32 points per CTA step), so this thread's
  // pixel (tx, ty) is fixed and step s is layer s.
  static_assert(TX * TY == ET_WARPS * ET_PPW && STEPS == PMVS_NUM_HYP, "edge_tile: one layer of the tile per step");
  const int tq = warp * ET_PPW + sub, tx = tq % TX, ty = tq / TX;
  // row of candidate code 0 = offset (-2, -2, -2) from the point of layer 0, in floats (negative: codes >= 2 layers)
  const int pb0 = ((-2 * G::HY + ty) * G::HX + tx) * ET_CP + cl;
  constexpr int LAYER = G::HY * G::HX * ET_CP;
  __syncthreads();

  unsigned loads = 0;  // TMA loads this CTA has waited for (mbarrier phase parity)
#pragma unroll 1
  for (int slab = 0; slab < SLABS; ++slab) {
    const int ch0 = slab * ET_CP;
    f32x2 n1_lo = pack2(0.f, 0.f), n1_hi = n1_lo, n2_lo = n1_lo, n2_hi = n1_lo;
#pragma unroll 1
    for (int tile = blockIdx.x; tile < tiles_per_group; tile += gridDim.x) {
    const int b = tile / tiles_per_cloud, tr = tile - b * tiles_per_cloud;
    const int y0 = (tr / tiles_x) * TY, x0 = (tr % tiles_x) * TX;
    const size_t cloud_base = (size_t)g * rows_per_group + (size_t)b * N;
    const bool ok = y0 + ty < gh && x0 + tx < gw;
    const int pq = (y0 + ty) * gw + x0 + tx;
    auto load_codes = [&](int s, uint4& c0, uint4& c1) {  // 16 x 16-bit neighbour codes of the point of layer s
      if (ok) {
        const uint4* cp = reinterpret_cast<const uint4*>(a.cand + (cloud_base + (size_t)(s * HW + pq)) * PMVS_KNN);
        c0 = __ldg(cp);
        c1 = __ldg(cp + 1);
      } else {
        c0 = c1 = make_uint4(0u, 0u, 0u, 0u);
      }
    };
    if (loads > 0) __syncthreads();  // every reader of the previous box is done before the TMA overwrites it
    if (tid == 0) {
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_addr), "r"((unsigned)G::BYTES)
                   : "memory");
      asm volatile(
          "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
          ::"r"(smem_u32(halo)), "l"(&tm), "r"(COUT + ch0), "r"(x0 - 2), "r"(y0 - 2),
          "r"((g * a.clouds_per_group + b) * PMVS_NUM_HYP), "r"(bar_addr)
          : "memory");
    }
    // the `local` rows of this thread's points (this slab's 32 channels), in flight while the tile loads
    float4 loc[STEPS];
#pragma unroll
    for (int s = 0; s < STEPS; ++s)
      loc[s] = ok ? ldg4(a.le + (cloud_base + (size_t)(s * HW + pq)) * LD + ch0 + cl) : make_float4(0.f, 0.f, 0.f, 0.f);
    {
      unsigned done = 0;
      const unsigned parity = loads & 1u;
      while (!done) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done)
            : "r"(bar_addr), "r"(parity)
            : "memory");
      }
      ++loads;
    }

    uint4 nx0, nx1;  // codes of the next point: in flight while the current one is processed
    load_codes(0, nx0, nx1);
#pragma unroll
    for (int s = 0; s < STEPS; ++s) {
      const uint4 ca = nx0, cb = nx1;
      if (s + 1 < STEPS) load_codes(s + 1, nx0, nx1);
      if (!ok) continue;
      const int n = s * HW + pq;
      const size_t row = cloud_base + (size_t)n;
      const float4 lc = loc[s];
      const bool esc = ((ca.x | ca.y | ca.z | ca.w | cb.x | cb.y | cb.z | cb.w) & 0x80008000u) != 0u;
      const float* hbase = halo + pb0 + s * LAYER;
      f32x2 o_lo = pack2(0.f, 0.f), o_hi = o_lo, A_lo = o_lo, A_hi = o_lo, c_lo = o_lo, c_hi = o_lo;
      const f32x2 l_lo = pack2(lc.x, lc.y), l_hi = pack2(lc.z, lc.w);
      if (APPLY) {
        const float4 A4 = *reinterpret_cast<const float4*>(&coef[ch0 + cl]);
        const float4 B4 = *reinterpret_cast<const float4*>(&coef[COUT + ch0 + cl]);
        A_lo = pack2(A4.x, A4.y); A_hi = pack2(A4.z, A4.w);
        // c0 = beta - (mean + loc) * A = (beta - mean * A) - loc * A
        c_lo = pack2(fmaf(-lc.x, A4.x, B4.x), fmaf(-lc.y, A4.y, B4.y));
        c_hi = pack2(fmaf(-lc.z, A4.z, B4.z), fmaf(-lc.w, A4.w, B4.w));
      }
      auto body = [&](const float4 e) {
        const f32x2 e_lo = pack2(e.x, e.y), e_hi = pack2(e.z, e.w);
        if (APPLY) {
          float t0, t1f, t2, t3;
          unpack2(fma2(e_lo, A_lo, c_lo), t0, t1f);
          unpack2(fma2(e_hi, A_hi, c_hi), t2, t3);
          o_lo = add2(o_lo, pack2(fmaxf(t0, 0.f), fmaxf(t1f, 0.f)));
          o_hi = add2(o_hi, pack2(fmaxf(t2, 0.f), fmaxf(t3, 0.f)));
        } else {
          const f32x2 d_lo = sub2(e_lo, l_lo), d_hi = sub2(e_hi, l_hi);
          n1_lo = add2(n1_lo, d_lo); n1_hi = add2(n1_hi, d_hi);
          n2_lo = fma2(d_lo, d_lo, n2_lo); n2_hi = fma2(d_hi, d_hi, n2_hi);
        }
      };
      auto code_of = [&](int k) -> unsigned {  // no indexable array: that would live in local memory
        const int wq = k >> 1;
        const unsigned wd = wq == 0 ? ca.x : wq == 1 ? ca.y : wq == 2 ? ca.z : wq == 3 ? ca.w
                          : wq == 4 ? cb.x : wq == 5 ? cb.y : wq == 6 ? cb.z : cb.w;
        return (k & 1) ? wd >> 16 : wd & 0xffffu;
      };
      if (!esc) {
        // 16 independent 128-bit gathers: row = base + code, i.e. one shift-add per address
#pragma unroll
        for (int k = 0; k < PMVS_KNN; ++k) body(*reinterpret_cast<const float4*>(hbase + code_of(k) * ET_CP));
      } else {
#pragma unroll 1
        for (int k = 0; k < PMVS_KNN; ++k) {
          const unsigned c = code_of(k);
          if (c & 0x8000u) {
            // out-of-grid candidate: the reference gathers row clamp(n + dd*HW + dh*W + dw) (torch_utils.py:51-59)
            const int j = (int)(c & 127u);
            int t = n + (j / 25 - 2) * HW + ((j % 25) / 5 - 2) * gw + (j % 5 - 2);
            t = t < 0 ? 0 : (t > N - 1 ? N - 1 : t);
            body(ldg4(a.le + (cloud_base + (size_t)t) * LD + COUT + ch0 + cl));
          } else {
            body(*reinterpret_cast<const float4*>(hbase + c * ET_CP));
          }
        }
      }
      if (APPLY) {
        float4 o;
        unpack2(o_lo, o.x, o.y);
        unpack2(o_hi, o.z, o.w);
        float* orow = a.out + row * a.ldo;
        if (a.concat_central) {
          const float4 m = *reinterpret_cast<const float4*>(&coef[2 * COUT + ch0 + cl]);
          const float4 is = *reinterpret_cast<const float4*>(&coef[3 * COUT + ch0 + cl]);
          const float4 gm = *reinterpret_cast<const float4*>(&coef[4 * COUT + ch0 + cl]);
          const float4 bt = *reinterpret_cast<const float4*>(&coef[5 * COUT + ch0 + cl]);
          float4 c;
          c.x = fmaxf(bn_apply(lc.x, m.x, is.x, gm.x, bt.x), 0.f);
          c.y = fmaxf(bn_apply(lc.y, m.y, is.y, gm.y, bt.y), 0.f);
          c.z = fmaxf(bn_apply(lc.z, m.z, is.z, gm.z, bt.z), 0.f);
          c.w = fmaxf(bn_apply(lc.w, m.w, is.w, gm.w, bt.w), 0.f);
          st4(orow + ch0 + cl, c);
          orow += COUT;
        }
        // mean over K = 16: x / 16 == x * 0.0625 exactly (power of two), without the division's slow path for 0
        constexpr float rk = 1.f / (float)PMVS_KNN;
        static_assert(PMVS_KNN == 16, "mean over K uses an exact power-of-two reciprocal");
        st4(orow + ch0 + cl, make_float4(__fmul_rn(o.x, rk), __fmul_rn(o.y, rk), __fmul_rn(o.z, rk), __fmul_rn(o.w, rk)));
      }
    }

    }  // tiles of this CTA

    if (!APPLY) {
      // per-thread fp32 partials (NPTS / 32 points x 16 values) -> shuffle over the 4 point slots of the warp ->
      // per-warp partials in shared memory -> fp64 per CTA -> one fp64 atomic per channel and statistic
      float v[8];
      unpack2(n1_lo, v[0], v[1]); unpack2(n1_hi, v[2], v[3]);
      unpack2(n2_lo, v[4], v[5]); unpack2(n2_hi, v[6], v[7]);
#pragma unroll
      for (int off = ET_LPP; off < 32; off <<= 1) {
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] += __shfl_xor_sync(0xffffffffu, v[q], off);
      }
      if (sub == 0) {
#pragma unroll
        for (int q = 0; q < 8; ++q) part[warp][(q >> 2) * ET_CP + cl + (q & 3)] = v[q];
      }
      __syncthreads();
      double* o = a.nstats + (size_t)g * 2 * COUT;
      if (tid < 2 * ET_CP) {
        double t = 0.0;
#pragma unroll
        for (int wq = 0; wq < ET_WARPS; ++wq) t += (double)part[wq][tid];
        atomicAdd(o + (tid / ET_CP) * COUT + ch0 + (tid % ET_CP), t);  // [sum_n | sumsq_n][COUT]
      }
    }
  }

  if (!APPLY) {
    // the LAST statistics CTA of the group turns the sums into the coefficients every apply CTA needs (instead of
    // ~2 us of serial fp64 arithmetic at the head of each of them)
    __threadfence();
    __syncthreads();
    if (tid == 0) {
      const unsigned t = atomicAdd(a.ticket + g, 1u);
      s_last = t == gridDim.x - 1;
    }
    __syncthreads();
    if (s_last) {
      __threadfence();
      const double* sc = a.cstats + (size_t)g * 4 * COUT;
      const double* sn = a.nstats + (size_t)g * 2 * COUT;
      float* cg = a.coef + (size_t)g * ET_COEF * COUT;
      const double cnt_c = (double)rows_per_group, cnt_n = (double)rows_per_group * PMVS_KNN;
      for (int c = tid; c < COUT; c += ET_THREADS) {
        const BnCoef kn = bn_coef(__ldcg(sn + c), __ldcg(sn + COUT + c), cnt_n, a.eps);
        const int gn = a.concat_central ? COUT + c : c;
        const float A = kn.invstd * a.gamma[gn];
        cg[c] = A;
        cg[COUT + c] = fmaf(-kn.mean, A, a.beta[gn]);
        if (a.concat_central) {
          const BnCoef kc = bn_coef(sc[c], sc[2 * COUT + c], cnt_c, a.eps);
          cg[2 * COUT + c] = kc.mean; cg[3 * COUT + c] = kc.invstd; cg[4 * COUT + c] = a.gamma[c]; cg[5 * COUT + c] = a.beta[c];
        }
      }
    }
  }
}

template <int COUT, bool APPLY, int TX, int TY>
int launch_variant(const EdgeTileArgs& a, cudaStream_t st) {
  using G = TileGeom<TX, TY>;
  EncodeTiledFn enc = encode_tiled_fn();
  if (enc == nullptr) {
    set_error("edge_tile: cuTensorMapEncodeTiled is not available from this driver");
    return PMVS_ERR_CUDA;
  }
  const int N = PMVS_NUM_HYP * a.gh * a.gw;
  const long long layers = (long long)a.groups * a.clouds_per_group * PMVS_NUM_HYP;
  PMVS_REQUIRE(a.groups <= 65535 && a.clouds_per_group <= 65535, "edge_tile: too many clouds");
  PMVS_REQUIRE(layers < (1ll << 31) && (long long)a.groups * a.clouds_per_group * N < (1ll << 40), "edge_tile: too large");
  PMVS_REQUIRE(((uintptr_t)a.le & 15) == 0, "edge_tile: LE must be 16-byte aligned");
  // LE [R, 2*cout] as (channel, x, y, cloud*5 + layer); box = 32 channels x (TX+4) x (TY+4) x 5 layers
  CUtensorMap tm;
  const cuuint64_t gdim[4] = {(cuuint64_t)(2 * COUT), (cuuint64_t)a.gw, (cuuint64_t)a.gh, (cuuint64_t)layers};
  const cuuint64_t gstr[3] = {(cuuint64_t)(2 * COUT) * 4, (cuuint64_t)a.gw * 2 * COUT * 4,
                              (cuuint64_t)a.gh * a.gw * 2 * COUT * 4};
  const cuuint32_t box[4] = {ET_CP, (cuuint32_t)G::HX, (cuuint32_t)G::HY, PMVS_NUM_HYP};
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  const CUresult r = enc(&tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, const_cast<float*>(a.le), gdim, gstr, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    set_error("edge_tile: cuTensorMapEncodeTiled failed (%d) for %dx%d, cout %d", (int)r, a.gh, a.gw, COUT);
    return PMVS_ERR_CUDA;
  }
  static unsigned long long smem_done = 0;
  PMVS_TRY(ensure_dyn_smem(edge_tile_kernel<COUT, APPLY, TX, TY>, G::SMEM, smem_done, "edge_tile"));
  // Statistics: persistent CTAs.  Every group (= one BatchNorm population) gets an equal share of the resident CTA
  // slots and each CTA walks its tiles, so the flush (shuffles, fp64 atomics, fence, ticket) is paid once per CTA
  // instead of once per tile.
  static int slots = 0;
  if (slots == 0) {
    slots = 3 * sm_count();  // __launch_bounds__(ET_THREADS, 3)
  }
  const int tiles_per_group = cdiv(a.gw, TX) * cdiv(a.gh, TY) * a.clouds_per_group;
  // The apply kernel has no per-CTA flush to amortise, so it keeps one tile per CTA.
  int ctas = APPLY ? tiles_per_group : std::min(tiles_per_group, std::max(1, slots / a.groups));
  ctas = cdiv(tiles_per_group, cdiv(tiles_per_group, ctas));  // same longest walk with fewer CTAs
  PMVS_REQUIRE(ctas <= 0x7fffffff / 2, "edge_tile: too many tiles");
  dim3 grid(ctas, 1, a.groups);
  static const char* const names[2][2] = {{"edge_stats_32", "edge_stats_64"}, {"edge_apply_32", "edge_apply_64"}};
  prof_begin(names[APPLY ? 1 : 0][COUT == 32 ? 0 : 1], st);
  edge_tile_kernel<COUT, APPLY, TX, TY><<<grid, ET_THREADS, G::SMEM, st>>>(tm, a);
  return check_launch(APPLY ? "edge_tile_apply_kernel" : "edge_tile_stats_kernel", st);
}

template <bool APPLY>
int launch_edge_tile(const EdgeTileArgs& a, int tile_w, cudaStream_t st) {
  // apply reads only the coefficient table, so it also serves a table written from running statistics
  PMVS_REQUIRE(a.le && a.cand && a.coef && (APPLY ? a.out != nullptr : (a.cstats && a.nstats && a.gamma && a.beta && a.ticket)),
               "edge_tile: NULL pointer");
  PMVS_REQUIRE(a.cout == 32 || a.cout == 64, "edge_tile: out_channels %d (supported: 32, 64)", a.cout);
  PMVS_REQUIRE(a.gh > 0 && a.gw > 0 && a.groups > 0 && a.clouds_per_group > 0, "edge_tile: bad cloud shape");
  // Tried and dropped before the H100 port (git history; not re-measured on H100): a 16 x 4 x 5 tile with 2 CTAs / SM,
  // and a ring variant - one persistent 21-warp CTA per SM, 3-deep ring of TMA boxes loaded two items ahead.
  (void)tile_w;
  return a.cout == 32 ? launch_variant<32, APPLY, 8, 4>(a, st) : launch_variant<64, APPLY, 8, 4>(a, st);
}

}  // namespace

int launch_edge_tile_stats(const EdgeTileArgs& a, int tile_w, cudaStream_t st) {
  return launch_edge_tile<false>(a, tile_w, st);
}
int launch_edge_tile_apply(const EdgeTileArgs& a, int tile_w, cudaStream_t st) {
  return launch_edge_tile<true>(a, tile_w, st);
}

}  // namespace pmvs
