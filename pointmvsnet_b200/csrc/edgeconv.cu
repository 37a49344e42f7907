// EdgeConv / EdgeConvNoC / flow_mlp building blocks on points-major fp32 data.
//
// Reference semantics: networks.py:9-81 (CUDA branches: conv1 -> local, conv2 -> edge,
// gather edge by kNN index, [central | neighbour - central], BatchNorm2d with BATCH
// statistics over (B, N, K) because test.py:58 keeps train mode, ReLU, mean over K) and
// model.py:40-43,218-227 (flow_mlp = 3 x [Conv1d + BatchNorm1d(batch stats) + ReLU] +
// Conv1d 16->1, softmax over the 5 hypotheses, expected offset).
//
// Design: the [B,C,N,K] tensors the reference materialises (gather, cat, BN, ReLU; 210 MB
// each at C=128) never exist.  Per layer:
//   gemm      : LE[n, 0:2*cout] = X[n, :] * [W1;W2]^T                 (points-major rows)
//   edgestats : per (group, channel) sum / sum-of-squares of local and of
//               (edge[idx[n,k]] - local[n]) accumulated in fp64 (grid reduction #1)
//   edgeapply : recomputes the gathered differences (L1/L2 hits), normalises, ReLU, mean over K
// The central half is constant over K, so its BN statistics equal the per-point statistics
// and its mean over K is the value itself.
#include "common.cuh"

namespace pmvs {

// =======================================================================================
// fp32 SIMT GEMM: Y[r, 0:cout] = f(X[r, 0:cin]) * W^T, optional fused input BN+ReLU and
// output column statistics.  128 rows x BN columns per CTA, 8-wide k chunks, register tile
// TM x 4, shared-memory operands stored k-major.
// =======================================================================================
constexpr int G_BM = 128, G_BK = 8, G_THREADS = 256;

template <int BN>
__global__ void __launch_bounds__(G_THREADS) gemm_kernel(const GemmArgs a) {
  constexpr int TX = BN / 4;           // threads along columns
  constexpr int TY = G_THREADS / TX;   // threads along rows
  constexpr int TM = G_BM / TY;        // rows per thread
  static_assert(TM >= 1 && TM * TY == G_BM, "tile");
  __shared__ __align__(16) float Xs[2][G_BK][G_BM + 4];
  __shared__ __align__(16) float Ws[2][G_BK][BN + 4];
  __shared__ float in_mean[224], in_istd[224], in_g[224], in_b[224];
  __shared__ double red[2][BN];

  const int g = blockIdx.y;
  const int row0 = blockIdx.x * G_BM;             // first row of the tile inside the group
  const int col0 = blockIdx.z * BN;               // first output column
  const int rows_valid = min(G_BM, a.rows_per_group - row0);
  const size_t grow0 = (size_t)g * a.rows_per_group + row0;
  const int tid = threadIdx.x;
  const int tx = tid % TX, ty = tid / TX;
  const bool in_bn = a.in_stats != nullptr;

  if (in_bn) {
    for (int c = tid; c < a.cin; c += G_THREADS) {
      const double* s = a.in_stats + (size_t)g * 2 * a.cin;
      BnCoef k = bn_coef(s[c], s[a.cin + c], a.in_count, a.eps);
      in_mean[c] = k.mean;
      in_istd[c] = k.invstd;
      in_g[c] = a.in_gamma[c];
      in_b[c] = a.in_beta[c];
    }
  }
  if (a.out_stats != nullptr && tid < BN) { red[0][tid] = 0.0; red[1][tid] = 0.0; }
  __syncthreads();

  // global->smem staging assignment
  // X chunk: 128 rows x 8 floats = 256 float4 -> one per thread
  const int xr = tid >> 1, xh = tid & 1;
  const bool xvalid = xr < rows_valid;
  const float* xsrc = a.x + (grow0 + (xvalid ? xr : 0)) * a.ldx + xh * 4;
  // W chunk: BN cols x 8 floats = 2*BN float4
  constexpr int WLOADS = (2 * BN + G_THREADS - 1) / G_THREADS;

  float acc[TM][4];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int nk = a.cin / G_BK;
  float4 xreg;
  float4 wreg[WLOADS];

  auto load_chunk = [&](int kc) {
    xreg = xvalid ? ldg4(xsrc + kc * G_BK) : make_float4(0.f, 0.f, 0.f, 0.f);
    if (in_bn && xvalid) {
      const int c = kc * G_BK + xh * 4;
      xreg.x = fmaxf(bn_apply(xreg.x, in_mean[c + 0], in_istd[c + 0], in_g[c + 0], in_b[c + 0]), 0.f);
      xreg.y = fmaxf(bn_apply(xreg.y, in_mean[c + 1], in_istd[c + 1], in_g[c + 1], in_b[c + 1]), 0.f);
      xreg.z = fmaxf(bn_apply(xreg.z, in_mean[c + 2], in_istd[c + 2], in_g[c + 2], in_b[c + 2]), 0.f);
      xreg.w = fmaxf(bn_apply(xreg.w, in_mean[c + 3], in_istd[c + 3], in_g[c + 3], in_b[c + 3]), 0.f);
    }
#pragma unroll
    for (int l = 0; l < WLOADS; ++l) {
      const int e = tid + l * G_THREADS;  // float4 id: col = e/2, half = e%2
      if (e < 2 * BN) {
        const int wc = e >> 1, wh = e & 1;
        const int oc = col0 + wc;
        wreg[l] = oc < a.cout ? ldg4(a.w + (size_t)oc * a.cin + kc * G_BK + wh * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
  };
  auto store_chunk = [&](int buf) {
    Xs[buf][xh * 4 + 0][xr] = xreg.x;
    Xs[buf][xh * 4 + 1][xr] = xreg.y;
    Xs[buf][xh * 4 + 2][xr] = xreg.z;
    Xs[buf][xh * 4 + 3][xr] = xreg.w;
#pragma unroll
    for (int l = 0; l < WLOADS; ++l) {
      const int e = tid + l * G_THREADS;
      if (e < 2 * BN) {
        const int wc = e >> 1, wh = e & 1;
        Ws[buf][wh * 4 + 0][wc] = wreg[l].x;
        Ws[buf][wh * 4 + 1][wc] = wreg[l].y;
        Ws[buf][wh * 4 + 2][wc] = wreg[l].z;
        Ws[buf][wh * 4 + 3][wc] = wreg[l].w;
      }
    }
  };

  load_chunk(0);
  store_chunk(0);
  __syncthreads();
  for (int kc = 0; kc < nk; ++kc) {
    const int buf = kc & 1;
    if (kc + 1 < nk) load_chunk(kc + 1);
#pragma unroll
    for (int k = 0; k < G_BK; ++k) {
      float xv[TM];
      if constexpr (TM >= 4) {
#pragma unroll
        for (int i = 0; i < TM; i += 4) {
          const float4 t = *reinterpret_cast<const float4*>(&Xs[buf][k][ty * TM + i]);
          xv[i] = t.x; xv[i + 1] = t.y; xv[i + 2] = t.z; xv[i + 3] = t.w;
        }
      } else {
#pragma unroll
        for (int i = 0; i < TM; ++i) xv[i] = Xs[buf][k][ty * TM + i];
      }
      const float4 wv = *reinterpret_cast<const float4*>(&Ws[buf][k][tx * 4]);
#pragma unroll
      for (int i = 0; i < TM; ++i) {
        acc[i][0] = fmaf(xv[i], wv.x, acc[i][0]);
        acc[i][1] = fmaf(xv[i], wv.y, acc[i][1]);
        acc[i][2] = fmaf(xv[i], wv.z, acc[i][2]);
        acc[i][3] = fmaf(xv[i], wv.w, acc[i][3]);
      }
    }
    if (kc + 1 < nk) store_chunk(buf ^ 1);
    __syncthreads();
  }

  // epilogue
  const int oc = col0 + tx * 4;
  float s1[4] = {0.f, 0.f, 0.f, 0.f}, s2[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int r = ty * TM + i;
    if (r < rows_valid && oc < a.cout) {
      st4(a.y + (grow0 + r) * a.ldy + oc, make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]));
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s1[j] += acc[i][j];
        s2[j] = fmaf(acc[i][j], acc[i][j], s2[j]);
      }
    }
  }
  if (a.out_stats != nullptr) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      atomicAdd(&red[0][tx * 4 + j], (double)s1[j]);
      atomicAdd(&red[1][tx * 4 + j], (double)s2[j]);
    }
    __syncthreads();
    if (tid < BN && col0 + tid < a.cout) {
      double* o = a.out_stats + (size_t)g * 2 * a.cout;
      atomicAdd(o + col0 + tid, red[0][tid]);
      atomicAdd(o + a.cout + col0 + tid, red[1][tid]);
    }
  }
}

int launch_gemm(const GemmArgs& a, cudaStream_t st) {
  PMVS_REQUIRE(a.cin % G_BK == 0 && a.cin <= 224, "gemm: cin=%d must be a multiple of 8 and <= 224", a.cin);
  PMVS_REQUIRE(a.cout % 4 == 0, "gemm: cout=%d must be a multiple of 4", a.cout);
  PMVS_REQUIRE(a.ldx % 4 == 0 && a.ldy % 4 == 0, "gemm: row strides must be multiples of 4 floats");
  PMVS_REQUIRE(a.groups <= 65535, "gemm: too many groups");
  const int tiles = cdiv(a.rows_per_group, G_BM);
  static const char* const names[] = {"gemm_136x64", "gemm_32x64", "gemm_64x128", "gemm_224x64",
                                      "gemm_64x64", "gemm_64x16", "gemm_other",
                                      // also the dX = dLE * W12 shapes of the model's EdgeConv backward (edge_bwd.cu)
                                      "gemm_64x136", "gemm_64x32", "gemm_128x64"};
  int ni = 6;
  if (a.cin == 136 && a.cout == 64) ni = 0;
  else if (a.cin == 32 && a.cout == 64) ni = 1;
  else if (a.cin == 64 && a.cout == 128) ni = 2;
  else if (a.cin == 224 && a.cout == 64) ni = 3;
  else if (a.cin == 64 && a.cout == 64) ni = 4;
  else if (a.cin == 64 && a.cout == 16) ni = 5;
  else if (a.cin == 64 && a.cout == 136) ni = 7;
  else if (a.cin == 64 && a.cout == 32) ni = 8;
  else if (a.cin == 128 && a.cout == 64) ni = 9;
  if (opt(OPT_GEMM) != 0 && pmvs_get_gemm_mode() == 3) {
    const int rc = launch_gemm_ws(a, st, names[ni]);
    if (rc >= 0) return rc;
  }
  {
    const int rc = launch_gemm_tc(a, st, names[ni]);
    if (rc >= 0) return rc;
  }
  prof_begin(names[ni], st);
  if (a.cout <= 16) {
    dim3 grid(tiles, a.groups, cdiv(a.cout, 16));
    gemm_kernel<16><<<grid, G_THREADS, 0, st>>>(a);
  } else {
    dim3 grid(tiles, a.groups, cdiv(a.cout, 64));
    gemm_kernel<64><<<grid, G_THREADS, 0, st>>>(a);
  }
  return check_launch("gemm_kernel", st);
}

// =======================================================================================
// EdgeConv statistics and apply.  Lane mapping: a "point group" of cout/4 lanes covers the
// cout channels of one point with float4s; a warp handles 32/(cout/4) points at a time.
// =======================================================================================
constexpr int E_THREADS = 256;
constexpr int E_PTS_PER_BLOCK = 128;  // points per CTA (contiguous -> neighbours overlap in L1)

// KT = compile-time neighbour count (16 on the hot path: indices are fetched as 4 x int4 and
// the 16 gathers are independent loads in flight); KT = 0 is the generic runtime-K path.
template <int COUT, bool APPLY, int KT>
__global__ void __launch_bounds__(E_THREADS) edge_kernel(const EdgeArgs a) {
  constexpr int LPP = COUT / 4;             // lanes per point
  constexpr int PPW = 32 / LPP;             // points per warp step
  constexpr int WARPS = E_THREADS / 32;
  constexpr int LD = 2 * COUT;
  __shared__ float part[APPLY ? 1 : WARPS][APPLY ? 1 : 4 * COUT];
  __shared__ float c_mean[2][COUT], c_istd[2][COUT], c_g[2][COUT], c_b[2][COUT];

  const int g = blockIdx.y;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane / LPP, cl = (lane % LPP) * 4;
  const int K = KT > 0 ? KT : a.K;

  if (APPLY) {
    const double* s = a.stats + (size_t)g * 4 * COUT;
    const double cnt_c = (double)a.rows_per_group, cnt_n = (double)a.rows_per_group * K;
    for (int c = tid; c < COUT; c += E_THREADS) {
      BnCoef kn = bn_coef(s[2 * COUT + c], s[3 * COUT + c], cnt_n, a.eps);
      const int gn = a.concat_central ? COUT + c : c;
      c_mean[1][c] = kn.mean; c_istd[1][c] = kn.invstd; c_g[1][c] = a.gamma[gn]; c_b[1][c] = a.beta[gn];
      if (a.concat_central) {
        BnCoef kc = bn_coef(s[c], s[COUT + c], cnt_c, a.eps);
        c_mean[0][c] = kc.mean; c_istd[0][c] = kc.invstd; c_g[0][c] = a.gamma[c]; c_b[0][c] = a.beta[c];
      }
    }
  }
  __syncthreads();

  float4 sc1 = make_float4(0.f, 0.f, 0.f, 0.f), sc2 = sc1, sn1 = sc1, sn2 = sc1;

  const int p0 = blockIdx.x * E_PTS_PER_BLOCK;
  const size_t gbase = (size_t)g * a.rows_per_group;
  for (int it = warp * PPW + sub; it < E_PTS_PER_BLOCK; it += WARPS * PPW) {
    const int r = p0 + it;  // row inside the group
    if (r >= a.rows_per_group) break;
    const size_t row = gbase + r;
    const size_t cloud_base = gbase + (size_t)(r / a.N) * a.N;
    const float4 loc = ldg4(a.le + row * LD + cl);
    const int32_t* ip = a.idx + row * K;
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    // apply: ((d - mean) * istd) * gamma + beta with d = e - loc is evaluated as fma(e, A, c0),
    // A = istd * gamma, c0 = beta - (mean + loc) * A  (one FFMA per gathered value; common.cuh edge_nb_*)
    float4 A4, c0;
    if (APPLY) {
      const float4 m = *reinterpret_cast<const float4*>(&c_mean[1][cl]);
      const float4 is = *reinterpret_cast<const float4*>(&c_istd[1][cl]);
      const float4 gm = *reinterpret_cast<const float4*>(&c_g[1][cl]);
      const float4 bt = *reinterpret_cast<const float4*>(&c_b[1][cl]);
      A4 = make_float4(edge_nb_scale(is.x, gm.x), edge_nb_scale(is.y, gm.y), edge_nb_scale(is.z, gm.z),
                       edge_nb_scale(is.w, gm.w));
      c0 = make_float4(edge_nb_offset(m.x, loc.x, A4.x, bt.x), edge_nb_offset(m.y, loc.y, A4.y, bt.y),
                       edge_nb_offset(m.z, loc.z, A4.z, bt.z), edge_nb_offset(m.w, loc.w, A4.w, bt.w));
    }
    auto body = [&](int nb) {
      const float4 e = ldg4(a.le + (cloud_base + nb) * LD + COUT + cl);
      if (APPLY) {
        o.x += fmaxf(edge_nb_pre(e.x, A4.x, c0.x), 0.f);
        o.y += fmaxf(edge_nb_pre(e.y, A4.y, c0.y), 0.f);
        o.z += fmaxf(edge_nb_pre(e.z, A4.z, c0.z), 0.f);
        o.w += fmaxf(edge_nb_pre(e.w, A4.w, c0.w), 0.f);
      } else {
        const float dx = __fsub_rn(e.x, loc.x), dy = __fsub_rn(e.y, loc.y);
        const float dz = __fsub_rn(e.z, loc.z), dw = __fsub_rn(e.w, loc.w);
        sn1.x += dx; sn1.y += dy; sn1.z += dz; sn1.w += dw;
        sn2.x = fmaf(dx, dx, sn2.x); sn2.y = fmaf(dy, dy, sn2.y);
        sn2.z = fmaf(dz, dz, sn2.z); sn2.w = fmaf(dw, dw, sn2.w);
      }
    };
    if constexpr (KT > 0) {
      static_assert(KT % 4 == 0, "KT");
      int nbs[KT];
#pragma unroll
      for (int q = 0; q < KT / 4; ++q) {
        const int4 t = __ldg(reinterpret_cast<const int4*>(ip) + q);
        nbs[4 * q] = t.x; nbs[4 * q + 1] = t.y; nbs[4 * q + 2] = t.z; nbs[4 * q + 3] = t.w;
      }
#pragma unroll
      for (int k = 0; k < KT; ++k) body(nbs[k]);
    } else {
      for (int k = 0; k < K; ++k) body(__ldg(ip + k));
    }
    if (APPLY) {
      const float kf = (float)K;
      float* orow = a.out + row * a.ldo;
      if (a.concat_central) {
        float4 c;
        c.x = fmaxf(bn_apply(loc.x, c_mean[0][cl + 0], c_istd[0][cl + 0], c_g[0][cl + 0], c_b[0][cl + 0]), 0.f);
        c.y = fmaxf(bn_apply(loc.y, c_mean[0][cl + 1], c_istd[0][cl + 1], c_g[0][cl + 1], c_b[0][cl + 1]), 0.f);
        c.z = fmaxf(bn_apply(loc.z, c_mean[0][cl + 2], c_istd[0][cl + 2], c_g[0][cl + 2], c_b[0][cl + 2]), 0.f);
        c.w = fmaxf(bn_apply(loc.w, c_mean[0][cl + 3], c_istd[0][cl + 3], c_g[0][cl + 3], c_b[0][cl + 3]), 0.f);
        st4(orow + cl, c);
        orow += COUT;
      }
      if ((K & (K - 1)) == 0) {  // power of two: x / K == x * (1 / K) exactly, without the division's slow path for 0
        const float rk = 1.f / kf;
        st4(orow + cl, make_float4(__fmul_rn(o.x, rk), __fmul_rn(o.y, rk), __fmul_rn(o.z, rk), __fmul_rn(o.w, rk)));
      } else {
        st4(orow + cl, make_float4(__fdiv_rn(o.x, kf), __fdiv_rn(o.y, kf), __fdiv_rn(o.z, kf), __fdiv_rn(o.w, kf)));
      }
    } else {
      sc1.x += loc.x; sc1.y += loc.y; sc1.z += loc.z; sc1.w += loc.w;
      sc2.x = fmaf(loc.x, loc.x, sc2.x); sc2.y = fmaf(loc.y, loc.y, sc2.y);
      sc2.z = fmaf(loc.z, loc.z, sc2.z); sc2.w = fmaf(loc.w, loc.w, sc2.w);
    }
  }

  if (!APPLY) {
    // per-thread fp32 partials (<= 32 points x K values) -> warp shuffle across the point
    // sub-groups -> per-warp partials in shared memory -> fp64 per CTA -> fp64 global atomics
    float v[16] = {sc1.x, sc1.y, sc1.z, sc1.w, sc2.x, sc2.y, sc2.z, sc2.w,
                   sn1.x, sn1.y, sn1.z, sn1.w, sn2.x, sn2.y, sn2.z, sn2.w};
#pragma unroll
    for (int off = LPP; off < 32; off <<= 1) {
#pragma unroll
      for (int q = 0; q < 16; ++q) v[q] += __shfl_xor_sync(0xffffffffu, v[q], off);
    }
    if (sub == 0) {
#pragma unroll
      for (int q = 0; q < 16; ++q) part[warp][(q >> 2) * COUT + cl + (q & 3)] = v[q];
    }
    __syncthreads();
    double* o = a.stats + (size_t)g * 4 * COUT;
    for (int c = tid; c < 4 * COUT; c += E_THREADS) {
      double t = 0.0;
#pragma unroll
      for (int wq = 0; wq < WARPS; ++wq) t += (double)part[wq][c];
      atomicAdd(o + c, t);
    }
  }
}

template <bool APPLY>
static int launch_edge(const EdgeArgs& a, cudaStream_t st) {
  PMVS_REQUIRE(a.groups <= 65535, "edgeconv: too many groups");
  PMVS_REQUIRE(a.rows_per_group % a.N == 0, "edgeconv: rows_per_group must be a multiple of N");
  dim3 grid(cdiv(a.rows_per_group, E_PTS_PER_BLOCK), a.groups);
  static const char* const names[2][4] = {{"edge_stats_16", "edge_stats_32", "edge_stats_64", "edge_stats_128"},
                                          {"edge_apply_16", "edge_apply_32", "edge_apply_64", "edge_apply_128"}};
  prof_begin(names[APPLY ? 1 : 0][a.cout == 16 ? 0 : (a.cout == 32 ? 1 : (a.cout == 64 ? 2 : 3))], st);
#define PMVS_EDGE_CASE(C)                                                        \
  case C:                                                                        \
    if (a.K == 16) edge_kernel<C, APPLY, 16><<<grid, E_THREADS, 0, st>>>(a);     \
    else edge_kernel<C, APPLY, 0><<<grid, E_THREADS, 0, st>>>(a);                \
    break;
  switch (a.cout) {
    PMVS_EDGE_CASE(16)
    PMVS_EDGE_CASE(32)
    PMVS_EDGE_CASE(64)
    PMVS_EDGE_CASE(128)
    default:
      set_error("edgeconv: unsupported out_channels=%d (supported: 16, 32, 64, 128)", a.cout);
      return PMVS_ERR_ARG;
  }
#undef PMVS_EDGE_CASE
  return check_launch(APPLY ? "edge_apply_kernel" : "edge_stats_kernel", st);
}
int launch_edge_stats(const EdgeArgs& a, cudaStream_t st) { return launch_edge<false>(a, st); }
int launch_edge_apply(const EdgeArgs& a, cudaStream_t st) { return launch_edge<true>(a, st); }

// =======================================================================================
// flow head: BN+ReLU of the 16-channel MLP output, Conv1d 16->1, softmax(-flow) over the 5
// hypotheses, expected offset, depth update and scatter back to the full-resolution grid
// (model.py:220-227, 256-266).  One thread per sub-cloud pixel.
// =======================================================================================

__global__ void __launch_bounds__(256) flow_head_kernel(const HeadArgs a) {
  __shared__ float cm[16], ci[16], cg[16], cb[16], cw[16];
  const int s = blockIdx.y;
  const int hs = a.h / a.ratio, ws = a.w / a.ratio;
  const int P = hs * ws, N = PMVS_NUM_HYP * P;
  if (threadIdx.x < 16) {
    const double* st = a.stats + (size_t)s * 32;
    BnCoef k = bn_coef(st[threadIdx.x], st[16 + threadIdx.x], (double)a.B * N, a.eps);
    cm[threadIdx.x] = k.mean;
    ci[threadIdx.x] = k.invstd;
    cg[threadIdx.x] = a.gamma[threadIdx.x];
    cb[threadIdx.x] = a.beta[threadIdx.x];
    cw[threadIdx.x] = a.w3[threadIdx.x];
  }
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= a.B * P) return;
  const int b = t / P, pp = t - b * P;
  const size_t cloud_row = ((size_t)s * a.B + b) * N;
  float raw[PMVS_NUM_HYP];
#pragma unroll
  for (int m = 0; m < PMVS_NUM_HYP; ++m) {
    const float* hrow = a.h2 + (cloud_row + (size_t)m * P + pp) * 16;
    float acc = 0.f;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = ldg4(hrow + q * 4);
      acc = fmaf(fmaxf(bn_apply(v.x, cm[q * 4 + 0], ci[q * 4 + 0], cg[q * 4 + 0], cb[q * 4 + 0]), 0.f), cw[q * 4 + 0], acc);
      acc = fmaf(fmaxf(bn_apply(v.y, cm[q * 4 + 1], ci[q * 4 + 1], cg[q * 4 + 1], cb[q * 4 + 1]), 0.f), cw[q * 4 + 1], acc);
      acc = fmaf(fmaxf(bn_apply(v.z, cm[q * 4 + 2], ci[q * 4 + 2], cg[q * 4 + 2], cb[q * 4 + 2]), 0.f), cw[q * 4 + 2], acc);
      acc = fmaf(fmaxf(bn_apply(v.w, cm[q * 4 + 3], ci[q * 4 + 3], cg[q * 4 + 3], cb[q * 4 + 3]), 0.f), cw[q * 4 + 3], acc);
    }
    raw[m] = acc;
  }
  flow_head_store(a, raw, s, b, pp);
}

int launch_flow_head(const HeadArgs& a, cudaStream_t st) {
  const int P = (a.h / a.ratio) * (a.w / a.ratio);
  dim3 grid(cdiv((long long)a.B * P, 256), a.S);
  prof_begin("flow_head", st);
  flow_head_kernel<<<grid, 256, 0, st>>>(a);
  return check_launch("flow_head_kernel", st);
}

// =======================================================================================
// BatchNorm running statistics, exactly as S sequential nn.BatchNorm train-mode calls:
// running = (1 - m) * running + m * batch_stat, unbiased variance for running_var.
// =======================================================================================
__global__ void bn_running_update_kernel(const RunUpdateBatch rb) {
  const RunUpdate& u = rb.u[blockIdx.x];
  if (threadIdx.x == 0 && u.nbt != nullptr) *u.nbt += rb.groups;
  for (int c = threadIdx.x; c < u.C; c += blockDim.x) {
    float rm = u.run_mean[c], rv = u.run_var[c];
    // the recurrence is sequential over the groups (S nn.BatchNorm calls in order), the loads are not: fetch the
    // sums of 8 groups at a time so that their latencies overlap
    for (int g0 = 0; g0 < rb.groups; g0 += 8) {
      double s1[8], s2[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        const bool ok = g0 + q < rb.groups;
        const double* s = u.stats + (size_t)(ok ? g0 + q : g0) * u.gstride;
        s1[q] = s[u.off_sum + c];
        s2[q] = s[u.off_sq + c];
      }
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (g0 + q < rb.groups) {
          const double mean = s1[q] / u.count;
          double var = s2[q] / u.count - mean * mean;
          if (var < 0.0) var = 0.0;
          const double unb = u.ncorr > 1.0 ? var * (u.ncorr / (u.ncorr - 1.0)) : var;
          rm = (1.f - rb.momentum) * rm + rb.momentum * (float)mean;
          rv = (1.f - rb.momentum) * rv + rb.momentum * (float)unb;
        }
      }
    }
    u.run_mean[c] = rm;
    u.run_var[c] = rv;
  }
}
int launch_bn_running_update(const RunUpdateBatch& rb, cudaStream_t st) {
  if (rb.n == 0) return PMVS_OK;
  prof_begin("bn_running_update", st);
  bn_running_update_kernel<<<rb.n, 128, 0, st>>>(rb);
  return check_launch("bn_running_update_kernel", st);
}

}  // namespace pmvs
