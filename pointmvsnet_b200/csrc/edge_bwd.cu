// EdgeConv / EdgeConvNoC backward on points-major data (pmvs_edgeconv_pm_backward).
//
// Forward (edgeconv.cu): LE = X * [W1;W2]^T = [l | e], d[n,k] = e[idx[n,k]] - l[n], y = mean_k ReLU(BN(d)) (and, for
// EdgeConv, the central half ReLU(BN(l)) in front).  With g = dy[n]/K * [pre > 0] and xhat = (d - mean) * invstd the
// BatchNorm backward is dd = A * (g - sum(g)/M - xhat * sum(g*xhat)/M), A = invstd * gamma, M = B*N*K; sum(g) and
// sum(g*xhat) are dbeta and dgamma.  In eval mode (frozen statistics) the two batch terms drop out.  The central half
// is the same over the B*N rows with g = dy * [pre > 0]: its K identical copies cancel the 1/K of the mean.
//
//   edge_bwd_stats   per-CTA partial sums of g and g*xhat of both halves over a fixed partition of the rows
//   edge_bwd_finish  fixed-order fp64 combination -> dgamma, dbeta and the coefficient table of edge_bwd_dle
//   inverse lists    build_inv_lists (gather_det.cu): for every point j, the (n, k) with idx[n,k] == j, ascending
//   edge_bwd_dle     row j of dLE = [dlocal | dedge]: dlocal = -sum_k dd[j,k] (+ central half), dedge = sum of dd over
//                    j's inverse list in ascending n*K + k, one fp32 rounding per add
//   dX  = dLE * W12  launch_gemm with W12^T (transposed into the workspace), or tile_gemm when 2*cout > 224
//   dW12 = dLE^T X   wgrad_wgmma_kernel (3xTF32 / TF32 like the forward; tile_gemm for other shapes or gemm mode 0)
//                    over fixed 1024-row slabs -> fp32 partial tiles -> fixed-order fp64 reduction
// Every sum has an order that depends only on the shapes, so the gradients are bit-reproducible on any H100.
// The ReLU mask is recomputed with the forward's own instruction sequence (common.cuh edge_nb_* and bn_apply) from
// the saved LE and statistics, so it is the forward's mask exactly.
#include <algorithm>

#include "common.cuh"
#include "wgmma.cuh"

namespace pmvs {

namespace {

constexpr int EB_THREADS = 256;
constexpr int EB_PTS = 128;    // points per CTA of the statistics and dLE passes (the statistics' fixed row partition)
constexpr int WG_SLAB = 1024;  // rows per weight-gradient slab: fixed, so the result does not depend on the SM count
constexpr int FIN_THREADS = 256;

// coefficient table [2][CF_ROWS][cout] floats, half 0 = central, 1 = neighbour
enum { CF_MEAN = 0, CF_ISTD, CF_GAMMA, CF_BETA, CF_GM, CF_GXM, CF_ROWS };

struct BwdArgs {
  const float* le;      // [R, 2*cout]
  const int32_t* idx;   // [R, K]
  const double* stats;  // [4*cout]: the sums the forward normalised with
  const float* gamma;
  const float* beta;
  float eps;
  int concat_central, bn_train;
  const float* dy;  // [R, lddy]
  int lddy;
  double* part;  // [ctas, 4*cout]: central sum g, sum g*xhat, neighbour sum g, sum g*xhat
  float* coef;   // [2, CF_ROWS, cout]
  float* dgamma;
  float* dbeta;
  const int* off;   // inverse lists
  const int* list;
  float* dle;  // [R, 2*cout]
  int R, N, K, cout;
  // NULL: the neighbour pre-activation is edge_nb_pre(e, A, edge_nb_offset(mean, l, A, beta)) (edge_kernel's sequence);
  // else the tile family's table (edge_tile.cu, [A | B | mean | invstd | gamma | beta] x cout): fma(e, A, fma(-l, A, B)),
  // the sequence it applied, and the central half's mean and invstd as it applied them
  const float* tcoef;
};

// c0 of the neighbour pre-activation pre = fma(e, A, c0) in the sequence of the family that ran the forward
__device__ __forceinline__ float bwd_nb_offset(const float* tcoef, int c, int cout, float mean, float l, float A,
                                               float beta) {
  return tcoef ? __fmaf_rn(-l, A, __ldg(tcoef + cout + c)) : edge_nb_offset(mean, l, A, beta);
}

// the central half's mean and invstd: the tile table's (with batch statistics the same bn_coef of the same sums; with
// running statistics the values the forward computed from them), else from the sums
__device__ __forceinline__ BnCoef central_coef(const BwdArgs& a, int c, int cout) {
  if (a.tcoef) return BnCoef{__ldg(a.tcoef + 2 * cout + c), __ldg(a.tcoef + 3 * cout + c)};
  return bn_coef(a.stats[c], a.stats[cout + c], (double)a.R, a.eps);
}

__device__ __forceinline__ float bwd_xhat(float d, float mean, float istd) { return __fmul_rn(__fsub_rn(d, mean), istd); }

// dd of one gathered value: the BatchNorm backward of the neighbour half at (n, k), e = e[idx[n,k]], l = l[n],
// c0 = edge_nb_offset(mean, l, A, beta), gk = dy[n] / K
__device__ __forceinline__ float bwd_dd(float e, float l, float c0, float gk, float A, float mean, float istd, float gm,
                                        float gxm) {
  const float g = edge_nb_pre(e, A, c0) > 0.f ? gk : 0.f;
  const float xh = bwd_xhat(__fsub_rn(e, l), mean, istd);
  return __fmul_rn(A, __fsub_rn(__fsub_rn(g, gm), __fmul_rn(xh, gxm)));
}

__device__ __forceinline__ float4 f4div(float4 v, float k) {
  return make_float4(__fdiv_rn(v.x, k), __fdiv_rn(v.y, k), __fdiv_rn(v.z, k), __fdiv_rn(v.w, k));
}

// KT = compile-time neighbour count (16 on the model's path), 0 = runtime K
template <int COUT, int KT>
__global__ void __launch_bounds__(EB_THREADS) edge_bwd_stats_kernel(const BwdArgs a) {
  constexpr int LPP = COUT / 4, PPW = 32 / LPP, WARPS = EB_THREADS / 32, LD = 2 * COUT;
  __shared__ float part[WARPS][4 * COUT];
  __shared__ float c_mean[2][COUT], c_istd[2][COUT], c_g[2][COUT], c_b[2][COUT];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane / LPP, cl = (lane % LPP) * 4;
  const int K = KT > 0 ? KT : a.K;
  for (int c = tid; c < COUT; c += EB_THREADS) {  // the forward's coefficients (edge_kernel APPLY)
    BnCoef kn = bn_coef(a.stats[2 * COUT + c], a.stats[3 * COUT + c], (double)a.R * K, a.eps);
    const int gn = a.concat_central ? COUT + c : c;
    c_mean[1][c] = kn.mean; c_istd[1][c] = kn.invstd; c_g[1][c] = a.gamma[gn]; c_b[1][c] = a.beta[gn];
    if (a.concat_central) {
      BnCoef kc = central_coef(a, c, COUT);
      c_mean[0][c] = kc.mean; c_istd[0][c] = kc.invstd; c_g[0][c] = a.gamma[c]; c_b[0][c] = a.beta[c];
    }
  }
  __syncthreads();
  const float kf = (float)K;
  const int nb_col = a.concat_central ? COUT : 0;
  float v[16];
#pragma unroll
  for (int q = 0; q < 16; ++q) v[q] = 0.f;
  const int p0 = blockIdx.x * EB_PTS;
  for (int it = warp * PPW + sub; it < EB_PTS; it += WARPS * PPW) {
    const int r = p0 + it;
    if (r >= a.R) break;
    const size_t cloud_base = (size_t)(r / a.N) * a.N;
    const float4 loc = ldg4(a.le + (size_t)r * LD + cl);
    const float4 gk = f4div(ldg4(a.dy + (size_t)r * a.lddy + nb_col + cl), kf);
    const float m[4] = {c_mean[1][cl], c_mean[1][cl + 1], c_mean[1][cl + 2], c_mean[1][cl + 3]};
    const float is[4] = {c_istd[1][cl], c_istd[1][cl + 1], c_istd[1][cl + 2], c_istd[1][cl + 3]};
    const float l4[4] = {loc.x, loc.y, loc.z, loc.w};
    const float g4[4] = {gk.x, gk.y, gk.z, gk.w};
    float A[4], c0[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      A[q] = a.tcoef ? __ldg(a.tcoef + cl + q) : edge_nb_scale(is[q], c_g[1][cl + q]);
      c0[q] = bwd_nb_offset(a.tcoef, cl + q, COUT, m[q], l4[q], A[q], c_b[1][cl + q]);
    }
    const int32_t* ip = a.idx + (size_t)r * K;
    auto body = [&](int nb) {
      const float4 e = ldg4(a.le + (cloud_base + nb) * LD + COUT + cl);
      const float e4[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float g = edge_nb_pre(e4[q], A[q], c0[q]) > 0.f ? g4[q] : 0.f;
        v[8 + q] += g;
        v[12 + q] = fmaf(g, bwd_xhat(__fsub_rn(e4[q], l4[q]), m[q], is[q]), v[12 + q]);
      }
    };
    if constexpr (KT > 0) {
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
    if (a.concat_central) {
      const float4 dc = ldg4(a.dy + (size_t)r * a.lddy + cl);
      const float d4[4] = {dc.x, dc.y, dc.z, dc.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int c = cl + q;
        const float pre = bn_apply(l4[q], c_mean[0][c], c_istd[0][c], c_g[0][c], c_b[0][c]);
        const float g = pre > 0.f ? d4[q] : 0.f;
        v[q] += g;
        v[4 + q] = fmaf(g, bwd_xhat(l4[q], c_mean[0][c], c_istd[0][c]), v[4 + q]);
      }
    }
  }
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
  double* o = a.part + (size_t)blockIdx.x * 4 * COUT;
  for (int c = tid; c < 4 * COUT; c += EB_THREADS) {
    double t = 0.0;
#pragma unroll
    for (int wq = 0; wq < WARPS; ++wq) t += (double)part[wq][c];
    o[c] = t;
  }
}

// one CTA per channel: the partials of all statistics CTAs in a fixed order (strided per thread, then a fixed tree)
__global__ void __launch_bounds__(FIN_THREADS) edge_bwd_finish_kernel(const BwdArgs a, int ctas) {
  __shared__ double red[FIN_THREADS];
  __shared__ double sums[4];
  const int c = blockIdx.x, tid = threadIdx.x, C = a.cout;
  for (int q = 0; q < 4; ++q) {
    double t = 0.0;
    for (int i = tid; i < ctas; i += FIN_THREADS) t += a.part[(size_t)i * 4 * C + q * C + c];
    red[tid] = t;
    __syncthreads();
    for (int s = FIN_THREADS / 2; s > 0; s >>= 1) {
      if (tid < s) red[tid] += red[tid + s];
      __syncthreads();
    }
    if (tid == 0) sums[q] = red[0];
    __syncthreads();
  }
  if (tid != 0) return;
  const double Mn = (double)a.R * a.K, Mc = (double)a.R;
  const int gn = a.concat_central ? C + c : c;
  BnCoef kn = bn_coef(a.stats[2 * C + c], a.stats[3 * C + c], Mn, a.eps);
  float* cn = a.coef + (size_t)CF_ROWS * C;
  cn[CF_MEAN * C + c] = kn.mean; cn[CF_ISTD * C + c] = kn.invstd;
  cn[CF_GAMMA * C + c] = a.gamma[gn]; cn[CF_BETA * C + c] = a.beta[gn];
  cn[CF_GM * C + c] = a.bn_train ? (float)(sums[2] / Mn) : 0.f;
  cn[CF_GXM * C + c] = a.bn_train ? (float)(sums[3] / Mn) : 0.f;
  a.dbeta[gn] = (float)sums[2];
  a.dgamma[gn] = (float)sums[3];
  if (a.concat_central) {
    BnCoef kc = central_coef(a, c, C);
    float* cc = a.coef;
    cc[CF_MEAN * C + c] = kc.mean; cc[CF_ISTD * C + c] = kc.invstd;
    cc[CF_GAMMA * C + c] = a.gamma[c]; cc[CF_BETA * C + c] = a.beta[c];
    cc[CF_GM * C + c] = a.bn_train ? (float)(sums[0] / Mc) : 0.f;
    cc[CF_GXM * C + c] = a.bn_train ? (float)(sums[1] / Mc) : 0.f;
    a.dbeta[c] = (float)sums[0];
    a.dgamma[c] = (float)sums[1];
  }
}

// one point group (COUT/4 lanes, a float4 each) per point j writes row j of dLE
template <int COUT, int KT>
__global__ void __launch_bounds__(EB_THREADS) edge_bwd_dle_kernel(const BwdArgs a) {
  constexpr int LPP = COUT / 4, PPW = 32 / LPP, WARPS = EB_THREADS / 32, LD = 2 * COUT;
  __shared__ __align__(16) float cf[2][CF_ROWS][COUT];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int sub = lane / LPP, cl = (lane % LPP) * 4;
  const int K = KT > 0 ? KT : a.K;
  for (int i = tid; i < 2 * CF_ROWS * COUT; i += EB_THREADS) (&cf[0][0][0])[i] = a.coef[i];
  __syncthreads();
  const float kf = (float)K;
  const int nb_col = a.concat_central ? COUT : 0;
  float m[4], is[4], A[4], bt[4], gm[4], gxm[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    m[q] = cf[1][CF_MEAN][cl + q]; is[q] = cf[1][CF_ISTD][cl + q]; bt[q] = cf[1][CF_BETA][cl + q];
    A[q] = a.tcoef ? __ldg(a.tcoef + cl + q) : edge_nb_scale(is[q], cf[1][CF_GAMMA][cl + q]);
    gm[q] = cf[1][CF_GM][cl + q]; gxm[q] = cf[1][CF_GXM][cl + q];
  }
  const int p0 = blockIdx.x * EB_PTS;
  for (int it = warp * PPW + sub; it < EB_PTS; it += WARPS * PPW) {
    const int r = p0 + it;
    if (r >= a.R) break;
    const int b = r / a.N, j = r - b * a.N;
    const size_t cloud_base = (size_t)b * a.N;
    const float4 loc = ldg4(a.le + (size_t)r * LD + cl);
    const float4 ej = ldg4(a.le + (size_t)r * LD + COUT + cl);
    const float4 gk = f4div(ldg4(a.dy + (size_t)r * a.lddy + nb_col + cl), kf);
    const float l4[4] = {loc.x, loc.y, loc.z, loc.w}, e4j[4] = {ej.x, ej.y, ej.z, ej.w};
    const float g4[4] = {gk.x, gk.y, gk.z, gk.w};
    float c0[4], dl[4] = {0.f, 0.f, 0.f, 0.f}, de[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int q = 0; q < 4; ++q) c0[q] = bwd_nb_offset(a.tcoef, cl + q, COUT, m[q], l4[q], A[q], bt[q]);
    // dlocal: -(sum over j's own K neighbours), k ascending
    const int32_t* ip = a.idx + (size_t)r * K;
    auto own = [&](int nb) {
      const float4 e = ldg4(a.le + (cloud_base + nb) * LD + COUT + cl);
      const float e4[4] = {e.x, e.y, e.z, e.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) dl[q] = __fadd_rn(dl[q], bwd_dd(e4[q], l4[q], c0[q], g4[q], A[q], m[q], is[q], gm[q], gxm[q]));
    };
    if constexpr (KT > 0) {
      int nbs[KT];
#pragma unroll
      for (int q = 0; q < KT / 4; ++q) {
        const int4 t = __ldg(reinterpret_cast<const int4*>(ip) + q);
        nbs[4 * q] = t.x; nbs[4 * q + 1] = t.y; nbs[4 * q + 2] = t.z; nbs[4 * q + 3] = t.w;
      }
#pragma unroll
      for (int k = 0; k < KT; ++k) own(nbs[k]);
    } else {
      for (int k = 0; k < K; ++k) own(__ldg(ip + k));
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) dl[q] = -dl[q];
    if (a.concat_central) {
      const float4 dc = ldg4(a.dy + (size_t)r * a.lddy + cl);
      const float d4[4] = {dc.x, dc.y, dc.z, dc.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int c = cl + q;
        const float mc = cf[0][CF_MEAN][c], ic = cf[0][CF_ISTD][c], gc = cf[0][CF_GAMMA][c];
        const float pre = bn_apply(l4[q], mc, ic, gc, cf[0][CF_BETA][c]);
        const float g = pre > 0.f ? d4[q] : 0.f;
        const float xh = bwd_xhat(l4[q], mc, ic);
        const float ddc = __fmul_rn(__fmul_rn(ic, gc), __fsub_rn(__fsub_rn(g, cf[0][CF_GM][c]), __fmul_rn(xh, cf[0][CF_GXM][c])));
        dl[q] = __fadd_rn(dl[q], ddc);
      }
    }
    // dedge: j's inverse list, ascending source position p = n*K + k
    const int lo = a.off[(size_t)b * (a.N + 1) + j], hi = a.off[(size_t)b * (a.N + 1) + j + 1];
    const int* lst = a.list + (size_t)b * a.N * K;
    for (int t = lo; t < hi; ++t) {
      const int p = __ldg(lst + t);
      const size_t rn = cloud_base + (size_t)(p / K);
      const float4 ln = ldg4(a.le + rn * LD + cl);
      const float4 gn = f4div(ldg4(a.dy + rn * a.lddy + nb_col + cl), kf);
      const float ln4[4] = {ln.x, ln.y, ln.z, ln.w}, gn4[4] = {gn.x, gn.y, gn.z, gn.w};
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float c0n = bwd_nb_offset(a.tcoef, cl + q, COUT, m[q], ln4[q], A[q], bt[q]);
        de[q] = __fadd_rn(de[q], bwd_dd(e4j[q], ln4[q], c0n, gn4[q], A[q], m[q], is[q], gm[q], gxm[q]));
      }
    }
    st4(a.dle + (size_t)r * LD + cl, make_float4(dl[0], dl[1], dl[2], dl[3]));
    st4(a.dle + (size_t)r * LD + COUT + cl, make_float4(de[0], de[1], de[2], de[3]));
  }
}

// fp32 SIMT tile contraction C[m, n] = sum_{k in slab} A(m, k) * B(k, n) with strided operands: 64 x 64 outputs per CTA,
// a 4 x 4 register tile per thread, k ascending in chunks of 16 staged in shared memory.  blockIdx.x = m tile + mt *
// slab, so the slabs of one launch cover [0, Kd) in fixed pieces of `kslab`; slab s writes its tile at c + s * c_slab.
struct TileGemm {
  const float* a;
  long long a_m, a_k;
  const float* b;
  long long b_k, b_n;
  float* c;
  long long ldc, c_slab;
  int M, Nn, Kd, kslab, mt;
};
constexpr int TG_BM = 64, TG_BN = 64, TG_BK = 16, TG_THREADS = 256;

__global__ void __launch_bounds__(TG_THREADS) tile_gemm_kernel(const TileGemm t) {
  __shared__ __align__(16) float As[TG_BK][TG_BM + 4];
  __shared__ __align__(16) float Bs[TG_BK][TG_BN + 4];
  const int tid = threadIdx.x, tx = tid % 16, ty = tid / 16;
  const int mtile = blockIdx.x % t.mt;
  const long long slab = blockIdx.x / t.mt;
  const int m0 = mtile * TG_BM, n0 = blockIdx.y * TG_BN;
  const long long k0 = slab * t.kslab, k1 = std::min<long long>(t.Kd, k0 + t.kslab);
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  for (long long kk = k0; kk < k1; kk += TG_BK) {
#pragma unroll
    for (int l = 0; l < (TG_BM * TG_BK) / TG_THREADS; ++l) {
      const int e = tid + l * TG_THREADS;
      int m, k;
      if (t.a_m == 1) { m = e % TG_BM; k = e / TG_BM; } else { k = e % TG_BK; m = e / TG_BK; }
      const long long gk = kk + k;
      As[k][m] = (m0 + m < t.M && gk < k1) ? __ldg(t.a + (m0 + m) * t.a_m + gk * t.a_k) : 0.f;
      int n, k2;
      if (t.b_n == 1) { n = e % TG_BN; k2 = e / TG_BN; } else { k2 = e % TG_BK; n = e / TG_BK; }
      const long long gk2 = kk + k2;
      Bs[k2][n] = (n0 + n < t.Nn && gk2 < k1) ? __ldg(t.b + gk2 * t.b_k + (n0 + n) * t.b_n) : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < TG_BK; ++k) {
      const float4 av = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      const float4 bv = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      const float a4[4] = {av.x, av.y, av.z, av.w}, b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a4[i], b4[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* c = t.c + slab * t.c_slab;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= t.M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < t.Nn) c[(long long)m * t.ldc + n] = acc[i][j];
    }
  }
}

// out[i] = sum over slabs s (ascending) of part[s * n + i], in fp64
__global__ void __launch_bounds__(256) slab_reduce_kernel(const float* __restrict__ part, float* __restrict__ out, int n,
                                                          int slabs) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int q = 0; q < slabs; ++q) s += (double)__ldg(part + (size_t)q * n + i);
  out[i] = (float)s;
}

// dW12 on the tensor cores: one CTA per fixed WG_SLAB-row slab writes the fp32 partial tile
// P[o, i] = sum over the slab's rows r of dLE[r, o] * X[r, i] (o < M2 = 2*cout, i < cin).  The contraction runs over
// rows, and tf32 wgmma reads shared-memory operands only K-major, so both row-major tensors are transposed while they
// are staged: per chunk of 32 rows, A = dLE^T [M2 x 32] and B = X^T [NP x 32] (NP = cin rounded up to 16, the padding
// rows zero) in the K-major SWIZZLE_128B layout of wgmma.cuh.  Warpgroup w owns output rows [64 w, 64 w + 64).
// NSPLIT = 3: 3xTF32 (A_lo*B_hi + A_hi*B_lo + A_hi*B_hi, the forward's arithmetic); NSPLIT = 1: plain TF32
// (pmvs_set_gemm_mode(1)).  The instruction sequence of a slab is fixed, so the partial tiles are reproducible.
constexpr int WG_KC = 32;  // rows per chunk = one 128-byte swizzle row of fp32

template <int M2, int NP, int NSPLIT>
struct WgradSmem {
  static constexpr int NPL = NSPLIT == 3 ? 2 : 1;
  static constexpr int A_PLANE = M2 * WG_KC * 4, B_PLANE = NP * WG_KC * 4;
  static constexpr int TOTAL = 1024 + NPL * (A_PLANE + B_PLANE);
};

__device__ __forceinline__ void wg_split(float x, float& hi, float& lo) {
  hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);  // the 10 mantissa bits the tensor core reads
  lo = __fsub_rn(x, hi);
}

template <int M2, int NP, int NSPLIT>
__global__ void __launch_bounds__(M2 * 2) wgrad_wgmma_kernel(const float* __restrict__ dle, const float* __restrict__ x,
                                                             int ldx, int cin, int R, float* __restrict__ part) {
  using S = WgradSmem<M2, NP, NSPLIT>;
  constexpr int THREADS = M2 * 2;  // one warpgroup per 64 output rows
  constexpr bool SPLIT = NSPLIT == 3;
  constexpr int BLK = (NP % 64 == 0) ? 64 : ((NP % 32 == 0) ? 32 : 16);
  constexpr int ACC = NP / 2;  // 64 x NP accumulator over 128 threads
  constexpr int A4 = M2 / 4;   // float4 per dLE row
  extern __shared__ unsigned char smem_raw[];
  unsigned char* smem = (unsigned char*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  unsigned char* sA = smem;                       // [plane][M2 x 128 B]
  unsigned char* sB = sA + S::NPL * S::A_PLANE;   // [plane][NP x 128 B]
  const int tid = threadIdx.x, wgi = tid >> 7, wtid = tid & 127;
  const long long r0 = (long long)blockIdx.x * WG_SLAB;
  const int rows = (int)min((long long)WG_SLAB, (long long)R - r0);
  const int nch = (rows + WG_KC - 1) / WG_KC;
  const int cin4 = cin / 4;

  // padding rows of B stay zero for the whole slab
  for (int e = tid; e < (NP - cin) * WG_KC; e += THREADS) {
    const int n = cin + e / WG_KC, k = e % WG_KC;
    const int off = wg::swz128(n, k >> 2) + (k & 3) * 4;
    *reinterpret_cast<float*>(sB + off) = 0.f;
    if (SPLIT) *reinterpret_cast<float*>(sB + S::B_PLANE + off) = 0.f;
  }
  // element (k, col) of a row-major chunk -> element (col, k) of a K-major plane; a warp covers 8 rows x 4 float4
  auto put = [&](unsigned char* plane, int plane_bytes, int k, int col0, float4 v) {
    const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int off = wg::swz128(col0 + j, k >> 2) + (k & 3) * 4;
      if (SPLIT) {
        float hi, lo;
        wg_split(vv[j], hi, lo);
        *reinterpret_cast<float*>(plane + off) = hi;
        *reinterpret_cast<float*>(plane + plane_bytes + off) = lo;
      } else {
        *reinterpret_cast<float*>(plane + off) = vv[j];
      }
    }
  };
  auto stage = [&](int c) {
    const long long rc = r0 + (long long)c * WG_KC;
    const int kvalid = min(WG_KC, rows - c * WG_KC);
    for (int e = tid; e < WG_KC * A4; e += THREADS) {
      const int k = e & 7 | ((e / (8 * 4)) % 4) << 3, col4 = (e >> 3) % 4 + 4 * (e / (8 * 4 * 4));
      const float4 v = k < kvalid ? ldg4(dle + (rc + k) * M2 + col4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      put(sA, S::A_PLANE, k, col4 * 4, v);
    }
    for (int e = tid; e < WG_KC * cin4; e += THREADS) {
      const int k = e % WG_KC, col4 = e / WG_KC;
      const float4 v = k < kvalid ? ldg4(x + (rc + k) * ldx + col4 * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      put(sB, S::B_PLANE, k, col4 * 4, v);
    }
  };

  float acc[ACC];
#pragma unroll
  for (int i = 0; i < ACC; ++i) acc[i] = 0.f;
  const uint32_t a_hi = wg::smem_u32(sA) + wgi * 64 * 128, a_lo = a_hi + S::A_PLANE;
  const uint32_t b_hi = wg::smem_u32(sB), b_lo = b_hi + S::B_PLANE;
  for (int c = 0; c < nch; ++c) {
    stage(c);
    wg::fence_proxy_async();
    __syncthreads();
    wg::fence();
#pragma unroll
    for (int j = 0; j < WG_KC / 8; ++j) {
      if (SPLIT) {
        wg::mma_tile<NP, BLK>(acc, a_lo + j * 32, b_hi + j * 32, 1u);
        wg::mma_tile<NP, BLK>(acc, a_hi + j * 32, b_lo + j * 32, 1u);
        wg::mma_tile<NP, BLK>(acc, a_hi + j * 32, b_hi + j * 32, 1u);
      } else {
        wg::mma_tile<NP, BLK>(acc, a_hi + j * 32, b_hi + j * 32, 1u);
      }
    }
    wg::commit();
    wg::wait_all();
    wg::fence_regs(acc);
    __syncthreads();  // every warpgroup has consumed the chunk before it is overwritten
  }
  // accumulator fragment (wgmma.cuh): acc[4 i + e] = D[16 w + l / 4 + 8 (e >> 1)][8 i + 2 (l % 4) + (e & 1)]
  const int warp = wtid >> 5, lane = wtid & 31;
  float* P = part + (size_t)blockIdx.x * M2 * cin;
#pragma unroll
  for (int i = 0; i < NP / 8; ++i) {
    const int col = 8 * i + 2 * (lane & 3);
    if (col < cin) {
      const int row = wgi * 64 + warp * 16 + (lane >> 2);
      *reinterpret_cast<float2*>(P + (size_t)row * cin + col) = make_float2(acc[4 * i], acc[4 * i + 1]);
      *reinterpret_cast<float2*>(P + (size_t)(row + 8) * cin + col) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
    }
  }
}

template <int M2, int NP, int NSPLIT>
int launch_wgrad_one(const float* dle, const float* x, int ldx, int cin, int R, int slabs, float* part, cudaStream_t st) {
  using S = WgradSmem<M2, NP, NSPLIT>;
  static unsigned long long smem_done = 0;
  PMVS_TRY((ensure_dyn_smem(wgrad_wgmma_kernel<M2, NP, NSPLIT>, S::TOTAL, smem_done, "wgrad_wgmma")));
  prof_begin(NSPLIT == 3 ? "edge_bwd_wgrad_3xtf32" : "edge_bwd_wgrad_tf32", st);
  wgrad_wgmma_kernel<M2, NP, NSPLIT><<<slabs, M2 * 2, S::TOTAL, st>>>(dle, x, ldx, cin, R, part);
  return check_launch("wgrad_wgmma_kernel", st);
}

// -1: the tensor-core path does not take this shape / mode (the caller runs tile_gemm_kernel)
int launch_wgrad_wgmma(const float* dle, const float* x, int ldx, int cin, int M2, int R, int slabs, float* part,
                       cudaStream_t st) {
  const int mode = pmvs_get_gemm_mode();
  if (mode != 1 && mode != 3) return -1;
  if (((uintptr_t)dle & 15) || ((uintptr_t)x & 15) || ldx % 4 != 0) return -1;
  const bool x3 = mode == 3;
#define PMVS_WG_CASE(MM, CIN, NPAD)                                                                              \
  if (M2 == MM && cin == CIN)                                                                                   \
    return x3 ? launch_wgrad_one<MM, NPAD, 3>(dle, x, ldx, cin, R, slabs, part, st)                             \
              : launch_wgrad_one<MM, NPAD, 1>(dle, x, ldx, cin, R, slabs, part, st);
  PMVS_WG_CASE(64, 136, 144)  // EdgeConvNoC 136 -> 32
  PMVS_WG_CASE(64, 32, 32)    // EdgeConv 32 -> 32
  PMVS_WG_CASE(128, 64, 64)   // EdgeConv 64 -> 64
  PMVS_WG_CASE(64, 64, 64)    // flow_mlp.0.1 (PointFlow backward)
  PMVS_WG_CASE(64, 224, 224)  // flow_mlp.0.0
  PMVS_WG_CASE(128, 32, 32)
  PMVS_WG_CASE(128, 136, 144)
#undef PMVS_WG_CASE
  return -1;
}

int launch_tile_gemm(const TileGemm& t, int slabs, const char* name, cudaStream_t st) {
  dim3 grid((unsigned)t.mt * (unsigned)slabs, cdiv(t.Nn, TG_BN));
  prof_begin(name, st);
  tile_gemm_kernel<<<grid, TG_THREADS, 0, st>>>(t);
  return check_launch("tile_gemm_kernel", st);
}

// scratch of one layer's backward (edge_layer_backward), and the stand-alone entry's workspace: the layer scratch, then
// the inverse lists and dLE
struct LayerPlan {
  int ctas, slabs;
  size_t part, coef, w12t, wpart, total;
};
LayerPlan layer_plan(long long R, long long cin, long long cout) {
  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  LayerPlan p{};
  p.ctas = (int)((R + EB_PTS - 1) / EB_PTS);
  p.slabs = (int)((R + WG_SLAB - 1) / WG_SLAB);
  size_t o = 0;
  p.part = o; o += up((size_t)p.ctas * 4 * cout * 8);
  p.coef = o; o += up((size_t)2 * CF_ROWS * cout * 4);
  p.w12t = o; o += up((size_t)cin * 2 * cout * 4);
  p.wpart = o; o += up((size_t)p.slabs * 2 * cout * cin * 4);
  p.total = o;
  return p;
}
struct BwdPlan {
  size_t inv, dle, total;
};
BwdPlan bwd_plan(long long B, long long N, long long K, long long cin, long long cout) {
  auto up = [](size_t x) { return (x + 255) & ~(size_t)255; };
  BwdPlan p{};
  size_t o = layer_plan(B * N, cin, cout).total;
  p.inv = o; o += up(inv_lists_bytes(B, N, K));
  p.dle = o; o += up((size_t)B * N * 2 * cout * 4);
  p.total = o;
  return p;
}

bool bwd_shape_ok(long long B, long long N, long long K, long long cin, long long cout) {
  return B > 0 && N > 0 && K > 0 && (cout == 16 || cout == 32 || cout == 64 || cout == 128) && cin > 0 &&
         cin % 8 == 0 && cin <= 224 && B * N * K < (1ll << 31) && B * (N + 1) < (1ll << 31);
}

}  // namespace

size_t weight_grad_scratch_bytes(long long R, int M2, int cin) {
  return (size_t)((R + WG_SLAB - 1) / WG_SLAB) * M2 * cin * sizeof(float);
}

int launch_weight_grad(const float* dy, const float* x, int ldx, int cin, int M2, int R, float* wpart, float* dw,
                       const char* simt_name, cudaStream_t st) {
  const int slabs = cdiv(R, WG_SLAB);
  const int rc = launch_wgrad_wgmma(dy, x, ldx, cin, M2, R, slabs, wpart, st);
  if (rc > 0) return rc;
  if (rc < 0) {
    TileGemm t{};
    t.a = dy; t.a_m = 1; t.a_k = M2; t.b = x; t.b_k = ldx; t.b_n = 1; t.c = wpart; t.ldc = cin;
    t.c_slab = (long long)M2 * cin; t.M = M2; t.Nn = cin; t.Kd = R; t.kslab = WG_SLAB; t.mt = cdiv(M2, TG_BM);
    PMVS_TRY(launch_tile_gemm(t, slabs, simt_name, st));
  }
  prof_begin("edge_bwd_wgrad_reduce", st);
  slab_reduce_kernel<<<cdiv((long long)M2 * cin, 256), 256, 0, st>>>(wpart, dw, M2 * cin, slabs);
  return check_launch("slab_reduce_kernel", st);
}

size_t edge_layer_bwd_scratch_bytes(long long R, int cin, int cout) { return layer_plan(R, cin, cout).total; }

int edge_layer_backward(const EdgeLayerBwd& L, cudaStream_t st) {
  const int cout = L.cout, cin = L.cin, R = L.B * L.N, C2 = 2 * cout;
  const LayerPlan p = layer_plan(R, cin, cout);
  auto at = [&](size_t off) { return L.scratch + off; };
  BwdArgs a{};
  a.le = L.le; a.idx = L.idx32; a.stats = L.stats; a.gamma = L.gamma; a.beta = L.beta; a.eps = L.eps;
  a.concat_central = L.concat_central ? 1 : 0; a.bn_train = L.bn_train ? 1 : 0; a.dy = L.dy; a.lddy = L.lddy;
  a.part = (double*)at(p.part); a.coef = (float*)at(p.coef); a.dgamma = L.dgamma; a.dbeta = L.dbeta;
  a.off = L.inv_off; a.list = L.inv_list;
  a.dle = L.dle; a.R = R; a.N = L.N; a.K = L.K; a.cout = cout; a.tcoef = L.tile_coef;

  // 1. sums of g and g * xhat -> dgamma, dbeta, coefficient table
  static const char* const sn[4] = {"edge_bwd_stats_16", "edge_bwd_stats_32", "edge_bwd_stats_64", "edge_bwd_stats_128"};
  static const char* const dn[4] = {"edge_bwd_dle_16", "edge_bwd_dle_32", "edge_bwd_dle_64", "edge_bwd_dle_128"};
  const int ci = cout == 16 ? 0 : (cout == 32 ? 1 : (cout == 64 ? 2 : 3));
  prof_begin(sn[ci], st);
#define PMVS_BWD_CASE(KERNEL, C)                                             \
  case C:                                                                    \
    if (L.K == 16) KERNEL<C, 16><<<p.ctas, EB_THREADS, 0, st>>>(a);          \
    else KERNEL<C, 0><<<p.ctas, EB_THREADS, 0, st>>>(a);                     \
    break;
  switch (cout) {
    PMVS_BWD_CASE(edge_bwd_stats_kernel, 16)
    PMVS_BWD_CASE(edge_bwd_stats_kernel, 32)
    PMVS_BWD_CASE(edge_bwd_stats_kernel, 64)
    PMVS_BWD_CASE(edge_bwd_stats_kernel, 128)
  }
  PMVS_TRY(check_launch("edge_bwd_stats_kernel", st));
  prof_begin("edge_bwd_finish", st);
  edge_bwd_finish_kernel<<<cout, FIN_THREADS, 0, st>>>(a, p.ctas);
  PMVS_TRY(check_launch("edge_bwd_finish_kernel", st));

  // 2. dLE
  prof_begin(dn[ci], st);
  switch (cout) {
    PMVS_BWD_CASE(edge_bwd_dle_kernel, 16)
    PMVS_BWD_CASE(edge_bwd_dle_kernel, 32)
    PMVS_BWD_CASE(edge_bwd_dle_kernel, 64)
    PMVS_BWD_CASE(edge_bwd_dle_kernel, 128)
  }
#undef PMVS_BWD_CASE
  PMVS_TRY(check_launch("edge_bwd_dle_kernel", st));

  // 3. dX = dLE * W12
  if (L.dx != nullptr) {
    if (C2 <= 224) {
      float* w12t = (float*)at(p.w12t);
      PMVS_TRY(launch_transpose(L.w12, w12t, 1, C2, cin, st));
      GemmArgs g{};
      g.x = a.dle; g.ldx = C2; g.w = w12t; g.y = L.dx; g.ldy = L.lddx;
      g.groups = 1; g.rows_per_group = R; g.cin = C2; g.cout = cin; g.eps = L.eps;
      PMVS_TRY(launch_gemm(g, st));
    } else {  // the contraction is longer than the GEMM kernels take
      TileGemm t{};
      t.a = a.dle; t.a_m = C2; t.a_k = 1; t.b = L.w12; t.b_k = cin; t.b_n = 1; t.c = L.dx; t.ldc = L.lddx; t.c_slab = 0;
      t.M = R; t.Nn = cin; t.Kd = C2; t.kslab = C2; t.mt = cdiv(R, TG_BM);
      PMVS_TRY(launch_tile_gemm(t, 1, "edge_bwd_dx_simt", st));
    }
  }

  // 4. dW12 = dLE^T X over fixed row slabs, then the slabs in order
  return launch_weight_grad(a.dle, L.x, L.ldx, cin, C2, R, (float*)at(p.wpart), L.dw12, "edge_bwd_wgrad_simt", st);
}

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_edgeconv_pm_backward_workspace_bytes(int B, int N, int K, int cin, int cout) {
  if (!bwd_shape_ok(B, N, K, cin, cout)) return 0;
  return bwd_plan(B, N, K, cin, cout).total;
}

extern "C" int pmvs_edgeconv_pm_backward(const float* x, int ldx, const int32_t* idx32, const int64_t* idx64,
                                         const float* w12, const float* gamma, const float* beta, float eps,
                                         int concat_central, int bn_train, const float* le, const double* stats,
                                         const float* dy, int lddy, float* dx, int lddx, float* dw12, float* dgamma,
                                         float* dbeta, void* workspace, size_t workspace_bytes, int B, int N, int K,
                                         int cin, int cout, pmvs_stream_t stream) {
  PMVS_REQUIRE(bwd_shape_ok(B, N, K, cin, cout),
               "edgeconv_backward: unsupported sizes B=%d N=%d K=%d in=%d out=%d (out in 16/32/64/128, in %% 8 == 0, "
               "in <= 224, B*N*K < 2^31)", B, N, K, cin, cout);
  const int ctot = concat_central ? 2 * cout : cout;
  PMVS_REQUIRE(ldx >= cin && ldx % 4 == 0 && lddy >= ctot && lddy % 4 == 0 && (dx == nullptr || (lddx >= cin && lddx % 4 == 0)),
               "edgeconv_backward: row strides must cover the row and be multiples of 4 floats");
  PMVS_REQUIRE(x && idx32 && idx64 && w12 && gamma && beta && le && stats && dy && dw12 && dgamma && dbeta,
               "edgeconv_backward: NULL pointer");
  const BwdPlan p = bwd_plan(B, N, K, cin, cout);
  PMVS_TRY(check_workspace("edgeconv_backward", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  EdgeLayerBwd L{};
  L.x = x; L.ldx = ldx; L.idx32 = idx32; L.w12 = w12; L.gamma = gamma; L.beta = beta; L.eps = eps;
  L.concat_central = concat_central; L.bn_train = bn_train; L.le = le; L.stats = stats; L.dy = dy; L.lddy = lddy;
  L.dx = dx; L.lddx = lddx; L.dw12 = dw12; L.dgamma = dgamma; L.dbeta = dbeta;
  L.dle = (float*)(ws + p.dle); L.B = B; L.N = N; L.K = K; L.cin = cin; L.cout = cout;
  PMVS_TRY(build_inv_lists(idx64, B, N, K, ws + p.inv, &L.inv_off, &L.inv_list, "edge_bwd_lists", st));
  L.scratch = ws;
  return edge_layer_backward(L, st);
}
