// Backward of one PointFlow iteration (pmvs_point_flow_backward): the train branch of the reference
// (model.py:150-204, 271-293: one cloud, ratio 1), from the gradients of depth_out and prob_out back to the 22 flow
// parameters, the three pyramid levels and the previous depth map.
//
// It reads what pmvs_point_flow_iter left in its workspace (camera blocks, warp source, xyz, neighbour codes or rows,
// ecat, h0-h2, the fp64 BatchNorm sums, the tile family's coefficient table, layer 2's LE) and never writes there.
// It recomputes F0 (the unfused fetch, bit-identical to what the fused fetch contracted) and the LE of layers 0 and 1
// (launch_gemm on the same inputs and weights).  Steps, in order:
//   head      dA2 = d relu(bn(h2)) through the expectation and softmax(-h3); dw3 over fixed row blocks
//   MLP x3    BatchNorm backward with the ReLU mask the forward applied (the head's or the contraction's form),
//             dW via launch_weight_grad, dX via launch_gemm (the last one is d ecat)
//   EdgeConv  layer 2 -> 0 with edge_layer_backward on inverse lists built once, each dX added into the d ecat
//             columns of the layer below (layer 0's dX is dF0)
//   fetch     dF0 -> d depth_up (skip + xyz columns) and d f_v per (pixel, hypothesis, view) with tap records;
//             the records sorted by texel (build_inv_lists) and summed per texel in record order; the transposes of
//             the bilinear and nearest resizes as gathers over fixed windows
// No floating-point atomics: every sum has an order fixed by the shapes, so two calls give the same bits.
//
// pmvs_point_flow_eval_backward is the same chain for a forward with running-statistics BatchNorm
// (pmvs_point_flow_eval_keep, which kept h0-h2, the raw flow_mlp outputs and a copy of the running statistics).  Each
// BatchNorm is then the affine map relu(fma(h, A, B)): dh = g A, dgamma = sum g xhat, dbeta = sum g with no batch
// terms, so
//   head      as above, from the kept raw outputs (the fused kernel's summation order) and the kept coefficient table
//   MLP x3    mlp_bwd_eval: dh and the per-CTA partial sums in one pass (nothing global to wait for)
//   EdgeConv  edge_layer_backward with bn_train = 0, the kept running statistics as sums (ec_run_sums_kernel) and the
//             forward's tile table for every ReLU mask
// and everything else (rows, inverse lists, F0, LE, fetch, resizes) is shared with the batch-statistics backward.
#include <algorithm>

#include "common.cuh"

namespace pmvs {

namespace {

constexpr int FB_ROWS = 128;  // rows per CTA of the BatchNorm-backward partial sums (the fixed row partition)
constexpr int HEAD_THREADS = 256;

// neighbour rows of the forward: from its 16-bit codes (tile family) or its int32 rows (gather family)
__global__ void __launch_bounds__(256) flow_idx_kernel(const unsigned short* __restrict__ cand,
                                                       const int32_t* __restrict__ idx_in, int32_t* __restrict__ idx32,
                                                       int64_t* __restrict__ idx64, long long total, int N, int HW, int W) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  int t;
  if (cand != nullptr) {
    // knn3d.cu knn_code16: inside the grid (dd+2)*96 + (dh+2)*12 + (dw+2), outside bit 15 + candidate id d*25+h*5+w;
    // the row is n + dd*HW + dh*W + dw clamped to the cloud (torch_utils.py:51-59)
    const int c = cand[e];
    const bool out = (c & 0x8000) != 0;
    const int j = c & 127;
    const int dd = (out ? j / 25 : c / 96) - 2, dh = (out ? (j % 25) / 5 : (c % 96) / 12) - 2,
              dw = (out ? j % 5 : c % 12) - 2;
    const int n = (int)((e / PMVS_KNN) % N);
    t = n + dd * HW + dh * W + dw;
    t = t < 0 ? 0 : (t > N - 1 ? N - 1 : t);
  } else {
    t = idx_in[e];
  }
  idx32[e] = t;
  idx64[e] = t;
}

// one thread per pixel: d prob and d depth through flow = sum_m softmax(-raw)_m (m - 2) interval (model.py:222-227) ->
// draw_m; dA2[row][c] = draw * w3[c]; per-CTA partials of dw3[c] = sum draw * relu(bn(h2))[c].
// EVAL: raw is the forward's (eraw [R]) and relu(bn(h2)) = relu(fma(h2, A2, B2)) from its table (ecoef [A2 | B2]).
template <bool EVAL>
__global__ void __launch_bounds__(HEAD_THREADS) head_bwd_kernel(const HeadArgs a, const float* __restrict__ dprob,
                                                                const float* __restrict__ ddepth, float* __restrict__ dA,
                                                                float* __restrict__ part, const float* __restrict__ eraw,
                                                                const float* __restrict__ ecoef) {
  __shared__ float cm[16], ci[16], cg[16], cb[16], cw[16];
  __shared__ float red[HEAD_THREADS / 32][16];
  const int P = a.h * a.w, N = PMVS_NUM_HYP * P;
  if (threadIdx.x < 16) {
    if constexpr (EVAL) {
      cm[threadIdx.x] = ecoef[threadIdx.x]; ci[threadIdx.x] = ecoef[16 + threadIdx.x];  // A2, B2
    } else {
      BnCoef k = bn_coef(a.stats[threadIdx.x], a.stats[16 + threadIdx.x], (double)a.B * N, a.eps);
      cm[threadIdx.x] = k.mean; ci[threadIdx.x] = k.invstd;
      cg[threadIdx.x] = a.gamma[threadIdx.x]; cb[threadIdx.x] = a.beta[threadIdx.x];
    }
    cw[threadIdx.x] = a.w3[threadIdx.x];
  }
  __syncthreads();
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  float dw[16];
#pragma unroll
  for (int c = 0; c < 16; ++c) dw[c] = 0.f;
  if (t < a.B * P) {
    const int b = t / P, pp = t - b * P;
    float act[PMVS_NUM_HYP][16], raw[PMVS_NUM_HYP];
#pragma unroll
    for (int m = 0; m < PMVS_NUM_HYP; ++m) {  // flow_head_kernel's arithmetic
      const size_t row = (size_t)b * N + (size_t)m * P + pp;
      const float* hrow = a.h2 + row * 16;
      float acc = 0.f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v = ldg4(hrow + q * 4);
        const float vv[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int c = q * 4 + r;
          if constexpr (EVAL) {
            act[m][c] = fmaxf(fmaf(vv[r], cm[c], ci[c]), 0.f);
          } else {
            act[m][c] = fmaxf(bn_apply(vv[r], cm[c], ci[c], cg[c], cb[c]), 0.f);
            acc = fmaf(act[m][c], cw[c], acc);
          }
        }
      }
      raw[m] = EVAL ? __ldg(eraw + row) : acc;
    }
    float mx = -raw[0];
#pragma unroll
    for (int m = 1; m < PMVS_NUM_HYP; ++m) mx = fmaxf(mx, -raw[m]);
    float e[PMVS_NUM_HYP], sum = 0.f;
#pragma unroll
    for (int m = 0; m < PMVS_NUM_HYP; ++m) {
      e[m] = expf(-raw[m] - mx);
      sum += e[m];
    }
    const float itv = __fmul_rn(a.interval_scale, a.interval[b]);
    const float gd = ddepth[(size_t)b * P + pp];
    float pr[PMVS_NUM_HYP], dpr[PMVS_NUM_HYP], s = 0.f;
#pragma unroll
    for (int m = 0; m < PMVS_NUM_HYP; ++m) {
      pr[m] = __fdiv_rn(e[m], sum);
      dpr[m] = __fmul_rn(gd, __fmul_rn((float)(m - 2), itv));
      if (dprob) dpr[m] = __fadd_rn(dpr[m], dprob[((size_t)b * PMVS_NUM_HYP + m) * P + pp]);
      s = fmaf(pr[m], dpr[m], s);
    }
#pragma unroll
    for (int m = 0; m < PMVS_NUM_HYP; ++m) {
      const float draw = -__fmul_rn(pr[m], __fsub_rn(dpr[m], s));  // d(-raw) = softmax backward
      float* drow = dA + ((size_t)b * N + (size_t)m * P + pp) * 16;
#pragma unroll
      for (int q = 0; q < 4; ++q)
        st4(drow + 4 * q, make_float4(__fmul_rn(draw, cw[4 * q]), __fmul_rn(draw, cw[4 * q + 1]),
                                      __fmul_rn(draw, cw[4 * q + 2]), __fmul_rn(draw, cw[4 * q + 3])));
#pragma unroll
      for (int c = 0; c < 16; ++c) dw[c] = fmaf(draw, act[m][c], dw[c]);
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1)
#pragma unroll
    for (int c = 0; c < 16; ++c) dw[c] += __shfl_xor_sync(0xffffffffu, dw[c], off);
  if ((threadIdx.x & 31) == 0)
#pragma unroll
    for (int c = 0; c < 16; ++c) red[threadIdx.x >> 5][c] = dw[c];
  __syncthreads();
  if (threadIdx.x < 16) {
    float v = 0.f;
    for (int wq = 0; wq < HEAD_THREADS / 32; ++wq) v += red[wq][threadIdx.x];
    part[(size_t)blockIdx.x * 16 + threadIdx.x] = v;
  }
}

// out[i] = sum over parts q (ascending) of part[q * n + i], in fp64
__global__ void __launch_bounds__(256) ordered_sum_kernel(const float* __restrict__ part, float* __restrict__ out, int n,
                                                          int parts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double s = 0.0;
  for (int q = 0; q < parts; ++q) s += (double)__ldg(part + (size_t)q * n + i);
  out[i] = (float)s;
}

// BatchNorm (batch statistics) + ReLU of the MLP: the pre-activation in the form the forward's consumer used
struct MlpBn {
  const float* h;       // [R, C] pre-BN
  const double* stats;  // [2C] sums / sums of squares
  const float* gamma;
  const float* beta;
  double count;
  float eps;
  int fma_form;  // 1: relu(fma(x, A, B)) (gemm_ws.cu), 0: ATen's ((x - mean) * invstd) * gamma + beta
  int R, C;
  // running statistics (the eval backward): the forward's [A | B] table and the running mean / variance it was built
  // from; stats and count are then not read, and the form is fma
  const float* ecoef;
  const float* rmean;
  const float* rvar;
};
struct MlpCoef {
  float mean, istd, A, B;
};
__device__ __forceinline__ MlpCoef mlp_coef(const MlpBn& a, int c) {
  if (a.ecoef) {
    MlpCoef o;
    o.mean = a.rmean[c];
    o.istd = (float)(1.0 / sqrt((double)a.rvar[c] + (double)a.eps));  // flow_eval_coef_kernel's
    o.A = a.ecoef[c];
    o.B = a.ecoef[a.C + c];
    return o;
  }
  const BnCoef k = bn_coef(a.stats[c], a.stats[a.C + c], a.count, a.eps);
  MlpCoef o;
  o.mean = k.mean; o.istd = k.invstd;
  o.A = __fmul_rn(k.invstd, a.gamma[c]);
  o.B = fmaf(-k.mean, o.A, a.beta[c]);
  return o;
}
__device__ __forceinline__ float mlp_pre(const MlpBn& a, const MlpCoef& k, float x, int c) {
  return a.fma_form ? fmaf(x, k.A, k.B) : bn_apply(x, k.mean, k.istd, a.gamma[c], a.beta[c]);
}

// act = relu(bn(h)), the input of the next contraction as the forward computed it
__global__ void __launch_bounds__(256) mlp_act_kernel(const MlpBn a, float* __restrict__ out) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)a.R * a.C) return;
  const int c = (int)(e % a.C);
  out[e] = fmaxf(mlp_pre(a, mlp_coef(a, c), a.h[e], c), 0.f);
}

// per-CTA partial sums of g = dA [pre > 0] and g * xhat over FB_ROWS rows: thread (row slot, channel)
__global__ void __launch_bounds__(256) mlp_bwd_stats_kernel(const MlpBn a, const float* __restrict__ dA,
                                                            double* __restrict__ part) {
  __shared__ float red[256][2];
  const int C = a.C, slots = 256 / C, c = threadIdx.x % C, slot = threadIdx.x / C;
  const MlpCoef k = mlp_coef(a, c);
  float s1 = 0.f, s2 = 0.f;
  const int r0 = blockIdx.x * FB_ROWS;
  for (int r = r0 + slot; r < min(r0 + FB_ROWS, a.R); r += slots) {
    const float x = a.h[(size_t)r * C + c];
    const float g = mlp_pre(a, k, x, c) > 0.f ? dA[(size_t)r * C + c] : 0.f;
    s1 += g;
    s2 = fmaf(g, __fmul_rn(__fsub_rn(x, k.mean), k.istd), s2);
  }
  red[threadIdx.x][0] = s1;
  red[threadIdx.x][1] = s2;
  __syncthreads();
  if (threadIdx.x < C) {
    double t1 = 0.0, t2 = 0.0;
    for (int q = 0; q < slots; ++q) {
      t1 += (double)red[q * C + threadIdx.x][0];
      t2 += (double)red[q * C + threadIdx.x][1];
    }
    part[(size_t)blockIdx.x * 2 * C + threadIdx.x] = t1;
    part[(size_t)blockIdx.x * 2 * C + C + threadIdx.x] = t2;
  }
}

// one CTA per channel: the partials in a fixed order -> dbeta, dgamma and coef[c] = (sum g / M, sum g xhat / M)
__global__ void __launch_bounds__(256) mlp_bwd_finish_kernel(const double* __restrict__ part, int ctas, int C,
                                                             double count, float* __restrict__ dgamma,
                                                             float* __restrict__ dbeta, float* __restrict__ coef) {
  __shared__ double red[256];
  __shared__ double sums[2];
  const int c = blockIdx.x, tid = threadIdx.x;
  for (int q = 0; q < 2; ++q) {
    double t = 0.0;
    for (int i = tid; i < ctas; i += 256) t += part[(size_t)i * 2 * C + q * C + c];
    red[tid] = t;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
      if (tid < s) red[tid] += red[tid + s];
      __syncthreads();
    }
    if (tid == 0) sums[q] = red[0];
    __syncthreads();
  }
  if (tid != 0) return;
  dbeta[c] = (float)sums[0];
  dgamma[c] = (float)sums[1];
  coef[2 * c] = (float)(sums[0] / count);
  coef[2 * c + 1] = (float)(sums[1] / count);
}

// dh = A (g - mean g - xhat mean(g xhat)), A = invstd * gamma
__global__ void __launch_bounds__(256) mlp_bwd_apply_kernel(const MlpBn a, const float* __restrict__ dA,
                                                            const float* __restrict__ coef, float* __restrict__ dh) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)a.R * a.C) return;
  const int c = (int)(e % a.C);
  const MlpCoef k = mlp_coef(a, c);
  const float x = a.h[e];
  const float g = mlp_pre(a, k, x, c) > 0.f ? dA[e] : 0.f;
  const float xh = __fmul_rn(__fsub_rn(x, k.mean), k.istd);
  dh[e] = __fmul_rn(k.A, __fsub_rn(__fsub_rn(g, coef[2 * c]), __fmul_rn(xh, coef[2 * c + 1])));
}

// running statistics: dh = A g, g = dA [pre > 0], and per-CTA partial sums of g and g * xhat over FB_ROWS rows (the
// layout of mlp_bwd_stats_kernel, for mlp_bwd_finish_kernel)
__global__ void __launch_bounds__(256) mlp_bwd_eval_kernel(const MlpBn a, const float* __restrict__ dA,
                                                           float* __restrict__ dh, double* __restrict__ part) {
  __shared__ float red[256][2];
  const int C = a.C, slots = 256 / C, c = threadIdx.x % C, slot = threadIdx.x / C;
  const MlpCoef k = mlp_coef(a, c);
  float s1 = 0.f, s2 = 0.f;
  const int r0 = blockIdx.x * FB_ROWS;
  for (int r = r0 + slot; r < min(r0 + FB_ROWS, a.R); r += slots) {
    const size_t e = (size_t)r * C + c;
    const float x = a.h[e];
    const float g = fmaf(x, k.A, k.B) > 0.f ? dA[e] : 0.f;
    dh[e] = __fmul_rn(k.A, g);
    s1 += g;
    s2 = fmaf(g, __fmul_rn(__fsub_rn(x, k.mean), k.istd), s2);
  }
  red[threadIdx.x][0] = s1;
  red[threadIdx.x][1] = s2;
  __syncthreads();
  if (threadIdx.x < C) {
    double t1 = 0.0, t2 = 0.0;
    for (int q = 0; q < slots; ++q) {
      t1 += (double)red[q * C + threadIdx.x][0];
      t2 += (double)red[q * C + threadIdx.x][1];
    }
    part[(size_t)blockIdx.x * 2 * C + threadIdx.x] = t1;
    part[(size_t)blockIdx.x * 2 * C + C + threadIdx.x] = t2;
  }
}

// the kept running statistics of the three EdgeConv layers as the sums edge_layer_backward reads, in the form the
// stand-alone EdgeConv's eval mode builds (networks.py): [m R | (v + m^2) R | m' R K | (v' + m'^2) R K] per layer at
// s4 + l * 4 * 64, m / v the central half's (channels [0, C)), m' / v' the neighbour half's
__global__ void __launch_bounds__(128) ec_run_sums_kernel(const float* __restrict__ run, double* __restrict__ s4,
                                                          double R) {
  const int l = blockIdx.x, C = flow_ec_cout(l), c = threadIdx.x;
  if (c >= C) return;
  const float* rm = run + flow_eval_run_offset(l);
  const int ctot = flow_eval_run_channels(l);
  const float* rv = rm + ctot;
  const int gn = l > 0 ? C + c : c;
  const double mc = rm[c], vc = rv[c], mn = rm[gn], vn = rv[gn];
  double* o = s4 + (size_t)l * 4 * 64;
  o[c] = mc * R;
  o[C + c] = (vc + mc * mc) * R;
  o[2 * C + c] = mn * (R * PMVS_KNN);
  o[3 * C + c] = (vn + mn * mn) * (R * PMVS_KNN);
}

// y[r, 0:n] += x[r, 0:n]  (row strides ldy, n)
__global__ void __launch_bounds__(256) add_cols_kernel(float* __restrict__ y, int ldy, const float* __restrict__ x, int n,
                                                       long long R) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= R * (n / 4)) return;
  const long long r = e / (n / 4);
  const int c = (int)(e % (n / 4)) * 4;
  float4 v = ldg4(x + r * n + c);
  float* yp = y + r * ldy + c;
  const float4 o = *reinterpret_cast<const float4*>(yp);
  st4(yp, make_float4(__fadd_rn(o.x, v.x), __fadd_rn(o.y, v.y), __fadd_rn(o.z, v.z), __fadd_rn(o.w, v.w)));
}

// transpose of the nearest resize (model.py:153-158, flow_head_kernel / fetch_describe's index rule): previous pixel
// (yp, xp) gathers the flow pixels Y, X with min(floor(Y * hp / h), hp - 1) == yp (and likewise in x), rows then
// columns ascending
__global__ void __launch_bounds__(256) nearest_bwd_kernel(const float* __restrict__ ddup, float* __restrict__ dprev,
                                                          int B, int h, int w, int hp, int wp) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= (long long)B * hp * wp) return;
  const int b = (int)(e / ((long long)hp * wp)), r = (int)(e % ((long long)hp * wp));
  const int yp = r / wp, xp = r - yp * wp;
  const float nsy = (float)hp / (float)h, nsx = (float)wp / (float)w;
  auto near = [](int o, float s, int n) {
    const int i = (int)floorf((float)o * s);
    return i < n - 1 ? i : n - 1;
  };
  const int ylo = max((int)floorf((float)yp / nsy) - 2, 0);
  const int yhi = yp == hp - 1 ? h - 1 : min((int)ceilf((float)(yp + 1) / nsy) + 1, h - 1);
  const int xlo = max((int)floorf((float)xp / nsx) - 2, 0);
  const int xhi = xp == wp - 1 ? w - 1 : min((int)ceilf((float)(xp + 1) / nsx) + 1, w - 1);
  float acc = 0.f;
  for (int Y = ylo; Y <= yhi; ++Y) {
    if (near(Y, nsy, hp) != yp) continue;
    for (int X = xlo; X <= xhi; ++X)
      if (near(X, nsx, wp) == xp) acc = __fadd_rn(acc, ddup[((size_t)b * h + Y) * w + X]);
  }
  dprev[e] = acc;
}

struct BwdFlowPlan {
  FlowPlan fwd;  // the forward's workspace, which the backward reads
  size_t npix, nrec;
  int head_ctas, mlp_ctas;
  size_t idx32, idx64, inv, f0, xyz, le, dle, decat, dtmp, df0, dA, dh, act, st4, wt, layer, wpart, hpart, mpart, mcoef;
  size_t ddup, dfv, rec_idx, rec_w, rec_inv, dsrc, total;
};

// the backward takes S = 1: the train branch (ratio 1) and the test branch at scale 0.125.  eval: the backward of
// pmvs_point_flow_eval_keep (bn_eval = 1)
int bwd_flow_plan(const pmvs_flow_shape* s, BwdFlowPlan& p, bool eval) {
  PMVS_REQUIRE(s != nullptr, "point_flow_backward: NULL shape");
  if (eval) {
    PMVS_REQUIRE(s->bn_eval == 1, "point_flow_eval_backward: bn_eval must be 1, got %d", s->bn_eval);
    // the keep forward runs on the tile EdgeConv family only, so its workspace has no gather-family rows or sums
    PMVS_REQUIRE(opt(OPT_EDGE) != 0, "point_flow_eval_backward: served by the tile EdgeConv kernels only (option "
                 "edge=%d)", opt(OPT_EDGE));
  } else {
    PMVS_REQUIRE(s->bn_eval == 0, "point_flow_backward: the forward ran with bn_eval = 1 (running-statistics "
                 "BatchNorm); its backward is pmvs_point_flow_eval_backward");
  }
  PMVS_REQUIRE(s->ratio == 1 && s->sub_count == 0 && s->sub_begin == 0,
               "point_flow_backward: only one cloud per call (ratio 1, no sub_count); got ratio %d, sub_count %d",
               s->ratio, s->sub_count);
  PMVS_TRY(flow_plan(s, p.fwd, eval));
  p.npix = (size_t)s->B * s->flow_h * s->flow_w;
  p.nrec = p.npix * PMVS_NUM_HYP * s->V * 4;
  PMVS_REQUIRE(p.fwd.R * PMVS_KNN < ((size_t)1 << 31) && p.nrec < ((size_t)1 << 31) &&
                   (size_t)s->B * (p.nrec / 4 + 1) < ((size_t)1 << 31),
               "point_flow_backward: problem too large");
  p.head_ctas = cdiv((long long)p.npix, HEAD_THREADS);
  p.mlp_ctas = cdiv((long long)p.fwd.R, FB_ROWS);
  const long long R = (long long)p.fwd.R;
  size_t lay = 0;
  for (int l = 0; l < 3; ++l) lay = std::max(lay, edge_layer_bwd_scratch_bytes(R, flow_ec_cin(l), flow_ec_cout(l)));
  size_t wp = 0;
  for (int l = 0; l < 3; ++l) wp = std::max(wp, weight_grad_scratch_bytes(R, flow_mlp_cout(l), flow_mlp_cin(l)));
  size_t o = 0;
  p.idx32 = o; o += up256(p.fwd.R * PMVS_KNN * 4);
  p.idx64 = o; o += up256(p.fwd.R * PMVS_KNN * 8);
  p.inv = o; o += up256(inv_lists_bytes(s->B, p.fwd.N, PMVS_KNN));
  p.f0 = o; o += up256(p.fwd.R * PMVS_FEAT_CH * 4);
  p.xyz = o; o += up256(p.fwd.R * 3 * 4);
  p.le = o; o += up256(p.fwd.R * 128 * 4);
  p.dle = o; o += up256(p.fwd.R * 128 * 4);
  p.decat = o; o += up256(p.fwd.R * 224 * 4);
  p.dtmp = o; o += up256(p.fwd.R * 64 * 4);
  p.df0 = o; o += up256(p.fwd.R * PMVS_FEAT_CH * 4);
  p.dA = o; o += up256(p.fwd.R * 64 * 4);
  p.dh = o; o += up256(p.fwd.R * 64 * 4);
  p.act = o; o += up256(p.fwd.R * 64 * 4);
  p.st4 = o; o += up256(3 * 4 * 64 * 8);
  p.wt = o; o += up256(224 * 64 * 4);
  p.layer = o; o += up256(lay);
  p.wpart = o; o += up256(wp);
  p.hpart = o; o += up256((size_t)p.head_ctas * 16 * 4);
  p.mpart = o; o += up256((size_t)p.mlp_ctas * 2 * 64 * 8);
  p.mcoef = o; o += up256(2 * 64 * 4);
  p.ddup = o; o += up256(p.npix * 4);
  p.dfv = o; o += up256(p.nrec / 4 * 112 * 4);
  p.rec_idx = o; o += up256(p.nrec * 8);
  p.rec_w = o; o += up256(p.nrec * 4);
  p.rec_inv = o; o += up256(inv_lists_bytes(s->B, (long long)(p.nrec / 4 / s->B), 4));
  p.dsrc = o; o += up256(warp_source_bytes(s->B, s->V, s->flow_h, s->flow_w));
  p.total = o;
  return PMVS_OK;
}

int mlp_layer_backward(const MlpBn& a, const float* dA, float* dh, double* part, float* coef, float* dgamma,
                       float* dbeta, int ctas, cudaStream_t st) {
  prof_begin("mlp_bwd_stats", st);
  mlp_bwd_stats_kernel<<<ctas, 256, 0, st>>>(a, dA, part);
  PMVS_TRY(check_launch("mlp_bwd_stats_kernel", st));
  prof_begin("mlp_bwd_finish", st);
  mlp_bwd_finish_kernel<<<a.C, 256, 0, st>>>(part, ctas, a.C, a.count, dgamma, dbeta, coef);
  PMVS_TRY(check_launch("mlp_bwd_finish_kernel", st));
  prof_begin("mlp_bwd_apply", st);
  mlp_bwd_apply_kernel<<<cdiv((long long)a.R * a.C, 256), 256, 0, st>>>(a, dA, coef, dh);
  return check_launch("mlp_bwd_apply_kernel", st);
}

int mlp_layer_backward_eval(const MlpBn& a, const float* dA, float* dh, double* part, float* coef, float* dgamma,
                            float* dbeta, int ctas, cudaStream_t st) {
  prof_begin("mlp_bwd_eval", st);
  mlp_bwd_eval_kernel<<<ctas, 256, 0, st>>>(a, dA, dh, part);
  PMVS_TRY(check_launch("mlp_bwd_eval_kernel", st));
  prof_begin("mlp_bwd_finish", st);
  mlp_bwd_finish_kernel<<<a.C, 256, 0, st>>>(part, ctas, a.C, 1.0, dgamma, dbeta, coef);
  return check_launch("mlp_bwd_finish_kernel", st);
}

int mlp_act(const MlpBn& a, float* out, cudaStream_t st) {
  prof_begin("mlp_bwd_act", st);
  mlp_act_kernel<<<cdiv((long long)a.R * a.C, 256), 256, 0, st>>>(a, out);
  return check_launch("mlp_act_kernel", st);
}

// dx [R, cin] = dy [R, cout] * w [cout, cin] through the forward contractions (w transposed into wt)
int contract_dx(const float* dy, int cout, const float* w, int cin, float* wt, float* dx, int ldx, int R, float eps,
                cudaStream_t st) {
  PMVS_TRY(launch_transpose(w, wt, 1, cout, cin, st));
  GemmArgs g{};
  g.x = dy; g.ldx = cout; g.w = wt; g.y = dx; g.ldy = ldx;
  g.groups = 1; g.rows_per_group = R; g.cin = cout; g.cout = cin; g.eps = eps;
  return launch_gemm(g, st);
}

int add_cols(float* y, int ldy, const float* x, int n, long long R, cudaStream_t st) {
  prof_begin("flow_bwd_add", st);
  add_cols_kernel<<<cdiv(R * (n / 4), 256), 256, 0, st>>>(y, ldy, x, n, R);
  return check_launch("add_cols_kernel", st);
}

// pmvs_point_flow_backward, and with eval pmvs_point_flow_eval_backward
int point_flow_backward(const pmvs_flow_shape* shape, const pmvs_flow_weights* wts, const float* const pyramids_cl[3],
                        const float* depth_prev, const float* cam_params, const float* interval, const float* mean,
                        const float* stdv, const void* fwd_workspace, const float* grad_depth_out,
                        const float* grad_prob_out, const pmvs_flow_grads* grads, void* workspace,
                        size_t workspace_bytes, pmvs_stream_t stream, bool eval) {
  BwdFlowPlan p;
  PMVS_TRY(bwd_flow_plan(shape, p, eval));
  PMVS_REQUIRE(wts && pyramids_cl && depth_prev && cam_params && interval && mean && stdv && fwd_workspace &&
                   grad_depth_out && grads && workspace,
               "point_flow_backward: NULL pointer");
  for (int l = 0; l < 3; ++l)
    PMVS_REQUIRE(grads->ec_dw12[l] && grads->ec_dgamma[l] && grads->ec_dbeta[l] && grads->mlp_dw[l] &&
                     grads->mlp_dgamma[l] && grads->mlp_dbeta[l] && pyramids_cl[l],
                 "point_flow_backward: NULL pointer");
  PMVS_REQUIRE(grads->mlp_dw[3] != nullptr, "point_flow_backward: NULL pointer");
  PMVS_REQUIRE(((uintptr_t)fwd_workspace & 255) == 0, "point_flow_backward: fwd_workspace must be 256-byte aligned");
  PMVS_TRY(check_workspace("point_flow_backward", workspace, workspace_bytes, p.total));
  (void)cam_params; (void)mean; (void)stdv;  // the forward's camera blocks already hold them
  const FlowPlan& fr = p.fwd;
  const bool gather = !fr.tile;  // the EdgeConv family of the forward (the options must not change between)
  cudaStream_t st = (cudaStream_t)stream;
  const char* fw = (const char*)fwd_workspace;
  char* ws = (char*)workspace;
  const int B = shape->B, N = fr.N, R = (int)fr.R, h = shape->flow_h, w = shape->flow_w;
  const float eps = wts->eps;
  const float* ecat = (const float*)(fw + fr.ecat);
  const float* h0 = (const float*)(fw + fr.h0);
  const float* h1 = (const float*)(fw + fr.h1);
  const float* h2 = (const float*)(fw + fr.h2);
  const float* le2 = (const float*)(fw + fr.le);  // the LE scratch holds the last EdgeConv layer's
  const double* stats = (const double*)(fw + fr.stats);
  const float* fcoef = (const float*)(fw + fr.coef);
  // eval: the forward's flow_mlp table, raw outputs and running statistics
  const float* ecoef = eval ? (const float*)(fw + fr.mlp_coef) : nullptr;
  const float* run = eval ? (const float*)(fw + fr.run) : nullptr;

  auto F = [&](size_t o) { return (float*)(ws + o); };
  double* part = (double*)(ws + p.mpart);
  float* mcoef = F(p.mcoef);
  const bool need_fetch = grads->ddepth_prev || grads->dpyramids_cl[0] || grads->dpyramids_cl[1] ||
                          grads->dpyramids_cl[2];
  const bool need_pyr = grads->dpyramids_cl[0] || grads->dpyramids_cl[1] || grads->dpyramids_cl[2];

  // ---- head
  HeadArgs ha = head_args(shape, fr, wts, depth_prev, interval, nullptr, nullptr);
  ha.h2 = h2; ha.stats = stats + fr.st_mlp[2]; ha.gamma = wts->mlp_gamma[2]; ha.beta = wts->mlp_beta[2];
  if (eval) {
    prof_begin("head_bwd_eval", st);
    head_bwd_kernel<true><<<p.head_ctas, HEAD_THREADS, 0, st>>>(ha, grad_prob_out, grad_depth_out, F(p.dA),
                                                                F(p.hpart), (const float*)(fw + fr.raw),
                                                                ecoef + flow_mlp_coef_offset(2));
  } else {
    prof_begin("head_bwd", st);
    head_bwd_kernel<false><<<p.head_ctas, HEAD_THREADS, 0, st>>>(ha, grad_prob_out, grad_depth_out, F(p.dA),
                                                                 F(p.hpart), nullptr, nullptr);
  }
  PMVS_TRY(check_launch("head_bwd_kernel", st));
  prof_begin("head_bwd_reduce", st);
  ordered_sum_kernel<<<1, 256, 0, st>>>(F(p.hpart), grads->mlp_dw[3], 16, p.head_ctas);
  PMVS_TRY(check_launch("ordered_sum_kernel", st));

  // ---- flow_mlp, layer 2 -> 0
  {
    const float* hs[3] = {h0, h1, h2};
    auto bn = [&](int l, int fma_form) {
      MlpBn a{};
      a.h = hs[l]; a.stats = stats + fr.st_mlp[l]; a.gamma = wts->mlp_gamma[l]; a.beta = wts->mlp_beta[l];
      a.count = (double)R; a.eps = eps; a.fma_form = fma_form; a.R = R; a.C = flow_mlp_cout(l);
      if (eval) {
        a.ecoef = ecoef + flow_mlp_coef_offset(l);
        a.rmean = run + flow_eval_run_offset(3 + l);
        a.rvar = a.rmean + flow_mlp_cout(l);
        a.fma_form = 1;
      }
      return a;
    };
    // the mask of layer l is the one its consumer applied: the head for layer 2, the contraction of layer l + 1
    auto consumer_fma = [&](int l) {
      if (l == 2 || eval) return 0;  // eval: the fused kernel's fma form (mlp_coef)
      GemmArgs g{};
      g.x = hs[l]; g.ldx = flow_mlp_cout(l); g.w = wts->mlp_w[l + 1]; g.y = (float*)hs[l + 1];
      g.ldy = flow_mlp_cout(l + 1); g.groups = 1; g.rows_per_group = R; g.cin = flow_mlp_cin(l + 1);
      g.cout = flow_mlp_cout(l + 1);
      return gemm_in_bn_fma_form(g) ? 1 : 0;
    };
    float* dA = F(p.dA);
    float* dh = F(p.dh);
    for (int l = 2; l >= 0; --l) {
      const MlpBn a = bn(l, consumer_fma(l));
      if (eval)
        PMVS_TRY(mlp_layer_backward_eval(a, dA, dh, part, mcoef, grads->mlp_dgamma[l], grads->mlp_dbeta[l], p.mlp_ctas,
                                         st));
      else
        PMVS_TRY(mlp_layer_backward(a, dA, dh, part, mcoef, grads->mlp_dgamma[l], grads->mlp_dbeta[l], p.mlp_ctas, st));
      const float* x = ecat;
      if (l > 0) {
        PMVS_TRY(mlp_act(bn(l - 1, consumer_fma(l - 1)), F(p.act), st));
        x = F(p.act);
      }
      const int cin = flow_mlp_cin(l), cout = flow_mlp_cout(l);
      PMVS_TRY(launch_weight_grad(dh, x, cin, cin, cout, R, F(p.wpart), grads->mlp_dw[l], "mlp_bwd_wgrad_simt", st));
      // dX: d act of layer l - 1 (into dA), or d ecat
      PMVS_TRY(contract_dx(dh, cout, wts->mlp_w[l], cin, F(p.wt), l > 0 ? dA : F(p.decat), cin, R, eps, st));
    }
  }

  // ---- neighbour rows, inverse lists (once for the three layers), F0
  {
    const long long total = (long long)fr.R * PMVS_KNN;
    prof_begin("flow_bwd_idx", st);
    flow_idx_kernel<<<cdiv(total, 256), 256, 0, st>>>(gather ? nullptr : (const unsigned short*)(fw + fr.cand),
                                                     gather ? (const int32_t*)(fw + fr.idx) : nullptr,
                                                     (int32_t*)(ws + p.idx32), (int64_t*)(ws + p.idx64), total, N,
                                                     h * w, w);
    PMVS_TRY(check_launch("flow_idx_kernel", st));
  }
  const int* inv_off = nullptr;
  const int* inv_list = nullptr;
  PMVS_TRY(build_inv_lists((const int64_t*)(ws + p.idx64), B, N, PMVS_KNN, ws + p.inv, &inv_off, &inv_list,
                           "flow_bwd_lists", st));
  // the forward's warp source and camera blocks; F0 and xyz go to this workspace
  FusedFetchParams ff = fetch_params(shape, fr, (char*)fw, depth_prev);
  ff.feature = F(p.f0); ff.xyz = F(p.xyz);
  PMVS_TRY(launch_fused_fetch(ff, st));

  // ---- flow_edge_conv, layer 2 -> 0
  {
    double* st4 = (double*)(ws + p.st4);
    if (eval) {  // the three layers' sums from the kept running statistics
      prof_begin("flow_bwd_run_sums", st);
      ec_run_sums_kernel<<<3, 128, 0, st>>>(run, st4, (double)R);
      PMVS_TRY(check_launch("ec_run_sums_kernel", st));
    }
    for (int l = 2; l >= 0; --l) {
      const int c = flow_ec_cout(l), cin = flow_ec_cin(l);
      double* s4 = st4 + (size_t)l * 4 * 64;
      if (!eval) {  // the forward's sums -> [sum_c | sumsq_c | sum_n | sumsq_n] (eval: ec_run_sums_kernel's are there)
        const RunUpdate cen = ec_sums(fr, stats, l, true), nb = ec_sums(fr, stats, l, false);
        const double* srcs[4] = {cen.stats + cen.off_sum, cen.stats + cen.off_sq, nb.stats + nb.off_sum,
                                 nb.stats + nb.off_sq};
        for (int q = (l > 0 ? 0 : 2); q < 4; ++q)
          if (cudaMemcpyAsync(s4 + q * c, srcs[q], c * sizeof(double), cudaMemcpyDeviceToDevice, st) != cudaSuccess) {
            set_error("point_flow_backward: copy failed");
            return PMVS_ERR_CUDA;
          }
      }
      const float* x = l == 0 ? F(p.f0) : ecat + flow_ec_in_off(l);
      const int ldx = l == 0 ? PMVS_FEAT_CH : 224;
      const float* le = le2;
      if (l < 2) {  // the forward's LE scratch holds layer 2's; recompute the others from the same inputs
        GemmArgs g{};
        g.x = x; g.ldx = ldx; g.w = wts->ec_w12[l]; g.y = F(p.le); g.ldy = 2 * c;
        g.groups = 1; g.rows_per_group = R; g.cin = cin; g.cout = 2 * c; g.eps = eps;
        PMVS_TRY(launch_gemm(g, st));
        le = F(p.le);
      }
      EdgeLayerBwd L{};
      L.x = x; L.ldx = ldx; L.idx32 = (const int32_t*)(ws + p.idx32); L.inv_off = inv_off; L.inv_list = inv_list;
      L.w12 = wts->ec_w12[l]; L.gamma = wts->ec_gamma[l]; L.beta = wts->ec_beta[l]; L.eps = eps;
      L.concat_central = l > 0; L.bn_train = eval ? 0 : 1; L.le = le; L.stats = s4;
      L.tile_coef = gather ? nullptr : fcoef + flow_ec_coef_offset(l, 1, 0);
      L.dy = F(p.decat) + flow_ec_out_off(l); L.lddy = 224;
      L.dx = l > 0 ? F(p.dtmp) : (need_fetch ? F(p.df0) : nullptr);
      L.lddx = l > 0 ? cin : PMVS_FEAT_CH;
      L.dw12 = grads->ec_dw12[l]; L.dgamma = grads->ec_dgamma[l]; L.dbeta = grads->ec_dbeta[l];
      L.dle = F(p.dle); L.scratch = ws + p.layer; L.B = B; L.N = N; L.K = PMVS_KNN; L.cin = cin; L.cout = c;
      PMVS_TRY(edge_layer_backward(L, st));
      if (l > 0) PMVS_TRY(add_cols(F(p.decat) + flow_ec_in_off(l), 224, F(p.dtmp), cin, R, st));
    }
  }
  if (!need_fetch) return PMVS_OK;

  // ---- fetch
  FetchBwdParams fb{};
  fb.f = ff;
  fb.f.feature = F(p.df0);
  fb.ddepth_out = grad_depth_out; fb.ddup = F(p.ddup);
  fb.dfv = need_pyr ? F(p.dfv) : nullptr;
  fb.rec_idx = (int64_t*)(ws + p.rec_idx); fb.rec_w = F(p.rec_w);
  PMVS_TRY(launch_fetch_backward(fb, st));
  if (grads->ddepth_prev) {
    const long long n = (long long)B * shape->prev_h * shape->prev_w;
    prof_begin("nearest_bwd", st);
    nearest_bwd_kernel<<<cdiv(n, 256), 256, 0, st>>>(F(p.ddup), grads->ddepth_prev, B, h, w, shape->prev_h,
                                                     shape->prev_w);
    PMVS_TRY(check_launch("nearest_bwd_kernel", st));
  }
  if (need_pyr) {
    const int T = shape->V * h * w, nrec = (int)(p.nrec / B);
    const int* roff = nullptr;
    const int* rlist = nullptr;
    PMVS_TRY(build_inv_lists((const int64_t*)(ws + p.rec_idx), B, nrec / 4, 4, ws + p.rec_inv, &roff, &rlist,
                             "flow_bwd_tap_lists", st));
    // d warp source [B][V*h*w + 1][112]: the layout of the forward's warp source
    PMVS_TRY(launch_texel_sum(roff, rlist, F(p.rec_w), F(p.dfv), F(p.dsrc), T, nrec, B, 112, (long long)(T + 1) * 112,
                              112, "texel_sum", st));
    PMVS_TRY(launch_warp_source_backward(F(p.dsrc), shape->pyr_h, shape->pyr_w, grads->dpyramids_cl, B, shape->V, h,
                                         w, st));
  }
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_point_flow_backward_workspace_bytes(const pmvs_flow_shape* shape) {
  BwdFlowPlan p;
  if (bwd_flow_plan(shape, p, false) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_point_flow_backward(const pmvs_flow_shape* shape, const pmvs_flow_weights* wts,
                                        const float* const pyramids_cl[3], const float* depth_prev,
                                        const float* cam_params, const float* interval, const float* mean,
                                        const float* stdv, const void* fwd_workspace, const float* grad_depth_out,
                                        const float* grad_prob_out, const pmvs_flow_grads* grads, void* workspace,
                                        size_t workspace_bytes, pmvs_stream_t stream) {
  return point_flow_backward(shape, wts, pyramids_cl, depth_prev, cam_params, interval, mean, stdv, fwd_workspace,
                             grad_depth_out, grad_prob_out, grads, workspace, workspace_bytes, stream, false);
}

extern "C" size_t pmvs_point_flow_eval_backward_workspace_bytes(const pmvs_flow_shape* shape) {
  BwdFlowPlan p;
  if (bwd_flow_plan(shape, p, true) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_point_flow_eval_backward(const pmvs_flow_shape* shape, const pmvs_flow_weights* wts,
                                             const float* const pyramids_cl[3], const float* depth_prev,
                                             const float* cam_params, const float* interval, const float* mean,
                                             const float* stdv, const void* fwd_workspace,
                                             const float* grad_depth_out, const float* grad_prob_out,
                                             const pmvs_flow_grads* grads, void* workspace, size_t workspace_bytes,
                                             pmvs_stream_t stream) {
  return point_flow_backward(shape, wts, pyramids_cl, depth_prev, cam_params, interval, mean, stdv, fwd_workspace,
                             grad_depth_out, grad_prob_out, grads, workspace, workspace_bytes, stream, true);
}

extern "C" int pmvs_point_flow_backward_debug_offsets(const pmvs_flow_shape* shape, int eval, size_t off[7]) {
  BwdFlowPlan p;
  PMVS_TRY(bwd_flow_plan(shape, p, eval != 0));
  PMVS_REQUIRE(off != nullptr, "point_flow_backward_debug_offsets: NULL pointer");
  off[0] = p.df0; off[1] = p.ddup; off[2] = p.dfv; off[3] = p.rec_idx; off[4] = p.rec_w; off[5] = p.dsrc;
  off[6] = p.total;
  return PMVS_OK;
}
