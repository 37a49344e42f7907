// Backward of ImageConv for every view at once, include/pmvs_b200.h, DESIGN 3.15.
//
// It reads the workspace of pmvs_image_conv_keep: every BatchNorm layer's pre-BatchNorm output y_l (NHWC) and its
// per-view scale / shift.  The layers are walked in reverse, conv3.2 down to conv0.0, and only as far up as the
// coarsest level that has a gradient.  For each layer l:
//   - BatchNorm + ReLU backward (l < 10), once dA_l, the gradient of its activation, is known: the data gradient of
//     layer l + 1, plus the gradient of the pyramid level l produces (conv0, conv1, conv2 at l = 1, 4, 7), added in
//     that order as it is loaded.  dz = dA * [y * scale_v + shift_v > 0] with the forward's own scale / shift; per-CTA
//     fp64 sums of dz and dz * (y - mean_v), a CTA never mixing two views (ic_bnb_reduce_kernel); one finalize per
//     channel that walks the views in order (per-view constants of G, and dgamma, dbeta summed over views in view
//     order); then G_l, the gradient of the pre-BatchNorm output, written over dA_l (ic_bnb_apply_kernel).  conv3.2's
//     G is the conv3 gradient itself.
//   - the weight gradient (ic_wgrad_kernel): CTAs own fixed pixel chunks of one image and sum G_l x act_in over them,
//     the input activation recomputed from the kept y_(l-1) with each view's scale / shift (conv0.0 reads the planar
//     image); a finalize adds the chunk partials in order into the PyTorch layout [Cout, Cin, K, K].
//   - the data gradient (l >= 1): a stride-1 layer's is the forward's convolution kernel (no BatchNorm prologue) on
//     G_l with flipped taps and Cin and Cout swapped; a 5x5 stride-2 layer's is a transposed convolution in gather
//     form (ic_dgrad_s2_kernel), one output parity class per CTA.
// The images get no gradient.  fp32 FMA products, fp64 sums across threads and CTAs, every sum in an order fixed by the
// shapes and no floating-point atomics: two calls give the same bits.
#include <float.h>

#include "image_conv.cuh"

namespace pmvs {

namespace {

constexpr int IB_THREADS = 256, IB_CHUNK = 16384;  // BatchNorm backward: about IB_CHUNK values of one image per CTA
constexpr int IW_TARGET_CTAS = 4224;               // weight gradients: 32 CTAs per SM of an H100 before splitting less
constexpr int IW_MIN_CHUNK = 1024;                 // ... and at least this many output pixels per CTA
constexpr int IW_CO = 8;                           // weight gradients: output channels per CTA

const char* const IB_DATA[IC_LAYERS] = {nullptr,      "icb_data0_1", "icb_data1_0", "icb_data1_1",
                                        "icb_data1_2", "icb_data2_0", "icb_data2_1", "icb_data2_2",
                                        "icb_data3_0", "icb_data3_1", "icb_data3_2"};
const char* const IB_WGRAD[IC_LAYERS] = {"icb_wgrad0_0", "icb_wgrad0_1", "icb_wgrad1_0", "icb_wgrad1_1",
                                         "icb_wgrad1_2", "icb_wgrad2_0", "icb_wgrad2_1", "icb_wgrad2_2",
                                         "icb_wgrad3_0", "icb_wgrad3_1", "icb_wgrad3_2"};

// The data gradient of a stride-1 layer: the forward's convolution on G without the BatchNorm prologue.
template <int K, int CIN, int COUT, int CO, int PX>
__global__ void __launch_bounds__(IC_THREADS) ic_dgrad_kernel(const IcArgs a) {
  ic_conv_body<K, 1, CIN, COUT, CO, PX, false>(a);
}

// The data gradient of a 5x5, stride-2, padding-2 layer in gather form: dx[i] = sum over (o, k) with 2 o - 2 + k = i
// of G[o] W[k], i.e. for i = 2 t + p the taps k = p, p + 2, ... at o = t + (p + 2 - k) / 2.  One CTA: IC_THREADS
// column groups of PX input pixels of one parity class (ph, pw) x CO channels of dx (group blockIdx.y);
// blockIdx.z = image * 4 + 2 ph + pw.  a.x = G [N, Hi, Wi, CIN] (the layer's output grid), a.y = dx [N, Ho, Wo, COUT]
// (its input grid), a.w = [25][CIN][COUT] (the forward's weights with Cin and Cout swapped, taps as they are).
template <int CIN, int COUT, int CO, int PX>
__global__ void __launch_bounds__(IC_THREADS) ic_dgrad_s2_kernel(const IcArgs a) {
  static_assert(CIN % 4 == 0 && CO % 4 == 0 && COUT % CO == 0, "channels are read and written four at a time");
  const int par = blockIdx.z & 3, n = blockIdx.z >> 2, ph = par >> 1, pw = par & 1, g = blockIdx.y;
  const int tp = blockIdx.x * IC_THREADS + threadIdx.x;
  const bool live = tp < a.tpix;
  const int th = live ? tp / a.ncg : 0, j0 = live ? (tp % a.ncg) * PX : 0;
  const int oh = 2 * th + ph;
  const float* wg = a.w + g * CO;

  float acc[PX][CO];
#pragma unroll
  for (int p = 0; p < PX; ++p)
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[p][c] = 0.f;

#pragma unroll 1
  for (int t = 0; t < 3; ++t) {
    const int kh = ph + 2 * t;
    if (kh > 4) break;
    const int gh = th + 1 - t;
    const bool okh = live && gh >= 0 && gh < a.Hi;
    const float* row = a.x + ((long long)n * a.Hi + gh) * a.Wi * CIN;
#pragma unroll
    for (int u = 0; u < 3; ++u) {
      const int kw = pw + 2 * u;
      if (kw > 4) break;
      const float* wt = wg + (kh * 5 + kw) * CIN * COUT;
#pragma unroll 1
      for (int c4 = 0; c4 < CIN; c4 += 4) {
        float xv[PX][4];
#pragma unroll
        for (int p = 0; p < PX; ++p) {
          const int gw = j0 + p + 1 - u;
          if (okh && gw >= 0 && gw < a.Wi) {
            const float4 q = ldg4(row + (long long)gw * CIN + c4);
            xv[p][0] = q.x; xv[p][1] = q.y; xv[p][2] = q.z; xv[p][3] = q.w;
          } else {
            xv[p][0] = xv[p][1] = xv[p][2] = xv[p][3] = 0.f;
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float wv[CO];
#pragma unroll
          for (int c = 0; c < CO; c += 4) {
            const float4 q = ldg4(wt + (c4 + j) * COUT + c);
            wv[c] = q.x; wv[c + 1] = q.y; wv[c + 2] = q.z; wv[c + 3] = q.w;
          }
#pragma unroll
          for (int p = 0; p < PX; ++p)
#pragma unroll
            for (int c = 0; c < CO; ++c) acc[p][c] = __fmaf_rn(xv[p][j], wv[c], acc[p][c]);
        }
      }
    }
  }
  if (!live || oh >= a.Ho) return;
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    const int ow = 2 * (j0 + p) + pw;
    if (ow >= a.Wo) continue;
    float* yp = a.y + (((long long)n * a.Ho + oh) * a.Wo + ow) * COUT + g * CO;
#pragma unroll
    for (int c = 0; c < CO; c += 4)
      *reinterpret_cast<float4*>(yp + c) = make_float4(acc[p][c], acc[p][c + 1], acc[p][c + 2], acc[p][c + 3]);
  }
}

// the incoming gradient of a BatchNorm layer's activation at NHWC element i = (n * P + pix) * C + c0 .. c0 + 3: the
// next layer's data gradient (NHWC, or NULL), then the gradient of the pyramid level this layer produces (in the
// layout the forward wrote it, or NULL), added in that order
__device__ __forceinline__ void ib_grad_in(const float* da, const float* lev, int lev_planar, long long i, long long n,
                                           long long pix, int c0, int C, long long P, float g[4]) {
  g[0] = g[1] = g[2] = g[3] = 0.f;
  if (da != nullptr) {
    const float4 t = ldg4(da + i);
    g[0] = t.x; g[1] = t.y; g[2] = t.z; g[3] = t.w;
  }
  if (lev != nullptr) {
    float l[4];
    if (lev_planar) {
      const float* q = lev + (n * C + c0) * P + pix;
#pragma unroll
      for (int j = 0; j < 4; ++j) l[j] = __ldg(q + j * P);
    } else {
      const float4 t = ldg4(lev + i);
      l[0] = t.x; l[1] = t.y; l[2] = t.z; l[3] = t.w;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) g[j] = da != nullptr ? g[j] + l[j] : l[j];
  }
}

struct IbBnArgs {
  const float* y;     // the kept pre-BatchNorm output [N, P, C]
  const float* da;    // the next layer's data gradient [N, P, C] or NULL
  const float* lev;   // the level gradient or NULL
  const float* ss;    // the kept scale [V][C], shift [V][C]
  const double* sums; // train: the forward's batch sums of this layer, view v at v * sums_stride
  const float* rs;    // eval: the kept running statistics [mean[C], var[C]]
  const float* k;     // apply: the per-view constants [V][4][C]
  float* G;           // apply: G (may be da: written in place)
  double* part;       // reduce: [V][2][C][B * nch]
  long long P, sums_stride;
  double count;
  int C, V, lev_planar, chunk, nch;
};

// Pass 1: per-CTA sums of dz and dz * (y - mean_v) over a chunk of pixels of one image, grid (nch, N).  Thread t
// handles channels 4 (t % C4) .. + 3 of every (IB_THREADS / C4)-th pixel; the CTA adds its threads in slot order.
__global__ void __launch_bounds__(IB_THREADS) ic_bnb_reduce_kernel(const IbBnArgs a) {
  __shared__ double red[IB_THREADS][8];
  const int n = blockIdx.y, v = n % a.V, C4 = a.C / 4, q = threadIdx.x % C4, slot = threadIdx.x / C4;
  const int slots = IB_THREADS / C4, c0 = 4 * q;
  float sc[4], sh[4];
  double mean[4], s[4], t[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    sc[j] = __ldg(a.ss + (long long)v * a.C + c0 + j);
    sh[j] = __ldg(a.ss + (long long)(a.V + v) * a.C + c0 + j);
    mean[j] = a.sums != nullptr ? a.sums[v * a.sums_stride + c0 + j] / a.count : (double)__ldg(a.rs + c0 + j);
    s[j] = t[j] = 0.0;
  }
  const long long p0 = (long long)blockIdx.x * a.chunk, p1 = min(a.P, p0 + a.chunk);
  for (long long pix = p0 + slot; pix < p1; pix += slots) {
    const long long i = ((long long)n * a.P + pix) * a.C + c0;
    float g[4];
    ib_grad_in(a.da, a.lev, a.lev_planar, i, n, pix, c0, a.C, a.P, g);
    const float4 y4 = ldg4(a.y + i);
    const float y[4] = {y4.x, y4.y, y4.z, y4.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float dz = __fmaf_rn(y[j], sc[j], sh[j]) > 0.f ? g[j] : 0.f;  // no gradient at exactly 0, as PyTorch's
      s[j] += (double)dz;
      t[j] += (double)dz * ((double)y[j] - mean[j]);
    }
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    red[threadIdx.x][j] = s[j];
    red[threadIdx.x][4 + j] = t[j];
  }
  __syncthreads();
  if (threadIdx.x < 2 * a.C) {
    const int stat = threadIdx.x / a.C, c = threadIdx.x % a.C;
    double r = 0.0;
    for (int k = 0; k < slots; ++k) r += red[k * C4 + c / 4][4 * stat + c % 4];
    const int b = n / a.V;
    const long long nparts = (long long)(gridDim.y / a.V) * a.nch;
    a.part[(((long long)v * 2 + stat) * a.C + c) * nparts + (long long)b * a.nch + blockIdx.x] = r;
  }
}

// One CTA per channel, the views in order: per view the batch statistics (train, from the forward's sums exactly as
// vc_bn_finalize_kernel recomputes them) or the kept running statistics (eval), and the constants of
// G = k1 dz + k2 (y - mean) + k3: train k1 = gamma invstd, k2 = -k1 invstd dgamma_v / n, k3 = -k1 dbeta_v / n; eval
// k1 = the forward's scale, k2 = k3 = 0.  dbeta = sum_v sum dz, dgamma = sum_v invstd_v sum dz (y - mean_v).
__global__ void __launch_bounds__(IB_THREADS)
    ic_bnb_finalize_kernel(const double* __restrict__ part, int nparts, int C, int V, double count,
                           const float* __restrict__ gamma, const double* __restrict__ sums, long long sums_stride,
                           const float* __restrict__ ss, const float* __restrict__ rs, float eps,
                           float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ k) {
  __shared__ double red[IB_THREADS];
  const int c = blockIdx.x;
  double dg_all = 0.0, db_all = 0.0;
  for (int v = 0; v < V; ++v) {
    const double* pv = part + (long long)v * 2 * C * nparts;
    double s = 0.0, t = 0.0;
    for (int i = threadIdx.x; i < nparts; i += IB_THREADS) {
      s += pv[(long long)c * nparts + i];
      t += pv[(long long)(C + c) * nparts + i];
    }
    s = block_sum<IB_THREADS>(s, red);
    t = block_sum<IB_THREADS>(t, red);
    if (threadIdx.x == 0) {
      double mean, var;
      if (sums != nullptr) {
        mean = sums[v * sums_stride + c] / count;
        var = fmax(sums[v * sums_stride + C + c] / count - mean * mean, 0.0);
      } else {
        mean = (double)rs[c];
        var = (double)rs[C + c];
      }
      const double invstd = 1.0 / sqrt(var + (double)eps);
      const double dg = t * invstd;
      float* kv = k + (long long)v * 4 * C;
      if (sums != nullptr) {
        const double k1 = (double)gamma[c] * invstd;
        kv[c] = (float)k1;
        kv[C + c] = (float)(-k1 * invstd * dg / count);
        kv[2 * C + c] = (float)(-k1 * s / count);
      } else {
        kv[c] = ss[(long long)v * C + c];
        kv[C + c] = 0.f;
        kv[2 * C + c] = 0.f;
      }
      kv[3 * C + c] = (float)mean;
      dg_all += dg;
      db_all += s;
    }
  }
  if (threadIdx.x == 0) {
    dgamma[c] = (float)dg_all;
    dbeta[c] = (float)db_all;
  }
}

// Pass 2: G = k1 dz + k2 (y - mean) + k3 with view v's constants, grid as ic_bnb_reduce_kernel's.
__global__ void __launch_bounds__(IB_THREADS) ic_bnb_apply_kernel(const IbBnArgs a) {
  const int n = blockIdx.y, v = n % a.V, C4 = a.C / 4, q = threadIdx.x % C4, slot = threadIdx.x / C4;
  const int slots = IB_THREADS / C4, c0 = 4 * q;
  const float* kv = a.k + (long long)v * 4 * a.C;
  float sc[4], sh[4], k1[4], k2[4], k3[4], mean[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    sc[j] = __ldg(a.ss + (long long)v * a.C + c0 + j);
    sh[j] = __ldg(a.ss + (long long)(a.V + v) * a.C + c0 + j);
    k1[j] = kv[c0 + j];
    k2[j] = kv[a.C + c0 + j];
    k3[j] = kv[2 * a.C + c0 + j];
    mean[j] = kv[3 * a.C + c0 + j];
  }
  const long long p0 = (long long)blockIdx.x * a.chunk, p1 = min(a.P, p0 + a.chunk);
  for (long long pix = p0 + slot; pix < p1; pix += slots) {
    const long long i = ((long long)n * a.P + pix) * a.C + c0;
    float g[4];
    ib_grad_in(a.da, a.lev, a.lev_planar, i, n, pix, c0, a.C, a.P, g);
    const float4 y4 = ldg4(a.y + i);
    const float y[4] = {y4.x, y4.y, y4.z, y4.w};
    float r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float dz = __fmaf_rn(y[j], sc[j], sh[j]) > 0.f ? g[j] : 0.f;
      r[j] = __fmaf_rn(k1[j], dz, __fmaf_rn(k2[j], __fsub_rn(y[j], mean[j]), k3[j]));
    }
    *reinterpret_cast<float4*>(a.G + i) = make_float4(r[0], r[1], r[2], r[3]);
  }
}

// the conv3 gradient [N, C, P] (the planar layout) -> NHWC [N, P, C]
__global__ void __launch_bounds__(256)
    ic_to_nhwc_kernel(const float* __restrict__ src, float* __restrict__ dst, int C, long long P, long long total) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const long long n = i / (P * C), r = i % (P * C), pix = r / C;
  const int c = (int)(r % C);
  dst[i] = __ldg(src + (n * C + c) * P + pix);
}

struct IcWgArgs {
  const float* x;   // the layer's forward input: the planar images (layer 0) or the producer's kept y, NHWC
  const float* ss;  // the producer's kept scale [V][Cin], shift [V][Cin]
  const float* g;   // G [N, Ho, Wo, Cout]
  double* part;     // [N * nch][Cout][Cin][K][K]
  int V, Hi, Wi, Ho, Wo;
  int nch;          // pixel chunks per image
  int chunk;        // output pixels per chunk
};

// dW[co][ci][kh][kw] = sum over (image, output pixel o) of G[o][co] act_in[S o - P + k][ci].  One CTA: one kernel row
// kh and four input channels (blockIdx.y = kh * CQ + quad), IW_CO output channels (group blockIdx.z) and one chunk of
// one image's output pixels (blockIdx.x = image * nch + chunk).  Each thread owns the K taps of the row x 4 x IW_CO
// products in fp32 over every IC_THREADS-th pixel of the chunk; the CTA then adds its threads in fp64 in a fixed order.
template <int K, int S, int CIN, int COUT>
__global__ void __launch_bounds__(IC_THREADS) ic_wgrad_kernel(const IcWgArgs a) {
  constexpr bool FIRST = CIN == 3;
  constexpr int CQ = FIRST ? 1 : CIN / 4, P = K / 2, E = COUT * CIN * K * K;
  const int n = blockIdx.x / a.nch, chunk = blockIdx.x % a.nch, v = n % a.V;
  const int kh = blockIdx.y / CQ, ci0 = 4 * (blockIdx.y % CQ), co0 = blockIdx.z * IW_CO;
  float sc[4] = {1.f, 1.f, 1.f, 1.f}, sh[4] = {0.f, 0.f, 0.f, 0.f};
  if (!FIRST) {
    const float4 s4 = ldg4(a.ss + (long long)v * CIN + ci0), h4 = ldg4(a.ss + (long long)(a.V + v) * CIN + ci0);
    sc[0] = s4.x; sc[1] = s4.y; sc[2] = s4.z; sc[3] = s4.w;
    sh[0] = h4.x; sh[1] = h4.y; sh[2] = h4.z; sh[3] = h4.w;
  }
  float acc[K][4][IW_CO];
#pragma unroll
  for (int kw = 0; kw < K; ++kw)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < IW_CO; ++c) acc[kw][j][c] = 0.f;

  const int Po = a.Ho * a.Wo;
  const int r0 = chunk * a.chunk, r1 = min(Po, r0 + a.chunk);
  const float* gn = a.g + (long long)n * Po * COUT + co0;
  for (int r = r0 + threadIdx.x; r < r1; r += IC_THREADS) {
    const int oh = r / a.Wo, ow = r - oh * a.Wo;
    const int ih = oh * S - P + kh;
    if (ih < 0 || ih >= a.Hi) continue;
    float g[IW_CO];
#pragma unroll
    for (int c = 0; c < IW_CO; c += 4) {
      const float4 t = ldg4(gn + (long long)r * COUT + c);
      g[c] = t.x; g[c + 1] = t.y; g[c + 2] = t.z; g[c + 3] = t.w;
    }
#pragma unroll
    for (int kw = 0; kw < K; ++kw) {
      const int iw = ow * S - P + kw;
      float x[4] = {0.f, 0.f, 0.f, 0.f};
      if (iw >= 0 && iw < a.Wi) {
        if (FIRST) {
#pragma unroll
          for (int j = 0; j < 3; ++j) x[j] = __ldg(a.x + (((long long)n * 3 + j) * a.Hi + ih) * a.Wi + iw);
        } else {
          const float4 t = ldg4(a.x + (((long long)n * a.Hi + ih) * a.Wi + iw) * CIN + ci0);
          x[0] = act(t.x, sc[0], sh[0]); x[1] = act(t.y, sc[1], sh[1]);
          x[2] = act(t.z, sc[2], sh[2]); x[3] = act(t.w, sc[3], sh[3]);
        }
      }
#pragma unroll
      for (int j = 0; j < 4; ++j)
#pragma unroll
        for (int c = 0; c < IW_CO; ++c) acc[kw][j][c] = __fmaf_rn(x[j], g[c], acc[kw][j][c]);
    }
  }

  // per tap: the 32 products of every thread through shared memory; 4 x 32 threads add 32 threads each in fp64, then
  // 32 threads add the four quarter sums in order
  __shared__ float red[4 * IW_CO][IC_THREADS + 1];
  __shared__ double red2[4][4 * IW_CO];
  double* part = a.part + (long long)blockIdx.x * E;
#pragma unroll
  for (int kw = 0; kw < K; ++kw) {
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int c = 0; c < IW_CO; ++c) red[j * IW_CO + c][threadIdx.x] = acc[kw][j][c];
    __syncthreads();
    {
      const int e = threadIdx.x & 31, qq = threadIdx.x >> 5;
      double s = 0.0;
#pragma unroll 8
      for (int i = 0; i < 32; ++i) s += (double)red[e][qq * 32 + i];
      red2[qq][e] = s;
    }
    __syncthreads();
    if (threadIdx.x < 4 * IW_CO) {
      const double s = ((red2[0][threadIdx.x] + red2[1][threadIdx.x]) + red2[2][threadIdx.x]) + red2[3][threadIdx.x];
      const int j = threadIdx.x / IW_CO, c = threadIdx.x % IW_CO;
      if (!FIRST || j < 3) part[(((long long)(co0 + c) * CIN + ci0 + j) * K + kh) * K + kw] = s;
    }
    __syncthreads();
  }
}

// dW in the PyTorch layout: the partials of the nparts chunks added in order
__global__ void ic_wgrad_finalize_kernel(const double* __restrict__ part, int nparts, int E, float* __restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= E) return;
  double s = 0.0;
  for (int k = 0; k < nparts; ++k) s += part[(long long)k * E + i];
  dw[i] = (float)s;
}

// ---- plan ---------------------------------------------------------------------------------------------------------

struct IbPlan {
  IcPlan f;                    // the forward's (keep) plan: the layout of fwd_workspace
  size_t wb[IC_LAYERS];        // packed data-gradient weights (layers 1 .. 10)
  size_t buf[2];               // ping-pong gradient buffers: dA_l, overwritten by G_l; the data gradient goes to the other
  size_t bn_part, kc, w_part, total;
  int bn_chunk[IC_BN], bn_nch[IC_BN];  // BatchNorm backward: pixels per CTA, CTAs per image
  int w_chunk[IC_LAYERS], w_nch[IC_LAYERS];  // weight gradients: output pixels per CTA, CTAs per image
};

int ib_plan(int B, int V, int H, int W, int base, IbPlan& p) {
  PMVS_TRY(ic_plan(B, V, H, W, base, 1, p.f));
  const long long N = (long long)B * V;
  size_t off = 0, bufmax = 0, bn_part = 0, w_part = 0;
  p.wb[0] = 0;
  for (int l = 1; l < IC_LAYERS; ++l) {
    const IcLayerPlan& q = p.f.L[l];
    const long long wn = (long long)q.k * q.k * q.cin * q.cout;
    p.wb[l] = off;
    off += up256(wn * 4);
  }
  for (int l = 0; l < IC_LAYERS; ++l) {
    const IcLayerPlan& q = p.f.L[l];
    const long long Po = (long long)q.Ho * q.Wo;
    bufmax = std::max(bufmax, (size_t)(N * Po * q.cout * 4));
    if (l < IC_BN) {
      p.bn_chunk[l] = std::max(1, IB_CHUNK / q.cout);
      p.bn_nch[l] = cdiv(Po, p.bn_chunk[l]);
      bn_part = std::max(bn_part, (size_t)V * 2 * q.cout * B * p.bn_nch[l] * 8);
    }
    const long long rows = (long long)q.k * (q.cin == 3 ? 1 : q.cin / 4) * (q.cout / IW_CO);
    const long long nch = std::max(1ll, std::min((long long)cdiv(IW_TARGET_CTAS, rows * N), (long long)cdiv(Po, IW_MIN_CHUNK)));
    p.w_chunk[l] = cdiv(Po, nch);
    p.w_nch[l] = cdiv(Po, p.w_chunk[l]);
    w_part = std::max(w_part, (size_t)q.k * q.k * q.cin * q.cout * (size_t)N * p.w_nch[l] * 8);
  }
  p.buf[0] = off;
  off += up256(bufmax);
  p.buf[1] = off;
  off += up256(bufmax);
  p.bn_part = off;
  off += up256(bn_part);
  p.kc = off;
  off += up256((size_t)V * 4 * IC_MAX_C * 4);
  p.w_part = off;
  off += up256(w_part);
  p.total = off;
  return PMVS_OK;
}

template <int K, int CIN, int COUT, int CO, int PX>
int launch_dgrad(const IcArgs& a, int N, const char* name, cudaStream_t st) {
  dim3 grid((unsigned)a.pix_blocks, (unsigned)(COUT / CO), (unsigned)N);
  prof_begin(name, st);
  ic_dgrad_kernel<K, CIN, COUT, CO, PX><<<grid, IC_THREADS, 0, st>>>(a);
  return check_launch(name, st);
}

template <int CIN, int COUT, int CO, int PX>
int launch_dgrad_s2(const IcArgs& a, int N, const char* name, cudaStream_t st) {
  dim3 grid((unsigned)a.pix_blocks, (unsigned)(COUT / CO), (unsigned)(4 * N));
  prof_begin(name, st);
  ic_dgrad_s2_kernel<CIN, COUT, CO, PX><<<grid, IC_THREADS, 0, st>>>(a);
  return check_launch(name, st);
}

// the data gradient of layer l (input G with the layer's Cout channels, output its Cin channels)
int ib_launch_data(int l, IcArgs& a, int N, cudaStream_t st) {
  const char* n = IB_DATA[l];
  const bool s2 = l == 2 || l == 5 || l == 8;
  const int px = l == 1 ? 8 : 4;
  a.ncg = cdiv(s2 ? (a.Wo + 1) / 2 : a.Wo, px);
  a.tpix = (s2 ? (a.Ho + 1) / 2 : a.Ho) * a.ncg;
  a.pix_blocks = cdiv(a.tpix, IC_THREADS);
  switch (l) {
    case 1: return launch_dgrad<3, 8, 8, 8, 8>(a, N, n, st);
    case 2: return launch_dgrad_s2<16, 8, 8, 4>(a, N, n, st);
    case 3: case 4: return launch_dgrad<3, 16, 16, 16, 4>(a, N, n, st);
    case 5: return launch_dgrad_s2<32, 16, 16, 4>(a, N, n, st);
    case 6: case 7: return launch_dgrad<3, 32, 32, 16, 4>(a, N, n, st);
    case 8: return launch_dgrad_s2<64, 32, 16, 4>(a, N, n, st);
    default: return launch_dgrad<3, 64, 64, 16, 4>(a, N, n, st);
  }
}

template <int K, int S, int CIN, int COUT>
int launch_wgrad(const IcWgArgs& a, int N, const char* name, cudaStream_t st) {
  dim3 grid((unsigned)(N * a.nch), (unsigned)(K * (CIN == 3 ? 1 : CIN / 4)), (unsigned)(COUT / IW_CO));
  prof_begin(name, st);
  ic_wgrad_kernel<K, S, CIN, COUT><<<grid, IC_THREADS, 0, st>>>(a);
  return check_launch(name, st);
}

int ib_launch_wgrad(int l, const IcWgArgs& a, int N, cudaStream_t st) {
  const char* n = IB_WGRAD[l];
  switch (l) {
    case 0: return launch_wgrad<3, 1, 3, 8>(a, N, n, st);
    case 1: return launch_wgrad<3, 1, 8, 8>(a, N, n, st);
    case 2: return launch_wgrad<5, 2, 8, 16>(a, N, n, st);
    case 3: case 4: return launch_wgrad<3, 1, 16, 16>(a, N, n, st);
    case 5: return launch_wgrad<5, 2, 16, 32>(a, N, n, st);
    case 6: case 7: return launch_wgrad<3, 1, 32, 32>(a, N, n, st);
    case 8: return launch_wgrad<5, 2, 32, 64>(a, N, n, st);
    default: return launch_wgrad<3, 1, 64, 64>(a, N, n, st);
  }
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_image_conv_backward_workspace_bytes(int B, int V, int H, int W, int base_channels) {
  IbPlan p;
  if (ib_plan(B, V, H, W, base_channels, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_image_conv_backward(const float* img, const pmvs_image_weights* wt, int train,
                                        const void* fwd_workspace, const double* batch_sums,
                                        const float* const* grad_level, int channels_last,
                                        const pmvs_image_grads* grads, void* workspace, size_t workspace_bytes, int B,
                                        int V, int H, int W, int base_channels, pmvs_stream_t stream) {
  PMVS_REQUIRE(img && wt && fwd_workspace && grad_level && grads && workspace,
               "image_conv_backward: NULL pointer");
  IbPlan p;
  PMVS_TRY(ib_plan(B, V, H, W, base_channels, p));
  for (int l = 0; l < IC_LAYERS; ++l) {
    PMVS_REQUIRE(wt->weight[l], "image_conv_backward: NULL weight of layer %d", l);
    PMVS_REQUIRE(grads->weight[l], "image_conv_backward: NULL weight gradient of layer %d", l);
  }
  for (int l = 0; l < IC_BN; ++l) {
    PMVS_REQUIRE(wt->gamma[l] && wt->beta[l], "image_conv_backward: NULL BatchNorm affine of layer %d", l);
    PMVS_REQUIRE(grads->gamma[l] && grads->beta[l], "image_conv_backward: NULL BatchNorm gradient of layer %d", l);
    PMVS_REQUIRE(finite_nonneg(wt->eps[l]), "image_conv_backward: eps of layer %d = %g (finite, >= 0)", l,
                 (double)wt->eps[l]);
  }
  PMVS_REQUIRE(!train || (long long)B * p.f.h[3] * p.f.w[3] >= 2,
               "image_conv_backward: train mode needs more than 1 value per channel at the coarsest level "
               "(B*h3*w3 = %lld)", (long long)B * p.f.h[3] * p.f.w[3]);
  PMVS_REQUIRE(!train || batch_sums, "image_conv_backward: train mode needs the forward's batch_sums");
  PMVS_REQUIRE(((uintptr_t)fwd_workspace & 255) == 0, "image_conv_backward: fwd_workspace must be 256-byte aligned");
  for (int k = 0; k < 4; ++k)
    PMVS_REQUIRE(((uintptr_t)grad_level[k] & 15) == 0, "image_conv_backward: grad_level[%d] must be 16-byte aligned",
                 k);
  PMVS_TRY(check_workspace("image_conv_backward", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  const char* fw = (const char*)fwd_workspace;
  char* ws = (char*)workspace;
  const IcLayerPlan* F = p.f.L;
  const int N = B * V;

  // the deepest layer a given level depends on; the layers above it get zeros and no kernels
  int top = -1;
  for (int k = 0; k < 4; ++k)
    if (grad_level[k] != nullptr) top = IC_LEVEL_LAYER[k];
  for (int l = top + 1; l < IC_LAYERS; ++l) {
    const IcLayerPlan& q = F[l];
    const char* what = "image_conv_backward";
    PMVS_TRY(memset_async(what, grads->weight[l], (size_t)q.k * q.k * q.cin * q.cout * sizeof(float), st));
    if (l < IC_BN) {
      PMVS_TRY(memset_async(what, grads->gamma[l], q.cout * sizeof(float), st));
      PMVS_TRY(memset_async(what, grads->beta[l], q.cout * sizeof(float), st));
    }
  }
  if (top < 0) return PMVS_OK;

  if (top >= 1) {
    // PyTorch Conv2d weights [Cout, Cin, K, K] -> [K*K][Cout][Cin], the packing of the data-gradient convolutions
    // (input G with Cout channels, output Cin channels) of layers 1 .. top; stride-1 layers with the taps flipped
    // (tap -> K*K - 1 - tap)
    PackTable pk;
    for (int l = 1; l <= top; ++l) {
      const IcLayerPlan& q = F[l];
      const int taps = q.k * q.k, flip = q.s == 1;
      pk.L[l - 1] = {wt->weight[l], (long long)(p.wb[l] / 4), {taps, q.cout, q.cin}, flip ? taps - 1 : 0,
                     {flip ? -1 : 1, q.cin * taps, taps}};
    }
    PMVS_TRY(launch_pack(pk, top, (float*)ws, "icb_pack", st));
  }

  size_t sums_at[IC_BN], sums_stride = 0;
  for (int l = 0; l < IC_BN; ++l) {
    sums_at[l] = sums_stride;
    sums_stride += 2 * (size_t)F[l].cout;
  }
  float* X = (float*)(ws + p.buf[0]);  // dA_l, then G_l in place
  float* Y = (float*)(ws + p.buf[1]);  // the data gradient dA_(l-1)
  double* bn_part = (double*)(ws + p.bn_part);
  double* w_part = (double*)(ws + p.w_part);
  float* kc = (float*)(ws + p.kc);

  for (int l = top; l >= 0; --l) {
    const IcLayerPlan& q = F[l];
    const long long Po = (long long)q.Ho * q.Wo;
    const float* G;
    if (l == IC_LAYERS - 1) {
      if (channels_last) {
        G = grad_level[3];
      } else {
        const long long total = (long long)N * Po * q.cout;
        prof_begin("icb_to_nhwc", st);
        ic_to_nhwc_kernel<<<cdiv(total, 256), 256, 0, st>>>(grad_level[3], X, q.cout, Po, total);
        PMVS_TRY(check_launch("ic_to_nhwc_kernel", st));
        G = X;
      }
    } else {
      IbBnArgs a;
      memset(&a, 0, sizeof(a));
      a.y = (const float*)(fw + p.f.y[l]);
      a.da = l < top ? X : nullptr;
      for (int k = 0; k < 3; ++k)
        if (IC_LEVEL_LAYER[k] == l) a.lev = grad_level[k];
      a.lev_planar = !channels_last;
      a.ss = (const float*)(fw + p.f.ss[l]);
      a.sums = train ? batch_sums + sums_at[l] : nullptr;
      a.rs = train ? nullptr : (const float*)(fw + p.f.rs) + p.f.rs_at[l];
      a.k = kc;
      a.G = X;
      a.part = bn_part;
      a.P = Po;
      a.sums_stride = (long long)sums_stride;
      a.count = (double)B * Po;
      a.C = q.cout;
      a.V = V;
      a.chunk = p.bn_chunk[l];
      a.nch = p.bn_nch[l];
      dim3 grid((unsigned)a.nch, (unsigned)N);
      prof_begin("icb_bn_reduce", st);
      ic_bnb_reduce_kernel<<<grid, IB_THREADS, 0, st>>>(a);
      PMVS_TRY(check_launch("ic_bnb_reduce_kernel", st));
      prof_begin("icb_bn_finalize", st);
      ic_bnb_finalize_kernel<<<q.cout, IB_THREADS, 0, st>>>(bn_part, B * a.nch, q.cout, V, a.count, wt->gamma[l],
                                                            a.sums, (long long)sums_stride, a.ss, a.rs, wt->eps[l],
                                                            grads->gamma[l], grads->beta[l], kc);
      PMVS_TRY(check_launch("ic_bnb_finalize_kernel", st));
      prof_begin("icb_bn_apply", st);
      ic_bnb_apply_kernel<<<grid, IB_THREADS, 0, st>>>(a);
      PMVS_TRY(check_launch("ic_bnb_apply_kernel", st));
      G = X;
    }

    // the weight gradient: the layer's input recomputed as the forward's prologue reads it
    IcWgArgs wa;
    memset(&wa, 0, sizeof(wa));
    wa.x = l == 0 ? img : (const float*)(fw + p.f.y[l - 1]);
    wa.ss = l == 0 ? nullptr : (const float*)(fw + p.f.ss[l - 1]);
    wa.g = G;
    wa.part = w_part;
    wa.V = V;
    wa.Hi = q.Hi; wa.Wi = q.Wi; wa.Ho = q.Ho; wa.Wo = q.Wo;
    wa.nch = p.w_nch[l];
    wa.chunk = p.w_chunk[l];
    PMVS_TRY(ib_launch_wgrad(l, wa, N, st));
    const int E = q.k * q.k * q.cin * q.cout;
    prof_begin("icb_wgrad_finalize", st);
    ic_wgrad_finalize_kernel<<<cdiv(E, 256), 256, 0, st>>>(w_part, N * wa.nch, E, grads->weight[l]);
    PMVS_TRY(check_launch("ic_wgrad_finalize_kernel", st));

    if (l == 0) break;  // the images get no gradient
    IcArgs a;
    memset(&a, 0, sizeof(a));
    a.x = G;
    a.w = (const float*)(ws + p.wb[l]);
    a.y = Y;
    a.V = V;
    a.Hi = q.Ho; a.Wi = q.Wo; a.Ho = q.Hi; a.Wo = q.Wi;
    PMVS_TRY(ib_launch_data(l, a, N, st));
    std::swap(X, Y);
  }
  return PMVS_OK;
}
