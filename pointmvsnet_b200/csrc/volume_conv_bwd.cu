// Backward of VolumeConv and of the coarse depth regression, include/pmvs_b200.h, DESIGN 3.13.
//
// The layers are walked in reverse dependency order (conv6_2 back to conv0_1 / conv1_0).  For each layer l:
//   - BatchNorm + ReLU backward, once the gradient dA_l of its activation is complete (the sum, in a fixed order, of
//     its consumers' data gradients): dz = dA * [y * scale + shift > 0] with the forward's own scale / shift, per-CTA
//     fp64 sums of dz and dz * (y - mean) (vc_bnb_reduce_kernel), one finalize per channel (dbeta, dgamma and the
//     constants of G), then G_l, the gradient of the pre-BatchNorm output, materialised (vc_bnb_apply_kernel);
//   - the weight gradient (vc_wgrad_kernel): per-CTA sums over fixed voxel chunks of act_in * G_l, the input activation
//     recomputed with the forward's prologue, then a fixed-order reduction into the PyTorch layout;
//   - the data gradient: one vconv_kernel launch on G_l.  A stride-1 layer's is the same convolution with the taps of
//     all three axes flipped, a stride-2 Conv3d's is the forward's transposed (VC_T2) formula, and a transposed
//     layer's is the stride-2 (VC_S2) formula, each with the roles of Cin and Cout swapped.
// No floating-point atomics: every sum has an order fixed by the shapes, so two calls give the same bits.
#include <float.h>
#include <math.h>

#include <algorithm>

#include "volume_conv.cuh"

namespace pmvs {

namespace {

constexpr int VB_THREADS = 256, VB_CHUNK = 4096;  // BatchNorm backward: VB_CHUNK values of one (b, c) plane per CTA
constexpr int VW_TARGET_CTAS = 4224;               // weight gradients: 32 CTAs per SM of an H100 before splitting less

const char* const VB_DATA[VC_LAYERS] = {"vcb_data0_1", "vcb_data1_0", "vcb_data2_0", "vcb_data3_0",
                                        "vcb_data1_1", "vcb_data2_1", "vcb_data3_1", "vcb_data4_0",
                                        "vcb_data5_0", "vcb_data6_0", "vcb_data6_2"};
const char* const VB_WGRAD[VC_LAYERS] = {"vcb_wgrad0_1", "vcb_wgrad1_0", "vcb_wgrad2_0", "vcb_wgrad3_0",
                                         "vcb_wgrad1_1", "vcb_wgrad2_1", "vcb_wgrad3_1", "vcb_wgrad4_0",
                                         "vcb_wgrad5_0", "vcb_wgrad6_0", "vcb_wgrad6_2"};
// reverse dependency order of the forward
const int VB_ORDER[VC_LAYERS] = {L6_2, L6_0, L5_0, L4_0, L3_1, L3_0, L2_1, L2_0, L1_1, L1_0, L0_1};

__device__ __forceinline__ float relu_grad(float y, float sc, float sh, const float* da, const float* db, long long i) {
  float g = __ldg(da + i);
  if (db != nullptr) g += __ldg(db + i);  // two consumers: their data gradients added in a fixed order
  return __fmaf_rn(y, sc, sh) > 0.f ? g : 0.f;  // ReLU passes no gradient at exactly 0, as PyTorch's
}

// Pass 1 of the BatchNorm + ReLU backward: per-CTA sums of dz and dz * (y - mean) over VB_CHUNK values of one (b, c)
// plane, grid (chunks, C, B); part [2][C][B * chunks].
__global__ void __launch_bounds__(VB_THREADS)
    vc_bnb_reduce_kernel(const float* __restrict__ y, const float* __restrict__ da, const float* __restrict__ db,
                         const float* __restrict__ ss, const double* __restrict__ sums,
                         const float* __restrict__ rmean, double count, int C, long long V,
                         double* __restrict__ part) {
  __shared__ double red[VB_THREADS];
  const int c = blockIdx.y, b = blockIdx.z;
  const float sc = __ldg(ss + c), sh = __ldg(ss + C + c);
  const double mean = sums != nullptr ? sums[c] / count : (double)rmean[c];
  const long long base = ((long long)b * C + c) * V;
  const long long e0 = (long long)blockIdx.x * VB_CHUNK, e1 = min(V, e0 + VB_CHUNK);
  double s = 0.0, t = 0.0;
  for (long long e = e0 + threadIdx.x; e < e1; e += VB_THREADS) {
    const float yv = __ldg(y + base + e);
    const float dz = relu_grad(yv, sc, sh, da, db, base + e);
    s += (double)dz;
    t += (double)dz * ((double)yv - mean);
  }
  const long long nparts = (long long)gridDim.x * gridDim.z, at = (long long)b * gridDim.x + blockIdx.x;
  s = block_sum<VB_THREADS>(s, red);
  if (threadIdx.x == 0) part[(long long)c * nparts + at] = s;
  t = block_sum<VB_THREADS>(t, red);
  if (threadIdx.x == 0) part[(long long)(C + c) * nparts + at] = t;
}

// One CTA per channel: dbeta = sum dz, dgamma = sum dz * xhat (partials added in a fixed order), and the constants of
// G = k1 * dz + k2 * (y - mean) + k3.  Train mode (n values, batch statistics):
// G = gamma * invstd * (dz - dbeta / n - xhat * dgamma / n); eval mode (running statistics): G = gamma * invstd * dz.
__global__ void __launch_bounds__(VB_THREADS)
    vc_bnb_finalize_kernel(const double* __restrict__ part, int nparts, int C, double count,
                           const float* __restrict__ gamma, const double* __restrict__ sums,
                           const float* __restrict__ rmean, const float* __restrict__ rvar, float eps,
                           float* __restrict__ dgamma, float* __restrict__ dbeta, float* __restrict__ k) {
  __shared__ double red[VB_THREADS];
  const int c = blockIdx.x;
  double s = 0.0, t = 0.0;
  for (int i = threadIdx.x; i < nparts; i += VB_THREADS) {
    s += part[(long long)c * nparts + i];
    t += part[(long long)(C + c) * nparts + i];
  }
  s = block_sum<VB_THREADS>(s, red);
  t = block_sum<VB_THREADS>(t, red);
  if (threadIdx.x != 0) return;
  double mean, var;
  if (sums != nullptr) {  // the forward's statistics, recomputed from its sums exactly as vc_bn_finalize_kernel does
    mean = sums[c] / count;
    var = fmax(sums[C + c] / count - mean * mean, 0.0);
  } else {
    mean = (double)rmean[c];
    var = (double)rvar[c];
  }
  const double invstd = 1.0 / sqrt(var + (double)eps);
  const double dg = t * invstd;
  const double k1 = (double)gamma[c] * invstd;
  dbeta[c] = (float)s;
  dgamma[c] = (float)dg;
  k[c] = (float)k1;
  k[C + c] = sums != nullptr ? (float)(-k1 * invstd * dg / count) : 0.f;
  k[2 * C + c] = sums != nullptr ? (float)(-k1 * s / count) : 0.f;
  k[3 * C + c] = (float)mean;
}

// Pass 2: G = k1 * dz + k2 * (y - mean) + k3, grid as vc_bnb_reduce_kernel's.
__global__ void __launch_bounds__(VB_THREADS)
    vc_bnb_apply_kernel(const float* __restrict__ y, const float* __restrict__ da, const float* __restrict__ db,
                        const float* __restrict__ ss, const float* __restrict__ k, int C, long long V,
                        float* __restrict__ G) {
  const int c = blockIdx.y, b = blockIdx.z;
  const float sc = __ldg(ss + c), sh = __ldg(ss + C + c);
  const float k1 = __ldg(k + c), k2 = __ldg(k + C + c), k3 = __ldg(k + 2 * C + c), mean = __ldg(k + 3 * C + c);
  const long long base = ((long long)b * C + c) * V;
  const long long e0 = (long long)blockIdx.x * VB_CHUNK, e1 = min(V, e0 + VB_CHUNK);
  for (long long e = e0 + threadIdx.x; e < e1; e += VB_THREADS) {
    const float yv = __ldg(y + base + e);
    const float dz = relu_grad(yv, sc, sh, da, db, base + e);
    G[base + e] = __fmaf_rn(k1, dz, __fmaf_rn(k2, __fsub_rn(yv, mean), k3));
  }
}

struct VcWgArgs {
  const float* xa;  // the layer's forward input, read as vconv_kernel reads it (VcArgs)
  const float* sa;
  const float* ha;
  const float* xb;
  const float* sb;
  const float* hb;
  const float* g;   // G [B, Cout, Do, Ho, Wo]
  double* part;     // [Cin][27][Cout][B * nchb]
  int Cin, Cout, Di, Hi, Wi, Do, Ho, Wo;
  int Pd, Ph, Pw;   // the grid a thread walks: the output (S1, S2) or the input (T2) of one batch element
  int nchb;         // voxel chunks per batch element
  int chunk;        // voxels per chunk
};

// dW[ci][tap][co] = sum over (b, voxel) of act_in * G at the tap's offset: S1 x[o - 1 + k] G[o], S2 x[2o - 1 + k] G[o],
// T2 x[i] G[2i - 1 + k].  One CTA: one input channel ci, one kd (blockIdx.y = 3 ci + kd), CO output channels (group
// blockIdx.z) and one chunk of one batch element's voxels (blockIdx.x = b * nchb + chunk); each thread owns the 9 (kh,
// kw) taps x CO channels in fp32 over a strided subset of the chunk, then the CTA adds its threads in fp64 in index order.
template <int MODE, int CO, int SRC>
__global__ void __launch_bounds__(VC_THREADS) vc_wgrad_kernel(const VcWgArgs a) {
  const int b = blockIdx.x / a.nchb, chunk = blockIdx.x % a.nchb;
  const int ci = blockIdx.y / 3, kd = blockIdx.y % 3;
  const int co0 = blockIdx.z * CO;
  float sa = 1.f, ha = 0.f, sb = 1.f, hb = 0.f;
  if (SRC >= 1) { sa = __ldg(a.sa + ci); ha = __ldg(a.ha + ci); }
  if (SRC == 2) { sb = __ldg(a.sb + ci); hb = __ldg(a.hb + ci); }
  const int HWp = a.Ph * a.Pw, P = a.Pd * HWp;
  const long long HWi = (long long)a.Hi * a.Wi, HWo = (long long)a.Ho * a.Wo, DHWo = HWo * a.Do;
  const long long xbase = ((long long)b * a.Cin + ci) * a.Di * HWi;
  const float* gb = a.g + ((long long)b * a.Cout + co0) * DHWo;

  float acc[9][CO];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[t][c] = 0.f;

  const int r0 = chunk * a.chunk, r1 = min(P, r0 + a.chunk);
  for (int r = r0 + threadIdx.x; r < r1; r += VC_THREADS) {
    const int pd = r / HWp, rem = r - pd * HWp;
    const int ph = rem / a.Pw, pw = rem - ph * a.Pw;
    if (MODE != VC_T2) {
      constexpr int S = MODE == VC_S1 ? 1 : 2;
      const int id = S * pd - 1 + kd;
      if (id < 0 || id >= a.Di) continue;
      float g[CO];
#pragma unroll
      for (int c = 0; c < CO; ++c) g[c] = __ldg(gb + c * DHWo + (long long)r);
      const long long xd = xbase + (long long)id * HWi;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int ih = S * ph - 1 + kh;
        const bool okh = ih >= 0 && ih < a.Hi;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int iw = S * pw - 1 + kw;
          float x = 0.f;
          if (okh && iw >= 0 && iw < a.Wi) {
            const long long off = xd + (long long)ih * a.Wi + iw;
            x = __ldg(a.xa + off);
            if (SRC >= 1) x = act(x, sa, ha);
            if (SRC == 2) x += act(__ldg(a.xb + off), sb, hb);
          }
#pragma unroll
          for (int c = 0; c < CO; ++c) acc[kh * 3 + kw][c] = __fmaf_rn(x, g[c], acc[kh * 3 + kw][c]);
        }
      }
    } else {
      const int od = 2 * pd - 1 + kd;
      if (od < 0 || od >= a.Do) continue;
      const long long off = xbase + (long long)r;
      float x = __ldg(a.xa + off);
      if (SRC >= 1) x = act(x, sa, ha);
      if (SRC == 2) x += act(__ldg(a.xb + off), sb, hb);
      const float* gd = gb + (long long)od * HWo;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh) {
        const int oh = 2 * ph - 1 + kh;
        const bool okh = oh >= 0 && oh < a.Ho;
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) {
          const int ow = 2 * pw - 1 + kw;
          if (!okh || ow < 0 || ow >= a.Wo) continue;
#pragma unroll
          for (int c = 0; c < CO; ++c)
            acc[kh * 3 + kw][c] = __fmaf_rn(x, __ldg(gd + c * DHWo + (long long)oh * a.Wo + ow), acc[kh * 3 + kw][c]);
        }
      }
    }
  }

  __shared__ float red[9 * CO][VC_THREADS + 1];
#pragma unroll
  for (int t = 0; t < 9; ++t)
#pragma unroll
    for (int c = 0; c < CO; ++c) red[t * CO + c][threadIdx.x] = acc[t][c];
  __syncthreads();
  if (threadIdx.x < 9 * CO) {
    double s = 0.0;
    for (int i = 0; i < VC_THREADS; ++i) s += (double)red[threadIdx.x][i];
    const int t = threadIdx.x / CO, c = threadIdx.x % CO;
    const long long nparts = gridDim.x;
    a.part[(((long long)ci * VC_TAPS + kd * 9 + t) * a.Cout + co0 + c) * nparts + blockIdx.x] = s;
  }
}

// dW in the PyTorch layout from the partials: Conv3d [Cout, Cin, 27], ConvTranspose3d [Cin, Cout, 27]
__global__ void vc_wgrad_finalize_kernel(const double* __restrict__ part, int nparts, int Cin, int Cout, int transposed,
                                         float* __restrict__ dw) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Cin * VC_TAPS * Cout) return;
  const int co = i % Cout, tap = (i / Cout) % VC_TAPS, ci = i / (Cout * VC_TAPS);
  double s = 0.0;
  for (int k = 0; k < nparts; ++k) s += part[(long long)i * nparts + k];
  dw[transposed ? (ci * Cout + co) * VC_TAPS + tap : (co * Cin + ci) * VC_TAPS + tap] = (float)s;
}

__global__ void vc_add_kernel(float4* __restrict__ dst, const float4* __restrict__ src, long long n4) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
    float4 a = dst[i];
    const float4 b = src[i];
    a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    dst[i] = a;
  }
}

__global__ void __launch_bounds__(256)
    coarse_depth_backward_kernel(const float* __restrict__ vol, const float* __restrict__ cams,
                                 const float* __restrict__ gdepth, int B, int V, int D, int HW,
                                 float* __restrict__ gvol) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * HW) return;
  const int b = (int)(idx / HW), p = (int)(idx % HW);
  // the forward's planes, maximum, fp64 normaliser and expectation (coarse_depth_kernel), recomputed
  const float* cam = cams + (long long)b * V * 32 + 16 + 12;
  const float start = __ldg(cam), interval = __ldg(cam + 1);
  const float end = __fadd_rn(start, __fmul_rn((float)(D - 1), interval));
  const float step = D > 1 ? __fdiv_rn(__fsub_rn(end, start), (float)(D - 1)) : 0.f;
  const float* x = vol + (long long)b * D * HW + p;
  float m = -INFINITY;
  for (int d = 0; d < D; ++d) m = fmaxf(m, -__ldg(x + (long long)d * HW));
  double S = 0.0, acc = 0.0;
  for (int d = 0; d < D; ++d) {
    const double e = (double)expf(__fsub_rn(-__ldg(x + (long long)d * HW), m));
    S += e;
    acc += (double)linspace_at(start, end, step, D, d) * e;
  }
  const double depth = acc / S;
  const double g = (double)__ldg(gdepth + idx) / S;
  // d/dx_d of sum_k z_k softmax(-x)_k = p_d (depth - z_d)
  float* gx = gvol + (long long)b * D * HW + p;
  for (int d = 0; d < D; ++d) {
    const double e = (double)expf(__fsub_rn(-__ldg(x + (long long)d * HW), m));
    gx[(long long)d * HW] = (float)(g * e * (depth - (double)linspace_at(start, end, step, D, d)));
  }
}

// ---- plan ---------------------------------------------------------------------------------------------------------

struct VbLayer {
  size_t wb;                   // packed data-gradient weights [Cout][27][Cin]
  size_t G, k;                 // BatchNorm layers: G (the pre-BatchNorm output's gradient), the constants [4][Cout]
  size_t din;                  // the data gradient [B, Cin, Di, Hi, Wi] (not conv1_0's: it goes to grad_x)
  int bn_chunks;               // vc_bnb_* CTAs per (b, c) plane
  int pd, ph, pw, nchb, chunk, co;  // vc_wgrad_kernel
};

struct VbPlan {
  VcPlan f;
  VbLayer L[VC_LAYERS];
  size_t bn_part, w_part, total;
};

int vb_plan(int B, int Cin, int base, int D, int H, int W, VbPlan& p) {
  PMVS_TRY(vc_plan(B, Cin, base, D, H, W, p.f));
  size_t off = 0, bn_part = 0, w_part = 0;
  for (int l = 0; l < VC_LAYERS; ++l) {
    const VcLayerPlan& q = p.f.L[l];
    VbLayer& r = p.L[l];
    const long long wn = (long long)q.cin * VC_TAPS * q.cout;
    r.wb = off;
    off += up256(wn * 4);
    r.co = l == L6_2 ? 1 : 8;
    if (q.mode == VC_T2) { r.pd = q.Di; r.ph = q.Hi; r.pw = q.Wi; }
    else { r.pd = q.Do; r.ph = q.Ho; r.pw = q.Wo; }
    const long long P = (long long)r.pd * r.ph * r.pw;
    const long long rows = 3ll * q.cin * (q.cout / r.co);
    r.nchb = (int)std::max(1ll, std::min((long long)cdiv(VW_TARGET_CTAS, rows * B), (long long)cdiv(P, 1024)));
    r.chunk = cdiv(P, r.nchb);
    w_part = std::max(w_part, (size_t)wn * B * r.nchb * 8);
  }
  for (int l = 0; l < VC_LAYERS; ++l) {
    const VcLayerPlan& q = p.f.L[l];
    VbLayer& r = p.L[l];
    r.G = r.k = r.din = 0;
    r.bn_chunks = 0;
    if (l != L6_2) {
      const long long V = (long long)q.Do * q.Ho * q.Wo;
      r.G = off;
      off += up256((size_t)B * q.cout * V * 4);
      r.k = off;
      off += up256((size_t)4 * q.cout * 4);
      r.bn_chunks = cdiv(V, VB_CHUNK);
      bn_part = std::max(bn_part, (size_t)2 * q.cout * B * r.bn_chunks * 8);
    }
    if (l != L1_0) {
      r.din = off;
      off += up256((size_t)B * q.cin * q.Di * q.Hi * q.Wi * 4);
    }
  }
  p.bn_part = off;
  off += up256(bn_part);
  p.w_part = off;
  off += up256(w_part);
  p.total = off;
  return PMVS_OK;
}

template <int MODE, int CO, int VD>
int launch_data(const VcArgs& a, int B, const char* name, cudaStream_t st) {
  const int npar = MODE == VC_T2 ? 4 : 1;
  dim3 grid((unsigned)(a.pix_blocks * cdiv(a.Do, VD)), (unsigned)(a.Cout / CO), (unsigned)(B * npar));
  prof_begin(name, st);
  vconv_kernel<MODE, CO, VD, 0><<<grid, VC_THREADS, 0, st>>>(a);
  return check_launch(name, st);
}

// the data gradient of layer l: its forward's transpose, blocked per layer (DESIGN 3.13)
int launch_data_layer(int l, const VcArgs& a, int B, cudaStream_t st) {
  const char* n = VB_DATA[l];
  switch (l) {
    case L6_2: case L0_1: return launch_data<VC_S1, 8, 8>(a, B, n, st);
    case L6_0: return launch_data<VC_S2, 8, 4>(a, B, n, st);
    case L5_0: case L4_0: return launch_data<VC_S2, 4, 2>(a, B, n, st);
    case L3_1: case L2_1: return launch_data<VC_S1, 4, 2>(a, B, n, st);
    case L3_0: return launch_data<VC_T2, 4, 2>(a, B, n, st);
    case L1_1: return launch_data<VC_S1, 8, 4>(a, B, n, st);
    default: return launch_data<VC_T2, 8, 4>(a, B, n, st);  // L2_0, L1_0
  }
}

template <int MODE, int CO, int SRC>
int launch_wgrad(const VcWgArgs& a, int B, int Cin, int Cout, const char* name, cudaStream_t st) {
  dim3 grid((unsigned)(B * a.nchb), (unsigned)(3 * Cin), (unsigned)(Cout / CO));
  prof_begin(name, st);
  vc_wgrad_kernel<MODE, CO, SRC><<<grid, VC_THREADS, 0, st>>>(a);
  return check_launch(name, st);
}

int launch_wgrad_layer(int l, const VcWgArgs& a, int B, cudaStream_t st) {
  const char* n = VB_WGRAD[l];
  switch (l) {
    case L6_2: return launch_wgrad<VC_S1, 1, 2>(a, B, a.Cin, a.Cout, n, st);
    case L6_0: case L5_0: return launch_wgrad<VC_T2, 8, 2>(a, B, a.Cin, a.Cout, n, st);
    case L4_0: return launch_wgrad<VC_T2, 8, 1>(a, B, a.Cin, a.Cout, n, st);
    case L3_1: case L2_1: case L1_1: return launch_wgrad<VC_S1, 8, 1>(a, B, a.Cin, a.Cout, n, st);
    case L3_0: case L2_0: return launch_wgrad<VC_S2, 8, 1>(a, B, a.Cin, a.Cout, n, st);
    case L1_0: return launch_wgrad<VC_S2, 8, 0>(a, B, a.Cin, a.Cout, n, st);
    default: return launch_wgrad<VC_S1, 8, 0>(a, B, a.Cin, a.Cout, n, st);  // L0_1
  }
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_volume_conv_backward_workspace_bytes(int B, int in_channels, int base_channels, int D, int H,
                                                            int W) {
  VbPlan p;
  if (vb_plan(B, in_channels, base_channels, D, H, W, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_volume_conv_backward(const float* x, const pmvs_volume_weights* wt, int train,
                                         const void* fwd_workspace, const double* batch_sums, const float* grad_out,
                                         float* grad_x, const pmvs_volume_grads* grads, void* workspace,
                                         size_t workspace_bytes, int B, int in_channels, int base_channels, int D,
                                         int H, int W, pmvs_stream_t stream) {
  PMVS_REQUIRE(x && wt && fwd_workspace && grad_out && grads && workspace, "volume_conv_backward: NULL pointer");
  VbPlan p;
  PMVS_TRY(vb_plan(B, in_channels, base_channels, D, H, W, p));
  for (int l = 0; l < VC_LAYERS; ++l) {
    PMVS_REQUIRE(wt->weight[l], "volume_conv_backward: NULL weight of layer %d", l);
    PMVS_REQUIRE(grads->weight[l], "volume_conv_backward: NULL weight gradient of layer %d", l);
  }
  for (int l = 0; l < VC_BN; ++l) {
    PMVS_REQUIRE(wt->gamma[l] && wt->beta[l], "volume_conv_backward: NULL BatchNorm affine of layer %d", l);
    PMVS_REQUIRE(grads->gamma[l] && grads->beta[l], "volume_conv_backward: NULL BatchNorm gradient of layer %d", l);
    PMVS_REQUIRE(train || (wt->running_mean[l] && wt->running_var[l]),
                 "volume_conv_backward: eval mode needs the running statistics of layer %d", l);
    PMVS_REQUIRE(finite_nonneg(wt->eps[l]), "volume_conv_backward: eps of layer %d = %g (finite, >= 0)", l,
                 (double)wt->eps[l]);
  }
  PMVS_REQUIRE(!train || batch_sums, "volume_conv_backward: train mode needs the forward's batch_sums");
  PMVS_REQUIRE(((uintptr_t)fwd_workspace & 255) == 0, "volume_conv_backward: fwd_workspace must be 256-byte aligned");
  PMVS_TRY(check_workspace("volume_conv_backward", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  const char* fw = (const char*)fwd_workspace;
  char* ws = (char*)workspace;
  const VcLayerPlan* F = p.f.L;

  // PyTorch layouts -> [Cout][27][Cin], the packing of the data-gradient convolutions (input G, output Cin channels):
  // ConvTranspose3d [Cin, Cout, 27], Conv3d [Cout, Cin, 27], stride-1 layers with the taps of all three axes flipped
  // (tap -> 26 - tap)
  PackTable pk;
  for (int l = 0; l < VC_LAYERS; ++l) {
    const VcLayerPlan& q = F[l];
    const bool t = q.mode == VC_T2, s1 = q.mode == VC_S1;
    pk.L[l] = {wt->weight[l], (long long)(p.L[l].wb / 4), {q.cout, VC_TAPS, q.cin}, s1 ? VC_TAPS - 1 : 0,
               {t ? VC_TAPS : q.cin * VC_TAPS, s1 ? -1 : 1, t ? q.cout * VC_TAPS : VC_TAPS}};
  }
  PMVS_TRY(launch_pack(pk, VC_LAYERS, (float*)ws, "vcb_pack", st));

  size_t sums_at[VC_BN], sums_off = 0;
  for (int l = 0; l < VC_BN; ++l) {
    sums_at[l] = sums_off;
    sums_off += 2 * (size_t)F[l].cout;
  }
  double* bn_part = (double*)(ws + p.bn_part);
  double* w_part = (double*)(ws + p.w_part);
  float* tmp = (float*)(ws + p.L[L0_1].din);  // conv0_1's share of grad_x, added to conv1_0's at the end

  for (int k = 0; k < VC_LAYERS; ++k) {
    const int l = VB_ORDER[k];
    const VcLayerPlan& q = F[l];
    const VbLayer& r = p.L[l];
    const float* G = grad_out;
    if (l != L6_2) {
      // dA_l: the data gradients of l's consumers (all done: they come later in the forward), in layer order
      const float* dA[2] = {nullptr, nullptr};
      int n = 0;
      for (int c = 0; c < VC_LAYERS; ++c)
        if (VC_SRCA[c] == l || VC_SRCB[c] == l) dA[n++] = (const float*)(ws + p.L[c].din);
      const float* y = (const float*)(fw + q.y);
      const float* ss = (const float*)(fw + q.ss);
      const double* sums = train ? batch_sums + sums_at[l] : nullptr;
      const long long V = (long long)q.Do * q.Ho * q.Wo;
      const double count = (double)B * V;
      float* kc = (float*)(ws + r.k);
      float* Gl = (float*)(ws + r.G);
      dim3 grid((unsigned)r.bn_chunks, (unsigned)q.cout, (unsigned)B);
      prof_begin("vcb_bn_reduce", st);
      vc_bnb_reduce_kernel<<<grid, VB_THREADS, 0, st>>>(y, dA[0], dA[1], ss, sums, wt->running_mean[l], count, q.cout,
                                                        V, bn_part);
      PMVS_TRY(check_launch("vc_bnb_reduce_kernel", st));
      prof_begin("vcb_bn_finalize", st);
      vc_bnb_finalize_kernel<<<q.cout, VB_THREADS, 0, st>>>(bn_part, B * r.bn_chunks, q.cout, count, wt->gamma[l],
                                                            sums, wt->running_mean[l], wt->running_var[l], wt->eps[l],
                                                            grads->gamma[l], grads->beta[l], kc);
      PMVS_TRY(check_launch("vc_bnb_finalize_kernel", st));
      prof_begin("vcb_bn_apply", st);
      vc_bnb_apply_kernel<<<grid, VB_THREADS, 0, st>>>(y, dA[0], dA[1], ss, kc, q.cout, V, Gl);
      PMVS_TRY(check_launch("vc_bnb_apply_kernel", st));
      G = Gl;
    }

    // the weight gradient: the layer's input recomputed as the forward's prologue reads it
    VcWgArgs wa;
    memset(&wa, 0, sizeof(wa));
    if (VC_SRCA[l] < 0) {
      wa.xa = x;
    } else {
      const VcLayerPlan& s = F[VC_SRCA[l]];
      wa.xa = (const float*)(fw + s.y);
      wa.sa = (const float*)(fw + s.ss);
      wa.ha = wa.sa + s.cout;
    }
    if (VC_SRCB[l] >= 0) {
      const VcLayerPlan& s = F[VC_SRCB[l]];
      wa.xb = (const float*)(fw + s.y);
      wa.sb = (const float*)(fw + s.ss);
      wa.hb = wa.sb + s.cout;
    }
    wa.g = G;
    wa.part = w_part;
    wa.Cin = q.cin; wa.Cout = q.cout;
    wa.Di = q.Di; wa.Hi = q.Hi; wa.Wi = q.Wi; wa.Do = q.Do; wa.Ho = q.Ho; wa.Wo = q.Wo;
    wa.Pd = r.pd; wa.Ph = r.ph; wa.Pw = r.pw;
    wa.nchb = r.nchb;
    wa.chunk = r.chunk;
    PMVS_TRY(launch_wgrad_layer(l, wa, B, st));
    const int wn = q.cin * VC_TAPS * q.cout;
    prof_begin("vcb_wgrad_finalize", st);
    vc_wgrad_finalize_kernel<<<cdiv(wn, 256), 256, 0, st>>>(w_part, B * r.nchb, q.cin, q.cout, q.mode == VC_T2,
                                                            grads->weight[l]);
    PMVS_TRY(check_launch("vc_wgrad_finalize_kernel", st));

    // the data gradient; conv1_0's and conv0_1's are grad_x's two terms
    if ((l == L1_0 || l == L0_1) && grad_x == nullptr) continue;
    VcArgs a;
    memset(&a, 0, sizeof(a));
    const int mode = q.mode == VC_S1 ? VC_S1 : (q.mode == VC_S2 ? VC_T2 : VC_S2);
    a.xa = G;
    a.w = (const float*)(ws + r.wb);
    a.y = l == L1_0 ? grad_x : (float*)(ws + r.din);
    a.part = nullptr;
    a.Cin = q.cout; a.Cout = q.cin;
    a.Di = q.Do; a.Hi = q.Ho; a.Wi = q.Wo; a.Do = q.Di; a.Ho = q.Hi; a.Wo = q.Wi;
    a.tw = mode == VC_T2 ? a.Wi : a.Wo;
    a.tpix = mode == VC_T2 ? a.Hi * a.Wi : a.Ho * a.Wo;
    a.pix_blocks = cdiv(a.tpix, VC_THREADS);
    PMVS_TRY(launch_data_layer(l, a, B, st));
  }
  if (grad_x != nullptr) {
    const long long n4 = (long long)B * F[L0_1].cin * F[L0_1].Di * F[L0_1].Hi * F[L0_1].Wi / 4;
    prof_begin("vcb_add", st);
    vc_add_kernel<<<(unsigned)std::min<long long>(cdiv(n4, 256), 8 * sm_count()), 256, 0, st>>>(
        (float4*)grad_x, (const float4*)tmp, n4);
    PMVS_TRY(check_launch("vc_add_kernel", st));
  }
  return PMVS_OK;
}

extern "C" int pmvs_coarse_depth_backward(const float* filtered, const float* cams, const float* grad_depth,
                                          float* grad_filtered, int B, int V, int D, int H, int W,
                                          pmvs_stream_t stream) {
  PMVS_REQUIRE(filtered && cams && grad_depth && grad_filtered, "coarse_depth_backward: NULL pointer");
  PMVS_REQUIRE(B >= 1 && V >= 1 && D >= 1 && H >= 1 && W >= 1,
               "coarse_depth_backward: bad shape B=%d V=%d D=%d H=%d W=%d", B, V, D, H, W);
  PMVS_REQUIRE((long long)B * D * H * W < (1ll << 40) && (long long)H * W < (1ll << 31),
               "coarse_depth_backward: volume too large");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * H * W;
  prof_begin("coarse_depth_backward", st);
  coarse_depth_backward_kernel<<<cdiv(n, 256), 256, 0, st>>>(filtered, cams, grad_depth, B, V, D, H * W,
                                                             grad_filtered);
  return check_launch("coarse_depth_backward_kernel", st);
}
