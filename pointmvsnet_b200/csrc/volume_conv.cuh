// The forward plan of VolumeConv (workspace layout, per-layer blocking) and its register-blocked direct convolution,
// shared by the forward (volume_conv.cu) and the backward (volume_conv_bwd.cu), so that one place knows the layout
// of the forward's workspace the backward reads.  DESIGN 3.12, 3.13.
#pragma once

#include <math.h>

#include "common.cuh"

namespace pmvs {

namespace {

constexpr int VC_LAYERS = 11, VC_BN = 10, VC_THREADS = 128, VC_TAPS = 27, VC_FIN_THREADS = 256;
enum { VC_S1 = 0, VC_S2 = 1, VC_T2 = 2 };  // Conv3d stride 1, Conv3d stride 2, ConvTranspose3d stride 2 (all 3^3, p1)

// the layers in the struct order of pmvs_volume_weights (the reference's attribute order)
enum { L0_1 = 0, L1_0, L2_0, L3_0, L1_1, L2_1, L3_1, L4_0, L5_0, L6_0, L6_2 };
// what each layer reads: act(source a) [+ act(source b)]; -1 is the U-Net's input x (a) or nothing (b)
const int VC_SRCA[VC_LAYERS] = {-1, -1, L1_0, L2_0, L1_0, L2_0, L3_0, L3_1, L4_0, L5_0, L6_0};
const int VC_SRCB[VC_LAYERS] = {-1, -1, -1, -1, -1, -1, -1, -1, L2_1, L1_1, L0_1};

struct VcArgs {
  const float* xa;  // source a [B, Cin, Di, Hi, Wi]
  const float* sa;  // its producer's BatchNorm as scale / shift per channel (SRC >= 1)
  const float* ha;
  const float* xb;  // source b (SRC == 2): the layer reads act(a) + act(b)
  const float* sb;
  const float* hb;
  const float* w;   // packed weights [Cin][27][Cout]
  float* y;         // [B, Cout, Do, Ho, Wo], before BatchNorm
  double* part;     // [2][Cout][nparts] per-CTA sums and sums of squares, or NULL
  int Cin, Cout, Di, Hi, Wi, Do, Ho, Wo;
  int tw;           // pixels per row of the thread grid: Wo (S1, S2) or Wi (T2, one output parity class per CTA)
  int tpix;         // pixels of the thread grid
  int pix_blocks;   // cdiv(tpix, VC_THREADS)
};

__device__ __forceinline__ float act(float x, float s, float h) { return fmaxf(__fmaf_rn(x, s, h), 0.f); }

// One CTA: VC_THREADS consecutive thread-grid pixels x VD output planes x CO output channels (group blockIdx.y) of
// one batch element (and, for T2, one (h, w) parity class), blockIdx.z = b * (T2 ? 4 : 1) + parity.
template <int MODE, int CO, int VD, int SRC>
__global__ void __launch_bounds__(VC_THREADS) vconv_kernel(const VcArgs a) {
  constexpr int NIN = MODE == VC_S1 ? VD + 2 : (MODE == VC_S2 ? 2 * VD + 1 : VD / 2 + 1);
  static_assert(MODE != VC_T2 || VD % 2 == 0, "transposed layers need an even VD (compile-time output parity)");
  constexpr int NPAR = MODE == VC_T2 ? 4 : 1;
  // small blockings keep two input channels in flight, so one's loads overlap the other's FMAs; conv0_1's 64
  // accumulators leave no registers for that
  constexpr int CI_UNROLL = CO * VD > 32 ? 1 : 2;
  const int pb = blockIdx.x % a.pix_blocks, td = blockIdx.x / a.pix_blocks;
  const int g = blockIdx.y;
  const int b = blockIdx.z / NPAR, par = blockIdx.z % NPAR;
  const int ph = par >> 1, pw = par & 1;
  const int tp = pb * VC_THREADS + threadIdx.x;
  const bool live = tp < a.tpix;
  const int th = live ? tp / a.tw : 0, tw = live ? tp % a.tw : 0;
  const int oh = MODE == VC_T2 ? 2 * th + ph : th, ow = MODE == VC_T2 ? 2 * tw + pw : tw;
  const int od0 = td * VD;
  const int id0 = MODE == VC_S1 ? od0 - 1 : (MODE == VC_S2 ? 2 * od0 - 1 : od0 / 2);
  unsigned dmask = 0;
#pragma unroll
  for (int j = 0; j < NIN; ++j)
    if (id0 + j >= 0 && id0 + j < a.Di) dmask |= 1u << j;
  const long long HWi = (long long)a.Hi * a.Wi, DHWi = HWi * a.Di;

  float acc[VD][CO];
#pragma unroll
  for (int v = 0; v < VD; ++v)
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[v][c] = 0.f;

#pragma unroll CI_UNROLL
  for (int ci = 0; ci < a.Cin; ++ci) {
    float sa = 1.f, ha = 0.f, sb = 1.f, hb = 0.f;
    if (SRC >= 1) { sa = __ldg(a.sa + ci); ha = __ldg(a.ha + ci); }
    if (SRC == 2) { sb = __ldg(a.sb + ci); hb = __ldg(a.hb + ci); }
    const long long cbase = ((long long)b * a.Cin + ci) * DHWi + (long long)id0 * HWi;
    const float* wci = a.w + (size_t)ci * VC_TAPS * a.Cout + g * CO;
#pragma unroll
    for (int kh = 0; kh < 3; ++kh) {
      int ih;
      if (MODE == VC_S1) ih = oh - 1 + kh;
      else if (MODE == VC_S2) ih = 2 * oh - 1 + kh;
      else {
        if ((ph + 1 - kh) & 1) continue;  // out[o] = sum over 2i - 1 + k = o: uniform per CTA
        ih = th + (ph + 1 - kh) / 2;
      }
      const bool okh = live && ih >= 0 && ih < a.Hi;
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        int iw;
        if (MODE == VC_S1) iw = ow - 1 + kw;
        else if (MODE == VC_S2) iw = 2 * ow - 1 + kw;
        else {
          if ((pw + 1 - kw) & 1) continue;
          iw = tw + (pw + 1 - kw) / 2;
        }
        const bool ok = okh && iw >= 0 && iw < a.Wi;
        const long long off = cbase + (long long)ih * a.Wi + iw;
        float xin[NIN];
#pragma unroll
        for (int j = 0; j < NIN; ++j) {
          float x = 0.f;
          if (ok && ((dmask >> j) & 1u)) {
            x = __ldg(a.xa + off + j * HWi);
            if (SRC >= 1) x = act(x, sa, ha);
            if (SRC == 2) x += act(__ldg(a.xb + off + j * HWi), sb, hb);
          }
          xin[j] = x;
        }
#pragma unroll
        for (int kd = 0; kd < 3; ++kd) {
          const float* wp = wci + (kd * 9 + kh * 3 + kw) * a.Cout;
          float wv[CO];
          if (CO % 4 == 0) {
#pragma unroll
            for (int c = 0; c < CO; c += 4) {
              const float4 t = ldg4(wp + c);
              wv[c] = t.x; wv[c + 1] = t.y; wv[c + 2] = t.z; wv[c + 3] = t.w;
            }
          } else {
#pragma unroll
            for (int c = 0; c < CO; ++c) wv[c] = __ldg(wp + c);
          }
#pragma unroll
          for (int v = 0; v < VD; ++v) {
            int j;
            if (MODE == VC_S1) j = v + kd;
            else if (MODE == VC_S2) j = 2 * v + kd;
            else {
              if ((v + 1 - kd) & 1 || v + 1 - kd < 0) continue;  // od0 is even: parity known at compile time
              j = (v + 1 - kd) / 2;
            }
#pragma unroll
            for (int c = 0; c < CO; ++c) acc[v][c] = __fmaf_rn(xin[j], wv[c], acc[v][c]);
          }
        }
      }
    }
  }

  // epilogue: store, then this CTA's per-channel sums in a fixed order (lanes by butterfly, warps in index order)
  const long long HWo = (long long)a.Ho * a.Wo;
  double s[CO], q[CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) {
    s[c] = 0.0;
    q[c] = 0.0;
    float* yc = a.y + ((long long)b * a.Cout + g * CO + c) * a.Do * HWo + (long long)oh * a.Wo + ow;
#pragma unroll
    for (int v = 0; v < VD; ++v) {
      if (live && od0 + v < a.Do) {
        const float r = acc[v][c];
        yc[(long long)(od0 + v) * HWo] = r;
        s[c] += (double)r;
        q[c] += (double)r * (double)r;
      }
    }
  }
  if (a.part == nullptr) return;
  __shared__ double red[VC_THREADS / 32][2 * CO];
#pragma unroll
  for (int c = 0; c < CO; ++c) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s[c] += __shfl_xor_sync(0xffffffffu, s[c], o);
      q[c] += __shfl_xor_sync(0xffffffffu, q[c], o);
    }
  }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (lane == 0) {
#pragma unroll
    for (int c = 0; c < CO; ++c) {
      red[warp][c] = s[c];
      red[warp][CO + c] = q[c];
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 * CO) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < VC_THREADS / 32; ++w) t += red[w][threadIdx.x];
    const int stat = threadIdx.x / CO, c = threadIdx.x % CO;
    const long long nparts = (long long)gridDim.x * gridDim.z;
    a.part[((long long)stat * a.Cout + g * CO + c) * nparts + (long long)blockIdx.z * gridDim.x + blockIdx.x] = t;
  }
}

// torch.linspace(start, end, D) as ATen's CUDA kernel computes it: step in fp32, the lower half counted up from
// start and the upper half down from end, each as one fused multiply-add.
__device__ __forceinline__ float linspace_at(float start, float end, float step, int D, int i) {
  if (D == 1) return start;
  if (i < D / 2) return __fmaf_rn(step, (float)i, start);
  return __fmaf_rn(-step, (float)(D - 1 - i), end);
}

// One CTA per (channel, view = blockIdx.y): the batch statistics from the CTA partials (fixed order), or the running
// statistics in eval mode, folded with the affine into the scale / shift the consumers apply: BN(y) = y * scale +
// shift.  View v reads part + v * 2 * Cout * nparts and writes scale / shift + v * Cout and sums + v * sums_stride;
// VolumeConv launches one view, ImageConv one per view (each view's BatchNorm has its own batch statistics).
__global__ void __launch_bounds__(VC_FIN_THREADS)
    vc_bn_finalize_kernel(const double* __restrict__ part, int nparts, int Cout, double count,
                          const float* __restrict__ gamma, const float* __restrict__ beta,
                          const float* __restrict__ rmean, const float* __restrict__ rvar, float eps,
                          float* __restrict__ scale, float* __restrict__ shift, double* __restrict__ sums,
                          long long sums_stride) {
  const int c = blockIdx.x, v = blockIdx.y;
  scale += (long long)v * Cout;
  shift += (long long)v * Cout;
  if (sums != nullptr) sums += (long long)v * sums_stride;
  double mean, var;
  if (part != nullptr) {
    __shared__ double rs[VC_FIN_THREADS], rq[VC_FIN_THREADS];
    double s = 0.0, q = 0.0;
    part += (long long)v * 2 * Cout * nparts;
    for (int i = threadIdx.x; i < nparts; i += VC_FIN_THREADS) {
      s += part[(long long)c * nparts + i];
      q += part[(long long)(Cout + c) * nparts + i];
    }
    rs[threadIdx.x] = s;
    rq[threadIdx.x] = q;
    __syncthreads();
    for (int o = VC_FIN_THREADS / 2; o > 0; o >>= 1) {
      if (threadIdx.x < o) {
        rs[threadIdx.x] += rs[threadIdx.x + o];
        rq[threadIdx.x] += rq[threadIdx.x + o];
      }
      __syncthreads();
    }
    if (threadIdx.x != 0) return;
    s = rs[0];
    q = rq[0];
    if (sums != nullptr) {
      sums[c] = s;
      sums[Cout + c] = q;
    }
    mean = s / count;
    var = fmax(q / count - mean * mean, 0.0);  // biased, for normalising (as nn.BatchNorm3d in train mode)
  } else {
    if (threadIdx.x != 0) return;
    mean = (double)rmean[c];
    var = (double)rvar[c];
  }
  const double sc = (double)gamma[c] / sqrt(var + (double)eps);
  scale[c] = (float)sc;
  shift[c] = (float)((double)beta[c] - mean * sc);
}

// fixed-order tree sum of one value per thread over a block of THREADS; `red` is free again when it returns
template <int THREADS>
__device__ __forceinline__ double block_sum(double v, double* red) {
  red[threadIdx.x] = v;
  __syncthreads();
  for (int o = THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) red[threadIdx.x] += red[threadIdx.x + o];
    __syncthreads();
  }
  const double r = red[0];
  __syncthreads();
  return r;
}

// The weight repacking of the conv towers (VolumeConv, ImageConv; forward and backward), every layer in one launch:
// dst[dst_off + (i0 * n1 + i1) * n2 + i2] = src[base + i0 * s0 + i1 * s1 + i2 * s2] for i < n.  A negative stride
// with base at the far end walks that axis backwards (the flipped taps of the stride-1 data gradients).
constexpr int PACK_MAX_LAYERS = 11;
struct PackLayer {
  const float* src;
  long long dst_off;
  int n[3];
  long long base, s[3];
};
struct PackTable {
  PackLayer L[PACK_MAX_LAYERS];
  long long end[PACK_MAX_LAYERS];  // running sum of the layers' element counts
};

__global__ void pack_kernel(const PackTable t, float* __restrict__ dst, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int l = 0;
    while (i >= t.end[l]) ++l;
    const PackLayer& L = t.L[l];
    const long long e = i - (l > 0 ? t.end[l - 1] : 0);
    const int i2 = (int)(e % L.n[2]), i1 = (int)((e / L.n[2]) % L.n[1]), i0 = (int)(e / ((long long)L.n[1] * L.n[2]));
    dst[L.dst_off + e] = __ldg(L.src + L.base + i0 * L.s[0] + i1 * L.s[1] + i2 * L.s[2]);
  }
}

// the first n layers of t (end is filled here)
int launch_pack(PackTable& t, int n, float* dst, const char* name, cudaStream_t st) {
  long long total = 0;
  for (int l = 0; l < n; ++l) {
    total += (long long)t.L[l].n[0] * t.L[l].n[1] * t.L[l].n[2];
    t.end[l] = total;
  }
  prof_begin(name, st);
  pack_kernel<<<cdiv(total, 256), 256, 0, st>>>(t, dst, total);
  return check_launch(name, st);
}

struct VcLayerPlan {
  int mode, cin, cout, co, vd, src;
  int Di, Hi, Wi, Do, Ho, Wo;
  int tw, tpix, pix_blocks, dtiles, groups, npar;
  long long nparts;
  size_t w, y, part, ss;  // workspace offsets
};

struct VcPlan {
  VcLayerPlan L[VC_LAYERS];
  size_t total;
};

int vc_plan(int B, int Cin, int base, int D, int H, int W, VcPlan& p) {
  PMVS_REQUIRE(Cin == 64 && base == 8,
               "volume_conv: (in_channels, base_channels) = (%d, %d); only (64, 8) is supported", Cin, base);
  PMVS_REQUIRE(B >= 1 && B <= 8192, "volume_conv: B = %d (1 <= B <= 8192)", B);
  PMVS_REQUIRE(D >= 8 && H >= 8 && W >= 8 && D % 8 == 0 && H % 8 == 0 && W % 8 == 0,
               "volume_conv: D, H, W = %d, %d, %d must be positive multiples of 8", D, H, W);
  PMVS_REQUIRE((long long)D * H * W <= (1ll << 30), "volume_conv: D*H*W = %lld (limit 2^30)", (long long)D * H * W);
  const int b = base;
  // mode, cin, cout, input level, output level, co, vd, src
  const int spec[VC_LAYERS][8] = {
      {VC_S1, Cin, b, 0, 0, 8, 8, 0},        {VC_S2, Cin, 2 * b, 0, 1, 8, 4, 0},
      {VC_S2, 2 * b, 4 * b, 1, 2, 4, 2, 1},  {VC_S2, 4 * b, 8 * b, 2, 3, 4, 2, 1},
      {VC_S1, 2 * b, 2 * b, 1, 1, 8, 4, 1},  {VC_S1, 4 * b, 4 * b, 2, 2, 4, 2, 1},
      {VC_S1, 8 * b, 8 * b, 3, 3, 4, 2, 1},  {VC_T2, 8 * b, 4 * b, 3, 2, 4, 2, 1},
      {VC_T2, 4 * b, 2 * b, 2, 1, 8, 4, 2},  {VC_T2, 2 * b, b, 1, 0, 8, 4, 2},
      {VC_S1, b, 1, 0, 0, 1, 8, 2}};
  size_t off = 0;
  for (int l = 0; l < VC_LAYERS; ++l) {
    VcLayerPlan& q = p.L[l];
    q.mode = spec[l][0]; q.cin = spec[l][1]; q.cout = spec[l][2];
    q.co = spec[l][5]; q.vd = spec[l][6]; q.src = spec[l][7];
    q.Di = D >> spec[l][3]; q.Hi = H >> spec[l][3]; q.Wi = W >> spec[l][3];
    q.Do = D >> spec[l][4]; q.Ho = H >> spec[l][4]; q.Wo = W >> spec[l][4];
    q.tw = q.mode == VC_T2 ? q.Wi : q.Wo;
    q.tpix = q.mode == VC_T2 ? q.Hi * q.Wi : q.Ho * q.Wo;
    q.pix_blocks = cdiv(q.tpix, VC_THREADS);
    q.dtiles = cdiv(q.Do, q.vd);
    q.groups = q.cout / q.co;
    q.npar = q.mode == VC_T2 ? 4 : 1;
    q.nparts = (long long)q.pix_blocks * q.dtiles * B * q.npar;
    const long long wn = (long long)q.cin * VC_TAPS * q.cout;
    q.w = off;
    off += up256(wn * 4);
  }
  for (int l = 0; l < VC_BN; ++l) {
    VcLayerPlan& q = p.L[l];
    q.y = off;
    off += up256((size_t)B * q.cout * q.Do * q.Ho * q.Wo * 4);
    q.part = off;
    off += up256((size_t)2 * q.cout * q.nparts * 8);
    q.ss = off;
    off += up256((size_t)2 * q.cout * 4);
  }
  p.L[L6_2].y = p.L[L6_2].part = p.L[L6_2].ss = 0;
  p.total = off;
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs
