// The forward plan of ImageConv (workspace layout, per-layer blocking) and its register-blocked direct convolution,
// shared by the forward (image_conv.cu) and the backward (image_conv_bwd.cu), so that one place knows the layout of
// the forward's workspace the backward reads.  DESIGN 3.14, 3.15.
#pragma once

#include <string.h>

#include <algorithm>

#include "volume_conv.cuh"

namespace pmvs {

namespace {

constexpr int IC_LAYERS = 11, IC_BN = 10, IC_THREADS = 128, IC_MAX_C = 64;

// the layers in module order (conv0.0, conv0.1, conv1.0 ... conv3.2) and the level (resolution) each one writes
const char* const IC_NAMES[IC_LAYERS] = {"ic_conv0_0", "ic_conv0_1", "ic_conv1_0", "ic_conv1_1",
                                         "ic_conv1_2", "ic_conv2_0", "ic_conv2_1", "ic_conv2_2",
                                         "ic_conv3_0", "ic_conv3_1", "ic_conv3_2"};
const int IC_OUT_LEVEL[IC_LAYERS] = {0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 3};
// the layer whose output is pyramid level k: ReLU(BN(.)) of it for conv0 .. conv2, the plain conv3_2 for conv3
const int IC_LEVEL_LAYER[4] = {1, 4, 7, 10};

struct IcArgs {
  const float* x;   // layer 0: the planar images [B, V, 3, Hi, Wi]; otherwise the producer's pre-BatchNorm output,
                    // NHWC [B*V, Hi, Wi, Cin]
  const float* ss;  // the producer's BatchNorm per view: scale [V][Cin], then shift [V][Cin] (not read by layer 0)
  const float* w;   // packed weights [K*K][Cin][Cout]
  float* y;         // [B*V, Ho, Wo, Cout] (or [B, V, Cout, Ho, Wo] with planar_out)
  double* part;     // [V][2][Cout][nparts] per-CTA sums and sums of squares (nparts = B * pix_blocks), or NULL
  int V, Hi, Wi, Ho, Wo;
  int ncg;          // column groups per output row: cdiv(Wo, PX)
  int tpix;         // Ho * ncg threads per image
  int pix_blocks;   // cdiv(tpix, IC_THREADS)
  int planar_out;
};

// One CTA: IC_THREADS column groups of PX output pixels x CO output channels (group blockIdx.y) of image blockIdx.z.
// BN_IN: the input is a producer's pre-BatchNorm output, activated as it is loaded (the forward); without it the
// input is read as it is (the backward's data gradients, which run this convolution on G with flipped taps).
template <int K, int S, int CIN, int COUT, int CO, int PX, bool BN_IN>
__device__ __forceinline__ void ic_conv_body(const IcArgs& a) {
  constexpr bool FIRST = CIN == 3;
  constexpr int P = K / 2;
  static_assert(FIRST || CIN % 4 == 0, "NHWC inputs are read four channels at a time");
  static_assert(CO % 4 == 0 && COUT % CO == 0, "output channels are written four at a time");
  const int g = blockIdx.y, n = blockIdx.z, v = n % a.V;
  const int tp = blockIdx.x * IC_THREADS + threadIdx.x;
  const bool live = tp < a.tpix;
  const int oh = live ? tp / a.ncg : 0, ow0 = live ? (tp % a.ncg) * PX : 0;
  const float* wg = a.w + g * CO;

  float acc[PX][CO];
#pragma unroll
  for (int p = 0; p < PX; ++p)
#pragma unroll
    for (int c = 0; c < CO; ++c) acc[p][c] = 0.f;

#pragma unroll 1
  for (int kh = 0; kh < K; ++kh) {
    const int ih = oh * S - P + kh;
    const bool okh = live && ih >= 0 && ih < a.Hi;
#pragma unroll
    for (int kw = 0; kw < K; ++kw) {
      const float* wt = wg + (kh * K + kw) * CIN * COUT;
      if (FIRST) {
#pragma unroll
        for (int ci = 0; ci < 3; ++ci) {
          const float* plane = a.x + (((long long)n * 3 + ci) * a.Hi + ih) * a.Wi;
          float xv[PX];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            const int iw = (ow0 + p) * S - P + kw;
            xv[p] = (okh && iw >= 0 && iw < a.Wi) ? __ldg(plane + iw) : 0.f;
          }
          float wv[CO];
#pragma unroll
          for (int c = 0; c < CO; c += 4) {
            const float4 t = ldg4(wt + ci * COUT + c);
            wv[c] = t.x; wv[c + 1] = t.y; wv[c + 2] = t.z; wv[c + 3] = t.w;
          }
#pragma unroll
          for (int p = 0; p < PX; ++p)
#pragma unroll
            for (int c = 0; c < CO; ++c) acc[p][c] = __fmaf_rn(xv[p], wv[c], acc[p][c]);
        }
      } else {
        const float* row = a.x + ((long long)n * a.Hi + ih) * a.Wi * CIN;
        const float* sc = a.ss + (long long)v * CIN;
        const float* sh = sc + (long long)a.V * CIN;
#pragma unroll 1
        for (int c4 = 0; c4 < CIN; c4 += 4) {
          float4 s4, h4;
          if (BN_IN) { s4 = ldg4(sc + c4); h4 = ldg4(sh + c4); }
          float xv[PX][4];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            const int iw = (ow0 + p) * S - P + kw;
            if (okh && iw >= 0 && iw < a.Wi) {
              const float4 t = ldg4(row + (long long)iw * CIN + c4);
              if (BN_IN) {
                xv[p][0] = act(t.x, s4.x, h4.x); xv[p][1] = act(t.y, s4.y, h4.y);
                xv[p][2] = act(t.z, s4.z, h4.z); xv[p][3] = act(t.w, s4.w, h4.w);
              } else {
                xv[p][0] = t.x; xv[p][1] = t.y; xv[p][2] = t.z; xv[p][3] = t.w;
              }
            } else {
              xv[p][0] = xv[p][1] = xv[p][2] = xv[p][3] = 0.f;  // padding of the activated tensor
            }
          }
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float wv[CO];
#pragma unroll
            for (int c = 0; c < CO; c += 4) {
              const float4 t = ldg4(wt + (c4 + j) * COUT + c);
              wv[c] = t.x; wv[c + 1] = t.y; wv[c + 2] = t.z; wv[c + 3] = t.w;
            }
#pragma unroll
            for (int p = 0; p < PX; ++p)
#pragma unroll
              for (int c = 0; c < CO; ++c) acc[p][c] = __fmaf_rn(xv[p][j], wv[c], acc[p][c]);
          }
        }
      }
    }
  }

  // epilogue: store, then this CTA's per-channel sums in a fixed order (pixels in order, lanes by butterfly, warps in
  // index order)
  const long long HWo = (long long)a.Ho * a.Wo;
#pragma unroll
  for (int p = 0; p < PX; ++p) {
    if (!live || ow0 + p >= a.Wo) continue;
    const long long pix = (long long)oh * a.Wo + ow0 + p;
    if (a.planar_out) {
      float* yp = a.y + ((long long)n * COUT + g * CO) * HWo + pix;
#pragma unroll
      for (int c = 0; c < CO; ++c) yp[c * HWo] = acc[p][c];
    } else {
      float* yp = a.y + ((long long)n * HWo + pix) * COUT + g * CO;
#pragma unroll
      for (int c = 0; c < CO; c += 4)
        *reinterpret_cast<float4*>(yp + c) = make_float4(acc[p][c], acc[p][c + 1], acc[p][c + 2], acc[p][c + 3]);
    }
  }
  if (a.part == nullptr) return;
  __shared__ double red[IC_THREADS / 32][2 * CO];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < CO; ++c) {
    double s = 0.0, q = 0.0;
#pragma unroll
    for (int p = 0; p < PX; ++p) {
      if (live && ow0 + p < a.Wo) {
        const double r = (double)acc[p][c];
        s += r;
        q += r * r;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      s += __shfl_xor_sync(0xffffffffu, s, o);
      q += __shfl_xor_sync(0xffffffffu, q, o);
    }
    if (lane == 0) {
      red[warp][c] = s;
      red[warp][CO + c] = q;
    }
  }
  __syncthreads();
  if (threadIdx.x < 2 * CO) {
    double t = 0.0;
#pragma unroll
    for (int w = 0; w < IC_THREADS / 32; ++w) t += red[w][threadIdx.x];
    const int stat = threadIdx.x / CO, c = threadIdx.x % CO;
    const long long nparts = (long long)(gridDim.z / a.V) * gridDim.x;
    const long long b = n / a.V;
    a.part[(((long long)v * 2 + stat) * COUT + g * CO + c) * nparts + b * gridDim.x + blockIdx.x] = t;
  }
}

template <int K, int S, int CIN, int COUT, int CO, int PX>
__global__ void __launch_bounds__(IC_THREADS) ic_conv_kernel(const IcArgs a) {
  ic_conv_body<K, S, CIN, COUT, CO, PX, true>(a);
}

struct IcLayerPlan {
  int k, s, cin, cout, co, px;
  int Hi, Wi, Ho, Wo;
  int ncg, tpix, pix_blocks, groups;
  long long nparts;  // per view: B * pix_blocks
  size_t w;          // workspace offset of the packed weights
};

// The forward's workspace.  Without keep, the pre-BatchNorm activations and the scale / shift sets ping-pong between
// two buffers (layer l uses y[l & 1], ss[l & 1]).  With keep (the forward of a training step), every BatchNorm layer
// has its own, so that the backward can read them all; in eval mode the running statistics the forward normalised
// with are copied too (rs: [mean[C_l], var[C_l]] per layer, at rs_at[l] floats), so an update of the module's buffers
// between forward and backward changes nothing.
struct IcPlan {
  IcLayerPlan L[IC_LAYERS];
  int h[4], w[4];  // level sizes
  int keep;
  size_t y[IC_BN], ss[IC_BN];  // workspace offsets of each BatchNorm layer's pre-BatchNorm output and scale / shift
  size_t part, rs, total;
  size_t rs_at[IC_BN];
};

int ic_plan(int B, int V, int H, int W, int base, int keep, IcPlan& p) {
  PMVS_REQUIRE(base == 8, "image_conv: base_channels = %d; only 8 is supported", base);
  PMVS_REQUIRE(B >= 1 && V >= 1 && (long long)B * V <= 65535, "image_conv: B = %d, V = %d (B >= 1, V >= 1, B*V <= 65535)",
               B, V);
  PMVS_REQUIRE(H >= 1 && W >= 1 && H <= 32768 && W <= 32768 && (long long)H * W <= (1ll << 28),
               "image_conv: H, W = %d, %d (1 .. 32768, H*W <= 2^28)", H, W);
  p.h[0] = H;
  p.w[0] = W;
  for (int k = 1; k < 4; ++k) {
    p.h[k] = (p.h[k - 1] + 1) / 2;  // 5x5, stride 2, padding 2: ceil(n / 2)
    p.w[k] = (p.w[k - 1] + 1) / 2;
  }
  const int b = base;
  // k, s, cin, cout, co, px
  const int spec[IC_LAYERS][6] = {{3, 1, 3, b, 8, 4},          {3, 1, b, b, 8, 8},
                                  {5, 2, b, 2 * b, 16, 4},     {3, 1, 2 * b, 2 * b, 16, 4},
                                  {3, 1, 2 * b, 2 * b, 16, 4}, {5, 2, 2 * b, 4 * b, 16, 4},
                                  {3, 1, 4 * b, 4 * b, 16, 4}, {3, 1, 4 * b, 4 * b, 16, 4},
                                  {5, 2, 4 * b, 8 * b, 16, 4}, {3, 1, 8 * b, 8 * b, 16, 4},
                                  {3, 1, 8 * b, 8 * b, 16, 4}};
  const long long N = (long long)B * V;
  size_t off = 0, ymax = 0, partmax = 0;
  p.keep = keep;
  for (int l = 0; l < IC_LAYERS; ++l) {
    IcLayerPlan& q = p.L[l];
    q.k = spec[l][0]; q.s = spec[l][1]; q.cin = spec[l][2]; q.cout = spec[l][3]; q.co = spec[l][4]; q.px = spec[l][5];
    const int lo = IC_OUT_LEVEL[l], li = q.s == 2 ? lo - 1 : lo;
    q.Hi = p.h[li]; q.Wi = p.w[li]; q.Ho = p.h[lo]; q.Wo = p.w[lo];
    q.ncg = cdiv(q.Wo, q.px);
    q.tpix = q.Ho * q.ncg;
    q.pix_blocks = cdiv(q.tpix, IC_THREADS);
    q.groups = q.cout / q.co;
    q.nparts = (long long)B * q.pix_blocks;
    const long long wn = (long long)q.k * q.k * q.cin * q.cout;
    q.w = off;
    off += up256(wn * 4);
    if (l < IC_BN) {
      ymax = std::max(ymax, (size_t)N * q.Ho * q.Wo * q.cout * 4);
      partmax = std::max(partmax, (size_t)V * 2 * q.cout * (size_t)q.nparts * 8);
    }
  }
  size_t rs_n = 0;
  for (int l = 0; l < IC_BN; ++l) {
    p.rs_at[l] = rs_n;
    rs_n += 2 * (size_t)p.L[l].cout;
  }
  if (!keep) {
    const size_t y0 = off, y1 = off + up256(ymax);
    p.part = y1 + up256(ymax);
    const size_t s0 = p.part + up256(partmax), s1 = s0 + up256((size_t)V * 2 * IC_MAX_C * 4);
    for (int l = 0; l < IC_BN; ++l) {
      p.y[l] = (l & 1) ? y1 : y0;
      p.ss[l] = (l & 1) ? s1 : s0;
    }
    p.rs = 0;
    p.total = s1 + up256((size_t)V * 2 * IC_MAX_C * 4);
    return PMVS_OK;
  }
  for (int l = 0; l < IC_BN; ++l) {
    const IcLayerPlan& q = p.L[l];
    p.y[l] = off;
    off += up256((size_t)N * q.Ho * q.Wo * q.cout * 4);
    p.ss[l] = off;
    off += up256((size_t)V * 2 * q.cout * 4);
  }
  p.part = off;
  off += up256(partmax);
  p.rs = off;
  off += up256(rs_n * 4);
  p.total = off;
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs
