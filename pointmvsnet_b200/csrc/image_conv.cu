// ImageConv (the image towers, reference networks.py:84-124): every view's feature pyramid in one call,
// include/pmvs_b200.h, DESIGN 3.14.
//
// Every layer is one register-blocked fp32 direct convolution (ic_conv_kernel).  Intermediates are NHWC, one image per
// (b, v), so a thread loads four input channels of a tap as one float4 and feeds each to CO output channels of PX
// consecutive output pixels of one row; the CO weights of a (tap, channel) are one uniform (broadcast) load per warp.
// The first layer reads the planar [B, V, 3, H, W] image directly.  A consumer applies its producer's BatchNorm + ReLU
// as it loads; a tap outside the image is zero after that, as the reference's zero padding of the activated tensor
// is.  A CTA covers pixels of one image only, so its fp64 per-channel sums and sums of squares belong to one view;
// vc_bn_finalize_kernel (shared with VolumeConv) adds the CTA partials of each view in a fixed order.  No
// floating-point atomics: two calls give the same bits.
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
template <int K, int S, int CIN, int COUT, int CO, int PX>
__global__ void __launch_bounds__(IC_THREADS) ic_conv_kernel(const IcArgs a) {
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
          const float4 s4 = ldg4(sc + c4), h4 = ldg4(sh + c4);
          float xv[PX][4];
#pragma unroll
          for (int p = 0; p < PX; ++p) {
            const int iw = (ow0 + p) * S - P + kw;
            if (okh && iw >= 0 && iw < a.Wi) {
              const float4 t = ldg4(row + (long long)iw * CIN + c4);
              xv[p][0] = act(t.x, s4.x, h4.x); xv[p][1] = act(t.y, s4.y, h4.y);
              xv[p][2] = act(t.z, s4.z, h4.z); xv[p][3] = act(t.w, s4.w, h4.w);
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

// a pyramid level conv0 .. conv2: ReLU(BN(y)) of its last layer, per view, into [B, V, h, w, C] (channels_last) or
// [B, V, C, h, w]; one thread per output element, in output order
__global__ void __launch_bounds__(256)
    ic_level_kernel(const float* __restrict__ y, const float* __restrict__ ss, float* __restrict__ out, int V, int C,
                    long long HW, long long total, int planar) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  long long src;
  int n, c;
  if (planar) {
    n = (int)(i / (C * HW));
    const long long r = i % (C * HW);
    c = (int)(r / HW);
    src = ((long long)n * HW + r % HW) * C + c;
  } else {
    n = (int)(i / (C * HW));
    c = (int)(i % C);
    src = i;
  }
  const int v = n % V;
  out[i] = act(__ldg(y + src), __ldg(ss + v * C + c), __ldg(ss + (V + v) * C + c));
}

// PyTorch Conv2d weights [Cout, Cin, K, K] -> [K*K][Cin][Cout] for every layer in one launch
struct IcPack {
  const float* src[IC_LAYERS];
  long long end[IC_LAYERS];  // running sum of the layers' element counts
  long long dst_off[IC_LAYERS];
  int cin[IC_LAYERS], cout[IC_LAYERS], taps[IC_LAYERS];
};

__global__ void ic_pack_kernel(const IcPack p, float* __restrict__ dst, long long total) {
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    int l = 0;
    while (i >= p.end[l]) ++l;
    const long long e = i - (l > 0 ? p.end[l - 1] : 0);
    const int cout = p.cout[l], cin = p.cin[l], taps = p.taps[l];
    const int co = (int)(e % cout), ci = (int)((e / cout) % cin), tap = (int)(e / ((long long)cout * cin));
    dst[p.dst_off[l] + e] = __ldg(p.src[l] + ((long long)co * cin + ci) * taps + tap);
  }
}

struct IcLayerPlan {
  int k, s, cin, cout, co, px;
  int Hi, Wi, Ho, Wo;
  int ncg, tpix, pix_blocks, groups;
  long long nparts;  // per view: B * pix_blocks
  size_t w;          // workspace offset of the packed weights
};

struct IcPlan {
  IcLayerPlan L[IC_LAYERS];
  int h[4], w[4];  // level sizes
  long long wtotal;
  size_t y[2], part, ss[2], total;  // workspace offsets: ping-pong activations, partials, ping-pong scale / shift
};

int ic_plan(int B, int V, int H, int W, int base, IcPlan& p) {
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
  p.wtotal = 0;
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
    p.wtotal += wn;
    if (l < IC_BN) {
      ymax = std::max(ymax, (size_t)N * q.Ho * q.Wo * q.cout * 4);
      partmax = std::max(partmax, (size_t)V * 2 * q.cout * (size_t)q.nparts * 8);
    }
  }
  p.y[0] = off;
  p.y[1] = off + up256(ymax);
  p.part = p.y[1] + up256(ymax);
  p.ss[0] = p.part + up256(partmax);
  p.ss[1] = p.ss[0] + up256((size_t)V * 2 * IC_MAX_C * 4);
  p.total = p.ss[1] + up256((size_t)V * 2 * IC_MAX_C * 4);
  return PMVS_OK;
}

template <int K, int S, int CIN, int COUT, int CO, int PX>
int launch_ic(const IcArgs& a, const IcLayerPlan& q, int N, const char* name, cudaStream_t st) {
  dim3 grid((unsigned)q.pix_blocks, (unsigned)q.groups, (unsigned)N);
  prof_begin(name, st);
  ic_conv_kernel<K, S, CIN, COUT, CO, PX><<<grid, IC_THREADS, 0, st>>>(a);
  return check_launch(name, st);
}

int ic_launch_layer(int l, const IcArgs& a, const IcLayerPlan& q, int N, cudaStream_t st) {
  const char* n = IC_NAMES[l];
  switch (l) {
    case 0: return launch_ic<3, 1, 3, 8, 8, 4>(a, q, N, n, st);
    case 1: return launch_ic<3, 1, 8, 8, 8, 8>(a, q, N, n, st);
    case 2: return launch_ic<5, 2, 8, 16, 16, 4>(a, q, N, n, st);
    case 3: case 4: return launch_ic<3, 1, 16, 16, 16, 4>(a, q, N, n, st);
    case 5: return launch_ic<5, 2, 16, 32, 16, 4>(a, q, N, n, st);
    case 6: case 7: return launch_ic<3, 1, 32, 32, 16, 4>(a, q, N, n, st);
    case 8: return launch_ic<5, 2, 32, 64, 16, 4>(a, q, N, n, st);
    default: return launch_ic<3, 1, 64, 64, 16, 4>(a, q, N, n, st);
  }
}

bool ic_finite_nonneg(float t) { return t >= 0.f && t <= 3.402823466e38f; }

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_image_conv_workspace_bytes(int B, int V, int H, int W, int base_channels) {
  IcPlan p;
  if (ic_plan(B, V, H, W, base_channels, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_image_conv(const float* img, const pmvs_image_weights* wt, int train, float* const* level_out,
                               int channels_last, double* batch_sums, void* workspace, size_t workspace_bytes, int B,
                               int V, int H, int W, int base_channels, pmvs_stream_t stream) {
  PMVS_REQUIRE(img && wt && level_out && workspace, "image_conv: NULL pointer");
  IcPlan p;
  PMVS_TRY(ic_plan(B, V, H, W, base_channels, p));
  for (int l = 0; l < IC_LAYERS; ++l) PMVS_REQUIRE(wt->weight[l], "image_conv: NULL weight of layer %d", l);
  for (int l = 0; l < IC_BN; ++l) {
    PMVS_REQUIRE(wt->gamma[l] && wt->beta[l], "image_conv: NULL BatchNorm affine of layer %d", l);
    PMVS_REQUIRE(train || (wt->running_mean[l] && wt->running_var[l]),
                 "image_conv: eval mode needs the running statistics of layer %d", l);
    PMVS_REQUIRE(ic_finite_nonneg(wt->eps[l]), "image_conv: eps of layer %d = %g (finite, >= 0)", l,
                 (double)wt->eps[l]);
  }
  PMVS_REQUIRE(!train || (long long)B * p.h[3] * p.w[3] >= 2,
               "image_conv: train mode needs more than 1 value per channel at the coarsest level (B*h3*w3 = %lld)",
               (long long)B * p.h[3] * p.w[3]);
  PMVS_REQUIRE(((uintptr_t)workspace & 255) == 0, "image_conv: workspace must be 256-byte aligned");
  for (int k = 0; k < 4; ++k)
    PMVS_REQUIRE(((uintptr_t)level_out[k] & 15) == 0, "image_conv: level output %d must be 16-byte aligned", k);
  if (workspace_bytes < p.total) {
    set_error("image_conv: workspace %zu bytes < required %zu", workspace_bytes, p.total);
    return PMVS_ERR_WORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  const int N = B * V;

  IcPack pk;
  long long run = 0;
  for (int l = 0; l < IC_LAYERS; ++l) {
    const IcLayerPlan& q = p.L[l];
    pk.src[l] = wt->weight[l];
    run += (long long)q.k * q.k * q.cin * q.cout;
    pk.end[l] = run;
    pk.dst_off[l] = (long long)(q.w / 4);
    pk.cin[l] = q.cin;
    pk.cout[l] = q.cout;
    pk.taps[l] = q.k * q.k;
  }
  prof_begin("ic_pack", st);
  ic_pack_kernel<<<cdiv(p.wtotal, 256), 256, 0, st>>>(pk, (float*)ws, p.wtotal);
  PMVS_TRY(check_launch("ic_pack_kernel", st));

  size_t sums_at[IC_BN], sums_stride = 0;
  for (int l = 0; l < IC_BN; ++l) {
    sums_at[l] = sums_stride;
    sums_stride += 2 * (size_t)p.L[l].cout;
  }
  for (int l = 0; l < IC_LAYERS; ++l) {
    const IcLayerPlan& q = p.L[l];
    const bool last = l == IC_LAYERS - 1;
    if (last && level_out[3] == nullptr) break;  // conv3_2 has no BatchNorm: nothing to do when conv3 is not asked for
    IcArgs a;
    memset(&a, 0, sizeof(a));
    a.x = l == 0 ? img : (const float*)(ws + p.y[(l - 1) & 1]);
    a.ss = l == 0 ? nullptr : (const float*)(ws + p.ss[(l - 1) & 1]);
    a.w = (const float*)(ws + q.w);
    a.y = last ? level_out[3] : (float*)(ws + p.y[l & 1]);
    a.part = (!last && train) ? (double*)(ws + p.part) : nullptr;
    a.V = V;
    a.Hi = q.Hi; a.Wi = q.Wi; a.Ho = q.Ho; a.Wo = q.Wo;
    a.ncg = q.ncg; a.tpix = q.tpix; a.pix_blocks = q.pix_blocks;
    a.planar_out = last && !channels_last;
    PMVS_TRY(ic_launch_layer(l, a, q, N, st));
    if (last) break;
    float* scale = (float*)(ws + p.ss[l & 1]);
    prof_begin("ic_bn_finalize", st);
    vc_bn_finalize_kernel<<<dim3(q.cout, V), VC_FIN_THREADS, 0, st>>>(
        a.part, (int)q.nparts, q.cout, (double)B * q.Ho * q.Wo, wt->gamma[l], wt->beta[l], wt->running_mean[l],
        wt->running_var[l], wt->eps[l], scale, scale + (size_t)V * q.cout,
        (train && batch_sums) ? batch_sums + sums_at[l] : nullptr, (long long)sums_stride);
    PMVS_TRY(check_launch("vc_bn_finalize_kernel", st));
    for (int k = 0; k < 3; ++k) {
      if (IC_LEVEL_LAYER[k] != l || level_out[k] == nullptr) continue;
      const long long HW = (long long)q.Ho * q.Wo, total = (long long)N * HW * q.cout;
      prof_begin("ic_level", st);
      ic_level_kernel<<<cdiv(total, 256), 256, 0, st>>>((const float*)(ws + p.y[l & 1]), scale, level_out[k], V,
                                                         q.cout, HW, total, channels_last ? 0 : 1);
      PMVS_TRY(check_launch("ic_level_kernel", st));
    }
  }
  return PMVS_OK;
}
