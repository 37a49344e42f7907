// VolumeConv (the coarse stage's 3-D U-Net, reference networks.py:127-167) and the coarse depth regression
// (model.py:117-130), include/pmvs_b200.h, DESIGN 3.12.
//
// Every layer is one register-blocked fp32 direct convolution (vconv_kernel).  A thread owns VD consecutive output
// planes along D of one output pixel and CO output channels, so every input value it loads feeds up to 3 * CO FMAs
// and the CO weights of a tap are one uniform (broadcast) load per warp.  Lanes take consecutive pixels, and every
// tensor is planar ([B, C, D, H, W], the layout build_cost_volume returns), so each load of a warp is one contiguous
// row segment.  A consumer applies its producer's BatchNorm + ReLU (and the skip sum) as it loads; a value outside
// the grid is zero after that, as the reference's zero padding of the activated tensor is.  Each CTA reduces its
// outputs' per-channel sums and sums of squares in fp64 in a fixed order; vc_bn_finalize_kernel then adds the CTA
// partials in a fixed order.  No floating-point atomics: two calls give the same bits.
#include <float.h>
#include <math.h>

#include "volume_conv.cuh"

namespace pmvs {

namespace {

const char* const VC_NAMES[VC_LAYERS] = {"vc_conv0_1", "vc_conv1_0", "vc_conv2_0", "vc_conv3_0",
                                         "vc_conv1_1", "vc_conv2_1", "vc_conv3_1", "vc_conv4_0",
                                         "vc_conv5_0", "vc_conv6_0", "vc_conv6_2"};
// dependency order of the forward
const int VC_ORDER[VC_LAYERS] = {L0_1, L1_0, L1_1, L2_0, L2_1, L3_0, L3_1, L4_0, L5_0, L6_0, L6_2};

// ---- depth regression: softmax(-x) over D, expectation against torch.linspace's planes, probability map ----------

__global__ void __launch_bounds__(256)
    coarse_depth_kernel(const float* __restrict__ vol, const float* __restrict__ cams, int B, int V, int D, int HW,
                        float* __restrict__ depth_out, float* __restrict__ prob_out) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (long long)B * HW) return;
  const int b = (int)(idx / HW), p = (int)(idx % HW);
  const float* cam = cams + (long long)b * V * 32 + 16 + 12;  // cam_params_list[b, 0, 1, 3, 0:3]
  const float start = __ldg(cam), interval = __ldg(cam + 1);
  const float end = __fadd_rn(start, __fmul_rn((float)(D - 1), interval));  // model.py:67, two fp32 roundings
  const float step = D > 1 ? __fdiv_rn(__fsub_rn(end, start), (float)(D - 1)) : 0.f;
  const float* x = vol + (long long)b * D * HW + p;
  float m = -INFINITY;
  for (int d = 0; d < D; ++d) m = fmaxf(m, -__ldg(x + (long long)d * HW));
  // S and the expectation accumulate in fp64 and divide once, so the regressed depth carries only the expf
  // roundings (a per-plane fp32 normalisation e_d / S would add ~1e-7 relative error per plane at depths of ~500)
  double S = 0.0, acc = 0.0;
  for (int d = 0; d < D; ++d) {
    const double e = (double)expf(__fsub_rn(-__ldg(x + (long long)d * HW), m));
    S += e;
    acc += (double)linspace_at(start, end, step, D, d) * e;
  }
  const float depth = (float)(acc / S);
  const float t = __fdiv_rn(__fsub_rn(depth, start), interval);
  const int lo = (int)fminf(fmaxf(floorf(t), 0.f), (float)(D - 1));
  const int hi = (int)fminf(fmaxf(ceilf(t), 0.f), (float)(D - 1));
  const double plo = (double)expf(__fsub_rn(-__ldg(x + (long long)lo * HW), m)) / S;
  const double phi = (double)expf(__fsub_rn(-__ldg(x + (long long)hi * HW), m)) / S;
  depth_out[idx] = depth;
  prob_out[idx] = (float)(plo + phi);
}

template <int MODE, int CO, int VD, int SRC>
int launch_vconv(const VcArgs& a, const VcLayerPlan& q, int B, const char* name, cudaStream_t st) {
  dim3 grid((unsigned)(q.pix_blocks * q.dtiles), (unsigned)q.groups, (unsigned)(B * q.npar));
  prof_begin(name, st);
  vconv_kernel<MODE, CO, VD, SRC><<<grid, VC_THREADS, 0, st>>>(a);
  return check_launch(name, st);
}

int launch_layer(int l, const VcArgs& a, const VcLayerPlan& q, int B, cudaStream_t st) {
  const char* n = VC_NAMES[l];
  switch (l) {
    case L0_1: return launch_vconv<VC_S1, 8, 8, 0>(a, q, B, n, st);
    case L1_0: return launch_vconv<VC_S2, 8, 4, 0>(a, q, B, n, st);
    case L2_0: case L3_0: return launch_vconv<VC_S2, 4, 2, 1>(a, q, B, n, st);
    case L1_1: return launch_vconv<VC_S1, 8, 4, 1>(a, q, B, n, st);
    case L2_1: case L3_1: return launch_vconv<VC_S1, 4, 2, 1>(a, q, B, n, st);
    case L4_0: return launch_vconv<VC_T2, 4, 2, 1>(a, q, B, n, st);
    case L5_0: case L6_0: return launch_vconv<VC_T2, 8, 4, 2>(a, q, B, n, st);
    default: return launch_vconv<VC_S1, 1, 8, 2>(a, q, B, n, st);
  }
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_volume_conv_workspace_bytes(int B, int in_channels, int base_channels, int D, int H, int W) {
  VcPlan p;
  if (vc_plan(B, in_channels, base_channels, D, H, W, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_volume_conv(const float* x, const pmvs_volume_weights* wt, int train, float* out,
                                double* batch_sums, void* workspace, size_t workspace_bytes, int B, int in_channels,
                                int base_channels, int D, int H, int W, pmvs_stream_t stream) {
  PMVS_REQUIRE(x && wt && out && workspace, "volume_conv: NULL pointer");
  VcPlan p;
  PMVS_TRY(vc_plan(B, in_channels, base_channels, D, H, W, p));
  for (int l = 0; l < VC_LAYERS; ++l) PMVS_REQUIRE(wt->weight[l], "volume_conv: NULL weight of layer %d", l);
  for (int l = 0; l < VC_BN; ++l) {
    PMVS_REQUIRE(wt->gamma[l] && wt->beta[l], "volume_conv: NULL BatchNorm affine of layer %d", l);
    PMVS_REQUIRE(train || (wt->running_mean[l] && wt->running_var[l]),
                 "volume_conv: eval mode needs the running statistics of layer %d", l);
    PMVS_REQUIRE(finite_nonneg(wt->eps[l]), "volume_conv: eps of layer %d = %g (finite, >= 0)", l, (double)wt->eps[l]);
  }
  PMVS_TRY(check_workspace("volume_conv", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;

  // PyTorch layouts -> [Cin][27][Cout]: Conv3d [Cout, Cin, 27], ConvTranspose3d [Cin, Cout, 27]
  PackTable pk;
  for (int l = 0; l < VC_LAYERS; ++l) {
    const VcLayerPlan& q = p.L[l];
    const bool t = q.mode == VC_T2;
    pk.L[l] = {wt->weight[l], (long long)(q.w / 4), {q.cin, VC_TAPS, q.cout}, 0,
               {t ? q.cout * VC_TAPS : VC_TAPS, 1, t ? VC_TAPS : q.cin * VC_TAPS}};
  }
  PMVS_TRY(launch_pack(pk, VC_LAYERS, (float*)ws, "vc_pack", st));

  size_t sums_off = 0;
  size_t sums_at[VC_BN];
  for (int l = 0; l < VC_BN; ++l) {
    sums_at[l] = sums_off;
    sums_off += 2 * (size_t)p.L[l].cout;
  }
  for (int k = 0; k < VC_LAYERS; ++k) {
    const int l = VC_ORDER[k];
    const VcLayerPlan& q = p.L[l];
    VcArgs a;
    memset(&a, 0, sizeof(a));
    if (VC_SRCA[l] < 0) {
      a.xa = x;
    } else {
      const VcLayerPlan& s = p.L[VC_SRCA[l]];
      a.xa = (const float*)(ws + s.y);
      a.sa = (const float*)(ws + s.ss);
      a.ha = a.sa + s.cout;
    }
    if (VC_SRCB[l] >= 0) {
      const VcLayerPlan& s = p.L[VC_SRCB[l]];
      a.xb = (const float*)(ws + s.y);
      a.sb = (const float*)(ws + s.ss);
      a.hb = a.sb + s.cout;
    }
    a.w = (const float*)(ws + q.w);
    a.y = l == L6_2 ? out : (float*)(ws + q.y);
    a.part = (l != L6_2 && train) ? (double*)(ws + q.part) : nullptr;
    a.Cin = q.cin; a.Cout = q.cout;
    a.Di = q.Di; a.Hi = q.Hi; a.Wi = q.Wi; a.Do = q.Do; a.Ho = q.Ho; a.Wo = q.Wo;
    a.tw = q.tw; a.tpix = q.tpix; a.pix_blocks = q.pix_blocks;
    PMVS_TRY(launch_layer(l, a, q, B, st));
    if (l == L6_2) break;
    float* scale = (float*)(ws + q.ss);
    const double count = (double)B * q.Do * q.Ho * q.Wo;
    prof_begin("vc_bn_finalize", st);
    vc_bn_finalize_kernel<<<q.cout, VC_FIN_THREADS, 0, st>>>(
        a.part, (int)q.nparts, q.cout, count, wt->gamma[l], wt->beta[l], wt->running_mean[l], wt->running_var[l],
        wt->eps[l], scale, scale + q.cout, (train && batch_sums) ? batch_sums + sums_at[l] : nullptr, 0);
    PMVS_TRY(check_launch("vc_bn_finalize_kernel", st));
  }
  return PMVS_OK;
}

extern "C" int pmvs_coarse_depth(const float* filtered, const float* cams, int B, int V, int D, int H, int W,
                                 float* depth_out, float* prob_out, pmvs_stream_t stream) {
  PMVS_REQUIRE(filtered && cams && depth_out && prob_out, "coarse_depth: NULL pointer");
  PMVS_REQUIRE(B >= 1 && V >= 1 && D >= 1 && H >= 1 && W >= 1, "coarse_depth: bad shape B=%d V=%d D=%d H=%d W=%d", B,
               V, D, H, W);
  PMVS_REQUIRE((long long)B * D * H * W < (1ll << 40) && (long long)H * W < (1ll << 31),
               "coarse_depth: volume too large");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)B * H * W;
  prof_begin("coarse_depth", st);
  coarse_depth_kernel<<<cdiv(n, 256), 256, 0, st>>>(filtered, cams, B, V, D, H * W, depth_out, prob_out);
  return check_launch("coarse_depth_kernel", st);
}
