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
// floating-point atomics: two calls give the same bits.  pmvs_image_conv_keep runs the same plan and launches with a
// workspace that keeps every BatchNorm layer's output for the backward (image_conv_bwd.cu; the layout: image_conv.cuh).
#include "image_conv.cuh"

namespace pmvs {

namespace {

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

// keep mode, eval: a copy of the running statistics the forward normalises with, [mean[C_l], var[C_l]] per layer
struct IcRunning {
  const float* mean[IC_BN];
  const float* var[IC_BN];
  int at[IC_BN + 1];  // running sum of 2 C_l
};

__global__ void ic_keep_running_kernel(const IcRunning r, float* __restrict__ dst) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= r.at[IC_BN]) return;
  int l = 0;
  while (i >= r.at[l + 1]) ++l;
  const int e = i - r.at[l], c = (r.at[l + 1] - r.at[l]) / 2;
  dst[i] = e < c ? __ldg(r.mean[l] + e) : __ldg(r.var[l] + e - c);
}

// the forward; with keep every BatchNorm layer's pre-BatchNorm output and scale / shift stay in the workspace
int ic_forward(const float* img, const pmvs_image_weights* wt, int train, float* const* level_out, int channels_last,
               double* batch_sums, void* workspace, size_t workspace_bytes, int B, int V, int H, int W,
               int base_channels, int keep, cudaStream_t st) {
  PMVS_REQUIRE(img && wt && level_out && workspace, "image_conv: NULL pointer");
  IcPlan p;
  PMVS_TRY(ic_plan(B, V, H, W, base_channels, keep, p));
  for (int l = 0; l < IC_LAYERS; ++l) PMVS_REQUIRE(wt->weight[l], "image_conv: NULL weight of layer %d", l);
  for (int l = 0; l < IC_BN; ++l) {
    PMVS_REQUIRE(wt->gamma[l] && wt->beta[l], "image_conv: NULL BatchNorm affine of layer %d", l);
    PMVS_REQUIRE(train || (wt->running_mean[l] && wt->running_var[l]),
                 "image_conv: eval mode needs the running statistics of layer %d", l);
    PMVS_REQUIRE(finite_nonneg(wt->eps[l]), "image_conv: eps of layer %d = %g (finite, >= 0)", l,
                 (double)wt->eps[l]);
  }
  PMVS_REQUIRE(!train || (long long)B * p.h[3] * p.w[3] >= 2,
               "image_conv: train mode needs more than 1 value per channel at the coarsest level (B*h3*w3 = %lld)",
               (long long)B * p.h[3] * p.w[3]);
  for (int k = 0; k < 4; ++k)
    PMVS_REQUIRE(((uintptr_t)level_out[k] & 15) == 0, "image_conv: level output %d must be 16-byte aligned", k);
  PMVS_TRY(check_workspace("image_conv", workspace, workspace_bytes, p.total));
  char* ws = (char*)workspace;
  const int N = B * V;

  // PyTorch Conv2d weights [Cout, Cin, K, K] -> [K*K][Cin][Cout]
  PackTable pk;
  for (int l = 0; l < IC_LAYERS; ++l) {
    const IcLayerPlan& q = p.L[l];
    const int taps = q.k * q.k;
    pk.L[l] = {wt->weight[l], (long long)(q.w / 4), {taps, q.cin, q.cout}, 0, {1, taps, q.cin * taps}};
  }
  PMVS_TRY(launch_pack(pk, IC_LAYERS, (float*)ws, "ic_pack", st));
  if (keep && !train) {
    IcRunning r;
    r.at[0] = 0;
    for (int l = 0; l < IC_BN; ++l) {
      r.mean[l] = wt->running_mean[l];
      r.var[l] = wt->running_var[l];
      r.at[l + 1] = r.at[l] + 2 * p.L[l].cout;
    }
    prof_begin("ic_keep_running", st);
    ic_keep_running_kernel<<<cdiv(r.at[IC_BN], 256), 256, 0, st>>>(r, (float*)(ws + p.rs));
    PMVS_TRY(check_launch("ic_keep_running_kernel", st));
  }

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
    a.x = l == 0 ? img : (const float*)(ws + p.y[l - 1]);
    a.ss = l == 0 ? nullptr : (const float*)(ws + p.ss[l - 1]);
    a.w = (const float*)(ws + q.w);
    a.y = last ? level_out[3] : (float*)(ws + p.y[l]);
    a.part = (!last && train) ? (double*)(ws + p.part) : nullptr;
    a.V = V;
    a.Hi = q.Hi; a.Wi = q.Wi; a.Ho = q.Ho; a.Wo = q.Wo;
    a.ncg = q.ncg; a.tpix = q.tpix; a.pix_blocks = q.pix_blocks;
    a.planar_out = last && !channels_last;
    PMVS_TRY(ic_launch_layer(l, a, q, N, st));
    if (last) break;
    float* scale = (float*)(ws + p.ss[l]);
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
      ic_level_kernel<<<cdiv(total, 256), 256, 0, st>>>((const float*)(ws + p.y[l]), scale, level_out[k], V, q.cout,
                                                         HW, total, channels_last ? 0 : 1);
      PMVS_TRY(check_launch("ic_level_kernel", st));
    }
  }
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_image_conv_workspace_bytes(int B, int V, int H, int W, int base_channels) {
  IcPlan p;
  if (ic_plan(B, V, H, W, base_channels, 0, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_image_conv(const float* img, const pmvs_image_weights* wt, int train, float* const* level_out,
                               int channels_last, double* batch_sums, void* workspace, size_t workspace_bytes, int B,
                               int V, int H, int W, int base_channels, pmvs_stream_t stream) {
  return ic_forward(img, wt, train, level_out, channels_last, batch_sums, workspace, workspace_bytes, B, V, H, W,
                    base_channels, 0, (cudaStream_t)stream);
}

extern "C" size_t pmvs_image_conv_keep_workspace_bytes(int B, int V, int H, int W, int base_channels) {
  IcPlan p;
  if (ic_plan(B, V, H, W, base_channels, 1, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_image_conv_keep(const float* img, const pmvs_image_weights* wt, int train,
                                    float* const* level_out, int channels_last, double* batch_sums, void* workspace,
                                    size_t workspace_bytes, int B, int V, int H, int W, int base_channels,
                                    pmvs_stream_t stream) {
  return ic_forward(img, wt, train, level_out, channels_last, batch_sums, workspace, workspace_bytes, B, V, H, W,
                    base_channels, 1, (cudaStream_t)stream);
}
