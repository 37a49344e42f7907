// Backward of the coarse-stage plane sweep (pmvs_cost_volume, reference model.py:81-113) with respect to the
// per-view features.  With s1 = f_0 + sum_{v>=1} f_v (view order), mean = s1 / V and cost = s2 / V - mean^2,
//   d cost / d f_v = 2 (f_v - mean) / V
// where f_0 is the un-warped reference feature (model.py:103-106: view 0's fetched samples are overwritten, so they get
// no gradient) and f_v, v >= 1, the bilinear sample of view v at the projection of plane point (d, y, x).  The fetch
// coordinates carry no gradient (feature_fetcher.py:29), so neither do the cameras.  Steps:
//   point   one thread per plane point: the forward's plane point and taps (projection.cuh, bit for bit), f_v and the
//           mean recomputed with the forward's arithmetic; writes d f_0 [B,C,D,h*w] and d f_v for v >= 1
//           channel-contiguous [B][D*h*w][V-1][C], with the 4 tap records (texel, weight) of every (point, view)
//   lists   build_inv_lists over the records: per source texel, its records in ascending (point, view, tap) order
//   texels  launch_texel_sum: per source texel, sum of weight * d f_v over its records, in list order, channels-last
//   finish  grad_features [B,V,C,h,w]: view 0 sums d f_0 over d in ascending order, views >= 1 take the texel sums
// No floating-point atomics: every sum has an order fixed by the shapes, so two calls give the same bits, and a batch
// element's gradient does not depend on the others.
#include "common.cuh"
#include "projection.cuh"

namespace pmvs {

namespace {

__global__ void __launch_bounds__(256)
    cv_bwd_point_kernel(const float* __restrict__ feat, const float* __restrict__ cam_params,
                        const float* __restrict__ cam_blocks, const float* __restrict__ grad_cost,
                        float* __restrict__ df0, float* __restrict__ dfv, int64_t* __restrict__ rec_idx,
                        float* __restrict__ rec_w, int V, int C, int h, int w, int D) {
  __shared__ float cam[cam_block_floats(PMVS_MAX_VIEWS)];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < cam_block_floats(V); i += blockDim.x)
    cam[i] = cam_blocks[(size_t)b * cam_block_floats(V) + i];
  __syncthreads();
  const int hw = h * w, N = D * hw;
  const int p = blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= N) return;
  const int d = p / hw, pix = p - d * hw;
  float wx, wy, wz;
  cv_world_point(cam, cam_params, b, V, D, h, w, p, wx, wy, wz);
  const float fV = (float)V;
  const size_t plane = (size_t)hw;
  const size_t row1 = ((size_t)b * N + p) * (V - 1);  // source row of (p, view 1); view v is row1 + v - 1
  // tap records: record 4 (row1 + v - 1) + tap holds the texel (v - 1) h w + y w + x of the tap, -1 if it is masked
  for (int v = 1; v < V; ++v) {
    const Taps tp = cv_view_taps(cam + CB_VIEW + v * CB_VSTRIDE, wx, wy, wz, w, h);
    const long long t00 = (long long)(v - 1) * hw + (long long)tp.y0 * w + tp.x0;
    const size_t r = (row1 + v - 1) * 4;
    rec_idx[r + 0] = tp.ok_n && tp.ok_w ? t00 : -1;
    rec_idx[r + 1] = tp.ok_n && tp.ok_e ? t00 + 1 : -1;
    rec_idx[r + 2] = tp.ok_s && tp.ok_w ? t00 + w : -1;
    rec_idx[r + 3] = tp.ok_s && tp.ok_e ? t00 + w + 1 : -1;
    rec_w[r + 0] = tp.nw; rec_w[r + 1] = tp.ne; rec_w[r + 2] = tp.sw; rec_w[r + 3] = tp.se;
  }
  for (int c0 = 0; c0 < C; c0 += CV_CH) {
    float mean[CV_CH], k[CV_CH];
    const float* ref = feat + ((size_t)(b * V) * C + c0) * plane + pix;
#pragma unroll
    for (int c = 0; c < CV_CH; ++c) mean[c] = __ldg(ref + c * plane);
    // the forward's sample and sum (cost_volume_kernel), so the mean is the one the forward used
    for (int v = 1; v < V; ++v) {
      const Taps tp = cv_view_taps(cam + CB_VIEW + v * CB_VSTRIDE, wx, wy, wz, w, h);
      const float* m = feat + ((size_t)(b * V + v) * C + c0) * plane + (size_t)tp.y0 * w + tp.x0;
#pragma unroll
      for (int c = 0; c < CV_CH; ++c) {
        const float* mc = m + c * plane;
        float acc = 0.f;
        if (tp.ok_n && tp.ok_w) acc = __fmul_rn(__ldg(mc), tp.nw);
        if (tp.ok_n && tp.ok_e) acc = fmaf(__ldg(mc + 1), tp.ne, acc);
        if (tp.ok_s && tp.ok_w) acc = fmaf(__ldg(mc + w), tp.sw, acc);
        if (tp.ok_s && tp.ok_e) acc = fmaf(__ldg(mc + w + 1), tp.se, acc);
        mean[c] = __fadd_rn(mean[c], acc);
      }
    }
    // d f = (2 g / V) (f - mean)
#pragma unroll
    for (int c = 0; c < CV_CH; ++c) {
      const size_t o = (((size_t)b * C + c0 + c) * D + d) * plane + pix;
      mean[c] = __fdiv_rn(mean[c], fV);
      k[c] = __fdiv_rn(__fmul_rn(2.f, __ldg(grad_cost + o)), fV);
      df0[o] = __fmul_rn(k[c], __fsub_rn(__ldg(ref + c * plane), mean[c]));
    }
    for (int v = 1; v < V; ++v) {
      const Taps tp = cv_view_taps(cam + CB_VIEW + v * CB_VSTRIDE, wx, wy, wz, w, h);
      const float* m = feat + ((size_t)(b * V + v) * C + c0) * plane + (size_t)tp.y0 * w + tp.x0;
      float* out = dfv + (row1 + v - 1) * C + c0;
#pragma unroll
      for (int c4 = 0; c4 < CV_CH; c4 += 4) {
        float g[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int c = c4 + j;
          const float* mc = m + c * plane;
          float acc = 0.f;
          if (tp.ok_n && tp.ok_w) acc = __fmul_rn(__ldg(mc), tp.nw);
          if (tp.ok_n && tp.ok_e) acc = fmaf(__ldg(mc + 1), tp.ne, acc);
          if (tp.ok_s && tp.ok_w) acc = fmaf(__ldg(mc + w), tp.sw, acc);
          if (tp.ok_s && tp.ok_e) acc = fmaf(__ldg(mc + w + 1), tp.se, acc);
          g[j] = __fmul_rn(k[c], __fsub_rn(acc, mean[c]));
        }
        st4(out + c4, make_float4(g[0], g[1], g[2], g[3]));
      }
    }
  }
}

// grad_features [B,V,C,h*w]: view 0 = sum over d (ascending) of d f_0; view v >= 1 = the texel sums
// tex [B][(V-1) h w][C]
__global__ void __launch_bounds__(256)
    cv_bwd_finish_kernel(const float* __restrict__ df0, const float* __restrict__ tex, float* __restrict__ grad, int V,
                         int C, int hw, int D, long long total) {
  const long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= total) return;
  const int pix = (int)(e % hw);
  const long long r = e / hw;
  const int c = (int)(r % C);
  const long long bv = r / C;
  const int v = (int)(bv % V);
  const long long b = bv / V;
  if (v == 0) {
    const float* s = df0 + ((b * C + c) * D) * hw + pix;
    float acc = 0.f;
    for (int d = 0; d < D; ++d) acc = __fadd_rn(acc, __ldg(s + (size_t)d * hw));
    grad[e] = acc;
  } else {
    grad[e] = __ldg(tex + ((b * (V - 1) + v - 1) * hw + pix) * C + c);
  }
}

struct CvBwdPlan {
  long long N, S;  // plane points and source rows (point, view >= 1) of a batch element
  size_t cam, df0, dfv, rec_idx, rec_w, lists, tex, total;
};

// workspace (each region rounded up to 256 bytes), with N = D h w and S = (V - 1) N:
//   camera blocks B (28 + 24 V) 4 | d f_0 4 B C N | d f_v 4 B S C | records 8 B 4 S + 4 B 4 S |
//   inverse lists inv_lists_bytes(B, S, 4) = 4 B S (1 + 1 + 4) + 4 B (S + 1) | texel sums 4 B (V - 1) h w C
int cv_bwd_plan(int B, int V, int C, int h, int w, int D, CvBwdPlan& p) {
  PMVS_TRY(cost_volume_check_shape("cost_volume_backward", B, V, C, h, w, D));
  p.N = (long long)D * h * w;
  p.S = (long long)(V - 1) * p.N;
  PMVS_REQUIRE(4 * p.S < (1ll << 31), "cost_volume_backward: (V-1)*4*D*h*w = %lld tap records per batch element (limit 2^31)",
               4 * p.S);
  size_t o = 0;
  p.cam = o; o += up256(cam_block_bytes(B, V));
  p.df0 = o; o += up256((size_t)B * C * p.N * 4);
  p.dfv = o; o += up256((size_t)B * p.S * C * 4);
  p.rec_idx = o; o += up256((size_t)B * p.S * 4 * 8);
  p.rec_w = o; o += up256((size_t)B * p.S * 4 * 4);
  p.lists = o; o += up256(inv_lists_bytes(B, p.S, 4));
  p.tex = o; o += up256((size_t)B * (V - 1) * h * w * C * 4);
  p.total = o;
  return PMVS_OK;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" size_t pmvs_cost_volume_backward_workspace_bytes(int B, int V, int C, int h, int w, int D) {
  CvBwdPlan p;
  if (cv_bwd_plan(B, V, C, h, w, D, p) != PMVS_OK) return 0;
  return p.total;
}

extern "C" int pmvs_cost_volume_backward(const float* features, const float* cam_params, const float* grad_cost,
                                         float* grad_features, void* workspace, size_t workspace_bytes, int B, int V,
                                         int C, int h, int w, int D, int is_test, pmvs_stream_t stream) {
  PMVS_REQUIRE(features && cam_params && grad_cost && grad_features && workspace, "cost_volume_backward: NULL pointer");
  CvBwdPlan p;
  PMVS_TRY(cv_bwd_plan(B, V, C, h, w, D, p));
  PMVS_TRY(check_workspace("cost_volume_backward", workspace, workspace_bytes, p.total));
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  auto F = [&](size_t off) { return (float*)(ws + off); };
  // the forward's camera blocks (pmvs_cost_volume): model.py:58-61
  PMVS_TRY(launch_cam_setup(cam_params, nullptr, nullptr, nullptr, F(p.cam), B, V, is_test ? 0.125f : 0.5f, 1.f, st));
  prof_begin("cv_bwd_point", st);
  cv_bwd_point_kernel<<<dim3(cdiv(p.N, 256), B), 256, 0, st>>>(features, cam_params, F(p.cam), grad_cost, F(p.df0),
                                                               F(p.dfv), (int64_t*)(ws + p.rec_idx), F(p.rec_w), V, C,
                                                               h, w, D);
  PMVS_TRY(check_launch("cv_bwd_point_kernel", st));
  if (V > 1) {
    const int* off = nullptr;
    const int* list = nullptr;
    const int S = (int)p.S, T = (V - 1) * h * w;
    PMVS_TRY(build_inv_lists((const int64_t*)(ws + p.rec_idx), B, S, 4, ws + p.lists, &off, &list, "cv_bwd_lists", st));
    PMVS_TRY(launch_texel_sum(off, list, F(p.rec_w), F(p.dfv), F(p.tex), T, 4 * S, B, C, (long long)T * C, C,
                              "cv_bwd_texel_sum", st));
  }
  const long long total = (long long)B * V * C * h * w;
  prof_begin("cv_bwd_finish", st);
  cv_bwd_finish_kernel<<<cdiv(total, 256), 256, 0, st>>>(F(p.df0), F(p.tex), grad_features, V, C, h * w, D, total);
  return check_launch("cv_bwd_finish_kernel", st);
}
