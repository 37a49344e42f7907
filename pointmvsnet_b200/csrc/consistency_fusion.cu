// Geometric-consistency fusion: a scene's V depth maps -> per-pixel consistent-view counts, averaged depths and fused
// points (include/pmvs_b200.h, DESIGN 3.21).  Every reference view r is checked against its own source list src[r]
// (S entries, -1 = none) in one launch; one thread per (r, pixel), and a block never spans two reference views, so the
// camera block of r, the list entry and the camera block of the source are warp-uniform loads.  Per valid pixel:
//   X = backproject(r, pixel centre, d); for each source s in list order:
//   (u, w, z) = project(s, X), z > 0; ds = bilinear depth[s] at index coordinates (u - .5, w - .5), valid;
//   (u', w', z') = project(r, backproject(s, u, w, ds));
//   consistent iff z' > 0, (u' - px)^2 + (w' - py)^2 <= reproj^2 and |z' - d| <= depth_thresh d.
// depth_avg = (d + sum z') / (count + 1) where count >= num_consistent (else 0);
// xyz = backproject(r, pixel centre, depth_avg) there (else 0).
// Every operation is one fp32 rounding (fusion_geometry.cuh: no FMA contraction), so the results equal the numpy
// float32 restatement the tests compare against, bit for bit.  No thread reads another thread's output: no atomics,
// and the outputs do not depend on thread or view order.
#include "common.cuh"
#include "fusion_geometry.cuh"

namespace pmvs {

namespace {

constexpr int CF_THREADS = 256;
constexpr float CF_MAX_COORD = 16777216.f;  // 2^24: beyond it a landing point is not consistent

// depth[s] at (i, j) for the bilinear taps: 0 off the map or where the depth is invalid
__device__ __forceinline__ float tap(const float* __restrict__ ds, int i, int j, int H, int W) {
  if (i < 0 || i >= W || j < 0 || j >= H) return 0.f;
  const float t = __ldg(ds + (size_t)j * W + i);
  return valid_depth(t) ? t : 0.f;
}

__global__ void __launch_bounds__(CF_THREADS)
    consistency_filter_kernel(const float* __restrict__ depth, const float* __restrict__ cams,
                              const int* __restrict__ src, int V, int S, int H, int W, int blocks_per_view,
                              int num_consistent, float depth_thresh, float reproj_thresh, int* __restrict__ count_out,
                              float* __restrict__ depth_out, float* __restrict__ xyz_out) {
  const int HW = H * W;
  const int r = blockIdx.x / blocks_per_view;
  const int p = (blockIdx.x - r * blocks_per_view) * CF_THREADS + threadIdx.x;
  if (p >= HW) return;
  const size_t rp = (size_t)r * HW + p;
  const float d = __ldg(depth + rp);
  if (!valid_depth(d)) {
    count_out[rp] = -1;
    depth_out[rp] = 0.f;
    if (xyz_out != nullptr) xyz_out[rp * 3 + 0] = xyz_out[rp * 3 + 1] = xyz_out[rp * 3 + 2] = 0.f;
    return;
  }
  const int x = p % W, y = p / W;
  const float px = __fadd_rn((float)x, 0.5f), py = __fadd_rn((float)y, 0.5f);
  const float* cbr = cams + (size_t)r * FB_STRIDE;
  float X0, X1, X2;
  backproject(cbr, px, py, d, X0, X1, X2);
  const float r2 = __fmul_rn(reproj_thresh, reproj_thresh);
  const float dlim = __fmul_rn(depth_thresh, d);
  const int* list = src + (size_t)r * S;
  float sum = d;
  int count = 0;
#pragma unroll 1
  for (int k = 0; k < S; ++k) {
    const int s = __ldg(list + k);
    if (s < 0 || s >= V || s == r) continue;  // -1 pads the list; the others are refused on the host, never read
    const float* cbs = cams + (size_t)s * FB_STRIDE;
    float u, w, z;
    project(cbs, X0, X1, X2, u, w, z);
    const float a = __fsub_rn(u, 0.5f), b = __fsub_rn(w, 0.5f);
    if (!(z > 0.f && fabsf(a) <= CF_MAX_COORD && fabsf(b) <= CF_MAX_COORD)) continue;  // NaN fails too
    const float fi = floorf(a), fj = floorf(b);
    const float fa = __fsub_rn(a, fi), fb = __fsub_rn(b, fj);
    const float ga = __fsub_rn(1.f, fa), gb = __fsub_rn(1.f, fb);
    const int i0 = (int)fi, j0 = (int)fj;
    const float* dsm = depth + (size_t)s * HW;
    const float t00 = tap(dsm, i0, j0, H, W), t01 = tap(dsm, i0 + 1, j0, H, W);
    const float t10 = tap(dsm, i0, j0 + 1, H, W), t11 = tap(dsm, i0 + 1, j0 + 1, H, W);
    const float ds = __fadd_rn(__fadd_rn(__fmul_rn(__fmul_rn(ga, gb), t00), __fmul_rn(__fmul_rn(fa, gb), t01)),
                               __fadd_rn(__fmul_rn(__fmul_rn(ga, fb), t10), __fmul_rn(__fmul_rn(fa, fb), t11)));
    if (!valid_depth(ds)) continue;
    float Y0, Y1, Y2, u2, w2, z2;
    backproject(cbs, u, w, ds, Y0, Y1, Y2);
    project(cbr, Y0, Y1, Y2, u2, w2, z2);
    const float du = __fsub_rn(u2, px), dw = __fsub_rn(w2, py);
    if (z2 > 0.f && __fadd_rn(__fmul_rn(du, du), __fmul_rn(dw, dw)) <= r2 && fabsf(__fsub_rn(z2, d)) <= dlim) {
      ++count;
      sum = __fadd_rn(sum, z2);
    }
  }
  count_out[rp] = count;
  const float davg = count >= num_consistent ? __fdiv_rn(sum, (float)(count + 1)) : 0.f;
  depth_out[rp] = davg;
  if (xyz_out == nullptr) return;
  X0 = X1 = X2 = 0.f;
  if (count >= num_consistent) backproject(cbr, px, py, davg, X0, X1, X2);
  xyz_out[rp * 3 + 0] = X0;
  xyz_out[rp * 3 + 1] = X1;
  xyz_out[rp * 3 + 2] = X2;
}

}  // namespace

}  // namespace pmvs

using namespace pmvs;

extern "C" int pmvs_consistency_filter(const float* depth, const float* cam_block, const int* src, int V, int S,
                                       int H, int W, int num_consistent, float depth_thresh, float reproj_thresh,
                                       int* count_out, float* depth_avg_out, float* xyz_out, pmvs_stream_t stream) {
  PMVS_REQUIRE(depth && cam_block && count_out && depth_avg_out && (src || S == 0),
               "consistency_filter: NULL pointer");
  PMVS_REQUIRE(V >= 1 && H >= 1 && W >= 1 && S >= 0, "consistency_filter: bad shape V=%d S=%d H=%d W=%d", V, S, H, W);
  PMVS_REQUIRE((long long)V * H * W < (1ll << 31), "consistency_filter: V*H*W = %lld (limit 2^31)",
               (long long)V * H * W);
  PMVS_REQUIRE(num_consistent >= 1, "consistency_filter: num_consistent = %d (must be >= 1)", num_consistent);
  PMVS_REQUIRE(finite_nonneg(depth_thresh) && finite_nonneg(reproj_thresh),
               "consistency_filter: thresholds must be finite and >= 0 (depth %g, reproj %g)", (double)depth_thresh,
               (double)reproj_thresh);
  const int HW = H * W;
  const int blocks_per_view = cdiv(HW, CF_THREADS);  // V * blocks_per_view <= V*H*W < 2^31 blocks
  cudaStream_t st = (cudaStream_t)stream;
  prof_begin("consistency_filter", st);
  consistency_filter_kernel<<<V * blocks_per_view, CF_THREADS, 0, st>>>(depth, cam_block, src, V, S, H, W,
                                                                        blocks_per_view, num_consistent, depth_thresh,
                                                                        reproj_thresh, count_out, depth_avg_out,
                                                                        xyz_out);
  return check_launch("consistency_filter_kernel", st);
}
